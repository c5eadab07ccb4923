"""Whole-step CUDA graph for a fixed-shape batch: forward -> loss -> backward captured once, replayed every step.

A WavLM-Large step is ~6400 kernel launches; enqueueing them through ctypes costs the host ~24 ms per 35 ms step.  That is off
the critical path while the GPU is the bottleneck, but it is host time the data loader does not get.  With the step captured in
one `torch.cuda.CUDAGraph` the host does, per step: sample the span mask with the reference's numpy sampler
(WavLM/WavLM.py:271-287) into a pinned buffer, enqueue two small copies and ONE graph launch.

What makes the capture legal (and what it requires):
  * every kernel goes to `torch.cuda.current_stream()` and every backward runs on its forward's stream (`wavlm._on_forward_stream`);
    the library itself never synchronises or allocates (csrc/: no cudaMalloc / cudaStreamSynchronize); all tensors created inside
    the capture come from the graph's private pool, so the TMA descriptors encoded at capture time stay valid on replay;
  * the batch shape and the set of executed layers are frozen: no padded samples (an all-False `padding_mask` is accepted and
    dropped, which is what the reference's own code path does with it), `encoder_layerdrop` must be 0, and the dropouts must be
    0 (their seeds are host-side kernel arguments);
  * the span mask is DATA, not structure: it lives in a static device tensor that the graph reads (`mask_indices=`); so does the
    channel mask of models with `mask_channel_prob > 0` (`mask_channel_indices=`, drawn right after the span mask).

`GraphedForwardBackward.step()` returns the static loss tensor of the replay; gradients are in `model.grad_buffer()` exactly as
after an eager `loss.backward()`.  Data-parallel runs keep the eager path (the bucketed NCCL exchange is issued from Python
between the backward stages, parallel.OverlappedGradSync).
"""
from __future__ import annotations

from typing import Callable, Optional

import torch

from .engine import ConvGeom


class GraphedForwardBackward:
    def __init__(self, model, loss_fn: Callable[[torch.Tensor], torch.Tensor], batch: int, samples: int, device,
                 padding_mask: Optional[torch.Tensor] = None, mask: bool = True):
        cfg = model.cfg
        if float(getattr(cfg, "encoder_layerdrop", 0.0)) > 0.0 and model.training:
            raise ValueError("GraphedForwardBackward: encoder_layerdrop > 0 changes the executed layers from step to step")
        for name in ("dropout", "attention_dropout", "activation_dropout", "dropout_input", "dropout_features"):
            if float(getattr(cfg, name, 0.0)) > 0.0 and model.training:
                raise ValueError(f"GraphedForwardBackward: {name} > 0 (dropout seeds are host-side kernel arguments)")
        if padding_mask is not None and padding_mask.device.type != "cpu":
            raise ValueError("GraphedForwardBackward: padding_mask must be a fixed host tensor")
        self.model, self.loss_fn, self.device, self.use_mask = model, loss_fn, torch.device(device), bool(mask)
        self.B, self.L = int(batch), int(samples)
        self.T = ConvGeom(model.conv_cfg, self.L).T[-1]
        if padding_mask is not None and bool(padding_mask.any()):
            # (a padded batch uploads its frame mask from pageable host memory inside extract_features: not capturable as is)
            raise ValueError("GraphedForwardBackward: padded batches take the eager path")
        self.pad, self.fpm_host = None, None
        self.wav = torch.zeros(self.B, self.L, dtype=torch.float32, device=self.device)
        self.mask_dev = torch.zeros(self.B, self.T, dtype=torch.bool, device=self.device)
        self.mask_host = torch.zeros(self.B, self.T, dtype=torch.bool).pin_memory()
        self.use_chan = self.use_mask and float(getattr(cfg, "mask_channel_prob", 0.0)) > 0.0
        self.chan_dev, self.chan_host = None, None
        if self.use_chan:
            self.chan_dev = torch.zeros(self.B, cfg.encoder_embed_dim, dtype=torch.bool, device=self.device)
            self.chan_host = torch.zeros(self.B, cfg.encoder_embed_dim, dtype=torch.bool).pin_memory()
        self.loss = torch.zeros((), dtype=torch.float32, device=self.device)
        self.graph: Optional[torch.cuda.CUDAGraph] = None
        self.capture_host_ms: Optional[float] = None

    # ---- the step body (identical in the eager warm-up and inside the capture)
    def _body(self):
        m = self.model
        if m._engine is not None and m._engine.flat is not None:
            m.zero_grad_buffer()
            m._engine.prepared_version = None  # parameters change between steps: re-derive the bf16 operands
        x, _ = m.extract_features(self.wav, padding_mask=self.pad, mask=self.use_mask,
                                  mask_indices=self.mask_dev if self.use_mask else None, mask_channel_indices=self.chan_dev)
        loss = self.loss_fn(x)
        loss.backward()
        self.loss.copy_(loss.detach().float().reshape(()))

    def sample_mask(self):
        """Host-side span (and channel) sampling of the reference into the pinned buffers, then small async copies to the static
        device masks."""
        if not self.use_mask:
            return
        idx, chan = self.model.sample_masks(self.B, self.T, self.fpm_host)
        if idx is None:
            self.mask_host.zero_()
        else:
            self.mask_host.copy_(idx)
        self.mask_dev.copy_(self.mask_host, non_blocking=True)
        if self.use_chan:
            self.chan_host.copy_(chan)
            self.chan_dev.copy_(self.chan_host, non_blocking=True)

    def capture(self, warmup: int = 2):
        """Eager warm-up on a side stream (lazy initialisation: kernel attributes, engine scratch, the flat gradient buffer), then
        the capture."""
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            for _ in range(max(1, warmup)):
                self.sample_mask()
                self._body()
        torch.cuda.current_stream(self.device).wait_stream(side)
        torch.cuda.synchronize(self.device)
        self.graph = torch.cuda.CUDAGraph()
        # capture on the SAME side stream as the warm-up: autograd remembers the stream a leaf's gradient accumulator was created
        # on, and a backward pass captured on another stream would have to wait on that (uncaptured) stream
        # (cudaErrorStreamCaptureIsolation)
        import time
        t0 = time.perf_counter()
        with torch.cuda.graph(self.graph, stream=side):
            self._body()
        # one-off cost: host time of the stream capture of one step (launch recording + graph-node creation; ~55 ms for WavLM-Large)
        self.capture_host_ms = (time.perf_counter() - t0) * 1e3
        return self

    def step(self, wav_host: Optional[torch.Tensor] = None) -> torch.Tensor:
        """One step: optional host->device copy of the batch (pinned `wav_host`), new span mask, graph replay."""
        if self.graph is None:
            raise RuntimeError("call capture() first")
        if wav_host is not None:
            self.wav.copy_(wav_host, non_blocking=True)
        self.sample_mask()
        self.graph.replay()
        return self.loss
