"""MFCC + delta features of HuBERT's first iteration on the library's kernels (`csrc/mfcc.cu`).

The HuBERT recipe (src/examples/hubert/simple_kmeans/dump_mfcc_feature.py) labels the first pre-training iteration with k-means
over 39-dim MFCC features at 100 Hz, computed on the CPU by

    mfcc = torchaudio.compliance.kaldi.mfcc(waveform=x, sample_frequency=16000, use_energy=False)   # [Tm, 13]
    delta = torchaudio.functional.compute_deltas(mfcc.T); ddelta = compute_deltas(delta)
    feats = torch.cat([mfcc, delta.T, ddelta.T], dim=-1)                                            # [Tm, 39]

and dumped to disk.  Here a whole padded batch is computed on the GPU and handed straight to `KMeans`::

    feats, pm, rows = mfcc(wav, padding_mask=pad, kmeans_rows=True)
    km = KMeans(100, ...).fit(rows[~pm])              # valid frames
    labels = km.predict(rows, pm)                     # int32 [B, Tm], -1 at padded frames
    model = HubertModel(HubertConfig(dict(cfg, label_rate=100)), [100])
    out = model(wav, target_list=[labels.long().clamp(min=0)], padding_mask=pad, mask=True)

Only the recipe's parameters exist: 16 kHz, no energy, no dither, no CMVN.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import ops

SAMPLE_RATE = 16000
WINDOW, SHIFT = 400, 160    # 25 ms frames every 10 ms
NUM_CEPS = 13
FEATURE_DIM = 3 * NUM_CEPS  # cepstra, deltas, delta-deltas
ROW_DIM = 64                # the k-means operand: FEATURE_DIM zero-padded to a multiple of 64


def num_frames(n: int) -> int:
    """Frames of an utterance of n samples (snip_edges): 1 + (n - 400) // 160, none below 400 samples."""
    return 1 + (n - WINDOW) // SHIFT if n >= WINDOW else 0


def mfcc(source: torch.Tensor, padding_mask: Optional[torch.Tensor] = None, kmeans_rows: bool = False,
         sample_rate: int = SAMPLE_RATE):
    """39-dim MFCC features of a padded batch, the inputs of `extract_features`.

    source: CUDA fp32 waveform [B, L] in [-1, 1] (as the recipe reads it, no normalisation).  padding_mask: bool [B, L], True at
    padded samples (the collater's mask, on the host or the device; valid samples are counted, no device read-back).
    Returns (feats fp32 [B, Tm, 39], frame padding mask bool [B, Tm] on the device or None) and, with `kmeans_rows`, the bf16
    [B, Tm, 64] operand of `KMeans` (feats rounded to bf16, zero columns 39..63).  Tm = num_frames(L); padded frames are zeros.
    An utterance shorter than 400 samples has no frames: its row of the mask is all True."""
    if sample_rate != SAMPLE_RATE:
        raise ValueError(f"sample_rate={sample_rate}: the MFCC features are built for {SAMPLE_RATE} Hz only")
    if not isinstance(source, torch.Tensor) or not source.is_cuda or source.dtype != torch.float32 or source.dim() != 2:
        raise TypeError(f"mfcc: expected a CUDA fp32 [B, L] waveform, got {getattr(source, 'dtype', type(source))} "
                        f"{list(getattr(source, 'shape', []))} on {getattr(source, 'device', '?')} (no CPU fallback)")
    B, L = source.shape
    wav = source if source.stride(1) == 1 else source.contiguous()
    dev = wav.device
    Tm = num_frames(L)
    if padding_mask is not None:
        if tuple(padding_mask.shape) != (B, L):
            raise ValueError(f"padding_mask must be [B, L] = [{B}, {L}]; got {list(padding_mask.shape)}")
        if padding_mask.device.type == "cpu":   # numpy's count is several times faster than torch's on a host bool mask
            n = L - torch.from_numpy(np.count_nonzero(padding_mask.bool().numpy(), axis=1)).to(torch.int32)
            n_dev = n.to(dev, non_blocking=True)
        else:
            n = n_dev = L - torch.count_nonzero(padding_mask.bool(), dim=1).to(torch.int32)
    else:
        n_dev = torch.full((B,), L, dtype=torch.int32, device=dev)
    feats = torch.empty(B, Tm, FEATURE_DIM, dtype=torch.float32, device=dev)
    rows = torch.empty(B, Tm, ROW_DIM, dtype=torch.bfloat16, device=dev) if kmeans_rows else None
    if Tm:
        ops.mfcc(wav, wav.stride(0), L, n_dev, B, Tm, feats, Tm * FEATURE_DIM, rows, Tm * ROW_DIM)
    fpm = None
    if padding_mask is not None:
        tb = torch.where(n >= WINDOW, (n - WINDOW) // SHIFT + 1, torch.zeros_like(n))
        fpm = (torch.arange(Tm, device=n.device).unsqueeze(0) >= tb.unsqueeze(1)).to(dev, non_blocking=True)
    return (feats, fpm, rows) if kmeans_rows else (feats, fpm)
