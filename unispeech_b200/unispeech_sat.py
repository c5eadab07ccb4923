"""UniSpeech-SAT pre-training model (BASELINE.json configs[3]): the WavLM-style encoder + masked-prediction head of
`pretrain.WavLMForPretraining` plus the UTTERANCE-CONTRASTIVE loss on the output of an intermediate layer and the Gumbel vector
quantizer of its targets, on the project's kernels (csrc/sat.cu + the wgmma GEMMs).

Mirrors src/fairseq/models/unispeech_sat/unispeech_sat.py: constructor tail :383-412 (state_dict keys `spk_proj.*`, `project_q.*`,
`quantizer.vars`, `quantizer.weight_proj.*`, `encoder.layer_norm_for_extract.*`), `forward` :585-760 (result keys `loss_spk_m`,
`mean_targets`, `contrastive_acc`, `loss_spk_u`, `prob_perplexity`, `code_perplexity`, `num_vars`, `temp`), `sample_instances`
:487-543 (host `torch.randint`, same call order: reproducible under `torch.manual_seed`), `compute_nce` :545-557,
`get_extra_losses` :795-820, `remove_pretraining_modules` :822-834, and `GumbelVectorQuantizer`
(src/fairseq/modules/gumbel_vector_quantizer.py:13-201: `set_num_updates` temperature schedule :85-88, forward :141-201); the
last two live in heads.py, shared with wav2vec 2.0.
Training-mode Gumbel noise comes from the library's counter-based hash (the reference's Philox stream cannot be reproduced;
the CPU checker restates this generator, as for dropout).
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import dropout as DR
from . import heads as H
from . import ops
from .engine import BF
from .heads import GumbelVectorQuantizer, _rows, sample_instances
from .pretrain import WavLMForPretraining, WavLMPretrainConfig
from .wavlm import _on_forward_stream

_SITE_GUMBEL = 0x7F000002  # noise site of the quantizer (distinct from every dropout site)


class UniSpeechSATConfig(WavLMPretrainConfig):
    """WavLMPretrainConfig + the utterance-contrastive fields of UniSpeechSATConfig (unispeech_sat.py:236-286)."""

    def __init__(self, cfg=None):
        self.utterance_contrastive_loss = True
        self.utterance_contrastive_layer = 6      # 1-based encoder layer whose output feeds the speaker loss
        self.num_instances = 0                    # `n_instances`: negatives drawn inside the utterance
        self.cross_sample_instances = 100         # negatives drawn over the whole local batch
        self.quantize_targets = False
        self.latent_vars = 320
        self.latent_groups = 2
        self.latent_dim = 0
        self.latent_temp = (2.0, 0.5, 0.999995)
        self.layer_norm_for_extract = True        # the SAT encoder owns `layer_norm_for_extract` when it is pre-LN (:1196-1197)
        super().__init__(cfg)


_DRAW_POOL = None


def _draw_pool():
    """One helper thread for the host side of the loss head (torch CPU ops release the GIL)."""
    global _DRAW_POOL
    if _DRAW_POOL is None:
        from concurrent.futures import ThreadPoolExecutor
        _DRAW_POOL = ThreadPoolExecutor(max_workers=1, thread_name_prefix="b200s-draw")
    return _DRAW_POOL


class _SpkNceFn(torch.autograd.Function):
    """loss_spk_m of unispeech_sat.py:699-745 on the selected frames.  spk2d: bf16 [B*T, D] (output of the contrastive layer)."""

    @staticmethod
    def forward(ctx, spk2d, anchor, model, rows_idx, inst_idx, same, S, N, gum_key, stats_out):
        ctx.fwd_stream = torch.cuda.current_stream()
        dev = spk2d.device
        Dp = model.final_dim
        sp, qz, pq = model.spk_proj, model.quantizer, model.project_q
        xs = H.gather(spk2d, rows_idx)
        wsp, wspT = H.linear_operands(sp.weight)
        proj = H.linear_rows(xs, wsp, sp.bias)
        y, qs = proj, None
        if qz is not None:
            q, qs = qz.forward_rows(xs, gum_key, stats_out)
            wpq, wpqT = H.linear_operands(pq.weight)
            y = H.linear_rows(q, wpq, pq.bias)
            qs.update(q=q, wpqT=wpqT)
        g = torch.empty(S, N + 1, dtype=torch.float32, device=dev)
        loss64 = torch.zeros(1, dtype=torch.float64, device=dev)
        stats = torch.zeros(2, dtype=torch.int32, device=dev)
        ops.sat_nce_fwd(proj, Dp, y, Dp, inst_idx, same, S, N, Dp, model.logit_temp, g, loss64, stats)
        tot = float(S * (N + 1))
        stats_out["contrastive_acc"] = stats[0].float() / tot
        stats_out["mean_targets"] = stats[1].float() / tot
        ctx.model, ctx.sel, ctx.rows = model, (rows_idx, inst_idx), spk2d.shape[0]
        ctx.st = dict(xs=xs, proj=proj, wspT=wspT, y=y, g=g, quant=qs)
        outs = [loss64.float().reshape(())]
        if qz is not None:
            outs.append(H.perplexity(qs["avg_probs"]).sum())  # prob_perplexity (differentiable below)
        return tuple(outs)

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dloss, dppl=None):
        model, st = ctx.model, ctx.st
        rows_idx, inst_idx = ctx.sel
        S, Dp = st["proj"].shape
        N = st["g"].shape[1] - 1
        dev = st["xs"].device
        g_ = model._engine.g
        qs = st["quant"]
        up = (dloss if dloss is not None else torch.zeros((), device=dev)).float().reshape(1).contiguous()
        dacc_p = torch.zeros(S, Dp, dtype=torch.float32, device=dev)
        dacc_y = dacc_p if qs is None else torch.zeros(S, Dp, dtype=torch.float32, device=dev)
        ops.sat_nce_bwd(st["proj"], Dp, st["y"], Dp, inst_idx, S, N, Dp, model.logit_temp, st["g"], up, dacc_p, dacc_y)
        dproj = _rows(S, Dp, BF, dev)
        ops.f32_to_bf16_rows(dacc_p, Dp, dproj, Dp, S, Dp)
        dxq = None
        if qs is not None:
            pq = model.project_q
            dy = _rows(S, Dp, BF, dev)
            ops.f32_to_bf16_rows(dacc_y, Dp, dy, Dp, S, Dp)
            dq = H.linear_rows_backward(dy, qs["q"], qs["wpqT"], g_(pq.weight), g_(pq.bias))
            dxq = model.quantizer.backward_rows(qs, dq, dppl, g_)
        # spk_proj's gradients come last: the quantizer's input gradient is added in the epilogue of spk_proj's input GEMM
        sp = model.spk_proj
        dxs = H.linear_rows_backward(dproj, st["xs"], st["wspT"], g_(sp.weight), g_(sp.bias), res=dxq)
        ctx.st = None
        return H.scatter(dxs, rows_idx, ctx.rows), None, None, None, None, None, None, None, None, None


class UniSpeechSATForPretraining(WavLMForPretraining):
    """UniSpeechSATModel: `WavLMForPretraining` + utterance-contrastive loss (+ optional quantized targets)."""

    def __init__(self, cfg: UniSpeechSATConfig, num_classes: List[int]):
        super().__init__(cfg, num_classes)
        D = cfg.encoder_embed_dim
        self.utterance_contrastive_loss = bool(cfg.utterance_contrastive_loss)
        self.utterance_contrastive_layer = None
        self.quantizer = None
        if self.utterance_contrastive_loss:
            self.utterance_contrastive_layer = int(cfg.utterance_contrastive_layer)
            assert 1 <= self.utterance_contrastive_layer <= cfg.encoder_layers
            self._extract_layer = self.utterance_contrastive_layer - 1
            self.n_instances = int(cfg.num_instances)
            self.cross_sample_instances = int(cfg.cross_sample_instances)
            assert self.final_dim % 4 == 0 and self.final_dim <= 1024
            if cfg.quantize_targets:
                vq_dim = cfg.latent_dim if cfg.latent_dim > 0 else self.final_dim
                assert (vq_dim // cfg.latent_groups) % 64 == 0, "vq_dim / latent_groups must be a multiple of 64 (GEMM K blocks)"
                assert (cfg.latent_vars * cfg.latent_groups) % 64 == 0, "latent_vars * latent_groups must be a multiple of 64 (GEMM K blocks)"
                self.quantizer = GumbelVectorQuantizer(D, cfg.latent_vars, tuple(cfg.latent_temp), cfg.latent_groups, vq_dim)
                self.project_q = nn.Linear(vq_dim, self.final_dim)
            else:
                self.project_q = nn.Linear(D, self.final_dim)   # present in the state_dict, unused without a quantizer (:405)
            self.spk_proj = nn.Linear(D, self.final_dim)
        self.noise_seed: Optional[int] = None  # an int pins the Gumbel noise (tests)

    def set_num_updates(self, num_updates: int):
        super().set_num_updates(num_updates)
        if self.quantizer is not None:
            self.quantizer.set_num_updates(num_updates)

    def get_extra_losses(self, net_output):
        """unispeech_sat.py:795-820 (order matters: `loss_weights` are positional)."""
        extra_losses, names = [], []
        if "features_pen" in net_output:
            extra_losses.append(net_output["features_pen"]); names.append("features_pen")
        if "loss_spk_m" in net_output:
            extra_losses.append(net_output["loss_spk_m"]); names.append("loss_spk_m")
        if "loss_spk_u" in net_output:
            extra_losses.append(net_output["loss_spk_u"]); names.append("loss_spk_u")
        if "prob_perplexity" in net_output:
            extra_losses.append((net_output["num_vars"] - net_output["prob_perplexity"]) / net_output["num_vars"])
            names.append("prob_perplexity")
        return extra_losses, names

    def remove_pretraining_modules(self):
        super().remove_pretraining_modules()
        if self.utterance_contrastive_loss:
            self.quantizer = None
            self.project_q = None
            self.spk_proj = None
            self.utterance_contrastive_loss = False
            self.utterance_contrastive_layer = None
            self._extract_layer = None
        if hasattr(self.encoder, "layer_norm_for_extract"):
            self.encoder.layer_norm_for_extract = None

    def _draw_instances(self, mi_h: torch.Tensor, pm_h: torch.Tensor, generator=None, device=None):
        """Host side of the utterance-contrastive loss: the selected (masked, unpadded) frames and the sampled instances
        (unispeech_sat.py:487-533, 742) as pinned host tensors.  Needs nothing from the encoder: `forward` runs it on a helper
        thread WHILE the main thread enqueues the encoder kernels -- the ~0.5 M host random draws take 4-15 ms, and a step whose
        ~6400 launches already cost the host as much as they cost the GPU cannot afford them on the launching thread (measured:
        +5 ms per step)."""
        if device is not None and device.type == "cuda":
            torch.cuda.set_device(device)   # (helper thread: pinned allocations must not touch another rank's GPU)
        B, T = mi_h.shape
        masked = ~pm_h & mi_h
        counts = masked.sum(1)
        num = int(counts[0])
        if not bool((counts == num).all()):
            raise RuntimeError("the utterance-contrastive loss needs the same number of masked frames in every utterance "
                               f"(`spk_x[masked].view(B, -1, C)`, unispeech_sat.py:742); got {counts.tolist()}")
        S = B * num
        rows_h = torch.nonzero(masked.reshape(-1), as_tuple=False).squeeze(1)
        N = self.n_instances + self.cross_sample_instances
        inst = sample_instances(B, num, self.n_instances, self.cross_sample_instances, generator)   # [B, N * num] host RNG
        inst_ns = inst.to(torch.int32).view(B, N, num).permute(1, 0, 2).reshape(N, S)    # instances.view(B, N, num, C).permute(1,0,2,3)
        utt = torch.div(torch.arange(S, dtype=torch.int32), num, rounding_mode="floor")
        same = torch.div(inst_ns, num, rounding_mode="floor") == utt.unsqueeze(0)        # instance from the positive's utterance
        pin = lambda t, dt: t.to(dt).contiguous().pin_memory()
        return dict(rows=pin(rows_h, torch.int32), inst=pin(inst_ns, torch.int32), same=pin(same, torch.uint8), S=S, N=N)

    def forward(self, source, target_list=None, padding_mask=None, mask=True, features_only=False, output_layer=None,
                mask_indices=None, mask_channel_indices=None):
        pre, fut, gen = None, None, None
        want_spk = not features_only and self.utterance_contrastive_loss and not self.skip_masked
        if want_spk and mask and (padding_mask is None or padding_mask.device.type == "cpu") and \
                (mask_indices is None or mask_indices.device.type == "cpu"):
            # everything the loss head needs from the host is known before the encoder runs: draw it now (see _draw_instances)
            from .engine import ConvGeom
            B = source.shape[0]
            L = source.shape[1]
            T = ConvGeom(self.conv_cfg, L).T[-1] if target_list is None else self.label_frames(L, target_list)
            pm_h = self.forward_padding_mask(T, padding_mask) if padding_mask is not None else torch.zeros(B, T, dtype=torch.bool)
            if mask_indices is None and mask_channel_indices is None:
                # the channel draw follows the span draw immediately, as in the reference's apply_mask
                mask_indices, mask_channel_indices = self.sample_masks(B, T, pm_h if padding_mask is not None else None)
            if mask_indices is not None:
                # The helper thread draws from a COPY of the global CPU generator (the values the global one would have produced);
                # the global state is moved to where that copy ended once the thread has been joined.
                gen = torch.Generator()
                gen.set_state(torch.get_rng_state())
                fut = _draw_pool().submit(self._draw_instances, mask_indices.bool(), pm_h, gen, source.device)
        out, res = self._forward(source, target_list=target_list, padding_mask=padding_mask, mask=mask, features_only=features_only,
                                 output_layer=output_layer, mask_indices=mask_indices, mask_channel_indices=mask_channel_indices)
        if fut is not None:
            pre = fut.result()
            torch.set_rng_state(gen.get_state())
        if features_only or not self.utterance_contrastive_loss:
            return out
        spk_x = res["spk_x"]                      # [B, T, D]: output of layer `utterance_contrastive_layer` (normalised for pre-LN)
        B, T, D = spk_x.shape
        dev = spk_x.device
        out["loss_spk_u"] = None
        if self.skip_masked:
            out.update(loss_spk_m=None, mean_targets=None, contrastive_acc=None)
            return out
        if pre is None:   # device-resident masks: the frame selection needs them on the host first
            assert res["mask_indices"] is not None, "the utterance-contrastive loss needs mask=True"
            mi_h, pm_h = self._host_masks(res)
            pre = self._draw_instances(mi_h.bool(), pm_h, None, dev)
        S, N = pre["S"], pre["N"]
        up = lambda t: t.to(dev, non_blocking=True)
        spk2d = H.bf16(spk_x.reshape(B * T, D))
        seed = self.noise_seed if self.noise_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
        stats: Dict = {}
        outs = _SpkNceFn.apply(spk2d, self.spk_proj.weight, self, up(pre["rows"]), up(pre["inst"]), up(pre["same"]), S, N,
                               DR.site_key(seed, _SITE_GUMBEL), stats)
        out["loss_spk_m"] = outs[0]
        out["mean_targets"] = stats["mean_targets"]
        out["contrastive_acc"] = stats["contrastive_acc"]
        if self.quantizer is not None:
            out["prob_perplexity"] = outs[1]
            out["code_perplexity"] = stats["code_perplexity"]
            out["num_vars"] = stats["num_vars"]
            out["temp"] = stats["temp"]
        return out
