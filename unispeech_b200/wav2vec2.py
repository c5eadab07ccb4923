"""wav2vec 2.0 pre-training model on the same kernels (SURVEY.md section 8f row 4): the encoder of `wavlm.WavLM` (no relative
position bias) + the quantizer of the targets + the contrastive (InfoNCE) head.

Mirrors src/fairseq/models/wav2vec/wav2vec2.py: constructor :304-418 (state_dict keys `quantizer.vars`,
`quantizer.weight_proj.*`, `project_q.*`, `final_proj.*`), `forward` :556-723 (targets are the LayerNorm'ed conv features of the
MASKED frames, quantised and projected; negatives drawn from them; x = `final_proj` of the encoder output at the same frames),
`sample_negatives` :474-531 (host `torch.randint`, same calls in the same order), `compute_preds` :533-553 (cosine logits / temp,
a negative that equals the positive gets -inf), `get_extra_losses` :752-767, and `Wav2vecCriterion.get_loss` with `infonce`
(src/fairseq/criterions/wav2vec_criterion.py:44-118).
Kernels: `b200s_gather_rows`, wgmma GEMMs (final_proj, quantizer logits, project_q), `b200s_vq_hard` (eval arg-max / training
Gumbel hard sample with the counter-based noise), `b200s_w2v_nce_fwd` (logits + -inf masking + cross entropy + accuracy in one pass;
nothing of size [N+1, S, Dp] exists), `b200s_sat_nce_bwd`, `b200s_vq_logits_bwd`, `b200s_vq_dvars`.  The gradient of the quantizer
branch reaches the conv stack through the LayerNorm output (`_ProjFn`'s third output).
Not built (raise): `quantize_input`, `negatives_from_everywhere`, `codebook_negatives`, `target_glu`, `dropout_features > 0`.
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
from .wavlm import WavLM, WavLMConfig, _on_forward_stream

_SITE_GUMBEL_W2V = 0x7F000003  # noise site of this model's quantizer


class Wav2Vec2Config(WavLMConfig):
    """WavLMConfig + the pre-training fields of Wav2Vec2Config (wav2vec2.py:35-228)."""

    def __init__(self, cfg=None):
        self.final_dim = 256
        self.quantize_targets = True
        self.quantize_input = False
        self.latent_vars = 320
        self.latent_groups = 2
        self.latent_dim = 0
        self.latent_temp = (2.0, 0.5, 0.999995)
        self.num_negatives = 100
        self.cross_sample_negatives = 0
        self.codebook_negatives = 0
        self.negatives_from_everywhere = False
        self.logit_temp = 0.1
        self.target_glu = False
        super().__init__(None)
        self.relative_position_embedding = False
        self.gru_rel_pos = False
        if cfg is not None:
            self.update(cfg)


class _W2vNceFn(torch.autograd.Function):
    """InfoNCE loss of the selected frames.  x2d: bf16 [B*T, D] encoder output; f2d: bf16 [B*T, C] LayerNorm'ed conv features."""

    @staticmethod
    def forward(ctx, x2d, f2d, anchor, model, rows_idx, neg_idx, S, N, gum_key, stats_out):
        ctx.fwd_stream = torch.cuda.current_stream()
        dev = x2d.device
        Dp = model.final_dim
        fp, qz, pq = model.final_proj, model.quantizer, model.project_q
        xs, ys = H.gather(x2d, rows_idx), H.gather(f2d, rows_idx)
        wfp, wfpT = H.linear_operands(fp.weight)
        proj = H.linear_rows(xs, wfp, fp.bias)
        wpq, wpqT = H.linear_operands(pq.weight)
        yin, qs = ys, None                        # project_q's input: the features, or their quantized codes
        if qz is not None:
            yin, qs = qz.forward_rows(ys, gum_key, stats_out)
            stats_out["codes"] = qs["codes"].view(S, qz.groups)   # `targets` of the reference's produce_targets
        y = H.linear_rows(yin, wpq, pq.bias)
        g = torch.empty(S, N + 1, dtype=torch.float32, device=dev)
        loss64 = torch.zeros(1, dtype=torch.float64, device=dev)
        stats = torch.zeros(2, dtype=torch.int32, device=dev)
        ops.w2v_nce_fwd(proj, Dp, y, Dp, neg_idx, S, N, Dp, model.logit_temp, g, loss64, stats)
        stats_out["correct"], stats_out["count"] = stats[0], stats[1]
        ctx.model, ctx.sel, ctx.rows = model, (rows_idx, neg_idx), x2d.shape[0]
        ctx.st = dict(xs=xs, proj=proj, wfpT=wfpT, yin=yin, wpqT=wpqT, y=y, g=g, quant=qs)
        outs = [loss64.float().reshape(())]
        if qz is not None:
            outs.append(H.perplexity(qs["avg_probs"]).sum())  # prob_perplexity (differentiable below)
        return tuple(outs)

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dloss, dppl=None):
        model, st = ctx.model, ctx.st
        rows_idx, neg_idx = ctx.sel
        S, Dp = st["proj"].shape
        N = st["g"].shape[1] - 1
        dev = st["xs"].device
        g_ = model._engine.g
        qs = st["quant"]
        fp, pq = model.final_proj, model.project_q
        up = (dloss if dloss is not None else torch.zeros((), device=dev)).float().reshape(1).contiguous()
        dacc_p = torch.zeros(S, Dp, dtype=torch.float32, device=dev)
        dacc_y = torch.zeros(S, Dp, dtype=torch.float32, device=dev)
        ops.sat_nce_bwd(st["proj"], Dp, st["y"], Dp, neg_idx, S, N, Dp, model.logit_temp, st["g"], up, dacc_p, dacc_y)
        # ---- x branch: final_proj
        dproj = _rows(S, Dp, BF, dev)
        ops.f32_to_bf16_rows(dacc_p, Dp, dproj, Dp, S, Dp)
        dx = H.scatter(H.linear_rows_backward(dproj, st["xs"], st["wfpT"], g_(fp.weight), g_(fp.bias)), rows_idx, ctx.rows)
        # ---- y branch: project_q (+ quantizer)
        dy = _rows(S, Dp, BF, dev)
        ops.f32_to_bf16_rows(dacc_y, Dp, dy, Dp, S, Dp)
        dys = H.linear_rows_backward(dy, st["yin"], st["wpqT"], g_(pq.weight), g_(pq.bias))
        if qs is not None:
            dys = model.quantizer.backward_rows(qs, dys, dppl, g_)
        df = None if dys is None else H.scatter(dys, rows_idx, ctx.rows)
        ctx.st = None
        return dx, df, None, None, None, None, None, None, None, None


class Wav2Vec2Model(WavLM):
    def __init__(self, cfg: Wav2Vec2Config):
        if getattr(cfg, "relative_position_embedding", False) or getattr(cfg, "gru_rel_pos", False):
            raise ValueError("wav2vec 2.0 has no relative position bias")
        for name, bad in (("quantize_input", bool(cfg.quantize_input)), ("negatives_from_everywhere", bool(cfg.negatives_from_everywhere)),
                          ("codebook_negatives", cfg.codebook_negatives > 0), ("target_glu", bool(cfg.target_glu))):
            if bad:
                raise NotImplementedError(f"wav2vec 2.0 head: {name} is not implemented")
        super().__init__(cfg)
        self._want_features_pen = True
        self._want_unmasked_features = True
        D, C = cfg.encoder_embed_dim, self.embed
        self.final_dim = cfg.final_dim if cfg.final_dim > 0 else D
        assert self.final_dim % 64 == 0 and self.final_dim <= 1024, "final_dim must be a multiple of 64 (GEMM K blocks), <= 1024"
        assert C % 64 == 0, "conv feature width must be a multiple of 64 (GEMM K blocks)"
        self.n_negatives, self.cross_sample_negatives = int(cfg.num_negatives), int(cfg.cross_sample_negatives)
        self.logit_temp = float(cfg.logit_temp)
        self.quantizer = None
        if cfg.quantize_targets:
            vq_dim = cfg.latent_dim if cfg.latent_dim > 0 else self.final_dim
            assert (vq_dim // cfg.latent_groups) % 64 == 0, "vq_dim / latent_groups must be a multiple of 64 (GEMM K blocks)"
            assert (cfg.latent_vars * cfg.latent_groups) % 64 == 0, "latent_vars * latent_groups must be a multiple of 64"
            self.quantizer = GumbelVectorQuantizer(C, cfg.latent_vars, tuple(cfg.latent_temp), cfg.latent_groups, vq_dim)
            self.project_q = nn.Linear(vq_dim, self.final_dim)
        else:
            self.project_q = nn.Linear(C, self.final_dim)
        self.final_proj = nn.Linear(D, self.final_dim)
        self.noise_seed: Optional[int] = None   # an int pins the Gumbel noise (tests)
        self.num_updates = 0

    # ---- BaseFairseqModel surface
    def set_num_updates(self, num_updates: int):
        self.num_updates = num_updates
        if self.quantizer is not None:
            self.quantizer.set_num_updates(num_updates)

    def upgrade_state_dict_named(self, state_dict, name):
        return state_dict

    def remove_pretraining_modules(self):
        self.quantizer = None
        self.project_q = None
        self.final_proj = None
        self._want_unmasked_features = False

    def get_extra_losses(self, net_output):
        """wav2vec2.py:752-767: [(num_vars - prob_perplexity) / num_vars, features_pen] (positional for `loss_weights`)."""
        pen = []
        if net_output.get("prob_perplexity") is not None:
            pen.append((net_output["num_vars"] - net_output["prob_perplexity"]) / net_output["num_vars"])
        if net_output.get("features_pen") is not None:
            pen.append(net_output["features_pen"])
        return pen

    def forward(self, source, padding_mask=None, mask=True, features_only=False, layer=None, mask_indices=None,
                mask_channel_indices=None):
        """Result keys of wav2vec2.py:633-723 except that `x` (the [N+1, B, T'] logits) is replaced by the fused loss:
        `loss_nce` (sum of cross entropies, device scalar), `sample_size`, `correct`, `count`."""
        if float(getattr(self.cfg, "dropout_features", 0.0)) > 0 and self.training and not features_only:
            raise NotImplementedError("dropout_features > 0 on the quantizer input is not implemented")
        # (`layer` is the 0-based index of the reference's TransformerEncoder.extract_features; extract_features here is 1-based)
        res = self._extract(source, padding_mask, mask, False, None if layer is None else layer + 1, mask_indices,
                            mask_channel_indices)
        if features_only:
            return {"x": res["x"], "padding_mask": res["padding_mask"], "features": res["unmasked_features"],
                    "layer_results": res["layer_results"]}
        x, unm, mi = res["x"], res["unmasked_features"], res["mask_indices"]
        assert mi is not None, "the contrastive loss needs mask=True"
        B, T, D = x.shape
        dev = x.device
        mi_h = mi.cpu().bool()
        counts = mi_h.sum(1)
        num = int(counts[0])
        if not bool((counts == num).all()):
            raise RuntimeError("wav2vec 2.0 needs the same number of masked frames in every utterance "
                               f"(`unmasked_features[mask_indices].view(B, -1, C)`, wav2vec2.py:621-623); got {counts.tolist()}")
        S = B * num
        N = self.n_negatives + self.cross_sample_negatives
        rows_h = torch.nonzero(mi_h.reshape(-1), as_tuple=False).squeeze(1)
        negs = sample_instances(B, num, self.n_negatives, self.cross_sample_negatives)      # [B, N * num], wav2vec2.py:488-523
        neg_ns = negs.to(torch.int32).view(B, num, N).permute(2, 0, 1).reshape(N, S)          # frame-major list -> [N, S] (:525-531)
        up = lambda t: t.contiguous().pin_memory().to(dev, non_blocking=True)
        x2d = H.bf16(x.reshape(B * T, D))
        f2d = unm.reshape(B * T, unm.shape[-1])
        seed = self.noise_seed if self.noise_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
        stats: Dict = {}
        outs = _W2vNceFn.apply(x2d, f2d, self.final_proj.weight, self, up(rows_h.to(torch.int32)), up(neg_ns), S, N,
                               DR.site_key(seed, _SITE_GUMBEL_W2V), stats)
        out = {"loss_nce": outs[0], "sample_size": S, "correct": stats["correct"], "count": stats["count"],
               "padding_mask": res["padding_mask"], "features_pen": res["features_pen"], "mask_indices": mi}
        if self.quantizer is not None:
            out.update(prob_perplexity=outs[1], code_perplexity=stats["code_perplexity"], num_vars=stats["num_vars"],
                       temp=stats["temp"], codes=stats["codes"])
        return out

    def criterion(self, net_output: Dict, loss_weights: Optional[List[float]] = None):
        """Wav2vecCriterion.get_loss with infonce (wav2vec_criterion.py:44-118): (loss, sample_size, logging_output)."""
        loss, ssz = net_output["loss_nce"], net_output["sample_size"]
        log = {"loss_0": loss.detach()}
        if loss_weights is not None:
            for i, p in H.weighted_extra_losses(self.get_extra_losses(net_output), loss_weights, ssz):
                loss = loss + p
                log[f"loss_{i + 1}"] = p.detach()
        log.update(loss=loss.detach(), ntokens=ssz, sample_size=ssz, correct=net_output["correct"], count=net_output["count"])
        for k in ("prob_perplexity", "code_perplexity", "temp"):
            if k in net_output:
                log[k] = net_output[k]
        return loss, ssz, log
