"""Pre-training surface of the fairseq WavLM model: encoder + masked-prediction head + criterion on the project's kernels.

Mirrors (SURVEY.md section 8b B2 / 8f row 1):
  * `WavLMModel.forward(source, target_list, padding_mask, mask, features_only, output_layer)`
    -- src/fairseq/models/wavlm/wavlm.py:465-576 (state_dict keys `final_proj.*`, `label_embs_concat` as there, :328-345)
  * `WavLMCriterion.get_loss`  -- src/fairseq/criterions/wavlm_criterion.py:52-138: sum-reduced cross entropy over the masked
    (x pred_masked_weight) and unmasked (x pred_nomask_weight) frames, `sample_size`, `features_pen` extra loss, accuracy counts.
The reference materialises `[C+1, S, final_dim]` expanded targets and `[S, C+1]` logits per label set; here the logits are one
wgmma GEMM against the row-normalised label embeddings and the softmax / cross entropy / backward operand come from one
row kernel (csrc/nce.cu), so the loss is a scalar produced on the device with no host synchronisation.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from . import heads as H
from . import ops
from .engine import BF
from .heads import _rows
from .wavlm import WavLM, WavLMConfig, _on_forward_stream


class WavLMPretrainConfig(WavLMConfig):
    """WavLMConfig + the pre-training fields of the fairseq dataclass (src/fairseq/models/wavlm/wavlm.py:50,104-135,223-230)."""

    def __init__(self, cfg=None):
        self.label_rate = 50
        self.sample_rate = 16000
        self.final_dim = 256
        self.untie_final_proj = False
        self.logit_temp = 0.1
        self.target_glu = False
        self.skip_masked = False
        self.skip_nomask = False
        super().__init__(cfg)


def _head_forward(model, x2d, w, b, label_embs, idx):
    """Shared front of the masked-prediction head: gather the selected frames, final_proj, and per label set the GEMM against the
    row-normalised label embeddings.  Returns the state both the fused criterion and the materialising logits path build on."""
    dev = x2d.device
    S = idx.numel()
    Dp = model.final_dim
    Dt = w.shape[0]
    untie = model.untie_final_proj
    wp, wpT = H.linear_operands(w)
    xs = H.gather(x2d, idx)
    proj = H.linear_rows(xs, wp, b)
    sets, off = [], 0
    for i, C in enumerate(model.num_classes):
        Cpad = (C + 63) // 64 * 64
        E = label_embs[off:off + C]
        en, en_t = _rows(Cpad, Dp, BF, dev), _rows(Dp, Cpad, BF, dev)
        invn = torch.empty(C, dtype=torch.float32, device=dev)
        ops.nce_prep(E, C, Cpad, Dp, en, en_t, invn)
        proj_i = proj[:, i * Dp:(i + 1) * Dp] if untie else proj
        zraw = _rows(S, Cpad, BF, dev)
        ops.gemm_rows(proj_i, 0, Dt, S, 1, Dp, en, Cpad, zraw, 0, Cpad, None)
        sets.append(dict(off=off, C=C, Cpad=Cpad, en_t=en_t, invn=invn, zraw=zraw))
        off += C
    return dict(xs=xs, proj=proj, wpT=wpT, sets=sets, shape=(x2d.shape[0], S, Dp, Dt, untie))


def _head_backward(st, label_embs, idx, Gs, pns, rvecs, grads):
    """Shared back of the head.  Gs[i] = d loss / d (proj . En^T) (bf16 [S, Cpad]), rvecs[i] = sum_c G_sc cos_sc, pns[i] = 1/|proj_s|:
    d proj = G En - rvec pn proj,  d En = G^T proj,  then final_proj's weight / bias / input gradients and the scatter back.
    `grads` = (d label_embs [sum C, Dp], d final_proj.weight, d final_proj.bias): fp32 views to accumulate into."""
    rows, S, Dp, Dt, untie = st["shape"]
    dev = st["xs"].device
    g_emb, g_w, g_b = grads
    dproj = _rows(S, Dt, BF, dev)
    for i, se in enumerate(st["sets"]):
        off, C, Cpad = se["off"], se["C"], se["Cpad"]
        proj_i = st["proj"][:, i * Dp:(i + 1) * Dp] if untie else st["proj"]
        first = untie or i == 0
        tgt = (dproj[:, i * Dp:(i + 1) * Dp] if untie else dproj) if first else _rows(S, Dp, BF, dev)
        ops.gemm_rows(Gs[i], 0, Cpad, S, 1, Cpad, se["en_t"], Dp, tgt, 0, tgt.stride(0), None)          # G En
        ops.nce_dproj(tgt, tgt.stride(0), proj_i, Dt, S, Dp, pns[i], rvecs[i])
        if not first:
            dproj.add_(tgt)  # tied final_proj shared by several label sets
        d_en = torch.zeros(Cpad, Dp, dtype=torch.float32, device=dev)
        ops.gemm_wgrad(Gs[i], 0, Cpad, proj_i, 0, Dt, S, 1, Cpad, Dp, d_en, Dp)                          # G^T proj
        ops.nce_dlabel(d_en, label_embs[off:off + C], se["invn"], C, Dp, g_emb[off:off + C])
    return H.scatter(H.linear_rows_backward(dproj, st["xs"], st["wpT"], g_w, g_b), idx, rows)


class _MaskedPredictionFn(torch.autograd.Function):
    """loss = sum over label sets of weight * CE(cos(final_proj(x[idx]), label_embs) / temp, target).  x: bf16 [B*T, D]."""

    @staticmethod
    def forward(ctx, x2d, w, b, label_embs, model, idx, targets, weight, stats, grads):
        ctx.fwd_stream = torch.cuda.current_stream()
        ctx.grad_views = grads
        dev = x2d.device
        st = _head_forward(model, x2d, w, b, label_embs, idx)
        S, Dp, Dt, untie = idx.numel(), model.final_dim, w.shape[0], model.untie_final_proj
        loss_sum = torch.zeros(1, dtype=torch.float64, device=dev)
        Gs, pns, rvecs = [], [], []
        for i, se in enumerate(st["sets"]):
            C, Cpad = se["C"], se["Cpad"]
            proj_i = st["proj"][:, i * Dp:(i + 1) * Dp] if untie else st["proj"]
            G = _rows(S, Cpad, BF, dev)
            pn = torch.empty(S, dtype=torch.float32, device=dev)
            rvec = torch.empty(S, dtype=torch.float32, device=dev)
            part = torch.zeros(1, dtype=torch.float64, device=dev)
            correct = torch.zeros(1, dtype=torch.int32, device=dev)
            ops.nce_ce(proj_i, Dt, Dp, se["zraw"], Cpad, targets[i], S, C, Cpad, model.logit_temp, weight, G, Cpad, pn, rvec, part, correct)
            loss_sum += part
            stats.append(dict(loss=part, correct=correct, count=S))
            se["zraw"] = None
            Gs.append(G); pns.append(pn); rvecs.append(rvec)
        ctx.idx, ctx.st, ctx.grads = idx, st, (Gs, pns, rvecs)
        ctx.save_for_backward(w, b, label_embs)
        return loss_sum.float().reshape(())

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dloss):
        w, b, label_embs = ctx.saved_tensors
        Gs, pns, rvecs = ctx.grads
        scale_bf, scale_f = dloss.to(BF), dloss.float()
        for G, rvec in zip(Gs, rvecs):
            G.mul_(scale_bf)     # upstream gradient of the scalar loss (device scalar, no sync): everything below is linear in G
            rvec.mul_(scale_f)
        dx = _head_backward(ctx.st, label_embs, ctx.idx, Gs, pns, rvecs, ctx.grad_views)
        ctx.st = ctx.grads = None
        return dx, None, None, None, None, None, None, None, None, None


class _LogitsFn(torch.autograd.Function):
    """Opt-in MATERIALISING path of the head: the `[S, C+1]` float logit lists of the reference (`compute_nce`,
    src/fairseq/models/wavlm/wavlm.py:426-438: column 0 = the positive, column 1 + c = class c, -inf where the class IS the
    positive), differentiable, so that the reference's own `WavLMCriterion.get_loss` (wavlm_criterion.py:52-103) can drive this
    model through `get_logits` / `get_targets`.  Same GEMMs as the fused criterion; the logits are assembled from their outputs."""

    @staticmethod
    def forward(ctx, x2d, w, b, label_embs, model, idx, targets, grads):
        ctx.fwd_stream = torch.cuda.current_stream()
        ctx.grad_views = grads
        st = _head_forward(model, x2d, w, b, label_embs, idx)
        Dp, untie = model.final_dim, model.untie_final_proj
        outs, pns = [], []
        for i, se in enumerate(st["sets"]):
            C = se["C"]
            proj_i = st["proj"][:, i * Dp:(i + 1) * Dp] if untie else st["proj"]
            pn = 1.0 / proj_i.float().norm(dim=-1).clamp_min(1e-8)                 # torch.cosine_similarity clamps each norm
            z = se["zraw"][:, :C].float() * (pn / model.logit_temp).unsqueeze(1)   # cos(proj_s, E_c) / temp
            t = targets[i].long().unsqueeze(1)
            pos = z.gather(1, t)
            outs.append(torch.cat([pos, z.scatter(1, t, float("-inf"))], dim=1))
            pns.append(pn)
        ctx.model, ctx.idx, ctx.st, ctx.pns, ctx.targets = model, idx, st, pns, targets
        ctx.save_for_backward(w, b, label_embs)
        return tuple(outs)

    @staticmethod
    @_on_forward_stream
    def backward(ctx, *dlogits):
        w, b, label_embs = ctx.saved_tensors
        model, st = ctx.model, ctx.st
        dev = st["xs"].device
        S = ctx.idx.numel()
        Gs, rvecs = [], []
        for i, se in enumerate(st["sets"]):
            C, Cpad = se["C"], se["Cpad"]
            dl = dlogits[i].float() if dlogits[i] is not None else torch.zeros(S, C + 1, device=dev)
            t = ctx.targets[i].long().unsqueeze(1)
            dz = dl[:, 1:].scatter(1, t, 0.0)            # the -inf entry receives no gradient ...
            dz.scatter_add_(1, t, dl[:, :1])             # ... the positive's gradient lands on its class column
            zs = (ctx.pns[i] / model.logit_temp).unsqueeze(1)
            Gf = dz * zs                                 # d / d (proj . En^T)
            cosv = se["zraw"][:, :C].float() * ctx.pns[i].unsqueeze(1)
            rvecs.append((Gf * cosv).sum(1).contiguous())
            G = torch.zeros(S, Cpad, dtype=BF, device=dev)
            G[:, :C] = Gf.to(BF)
            Gs.append(G)
        dx = _head_backward(st, label_embs, ctx.idx, Gs, ctx.pns, rvecs, ctx.grad_views)
        ctx.st = None
        return dx, None, None, None, None, None, None, None


class WavLMForPretraining(WavLM):
    """`WavLM` + `final_proj` / `label_embs_concat` (same state_dict keys as the fairseq model) and the fused criterion."""

    def __init__(self, cfg: WavLMPretrainConfig, num_classes: List[int]):
        super().__init__(cfg)
        self._want_features_pen = True
        if cfg.target_glu:
            raise NotImplementedError("target_glu is not implemented in the fused masked-prediction head")
        D = cfg.encoder_embed_dim
        self.final_dim = cfg.final_dim if cfg.final_dim > 0 else D
        assert self.final_dim % 64 == 0, "final_dim must be a multiple of 64"
        self.num_classes = [int(c) for c in num_classes]
        assert all(0 < c <= 1024 for c in self.num_classes), "label sets of 1..1024 classes are supported"
        self.untie_final_proj = bool(cfg.untie_final_proj)
        self.logit_temp = float(cfg.logit_temp)
        self.skip_masked, self.skip_nomask = bool(cfg.skip_masked), bool(cfg.skip_nomask)
        self.feat2tar_ratio = cfg.label_rate * 320 / cfg.sample_rate  # label_rate * feature_ds_rate / sample_rate, wavlm.py:277-279
        self.final_proj = nn.Linear(D, self.final_dim * (len(self.num_classes) if self.untie_final_proj else 1))
        self.label_embs_concat = nn.Parameter(torch.empty(sum(self.num_classes), self.final_dim))
        nn.init.uniform_(self.label_embs_concat)  # wavlm.py:345

    # ---- reference helpers
    def forward_targets(self, T: int, target_list: List[torch.Tensor]) -> List[torch.Tensor]:
        """Label sub-sampling of wavlm.py:440-451 (features are never trimmed here: the labels must cover every frame)."""
        targ_tsz = min(t.size(1) for t in target_list)
        if self.feat2tar_ratio * T > targ_tsz:
            raise NotImplementedError(f"labels ({targ_tsz} per utterance) are shorter than the {T} feature frames: trimming the "
                                      "features is not implemented")
        inds = (torch.arange(T).float() * self.feat2tar_ratio).long()
        return [t[:, inds.to(t.device)] for t in target_list]

    def label_frames(self, L: int, target_list: List[torch.Tensor]) -> int:
        """Frames the model runs on for waveforms of L samples: the conv frame count T, or int(targ_tsz / feat2tar_ratio) when the
        shortest label sequence does not cover T frames (the feature trimming of wavlm.py:440-451 / fairseq HubertModel: at
        label_rate 100 the 100 Hz labels of an utterance are one short whenever (L - 400) mod 320 < 160)."""
        from .engine import ConvGeom
        T = ConvGeom(self.conv_cfg, L).T[-1]
        targ_tsz = min(t.size(1) for t in target_list)
        if self.feat2tar_ratio * T > targ_tsz:
            T = int(targ_tsz / self.feat2tar_ratio)
            if T <= 0:
                raise ValueError(f"labels of {targ_tsz} frames leave no feature frame at feat2tar_ratio {self.feat2tar_ratio}")
        return T

    def remove_pretraining_modules(self):
        self.final_proj = None
        self.label_embs_concat = None

    # ---- BaseFairseqModel surface the trainer / criterion touch (src/fairseq/models/fairseq_model.py:102-158, wavlm.py:599-627)
    def set_num_updates(self, num_updates: int):
        self.num_updates = num_updates

    def upgrade_state_dict_named(self, state_dict, name):
        return state_dict

    def get_extra_losses(self, net_output):
        """(losses, names) exactly as wavlm.py:611-620: the feature penalty when the forward pass produced it."""
        extra_losses, names = [], []
        if net_output.get("features_pen") is not None:
            extra_losses.append(net_output["features_pen"])
            names.append("features_pen")
        return extra_losses, names

    # ---- frame selection (host), shared by the criterion and the materialising logits path
    @staticmethod
    def _host_masks(out):
        """Host copies of the span mask and the frame padding mask of a forward result.  Frames are selected on the host, like
        the reference's collater-side masks: with a host padding mask there is no device round trip at all (a device-only mask
        costs one synchronising copy here)."""
        mi_h = out["mask_indices"].cpu()
        pm, pm_h = out["padding_mask"], out.get("padding_mask_host")
        if pm_h is None:
            pm_h = torch.zeros(mi_h.shape, dtype=torch.bool) if pm is None else pm.cpu()
        return mi_h, pm_h

    def _plans(self, net_output, pred_masked_weight, pred_nomask_weight):
        """(tag, host frame selection, weight) of the masked ("m") and unmasked ("u") terms that are switched on."""
        assert net_output["mask_indices"] is not None and net_output["target_list"] is not None, \
            "forward(..., target_list=..., mask=True) must run first"
        mi_h, pm_h = self._host_masks(net_output)
        plans = []
        if not self.skip_masked and pred_masked_weight > 0:
            plans.append(("m", torch.logical_and(~pm_h, mi_h), pred_masked_weight))
        if not self.skip_nomask and pred_nomask_weight > 0:
            plans.append(("u", torch.logical_and(~pm_h, ~mi_h), pred_nomask_weight))
        return plans

    @staticmethod
    def _select(sel, targets, dev):
        """Flat indices of the selected frames (host, and int32 on the device) and their labels (int32, device)."""
        idx_h = torch.nonzero(sel.reshape(-1), as_tuple=False).squeeze(1)
        idx = idx_h.to(torch.int32).to(dev, non_blocking=True)
        tg = [t.reshape(-1).to(dev)[idx.long()].to(torch.int32).contiguous() if t.device.type != "cpu"
              else t.reshape(-1)[idx_h].to(torch.int32).to(dev, non_blocking=True) for t in targets]
        return idx_h, idx, tg

    def _heads(self, net_output):
        """Each masked-prediction head: (bf16 [B*T, D] rows it reads, final_proj weight, bias, label embeddings, the fp32 gradient
        views of those three, weight of its loss or None).  One head here, on the encoder output."""
        g = self._engine.g
        fp, emb = self.final_proj, self.label_embs_concat
        x = net_output["x"]
        yield H.bf16(x.reshape(-1, x.shape[-1])), fp.weight, fp.bias, emb, (g(emb), g(fp.weight), g(fp.bias)), None

    def get_logits(self, net_output, is_masked=True):
        """`[S, C+1]` float logit list of the reference (wavlm.py:599-607), one per head and label set (head-major), positives in
        column 0.  Opt-in materialising path (the fused `criterion` never builds these); differentiable, cached in `net_output`."""
        key = "logit_m_list" if is_masked else "logit_u_list"
        if net_output.get(key) is None:
            plans = self._plans(net_output, float(is_masked), float(not is_masked))
            idx_h, idx, tg = self._select(plans[0][1], net_output["target_list"], net_output["x"].device) if plans else (None,) * 3
            lst = []
            for x2d, w, b, emb, grads, _ in self._heads(net_output):
                lst += (_LogitsFn.apply(x2d, w, b, emb, self, idx, tg, grads) if idx_h is not None and idx_h.numel()
                        else [None] * len(self.num_classes))
            net_output[key] = lst
        return [lg.float() for lg in net_output[key] if lg is not None]

    def get_targets(self, net_output, is_masked=True):
        """All-zero class indices: the positive sits in column 0 (wavlm.py:608-610)."""
        return [lg.new_zeros(lg.size(0), dtype=torch.long) for lg in self.get_logits(net_output, is_masked)]

    def forward(self, source, target_list=None, padding_mask=None, mask=True, features_only=False, output_layer=None,
                mask_indices=None, mask_channel_indices=None):
        """fairseq WavLMModel.forward.  With `features_only=False` the result carries everything the criterion needs
        (`x`, `padding_mask`, `mask_indices`, the frame-aligned `target_list`, `features_pen`); logits are never materialised.
        Labels shorter than the conv frames trim the features first (`label_frames`): everything after the conv stack, the
        feature penalty included, runs on the kept frames, and the trimmed frames get a zero gradient."""
        return self._forward(source, target_list, padding_mask, mask, features_only, output_layer, mask_indices,
                             mask_channel_indices)[0]

    def _forward(self, source, target_list, padding_mask, mask, features_only, output_layer, mask_indices, mask_channel_indices):
        """`forward`, and the full result dict of the extraction call it made (for the subclasses' loss heads): (out, res)."""
        frames = self.label_frames(source.shape[1], target_list) if target_list is not None and not features_only else None
        res = self._extract(source, padding_mask, mask, False, output_layer, mask_indices, mask_channel_indices, frames)
        out = {"x": res["x"], "padding_mask": res["padding_mask"], "features": res["features"],
               "layer_results": res["layer_results"]}
        if features_only:
            return out, res
        T = res["x"].shape[1]
        out["mask_indices"] = res["mask_indices"]
        out["padding_mask_host"] = res["padding_mask_host"]  # host copy of the frame mask when the caller's mask was on the host
        out["target_list"] = self.forward_targets(T, target_list) if target_list is not None else None
        out["features_pen"] = res["features_pen"]  # mean(features^2) after GradMultiply, wavlm.py:477-484 (kernel, inside _ConvFn)
        return out, res

    def criterion(self, net_output: Dict, pred_masked_weight: float = 1.0, pred_nomask_weight: float = 0.0,
                  loss_weights: Optional[List[float]] = None):
        """WavLMCriterion.get_loss (wavlm_criterion.py:52-138; for several heads HubertCriterion.get_loss over the head-major list,
        hubert_criterion.py:52-110): returns (loss, sample_size, logging_output) with `loss` a device scalar; logging values stay
        device tensors (call `.item()` when you log)."""
        x = net_output["x"]
        loss, sample_size, log = 0.0, 0, {}
        plans = self._plans(net_output, pred_masked_weight, pred_nomask_weight)
        heads = list(self._heads(net_output))
        for tag, sel, wgt in plans:
            idx_h, idx, tg = self._select(sel, net_output["target_list"], x.device)
            if idx_h.numel() == 0:
                continue
            k = 0
            for x2d, w, b, emb, grads, lw in heads:
                stats = []
                part = _MaskedPredictionFn.apply(x2d, w, b, emb, self, idx, tg, float(wgt), stats, grads)
                loss = loss + (part if lw is None else lw * part)
                for st in stats:
                    log[f"loss_{tag}_{k}"] = st["loss"] / wgt
                    log[f"correct_{tag}_{k}"] = st["correct"]
                    log[f"count_{tag}_{k}"] = st["count"]
                    k += 1
            sample_size += idx_h.numel()   # once per plan, whatever the number of heads (hubert_criterion.py:75, 91)
        if loss_weights is not None:  # every extra loss the model reports, weight x value x sample_size
            extra_losses, names = self.get_extra_losses(net_output)
            for i, p in H.weighted_extra_losses(extra_losses, loss_weights, sample_size):
                loss = loss + p
                log[f"loss_{names[i]}"] = p.detach()
        log.update(ntokens=sample_size, sample_size=sample_size, nsentences=x.shape[0])
        log["loss"] = loss.detach() if torch.is_tensor(loss) else loss
        return loss, sample_size, log
