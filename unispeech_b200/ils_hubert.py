"""ILS-HuBERT (intermediate layer supervision) on the same kernels -- SURVEY.md section 8f row 4.

Mirrors `ILSHubertModel` (src/fairseq/models/hubert/ils_hubert.py:58-330):
  * `predict_layers` (1-based): the encoder returns the outputs of these layers (`layer=self.predict_layers`, :167-171; no final
    encoder LayerNorm then), pre-LN models normalise each with its own `post_layer_norm[i]` (:187-188);
  * every predicted layer gets the masked-prediction head of HuBERT (:190-270): `final_proj` is shared or, with
    `separate_label_embeds`, an `nn.Sequential` of one Linear per layer; `label_embs_concat` is `[layer_dim, sum(C), final_dim]`
    with `layer_dim = len(predict_layers)` when the label embeddings are separate, else 1;
  * the logit list is layer-major (`logit_m_list`: for each layer, for each label set), and `HubertCriterion.get_loss`
    (src/fairseq/criterions/hubert_criterion.py:52-110) sums the cross entropies of ALL entries (optionally weighted by
    `softmax(weights)` per layer, `weighted_sum`) while `sample_size` counts the selected frames ONCE.
State_dict keys are the reference's (`post_layer_norm.{i}.*`, `final_proj.{i}.*` or `final_proj.*`, `label_embs_concat`, `weights`).
Each head is the fused head of pretrain.py (gather -> final_proj GEMM -> cosine logits GEMM -> softmax / CE kernel), attached to
the layer output it supervises: autograd adds its input gradient to the one arriving from the layers above.
`separate_layer_targets` (one label set per layer) is not built.
"""
from __future__ import annotations

from typing import Dict, List, Optional

import torch
import torch.nn as nn

from .engine import BF
from .hubert import HubertConfig
from .pretrain import WavLMForPretraining, _LogitsFn, _MaskedPredictionFn
from .wavlm import _LNFn


class ILSHubertConfig(HubertConfig):
    """HubertConfig + the ILS fields (ils_hubert.py:27-55); the bucketed relative position bias of that config is allowed."""

    def __init__(self, cfg=None):
        self.predict_layers = "[12]"
        self.separate_label_embeds = False
        self.separate_layer_targets = False
        self.weighted_sum = False
        super().__init__(None)
        if cfg is not None:
            self.update(cfg)


class ILSHubertModel(WavLMForPretraining):
    def __init__(self, cfg: ILSHubertConfig, num_classes: List[int]):
        super().__init__(cfg, num_classes)
        if getattr(cfg, "separate_layer_targets", False):
            raise NotImplementedError("separate_layer_targets (one label set per predicted layer) is not implemented")
        pl = cfg.predict_layers
        self.predict_layers = [int(v) for v in (eval(pl) if isinstance(pl, str) else pl)]
        n = len(self.predict_layers)
        assert n >= 1 and all(1 <= v <= cfg.encoder_layers for v in self.predict_layers), self.predict_layers
        assert self.predict_layers == sorted(self.predict_layers), "predict_layers must be increasing (the encoder collects them in order)"
        self._predict_layers = self.predict_layers          # read by WavLM.extract_features
        self.separate_label_embeds = bool(cfg.separate_label_embeds)
        self.weighted_sum = bool(cfg.weighted_sum)
        D = cfg.encoder_embed_dim
        self.layer_norm_first = bool(cfg.layer_norm_first)
        if self.layer_norm_first:
            self.post_layer_norm = nn.Sequential(*[nn.LayerNorm(D) for _ in range(n)])
        out_dim = self.final_dim * (len(self.num_classes) if self.untie_final_proj else 1)
        if self.separate_label_embeds:
            self.final_proj = nn.Sequential(*[nn.Linear(D, out_dim) for _ in range(n)])
        else:
            self.final_proj = nn.Linear(D, out_dim)
        layer_dim = n if self.separate_label_embeds else 1
        self.label_embs_concat = nn.Parameter(torch.empty(layer_dim, sum(self.num_classes), self.final_dim))
        nn.init.uniform_(self.label_embs_concat)
        if self.weighted_sum:
            self.weights = nn.Parameter(torch.zeros(n))

    # ---- per-layer head parameters and their gradient views
    def _head_params(self, i: int):
        fp = self.final_proj[i] if self.separate_label_embeds else self.final_proj
        j = i if self.separate_label_embeds else 0
        g = self._engine.g
        grads = (g(self.label_embs_concat)[j], g(fp.weight), g(fp.bias))
        return fp.weight, fp.bias, self.label_embs_concat[j], grads

    def remove_pretraining_modules(self):
        self.final_proj = None
        self.label_embs_concat = None

    def forward(self, source, target_list=None, padding_mask=None, mask=True, features_only=False, output_layer=None,
                mask_indices=None, mask_channel_indices=None):
        out = super().forward(source, target_list=target_list, padding_mask=padding_mask, mask=mask, features_only=features_only,
                              output_layer=output_layer, mask_indices=mask_indices, mask_channel_indices=mask_channel_indices)
        eng = self._engine
        if features_only:
            if self.layer_norm_first and output_layer is not None:   # ils_hubert.py:176-178
                x = out["x"]
                xb = x if (x.dtype == BF and x.is_contiguous()) else x.to(BF).contiguous()
                out["x"] = _LNFn.apply(xb, eng, self.post_layer_norm[-1])
            return out
        lrs = [h.transpose(0, 1) for h, _ in out["layer_results"]]      # T x B x C -> B x T x C
        assert len(lrs) == len(self.predict_layers), (len(lrs), self.predict_layers)
        if self.layer_norm_first:
            normed = []
            for h, ln in zip(lrs, self.post_layer_norm):
                hb = h if (h.dtype == BF and h.is_contiguous()) else h.to(BF).contiguous()
                normed.append(_LNFn.apply(hb, eng, ln))
            lrs = normed
        out["ils_layers"] = lrs
        return out

    # ---- frame selection (host), shared by the criterion and the materialising logits path
    def _plans(self, net_output, pred_masked_weight, pred_nomask_weight):
        x = net_output["x"]
        B, T, _ = x.shape
        mi, pm = net_output["mask_indices"], net_output["padding_mask"]
        assert mi is not None and net_output["target_list"] is not None, "forward(..., target_list=..., mask=True) must run first"
        mi_h = mi.cpu() if mi.device.type != "cpu" else mi
        pm_h = net_output.get("padding_mask_host")
        if pm_h is None:
            pm_h = torch.zeros(B, T, dtype=torch.bool) if pm is None else (pm.cpu() if pm.device.type != "cpu" else pm)
        plans = []
        if not self.skip_masked and pred_masked_weight > 0:
            plans.append(("m", torch.logical_and(~pm_h, mi_h), pred_masked_weight))
        if not self.skip_nomask and pred_nomask_weight > 0:
            plans.append(("u", torch.logical_and(~pm_h, ~mi_h), pred_nomask_weight))
        return plans

    def _select(self, sel, targets, dev):
        idx_h = torch.nonzero(sel.reshape(-1), as_tuple=False).squeeze(1)
        idx = idx_h.to(torch.int32).to(dev, non_blocking=True)
        tg = [t.reshape(-1).to(dev)[idx.long()].to(torch.int32).contiguous() if t.device.type != "cpu"
              else t.reshape(-1)[idx_h].to(torch.int32).to(dev, non_blocking=True) for t in targets]
        return idx_h, idx, tg

    @staticmethod
    def _rows2d(h):
        h2 = h.reshape(-1, h.shape[-1])
        return h2 if (h2.dtype == BF and h2.is_contiguous()) else h2.to(BF).contiguous()

    def get_logits(self, net_output, is_masked=True):
        """Layer-major `[S, C+1]` float logit list (ils_hubert.py:213-272, 290-296); differentiable, cached in `net_output`."""
        key = "logit_m_list" if is_masked else "logit_u_list"
        if net_output.get(key) is None:
            skip = self.skip_masked if is_masked else self.skip_nomask
            mi_h = net_output["mask_indices"]
            mi_h = mi_h.cpu() if mi_h.device.type != "cpu" else mi_h
            plans = self._plans(net_output, 1.0 if is_masked else 0.0, 0.0 if is_masked else 1.0)
            lst = []
            if skip or not plans:
                lst = [None for _ in self.predict_layers for _ in self.num_classes]
            else:
                _, sel, _ = plans[0]
                idx_h, idx, tg = self._select(sel, net_output["target_list"], net_output["x"].device)
                for i, h in enumerate(net_output["ils_layers"]):
                    w, b, emb, grads = self._head_params(i)
                    lst += list(_LogitsFn.apply(self._rows2d(h), w, b, emb, self, idx, tg, grads)) if idx_h.numel() else \
                        [None for _ in self.num_classes]
            net_output[key] = lst
        return [lg.float() for lg in net_output[key] if lg is not None]

    def criterion(self, net_output: Dict, pred_masked_weight: float = 1.0, pred_nomask_weight: float = 0.0,
                  loss_weights: Optional[List[float]] = None):
        """HubertCriterion.get_loss over the layer-major logit list, fused: returns (loss, sample_size, logging_output)."""
        x = net_output["x"]
        B = x.shape[0]
        dev = x.device
        loss, sample_size, log = 0.0, 0, {}
        lw_layers = torch.softmax(self.weights, dim=-1) if self.weighted_sum else None
        for tag, sel, wgt in self._plans(net_output, pred_masked_weight, pred_nomask_weight):
            idx_h, idx, tg = self._select(sel, net_output["target_list"], dev)
            if idx_h.numel() == 0:
                continue
            k = 0
            for i, h in enumerate(net_output["ils_layers"]):
                w, b, emb, grads = self._head_params(i)
                stats = []
                part = _MaskedPredictionFn.apply(self._rows2d(h), w, b, emb, self, idx, tg, float(wgt), stats, grads)
                loss = loss + (part if lw_layers is None else lw_layers[i] * part)
                for st in stats:
                    log[f"loss_{tag}_{k}"] = st["loss"] / wgt
                    log[f"correct_{tag}_{k}"] = st["correct"]
                    log[f"count_{tag}_{k}"] = st["count"]
                    k += 1
            sample_size += idx_h.numel()       # once per plan, whatever the number of layers (hubert_criterion.py:75, 91)
        if loss_weights is not None:
            extra_losses, names = self.get_extra_losses(net_output)
            lw = list(loss_weights)
            if len(lw) == 1 and len(extra_losses) != 1:
                lw = [lw[0]] * len(extra_losses)
            assert len(extra_losses) == len(lw), f"{len(extra_losses)}, {len(lw)}"
            for p, n, coef in zip(extra_losses, names, lw):
                if coef != 0 and p is not None:
                    p = coef * p.float() * sample_size
                    loss = loss + p
                    log[f"loss_{n}"] = p.detach()
        log.update(ntokens=sample_size, sample_size=sample_size, nsentences=B)
        log["loss"] = loss.detach() if torch.is_tensor(loss) else loss
        return loss, sample_size, log
