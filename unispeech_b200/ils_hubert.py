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

from typing import List

import torch
import torch.nn as nn

from . import heads as H
from .hubert import HubertConfig
from .pretrain import WavLMForPretraining
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

    def forward(self, source, target_list=None, padding_mask=None, mask=True, features_only=False, output_layer=None,
                mask_indices=None, mask_channel_indices=None):
        out = super().forward(source, target_list=target_list, padding_mask=padding_mask, mask=mask, features_only=features_only,
                              output_layer=output_layer, mask_indices=mask_indices, mask_channel_indices=mask_channel_indices)
        eng = self._engine
        if features_only:
            if self.layer_norm_first and output_layer is not None:   # ils_hubert.py:176-178
                out["x"] = _LNFn.apply(H.bf16(out["x"]), eng, self.post_layer_norm[-1])
            return out
        lrs = [h.transpose(0, 1) for h, _ in out["layer_results"]]      # T x B x C -> B x T x C
        assert len(lrs) == len(self.predict_layers), (len(lrs), self.predict_layers)
        if self.layer_norm_first:
            lrs = [_LNFn.apply(H.bf16(h), eng, ln) for h, ln in zip(lrs, self.post_layer_norm)]
        out["ils_layers"] = lrs
        return out

    def _heads(self, net_output):
        """One head per predicted layer (layer-major, ils_hubert.py:213-272), each weighted by softmax(weights) with
        `weighted_sum`."""
        g = self._engine.g
        lw = torch.softmax(self.weights, dim=-1) if self.weighted_sum else None
        for i, h in enumerate(net_output["ils_layers"]):
            fp = self.final_proj[i] if self.separate_label_embeds else self.final_proj
            j = i if self.separate_label_embeds else 0
            yield (H.bf16(h.reshape(-1, h.shape[-1])), fp.weight, fp.bias, self.label_embs_concat[j],
                   (g(self.label_embs_concat)[j], g(fp.weight), g(fp.bias)), None if lw is None else lw[i])
