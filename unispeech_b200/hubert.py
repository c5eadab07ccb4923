"""HuBERT on the same kernels (SURVEY.md section 8f row 4).

The fairseq `HubertModel` (src/fairseq/models/hubert/hubert.py:234-310: `feature_extractor`, `post_extract_proj`, `mask_emb`,
wav2vec2's `TransformerEncoder`, `layer_norm`, `final_proj`, `label_embs_concat`) is the WavLM pre-training model without the
gated relative-position bias: identical module tree and state_dict keys minus `relative_attention_bias`, `grep_linear` and
`grep_a`.  The attention kernels take `tab = NULL` for it (tests: the `relative_position_embedding=False` golden fixture of
tests/test_model_gpu.py and the dropout / pre-training cases built on that configuration).
"""
from __future__ import annotations

from typing import List

from .pretrain import WavLMForPretraining, WavLMPretrainConfig


class HubertConfig(WavLMPretrainConfig):
    def __init__(self, cfg=None):
        super().__init__(cfg)
        self.relative_position_embedding = False
        self.gru_rel_pos = False


class HubertModel(WavLMForPretraining):
    """`HubertModel.forward(source, target_list, padding_mask, mask, features_only, output_layer)` and the masked-prediction
    criterion (src/fairseq/criterions/hubert_criterion.py has the same get_loss as wavlm_criterion.py) on the project's kernels."""

    def __init__(self, cfg: HubertConfig, num_classes: List[int]):
        if getattr(cfg, "relative_position_embedding", False) or getattr(cfg, "gru_rel_pos", False):
            raise ValueError("HuBERT has no relative position bias: use WavLMForPretraining for configurations that enable it")
        super().__init__(cfg, num_classes)
