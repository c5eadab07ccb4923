"""Synthetic workloads of BASELINE.json (model configurations, per-GPU batches, algorithmic flop counts) for bench.py and the
examples: product-side, so the benchmark builds what it times without the CPU checker.

Configurations: `WavLM/README.md` model table / the released checkpoints' cfg (SURVEY.md section 8): WavLM-Base = 12 x 768 / 3072 /
12 heads, post-LN, GroupNorm extractor; WavLM-Large = 24 x 1024 / 4096 / 16 heads, pre-LN, LayerNorm extractor, normalised
input; both with the gated relative-position bias (320 buckets, max distance 800).
"""
from __future__ import annotations

from typing import Dict, Tuple

SR = 16000

_COMMON = dict(
    extractor_mode="default", encoder_layers=12, encoder_embed_dim=768, encoder_ffn_embed_dim=3072, encoder_attention_heads=12,
    activation_fn="gelu", layer_norm_first=False, conv_feature_layers="[(512,10,5)] + [(512,3,2)] * 4 + [(512,2,2)] * 2",
    conv_bias=False, feature_grad_mult=1.0, normalize=False, dropout=0.0, attention_dropout=0.0, activation_dropout=0.0,
    encoder_layerdrop=0.0, dropout_input=0.0, dropout_features=0.0, mask_length=10, mask_prob=0.65, mask_selection="static",
    mask_other=0, no_mask_overlap=False, mask_min_space=1, mask_channel_length=10, mask_channel_prob=0.0,
    mask_channel_selection="static", mask_channel_other=0, no_mask_channel_overlap=False, mask_channel_min_space=1, conv_pos=128,
    conv_pos_groups=16, relative_position_embedding=True, num_buckets=320, max_distance=800, gru_rel_pos=True,
)

_MODELS: Dict[str, Tuple[dict, int, int]] = {
    # name -> (config overrides, utterances per GPU, seconds per utterance)   BASELINE.json configs[1] / configs[2]
    "base": (dict(), 16, 15),
    "large": (dict(extractor_mode="layer_norm", encoder_layers=24, encoder_embed_dim=1024, encoder_ffn_embed_dim=4096,
                   encoder_attention_heads=16, layer_norm_first=True, normalize=True), 8, 20),
    # XLS-R 1B / MMS-1B (HuBERT X-Large has the same encoder shape): head width 80, pos_conv groups of 80 channels, no
    # relative-position bias, conv biases in the extractor
    "xlsr1b": (dict(extractor_mode="layer_norm", encoder_layers=48, encoder_embed_dim=1280, encoder_ffn_embed_dim=5120,
                    encoder_attention_heads=16, layer_norm_first=True, normalize=True, conv_bias=True,
                    relative_position_embedding=False, gru_rel_pos=False), 8, 20),
    # XLS-R 2B: head width 120, pos_conv groups of 120 channels, otherwise as xlsr1b.  8 x 20 s per GPU fits one 80 GB card:
    # the fine-tuning step peaks at 64.6 GiB allocated (tools/bench_wide.py --workload xlsr2b, H100 80GB HBM3)
    "xlsr2b": (dict(extractor_mode="layer_norm", encoder_layers=48, encoder_embed_dim=1920, encoder_ffn_embed_dim=7680,
                    encoder_attention_heads=16, layer_norm_first=True, normalize=True, conv_bias=True,
                    relative_position_embedding=False, gru_rel_pos=False), 8, 20),
    "tiny": (dict(encoder_layers=2, encoder_embed_dim=128, encoder_ffn_embed_dim=256, encoder_attention_heads=2,
                  conv_feature_layers="[(64,10,5)] + [(64,3,2)] * 4 + [(64,2,2)] * 2"), 4, 2),
}


def model_config(name: str) -> Tuple[dict, int, int]:
    """(WavLMConfig fields, utterances per GPU, seconds per utterance) of a named workload."""
    over, B, secs = _MODELS[name]
    return dict(_COMMON, **over), B, secs


def num_frames(L: int, cfg: dict) -> int:
    for (_, k, s) in eval(cfg["conv_feature_layers"]):
        L = (L - k) // s + 1
    return L


def forward_flops(L: int, cfg: dict) -> float:
    """Algorithmic GEMM flops of one forward pass of one utterance of L samples (SURVEY.md section 8d):
    sum_l 2 T_l 512 Cin_l k_l + 2 T 512 D + 2 T D (D/16) 128 + N (8 T D^2 + 4 T^2 D + 4 T D F + 2 T H (D/H) 8); a step is 3x this."""
    D, Fd, H = cfg["encoder_embed_dim"], cfg["encoder_ffn_embed_dim"], cfg["encoder_attention_heads"]
    fl, cin, t = 0.0, 1, L
    for (dim, k, s) in eval(cfg["conv_feature_layers"]):
        t = (t - k) // s + 1
        fl += 2.0 * t * dim * cin * k
        cin = dim
    T = t
    fl += 2.0 * T * cin * D
    fl += 2.0 * T * D * (D // cfg["conv_pos_groups"]) * cfg["conv_pos"]
    fl += cfg["encoder_layers"] * (8.0 * T * D * D + 4.0 * T * T * D + 4.0 * T * D * Fd + 2.0 * T * H * (D // H) * 8)
    return fl
