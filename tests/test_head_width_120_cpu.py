"""Head width 120 (XLS-R 2B: D = 1920, 16 heads, pos_conv groups of 120 channels) is accepted at model construction without the
relative-position bias and refused with it; the attention entry points still refuse head widths 72 and 96 (the argument checks
run before any device work, so no GPU is needed).  Width 120 itself runs in tests/test_attn_hd120_gpu.py."""
import pytest

from oracle import wavlm_oracle as O


def _cfg(**kw):
    from unispeech_b200.wavlm import WavLMConfig
    cfg = vars(O.tiny_config(pre_ln=True))
    cfg.update(dict(encoder_embed_dim=1920, encoder_ffn_embed_dim=7680, encoder_attention_heads=16, conv_pos_groups=16), **kw)
    return WavLMConfig(cfg)


def test_head_width_120_accepted():
    from unispeech_b200.wavlm import _check_supported
    assert _check_supported(_cfg(relative_position_embedding=False, gru_rel_pos=False)) == []


def test_head_width_120_rejects_bias():
    from unispeech_b200.wavlm import WavLM, _check_supported
    cfg = _cfg(relative_position_embedding=True)
    assert any("relative_position_embedding" in b for b in _check_supported(cfg))
    with pytest.raises(NotImplementedError, match="relative_position_embedding"):
        WavLM(cfg)


def test_xlsr2b_workload():
    from unispeech_b200 import workloads as W
    from unispeech_b200.wavlm import WavLMConfig, _check_supported
    cfg, B, secs = W.model_config("xlsr2b")
    assert (cfg["encoder_layers"], cfg["encoder_embed_dim"], cfg["encoder_ffn_embed_dim"], cfg["encoder_attention_heads"]) == \
        (48, 1920, 7680, 16)
    assert _check_supported(WavLMConfig(cfg)) == []


@pytest.mark.parametrize("hd", [72, 96])
def test_entry_points_reject_head_dim(hd):
    from unispeech_b200 import _lib as L
    lib = L.load()
    fake = 256   # never dereferenced: the head_dim check returns first
    B, T, H, scale = 1, 8, 2, hd ** -0.5
    calls = {
        "b200s_attn_fwd": (fake, 0, 0, 0, fake, fake, B, T, H, scale, hd, 0),
        "b200s_attn_fwd_dropout": (fake, 0, 0, 0, fake, fake, B, T, H, scale, 0.0, 0, 0, 0, hd, 0),
        "b200s_attn_bwd": (fake, fake, fake, 0, 0, 0, fake, fake, fake, 0, 0, B, T, H, scale, hd, 0),
        "b200s_attn_bwd_fused": (fake, fake, fake, 0, 0, 0, fake, fake, fake, fake, 0, 0, B, T, H, scale, hd, 0),
        "b200s_attn_bwd_fused_dropout": (fake, fake, fake, 0, 0, 0, fake, fake, fake, fake, 0, 0, B, T, H, scale, 0.0, 0, hd, 0),
    }
    for name, args in calls.items():
        rc = getattr(lib, name)(*args)
        assert rc != 0, name
        assert f"head_dim={hd}".encode() in lib.b200s_last_error(), name
