"""Head widths the kernels do not take are refused: at model construction with NotImplementedError, and by every attention
entry point with an error (the argument checks run before any device work, so no GPU is needed)."""
import pytest

from oracle import wavlm_oracle as O


def _cfg(**kw):
    from unispeech_b200.wavlm import WavLMConfig
    cfg = vars(O.tiny_config(pre_ln=True))
    cfg.update(kw)
    return WavLMConfig(cfg)


@pytest.mark.parametrize("kw,msg", [
    (dict(encoder_embed_dim=192, encoder_attention_heads=2, relative_position_embedding=False), "head width"),   # 96
    (dict(encoder_embed_dim=160, encoder_attention_heads=2, relative_position_embedding=True, conv_pos_groups=4),
     "relative_position_embedding"),
    (dict(encoder_embed_dim=1280, encoder_attention_heads=16, relative_position_embedding=False, conv_pos_groups=8),
     "pos_conv groups"),   # 160 channels per group, head width 80
])
def test_construction_rejects(kw, msg):
    from unispeech_b200.wavlm import WavLM, _check_supported
    cfg = _cfg(**kw)
    assert any(msg in b for b in _check_supported(cfg))
    with pytest.raises(NotImplementedError, match=msg):
        WavLM(cfg)


def test_head_width_80_accepted():
    from unispeech_b200.wavlm import _check_supported
    assert _check_supported(_cfg(encoder_embed_dim=160, encoder_attention_heads=2, relative_position_embedding=False,
                                 conv_pos_groups=4)) == []


def test_entry_points_reject_head_dim_72():
    from unispeech_b200 import _lib as L
    lib = L.load()
    fake = 256   # never dereferenced: the head_dim check returns first
    B, T, H, scale, hd = 1, 8, 2, 72 ** -0.5, 72
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
        assert b"head_dim=72" in lib.b200s_last_error(), name
