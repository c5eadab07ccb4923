"""Host side of `conv_bias=True` (no GPU): the reference's state_dict layout and the place of the bias gradients in the flat
gradient buffer."""
import pytest

from oracle import wavlm_oracle as O


CONFIGS = {
    "w2v_large_style": lambda: O.large_config(encoder_layers=2, conv_bias=True, relative_position_embedding=False,
                                              gru_rel_pos=False),
    "default_mode_bias": lambda: O.base_config(encoder_layers=2, conv_bias=True),
}


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_state_dict_matches_reference_layout_and_loads(name):
    from unispeech_b200.wavlm import WavLM, WavLMConfig, _check_supported
    cfg = CONFIGS[name]()
    wcfg = WavLMConfig(vars(cfg))
    assert _check_supported(wcfg) == []
    m = WavLM(wcfg)
    shapes = {k: tuple(v.shape) for k, v in m.state_dict().items()}
    assert shapes == O.parameter_shapes(cfg)
    m.load_state_dict(O.deterministic_state_dict(cfg), strict=True)


@pytest.mark.parametrize("name", sorted(CONFIGS))
def test_bias_gradients_are_views_into_the_conv_range(name):
    from unispeech_b200.engine import build_flat_grads
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    cfg = CONFIGS[name]()
    m = WavLM(WavLMConfig(vars(cfg)))
    flat, ranges, order = build_flat_grads(m, "cpu")
    assert order[-1] == "conv"
    c0, c1 = ranges["conv"]
    for i, blk in enumerate(m.feature_extractor.conv_layers):
        b = blk[0].bias
        off = flat.offsets[id(b)]
        assert c0 <= off and off + b.numel() <= c1, i
        v = flat.view(b)
        assert v.shape == b.shape and v.data_ptr() == flat.flat.data_ptr() + 4 * off
