"""Host side of channel masking (no GPU): the masks the models draw from numpy's global RNG are the reference's two
compute_mask_indices calls in the reference's order (apply_mask, WavLM/WavLM.py:271-309: the span mask over (B, T) with min_masks 2,
then the channel mask over (B, encoder_embed_dim) with no padding mask and min_masks 0)."""
import numpy as np
import pytest
import torch

from oracle import wavlm_oracle as O


def _reference_draws(seed, B, T, D, cfg, fpm):
    from unispeech_b200.masking import compute_mask_indices
    np.random.seed(seed)
    mi = compute_mask_indices((B, T), fpm, cfg.mask_prob, cfg.mask_length, cfg.mask_selection, cfg.mask_other, min_masks=2,
                              no_overlap=cfg.no_mask_overlap, min_space=cfg.mask_min_space)
    ci = compute_mask_indices((B, D), None, cfg.mask_channel_prob, cfg.mask_channel_length, cfg.mask_channel_selection,
                              cfg.mask_channel_other, no_overlap=cfg.no_mask_channel_overlap, min_space=cfg.mask_channel_min_space)
    return torch.from_numpy(mi), torch.from_numpy(ci)


def _padding(B, L, lengths):
    pm = torch.zeros(B, L, dtype=torch.bool)
    for b, n in enumerate(lengths):
        pm[b, n:] = True
    return pm


@pytest.mark.parametrize("padded", [False, True])
@pytest.mark.parametrize("selection,no_overlap", [("static", False), ("uniform", True)])
def test_wavlm_draws_span_then_channel_mask(padded, selection, no_overlap):
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    cfg = O.tiny_config(mask_channel_prob=0.5, mask_channel_length=16, mask_channel_selection=selection, mask_channel_other=4,
                        no_mask_channel_overlap=no_overlap)
    m = WavLM(WavLMConfig(vars(cfg)))
    B, L = 3, 16000
    T, D = O.num_frames(L, cfg), cfg.encoder_embed_dim
    fpm = m.forward_padding_mask(T, _padding(B, L, [L, 12000, 9000])) if padded else None
    for seed in (0, 7, 1234):
        np.random.seed(seed)
        mi, ci = m.sample_masks(B, T, fpm)
        after = np.random.random()
        want_mi, want_ci = _reference_draws(seed, B, T, D, cfg, fpm)
        assert torch.equal(mi, want_mi) and torch.equal(ci, want_ci)
        assert np.random.random() == after            # and nothing else consumed from the global state
        assert ci.shape == (B, D) and ci.any()


def test_no_channel_draw_without_channel_prob():
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    cfg = O.tiny_config()
    m = WavLM(WavLMConfig(vars(cfg)))
    np.random.seed(3)
    mi, ci = m.sample_masks(2, 49, None)
    after = np.random.random()
    np.random.seed(3)
    assert torch.equal(mi, m.apply_mask(2, 49, None)) and ci is None
    assert np.random.random() == after


@pytest.mark.parametrize("padded", [False, True])
def test_sat_early_draws_reach_the_extraction_call_in_the_reference_order(monkeypatch, padded):
    """UniSpeech-SAT draws its masks before the encoder runs (for the instance-sampling helper thread): the channel draw must
    follow the span draw there, and both must reach the encoder."""
    from unispeech_b200.pretrain import WavLMForPretraining
    from unispeech_b200.unispeech_sat import UniSpeechSATConfig, UniSpeechSATForPretraining
    cfg = O.tiny_config(pre_ln=True, layer_norm_for_extract=True, relative_position_embedding=False, gru_rel_pos=False,
                        mask_channel_prob=0.5, mask_channel_length=16)
    scfg = UniSpeechSATConfig(dict(vars(cfg), final_dim=64, utterance_contrastive_layer=1, num_instances=3,
                                   cross_sample_instances=5))
    m = UniSpeechSATForPretraining(scfg, [30])
    seen = {}

    class _Stop(Exception):
        pass

    def fake_forward(self, source, **kw):
        seen.update(kw)
        raise _Stop

    monkeypatch.setattr(WavLMForPretraining, "_forward", fake_forward)
    B, L = 2, 16000
    T, D = O.num_frames(L, cfg), cfg.encoder_embed_dim
    pm = _padding(B, L, [L, 11000]) if padded else None
    np.random.seed(99)
    with pytest.raises(_Stop):
        m.forward(torch.zeros(B, L), padding_mask=pm, mask=True)
    want_mi, want_ci = _reference_draws(99, B, T, D, cfg, m.forward_padding_mask(T, pm) if padded else None)
    assert torch.equal(seen["mask_indices"], want_mi)
    assert torch.equal(seen["mask_channel_indices"], want_ci)


def test_channel_masking_is_a_supported_configuration():
    from unispeech_b200.wavlm import _check_supported, WavLMConfig
    cfg = WavLMConfig(vars(O.tiny_config(mask_channel_prob=0.5, mask_channel_length=64)))
    assert _check_supported(cfg) == []
