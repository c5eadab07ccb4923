"""Host side of HuBERT's first iteration: the float64 MFCC oracle (oracle/mfcc_oracle.py) against the recipe's own call
(`torchaudio.compliance.kaldi.mfcc(x, sample_frequency=16000, use_energy=False)` + `compute_deltas` twice, fp32), the frame
count, and the label-driven feature trimming of the pre-training forward (frame count and T'-frame padding mask).

Tolerance: torchaudio runs in fp32, and its fp32 result differs from its own float64 run by up to 9.1e-5 on the speech fixture
(features up to 74); 5e-4 leaves room for that and for the oracle's different summation order, and is still far below what a
wrong constant moves: a window exponent of 0.8 instead of 0.85 moves the fixture's features by 1.2, and float64's log floor
(2.2e-16) instead of float32's moves those of digital silence by 96."""
import os

import numpy as np
import pytest
import torch

from oracle import mfcc_oracle as MO
from oracle import trim_oracle as TO
from oracle import wavlm_oracle as O

GOLD = os.path.join(os.path.dirname(__file__), "golden", "vox_real_large2l.npz")
TOL = 5e-4


def recipe_features(x: np.ndarray) -> np.ndarray:
    """dump_mfcc_feature.py's MfccFeatureReader.get_feats, fp32 (the recipe's dtype)."""
    ta = pytest.importorskip("torchaudio")
    wav = torch.from_numpy(np.asarray(x, np.float32)).view(1, -1)
    mfcc = ta.compliance.kaldi.mfcc(waveform=wav, sample_frequency=16000, use_energy=False)   # [Tm, 13]
    mfcc = mfcc.transpose(0, 1)
    delta = ta.functional.compute_deltas(mfcc)
    ddelta = ta.functional.compute_deltas(delta)
    return torch.cat([mfcc, delta, ddelta], dim=0).transpose(0, 1).contiguous().numpy()


def _vox():
    g = np.load(GOLD)
    return [g["pcm"][b, :int(n)].astype(np.float64) / 32768.0 for b, n in enumerate(g["lengths"])]


def test_oracle_matches_recipe_on_real_speech():
    worst = 0.0
    for x in _vox():
        want = recipe_features(x)
        got = MO.mfcc39(x)
        assert got.shape == want.shape == (MO.num_frames(len(x)), 39)
        worst = max(worst, float(np.abs(got - want).max()))
    assert worst <= TOL, worst


def _edge_cases():
    rng = np.random.default_rng(7)
    speech = _vox()[0]
    t = np.arange(4000)
    return {
        "n400": rng.uniform(-0.5, 0.5, 400),
        "n559": speech[:559],
        "n560": speech[:560],
        "n723": speech[1000:1723],
        "dc_offset": speech[:8000] * 0.3 + 0.4,
        "silence": np.zeros(4000),
        "square_full_scale": np.where((t // 20) % 2 == 0, 1.0, -1.0),
    }


@pytest.mark.parametrize("case", list(_edge_cases()))
def test_oracle_matches_recipe_on_edge_cases(case):
    x = _edge_cases()[case]
    want, got = recipe_features(x), MO.mfcc39(x)
    assert got.shape == want.shape
    err = float(np.abs(got - want).max())
    assert err <= TOL, (case, err)


def test_single_frame_has_zero_deltas():
    got = MO.mfcc39(_vox()[1][:400])
    assert got.shape == (1, 39)
    assert np.all(got[:, 13:] == 0.0)
    assert np.abs(got - recipe_features(_vox()[1][:400])).max() <= TOL


def test_frame_count():
    for n in list(range(0, 2000, 7)) + [160_000, 160_160, 250_000]:
        want = 0 if n < 400 else int(np.floor((n - 400) / 160)) + 1
        assert MO.num_frames(n) == want
        if n >= 400:
            assert MO.mfcc39(np.zeros(n)).shape[0] == want
    from unispeech_b200.mfcc import num_frames
    assert all(num_frames(n) == MO.num_frames(n) for n in range(0, 3000))
    assert MO.mfcc39(np.zeros(399)).shape == (0, 39)


def _hubert(label_rate):
    from unispeech_b200.hubert import HubertConfig, HubertModel
    cfg = O.tiny_config(pre_ln=False, relative_position_embedding=False, gru_rel_pos=False)
    return HubertModel(HubertConfig(dict(vars(cfg), final_dim=64, label_rate=label_rate)), [100]), cfg


def test_trimmed_frame_count_matches_the_reference_rule():
    """label_rate 100: T conv frames against Tm = num_frames(L) labels; 2T = Tm + 1 (one label short) whenever
    (L - 400) mod 320 < 160, and the model then runs on T - 1 frames.  label_rate 50 with cropped labels trims to their count."""
    m, cfg = _hubert(100)
    short = 0
    for L in list(range(16000, 16 * 16000, 37)) + [160_000, 160_160, 250_000]:
        T, Tm = O.num_frames(L, cfg), MO.num_frames(L)
        want = TO.trimmed_frames(T, Tm, 2.0)
        assert m.label_frames(L, [torch.zeros(1, Tm)]) == want
        assert want == (T - 1 if (L - 400) % 320 < 160 else T)
        short += want < T
    assert short > 3000
    assert m.label_frames(250_000, [torch.zeros(1, 1561)]) == 780
    assert m.label_frames(160_160, [torch.zeros(1, MO.num_frames(160_160))]) == O.num_frames(160_160, cfg) - 1
    assert m.label_frames(160_000, [torch.zeros(1, MO.num_frames(160_000))]) == O.num_frames(160_000, cfg)
    m50, _ = _hubert(50)
    assert m50.label_frames(8000, [torch.zeros(1, 23), torch.zeros(1, 30)]) == 23
    assert m50.label_frames(8000, [torch.zeros(1, 30)]) == O.num_frames(8000, cfg)
    with pytest.raises(ValueError):
        m.label_frames(8000, [torch.zeros(1, 1)])
    # forward_targets itself is unchanged: it still refuses a T the labels do not cover
    with pytest.raises(NotImplementedError):
        m.forward_targets(O.num_frames(160_160, cfg), [torch.zeros(1, MO.num_frames(160_160))])


@pytest.mark.parametrize("L,lengths", [(160_160, [160_160, 97_000]), (250_000, [250_000, 123_457, 40_001])])
def test_trimmed_padding_mask_matches_the_reference(L, lengths):
    """forward_padding_mask on T' frames chunks the L samples by L // T' (not by the conv stride), as the reference does."""
    m, cfg = _hubert(100)
    T2 = m.label_frames(L, [torch.zeros(1, MO.num_frames(L))])
    pm = torch.zeros(len(lengths), L, dtype=torch.bool)
    for b, n in enumerate(lengths):
        pm[b, n:] = True
    got = m.forward_padding_mask(T2, pm)
    want = TO.frame_padding_mask(pm.numpy(), T2)
    assert got.shape == (len(lengths), T2)
    assert np.array_equal(got.numpy(), want)
