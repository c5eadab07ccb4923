"""Float64 numpy restatement of the HuBERT recipe's first-iteration features (src/examples/hubert/simple_kmeans/
dump_mfcc_feature.py): `torchaudio.compliance.kaldi.mfcc(x, sample_frequency=16000, use_energy=False)` followed by
`compute_deltas` twice and the concatenation [Tm, 13 + 13 + 13].  No torch in the arithmetic."""
from __future__ import annotations

import numpy as np

EPS32 = float(np.finfo(np.float32).eps)   # log floor of the fp32 recipe (a float64 torchaudio run floors at 2.2e-16)


def num_frames(n: int) -> int:
    """snip_edges framing: 400-sample frames every 160 samples; an utterance shorter than one frame has none."""
    return 1 + (n - 400) // 160 if n >= 400 else 0


def mel_banks() -> np.ndarray:
    """[23, 256] triangle weights of FFT bins 0..255 (bin 256 has weight 0): edges equally spaced in mel(f) = 1127 ln(1 + f/700)
    from 20 Hz to 8 kHz."""
    mel = lambda f: 1127.0 * np.log(1.0 + f / 700.0)
    lo, hi = mel(20.0), mel(8000.0)
    d = (hi - lo) / 24
    b = np.arange(23)[:, None]
    left, center, right = lo + b * d, lo + (b + 1) * d, lo + (b + 2) * d
    m = mel(31.25 * np.arange(256))[None, :]
    return np.maximum(0.0, np.minimum((m - left) / (center - left), (right - m) / (right - center)))


def dct_lifter() -> np.ndarray:
    """[23, 13]: orthonormal DCT-II (column 0 = sqrt(1/23)) times the lifter 1 + 11 sin(pi i / 22)."""
    k = np.arange(23)
    dct = np.sqrt(2 / 23) * np.cos(np.pi / 23 * (k[:, None] + 0.5) * np.arange(13)[None, :])
    dct[:, 0] = np.sqrt(1 / 23)
    return dct * (1 + 11 * np.sin(np.pi * np.arange(13) / 22))[None, :]


def deltas(v: np.ndarray) -> np.ndarray:
    """compute_deltas(win_length=5): sum_{k=1,2} k (v[t+k] - v[t-k]) / 10, frame indices clamped to [0, T - 1]."""
    T = v.shape[0]
    idx = lambda o: np.clip(np.arange(T) + o, 0, T - 1)
    return sum(k * (v[idx(k)] - v[idx(-k)]) for k in (1, 2)) / 10.0


def mfcc39(x) -> np.ndarray:
    """[Tm, 39] features of one utterance (float samples in [-1, 1])."""
    x = np.asarray(x, np.float64)
    T = num_frames(x.shape[0])
    if T == 0:
        return np.zeros((0, 39))
    fr = np.stack([x[t * 160:t * 160 + 400] for t in range(T)])
    fr = fr - fr.mean(1, keepdims=True)                                   # remove_dc_offset
    fr = fr - 0.97 * np.concatenate([fr[:, :1], fr[:, :-1]], 1)            # pre-emphasis, the first sample uses itself
    fr = fr * (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(400) / 399)) ** 0.85   # Povey window
    spec = np.fft.rfft(fr, n=512)
    power = spec.real ** 2 + spec.imag ** 2
    le = np.log(np.maximum(power[:, :256] @ mel_banks().T, EPS32))
    c = le @ dct_lifter()
    dl = deltas(c)
    return np.concatenate([c, dl, deltas(dl)], 1)

