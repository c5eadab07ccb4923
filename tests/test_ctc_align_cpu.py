"""CTC forced alignment without a GPU: the fp32 numpy oracle (oracle/align_oracle.py) against
torchaudio.functional.forced_align bit for bit (paths and frame scores, ties included), `token_spans` against
torchaudio.functional.merge_tokens, the workspace-size formula and the C entry point's argument checks (which return before any
launch, so they run without a device)."""
import numpy as np
import pytest
import torch

from oracle import align_oracle as AO

F = pytest.importorskip("torchaudio.functional")


def _lp(T, V, seed, quant=None):
    """fp32 log-probabilities [T, V] of random logits, rounded to multiples of `quant` first (many exact ties)."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((T, V)).astype(np.float32) * 2
    if quant is not None:
        x = np.round(x / quant) * quant if quant > 0 else np.zeros_like(x)
    x = torch.from_numpy(x)
    return (x - torch.logsumexp(x, dim=-1, keepdim=True)).numpy()


def _ta(lp, targets, blank=0):
    p, s = F.forced_align(torch.from_numpy(lp)[None], torch.tensor([list(targets)], dtype=torch.int32), blank=blank)
    return p[0].numpy().astype(np.int32), s[0].numpy().astype(np.float32)


def _same(lp, targets, blank=0):
    labels, fs, score = AO.viterbi(lp, targets, blank)
    want_l, want_s = _ta(lp, targets, blank)
    np.testing.assert_array_equal(labels, want_l)
    np.testing.assert_array_equal(fs.view(np.int32), want_s.view(np.int32))
    assert abs(float(score) - float(fs.astype(np.float64).sum())) <= 1e-5 * max(1.0, abs(float(score)))
    return labels, fs


CASES = {
    # name: (T, V, targets, blank, quant)
    "random": (60, 12, [3, 7, 1, 1, 9, 4, 2, 11, 5], 0, None),
    "random_blank_last": (45, 8, [2, 0, 5, 1, 1, 3], 7, None),
    "quantised": (50, 6, [1, 2, 3, 2, 1, 4, 5], 0, 0.5),
    "all_tie": (20, 5, [1, 2, 3, 4], 0, 0.0),
    "all_tie_repeats": (16, 4, [1, 1, 2, 2, 3, 3], 0, 0.0),
    "repeats_force_blanks": (12, 5, [2, 2, 2, 2, 2, 2], 0, None),
    "min_feasible": (8, 6, [1, 1, 2, 3, 3, 4], 0, None),          # 6 labels + one blank per repeat: 8 frames
    "min_feasible_tie": (5, 4, [1, 1, 1], 0, 0.0),               # 3 labels + 2 blanks
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_matches_torchaudio(name):
    T, V, targets, blank, quant = CASES[name]
    if name.startswith("min_feasible"):
        T = AO.min_frames(targets)
    _same(_lp(T, V, seed=sum(map(ord, name)), quant=quant), targets, blank)


def test_oracle_matches_torchaudio_random_sweep():
    """Many small cases at and just above the minimum length, logits quantised to 0, 1/4 or not at all."""
    rng = np.random.default_rng(7)
    for it in range(400):
        V = int(rng.integers(3, 7))
        S = int(rng.integers(1, 9))
        targets = rng.integers(1, V, size=S).tolist()
        T = AO.min_frames(targets) + int(rng.integers(0, 4))
        _same(_lp(T, V, seed=it, quant=[None, 0.25, 0.0][it % 3]), targets)


def test_tie_rule_advance_equal_to_skip_takes_stay():
    """advance == skip > stay picks stay (both strict tests fail): frame 2 of label 2 stays, where a plain max would advance."""
    x = torch.tensor([[0.0, 0.0, 0.0], [3.0, 3.0, 0.0], [0.0, 0.0, 5.0]])
    lp = (x - torch.logsumexp(x, -1, keepdim=True)).numpy()
    labels, _ = _same(lp, [1, 2])
    assert labels.tolist() == [1, 2, 2]


def test_empty_target_aligns_to_blank():
    lp = _lp(7, 5, seed=3)
    labels, fs, score = AO.viterbi(lp, [], blank=2)
    assert labels.tolist() == [2] * 7
    np.testing.assert_array_equal(fs, lp[:, 2])
    b_lab, b_fs, b_score = AO.align_batch(lp[None], [7], np.zeros((1, 1), np.int64), [0], blank=2)
    assert b_lab[0].tolist() == [2] * 7 and b_score[0] == score


def test_batch_semantics_padding_and_infeasible():
    B, T, V = 5, 12, 6
    lp = np.stack([_lp(T, V, seed=b) for b in range(B)])
    targets = np.array([[1, 2, 3], [1, 1, 1], [1, 0, 2], [1, 7, 2], [4, 4, 4]])
    tl = [3, 3, 3, 3, 4]
    il = [10, 4, 12, 12, 12]
    labels, fs, score = AO.align_batch(lp, il, targets, tl, blank=0)
    want_l, want_s = _ta(lp[0, :10], [1, 2, 3])
    assert labels[0, :10].tolist() == want_l.tolist() and labels[0, 10:].tolist() == [-1, -1]
    assert fs[0, 10:].tolist() == [0.0, 0.0]
    # [1, 1, 1] needs 5 frames; a blank label; a label >= V; target_len > Smax
    for b in (1, 2, 3, 4):
        assert labels[b].tolist() == [-1] * T and score[b] == -np.inf and not fs[b].any()


def test_token_spans_match_merge_tokens():
    from unispeech_b200.ctc import token_spans
    cases = [(CASES["random"], 0), (CASES["all_tie_repeats"], 0), (CASES["repeats_force_blanks"], 0),
             (CASES["random_blank_last"], 7)]
    T = max(c[0][0] for c in cases)
    labels = torch.full((len(cases), T), -1, dtype=torch.int32)
    scores = torch.zeros(len(cases), T)
    lens = []
    for i, ((t, V, tg, blank, quant), _) in enumerate(cases):
        lab, fs = _same(_lp(t, V, seed=i, quant=quant), tg, blank)
        labels[i, :t], scores[i, :t] = torch.from_numpy(lab), torch.from_numpy(fs)
        lens.append(t)
    for i, (c, blank) in enumerate(cases):
        got = token_spans(labels[i:i + 1], scores[i:i + 1], [lens[i]], blank=blank)[0]
        want = F.merge_tokens(labels[i, :lens[i]], scores[i, :lens[i]], blank=blank)
        assert [(s.token, s.start, s.end) for s in got] == [(s.token, s.start, s.end) for s in want]
        assert [s.score for s in got] == [s.score for s in want]
        assert [s.token for s in got] == c[2]


def test_token_spans_infeasible_and_empty():
    from unispeech_b200.ctc import token_spans
    labels = torch.tensor([[-1, -1, -1], [0, 0, 0], [0, 3, -1]], dtype=torch.int32)
    scores = torch.tensor([[0.0, 0.0, 0.0], [-0.1, -0.2, -0.3], [-0.5, -0.25, 0.0]])
    assert token_spans(labels, scores, [3, 3, 2]) == [[], [], [(3, 1, 2, -0.25)]]


def test_workspace_formula():
    from unispeech_b200 import ops
    for B, T, S in [(1, 1, 0), (8, 999, 300), (3, 17, 7), (1, 90000, 6000), (2, 5, 8191)]:
        assert ops.ctc_align_workspace_bytes(B, T, S) == B * T * ((2 * S + 1 + 15) // 16) * 4
    assert ops.ctc_align_workspace_bytes(1, 90000, 6000) == 270_360_000
    for B, T, S in [(0, 5, 1), (1, 0, 1), (1, 5, -1), (1, 5, 8192)]:
        assert ops.ctc_align_workspace_bytes(B, T, S) == -1


def _call_align(**over):
    """b200s_ctc_align with dummy (never dereferenced) addresses: every argument check runs on the host before any launch."""
    from unispeech_b200 import _lib as L
    a = dict(logits=16, fs=32, bs=320, lse=16, il=16, tg=16, Smax=4, tl=16, B=2, T=10, V=32, blank=0, ws=16, ws_bytes=1 << 20,
             labels=16, fscores=16, score=16)
    a.update(over)
    L.call("b200s_ctc_align", a["logits"], a["fs"], a["bs"], a["lse"], a["il"], a["tg"], a["Smax"], a["tl"], a["B"], a["T"],
           a["V"], a["blank"], a["ws"], a["ws_bytes"], a["labels"], a["fscores"], a["score"], 0)


@pytest.mark.parametrize("over,msg", [
    (dict(Smax=8192), "Smax=8192 outside [0, 8191]"),
    (dict(Smax=-1), "Smax=-1 outside"),
    (dict(V=1025), "V=1025 outside [1, 1024]"),
    (dict(blank=32), "blank=32 outside [0, V=32)"),
    (dict(blank=-1), "blank=-1 outside"),
    (dict(B=0), "need B > 0"),
    (dict(labels=0), "null pointer"),
    (dict(ws=0), "null pointer"),
    (dict(tg=0), "null targets"),
    (dict(ws_bytes=2 * 10 * 1 * 4 - 1), "workspace of 79 bytes, need 80"),
])
def test_argument_checks(over, msg):
    with pytest.raises(RuntimeError, match=msg.replace("[", r"\[").replace("(", r"\(").replace(")", r"\)")):
        _call_align(**over)
