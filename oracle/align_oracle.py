"""fp32 numpy restatement of CTC forced alignment (Viterbi over the extended label sequence), with the tie rule of
`torchaudio.functional.forced_align` (CPU), which it reproduces bit for bit.

Extended sequence l' = (blank, l_1, blank, ..., l_S, blank), L = 2S + 1 positions.  With lp [T, V] fp32 log-probabilities:
  alpha_0(0) = lp[0, blank], alpha_0(1) = lp[0, l_1], every other position -inf;
  alpha_t(s) = pick(stay = alpha_{t-1}(s), advance = alpha_{t-1}(s-1), skip = alpha_{t-1}(s-2) if s is a label position
               whose label differs from the previous label, else -inf) + lp[t, l'_s]   (fp32 add)
  pick: skip   if skip > advance and skip > stay,
        else advance if advance > stay and advance > skip,
        else stay.
Every comparison is strict, so an exact tie goes to stay before advance before skip -- and when advance == skip > stay, neither
wins its strict test and stay is taken although it is smaller.  The end position is L-1 (final blank) if
alpha_{T-1}(L-1) > alpha_{T-1}(L-2), else L-2 (ties to the last label); with S = 0 it is position 0.  The path is walked back
from there through the recorded choices.

torchaudio also restricts each frame to a window of positions that can still be reached from frame 0 and can still reach the
end.  Positions outside it are -inf there but can never be on the path nor feed a position that is, so the plain recursion here
(and in csrc/ctc_align.cu) gives the same path and scores.
"""
from __future__ import annotations

import numpy as np

NEG_INF = np.float32(-np.inf)


def min_frames(targets) -> int:
    """Fewest frames a path through `targets` needs: one per label plus one blank between each pair of equal neighbours."""
    t = list(targets)
    return len(t) + sum(1 for i in range(1, len(t)) if t[i] == t[i - 1])


def feasible(T: int, targets, V: int, blank: int) -> bool:
    return all(0 <= int(c) < V and int(c) != blank for c in targets) and T >= min_frames(targets)


def viterbi(lp: np.ndarray, targets, blank: int = 0):
    """lp: fp32 [T, V] (T >= 1), targets: S labels (a feasible alignment).  Returns (labels int32 [T], frame_scores fp32 [T],
    score fp32): the class per frame on the best path, lp at it, and alpha_{T-1} at the end position."""
    lp = np.asarray(lp, dtype=np.float32)
    T = lp.shape[0]
    tg = np.asarray(list(targets), dtype=np.int64)
    S = len(tg)
    L = 2 * S + 1
    ext = np.full(L, blank, dtype=np.int64)
    ext[1::2] = tg
    skip = np.zeros(L, dtype=bool)
    if S > 1:
        skip[3::2] = tg[1:] != tg[:-1]
    bp = np.zeros((T, L), dtype=np.int8)
    a = np.full(L, NEG_INF, dtype=np.float32)
    a[0] = lp[0, blank]
    if L > 1:
        a[1] = lp[0, ext[1]]
    for t in range(1, T):
        x0 = a
        x1 = np.concatenate(([NEG_INF], a[:-1]))
        x2 = np.where(skip, np.concatenate(([NEG_INF, NEG_INF], a[:-2]))[:L], NEG_INF)
        c2 = (x2 > x1) & (x2 > x0)
        c1 = ~c2 & (x1 > x0) & (x1 > x2)
        v = np.where(c2, x2, np.where(c1, x1, x0)).astype(np.float32)
        bp[t] = np.where(c2, 2, np.where(c1, 1, 0))
        a = (v + lp[t, ext]).astype(np.float32)
    pos = 0 if L == 1 else (L - 1 if a[L - 1] > a[L - 2] else L - 2)
    score = np.float32(a[pos])
    path = np.empty(T, dtype=np.int64)
    for t in range(T - 1, -1, -1):
        path[t] = pos
        pos -= int(bp[t, pos])
    labels = ext[path].astype(np.int32)
    return labels, lp[np.arange(T), labels].astype(np.float32), score


def align_batch(lp: np.ndarray, input_len, targets, target_len, blank: int = 0):
    """Batched semantics of `unispeech_b200.ctc.forced_align` over fp32 lp [B, T, V]: padded frames get (-1, 0); an infeasible
    utterance gets -1 on every frame, frame scores 0 and score -inf."""
    B, T, V = lp.shape
    Smax = targets.shape[1]
    labels = np.full((B, T), -1, dtype=np.int32)
    fs = np.zeros((B, T), dtype=np.float32)
    score = np.full(B, NEG_INF, dtype=np.float32)
    for b in range(B):
        n, s = min(max(int(input_len[b]), 0), T), int(target_len[b])
        if s < 0 or s > Smax:
            continue
        tg = [int(c) for c in targets[b, :s]]
        if not feasible(n, tg, V, blank):
            continue
        if n == 0:
            score[b] = 0.0
            continue
        labels[b, :n], fs[b, :n], score[b] = viterbi(lp[b, :n], tg, blank)
    return labels, fs, score
