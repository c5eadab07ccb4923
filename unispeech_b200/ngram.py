"""Word n-gram LM for `ctc.ctc_beam_search`: an ARPA file parsed on the host, hashed into device tables by the library's own
kernel (csrc/ctc_decode.cu, `b200s_ctc_lm_table_build`).

  * n-gram table: key = hash of the word ids (oldest first) -> (log10 p, log10 backoff);
  * spelling table: key = hash of a word's class ids -> word id.  Each character of a word maps to the class whose symbol is
    that character; words with a character no single-character symbol spells are left out (`dropped` counts them).

`NgramLM.start_ln` (host, fp32 per word id) holds ln P(w | <s>), from which `lexicon.Lexicon` builds its look-ahead.
Word ids are the order of the unigram section.  <s> and </s> must be unigrams; <unk> is optional (without it an unknown spelling
has no LM term, only `unk_score`).  Limits: order <= 5, fewer than 2^24 words.  A malformed file raises ValueError.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

from . import ops

MAX_ORDER = 5        # B200S_CTC_LM_MAX_ORDER
MAX_WORDS = 1 << 24
SPECIAL = ("<s>", "</s>", "<unk>")


def parse_arpa(path) -> Tuple[int, List[Dict[Tuple[str, ...], Tuple[float, float]]]]:
    """-> (order, [ {words: (log10 p, log10 backoff)} for n = 1..order ]).  Raises ValueError on a malformed file, an order
    above MAX_ORDER, MAX_WORDS words or more, a duplicate n-gram, a missing <s> or </s>, or an n-gram over a non-unigram."""
    with open(path, encoding="utf-8") as f:
        lines = f.read().splitlines()
    i = 0
    while i < len(lines) and lines[i].strip() != "\\data\\":
        i += 1
    if i == len(lines):
        raise ValueError(f"{path}: no \\data\\ section")
    i += 1
    counts = {}
    while i < len(lines) and lines[i].strip().startswith("ngram "):
        try:
            n, c = lines[i].strip()[6:].split("=")
            counts[int(n)] = int(c)
        except ValueError:
            raise ValueError(f"{path}:{i + 1}: bad count line {lines[i]!r}") from None
        i += 1
    if not counts or sorted(counts) != list(range(1, max(counts) + 1)):
        raise ValueError(f"{path}: the \\data\\ section must give the counts of orders 1..N, got {sorted(counts)}")
    order = max(counts)
    if order > MAX_ORDER:
        raise ValueError(f"{path}: LM order {order} is above the supported {MAX_ORDER}")
    grams: List[Dict[Tuple[str, ...], Tuple[float, float]]] = []
    for n in range(1, order + 1):
        while i < len(lines) and not lines[i].strip():
            i += 1
        if i == len(lines) or lines[i].strip() != f"\\{n}-grams:":
            raise ValueError(f"{path}:{i + 1}: expected \\{n}-grams:")
        i += 1
        table: Dict[Tuple[str, ...], Tuple[float, float]] = {}
        while i < len(lines) and lines[i].strip() and not lines[i].startswith("\\"):
            parts = lines[i].split()
            if len(parts) not in (n + 1, n + 2):
                raise ValueError(f"{path}:{i + 1}: a {n}-gram line needs log10 p, {n} words and an optional backoff")
            try:
                p = float(parts[0])
                bo = float(parts[n + 1]) if len(parts) == n + 2 else 0.0
            except ValueError:
                raise ValueError(f"{path}:{i + 1}: bad number in {lines[i]!r}") from None
            words = tuple(parts[1:n + 1])
            if words in table:
                raise ValueError(f"{path}:{i + 1}: duplicate {n}-gram {' '.join(words)}")
            table[words] = (p, bo)
            i += 1
        if len(table) != counts[n]:
            raise ValueError(f"{path}: {len(table)} {n}-grams, the header says {counts[n]}")
        grams.append(table)
    while i < len(lines) and not lines[i].strip():
        i += 1
    if i == len(lines) or lines[i].strip() != "\\end\\":
        raise ValueError(f"{path}:{i + 1}: expected \\end\\")
    if len(grams[0]) >= MAX_WORDS:
        raise ValueError(f"{path}: {len(grams[0])} words, the limit is {MAX_WORDS - 1}")
    for s in ("<s>", "</s>"):
        if (s,) not in grams[0]:
            raise ValueError(f"{path}: {s} is not a unigram")
    for n in range(2, order + 1):
        for g in grams[n - 1]:
            if any((w,) not in grams[0] for w in g):
                raise ValueError(f"{path}: the {n}-gram {' '.join(g)} has a word that is not a unigram")
    return order, grams


def spellings(words: Sequence[str], symbols: Sequence[str], word_boundary: int):
    """-> (class-id spellings, their word ids, number of words left out).  A character is spelled by the first single-character
    symbol equal to it (the boundary class excluded); <s>, </s> and <unk> are not spelled."""
    char_class: Dict[str, int] = {}
    for c, s in enumerate(symbols):
        if len(s) == 1 and c != word_boundary:
            char_class.setdefault(s, c)
    spelled, ids, dropped = [], [], 0
    for i, w in enumerate(words):
        if w in SPECIAL:
            continue
        if all(ch in char_class for ch in w):
            spelled.append([char_class[ch] for ch in w])
            ids.append(i)
        else:
            dropped += 1
    return spelled, ids, dropped


def _capacity(n: int) -> int:
    c = 2
    while c < 2 * n:
        c *= 2
    return c


def _table(seqs: np.ndarray, v0: np.ndarray, v1, dev):
    n = seqs.shape[0]
    cap = _capacity(n)
    keys = torch.zeros(cap, dtype=torch.int64, device=dev)
    vals = torch.zeros(cap, 2, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    s = torch.from_numpy(np.ascontiguousarray(seqs, dtype=np.int32)).to(dev)
    a = torch.from_numpy(np.ascontiguousarray(v0).view(np.int32)).to(dev)
    b = None if v1 is None else torch.from_numpy(np.ascontiguousarray(v1).view(np.int32)).to(dev)
    ops.ctc_lm_table_build(s, n, seqs.shape[1], a, b, keys, vals, status)
    return keys, vals, status


class NgramLM:
    """Device tables of a word n-gram LM.  `NgramLM.from_arpa(path, symbols, word_boundary)`; `symbols[c]` is the string of class
    c (a fairseq letter dictionary), `word_boundary` the class that separates words (fairseq's "|")."""

    def __init__(self, order, words, word_ids, ngram_keys, ngram_vals, spell_keys, spell_vals, has_unk, dropped, word_boundary):
        self.order, self.words, self.word_ids = order, words, word_ids
        self.ngram_keys, self.ngram_vals, self.spell_keys, self.spell_vals = ngram_keys, ngram_vals, spell_keys, spell_vals
        self.has_unk, self.dropped, self.word_boundary = has_unk, dropped, word_boundary
        self.bos, self.eos = word_ids["<s>"], word_ids["</s>"]
        self.unk = word_ids["<unk>"] if has_unk else len(words)   # without <unk>: an id no n-gram contains

    @classmethod
    def from_arpa(cls, path, symbols: Sequence[str], word_boundary: int, device=None) -> "NgramLM":
        order, grams = parse_arpa(path)
        if not 0 <= word_boundary < len(symbols):
            raise ValueError(f"word_boundary={word_boundary} is not a class of the {len(symbols)} symbols")
        words = [w[0] for w in grams[0]]
        word_ids = {w: i for i, w in enumerate(words)}
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        # n-grams: word ids padded with -1, (log10 p, log10 backoff) as fp32
        n_all = sum(len(g) for g in grams)
        seqs = np.full((n_all, order), -1, dtype=np.int32)
        lp = np.zeros(n_all, dtype=np.float32)
        bo = np.zeros(n_all, dtype=np.float32)
        r = 0
        for g in grams:
            for ws, (p, b) in g.items():
                seqs[r, :len(ws)] = [word_ids[w] for w in ws]
                lp[r], bo[r] = p, b
                r += 1
        spelled, ids, dropped = spellings(words, symbols, word_boundary)
        if spelled:
            sp = np.full((len(spelled), max(len(s) for s in spelled)), -1, dtype=np.int32)
            for k, s in enumerate(spelled):
                sp[k, :len(s)] = s
            sp_keys, sp_vals, sp_status = _table(sp, np.asarray(ids, dtype=np.int32), None, dev)
        else:   # no word can be spelled: an empty table, every lookup misses
            sp_keys = torch.zeros(2, dtype=torch.int64, device=dev)
            sp_vals = torch.zeros(2, 2, dtype=torch.int32, device=dev)
            sp_status = torch.zeros(1, dtype=torch.int32, device=dev)
        ng_keys, ng_vals, ng_status = _table(seqs, lp, bo, dev)
        st = int(ng_status.item()) | int(sp_status.item())
        if st:
            raise ValueError(f"{path}: the 64-bit hash of two different n-grams or spellings collided (status {st}); "
                             "the tables cannot hold this LM")
        lm = cls(order, words, word_ids, ng_keys, ng_vals, sp_keys, sp_vals, ("<unk>",) in grams[0], dropped, word_boundary)
        lm.start_ln = start_log_probs(order, grams, words)
        return lm


def start_log_probs(order: int, grams, words: Sequence[str]) -> np.ndarray:
    """fp32 [len(words)]: ln P(w | <s>) of every word id, in the device's `ln_prob` order (log10 backoff of <s> when the bigram
    (<s>, w) is missing, then the log10 p, summed in fp32 from 0, then * ln 10 in fp32).  The look-ahead of a lexicon's trie
    (`lexicon.Lexicon`) is built from these."""
    f32 = np.float32
    p1 = np.asarray([grams[0][(w,)][0] for w in words], dtype=f32)
    if order > 1:
        acc = (f32(0.0) + f32(grams[0][("<s>",)][1])) + p1
        ids = {w: i for i, w in enumerate(words)}
        for (a, w), (p, _) in grams[1].items():
            if a == "<s>":
                acc[ids[w]] = f32(0.0) + f32(p)
    else:
        acc = f32(0.0) + p1
    return (acc.astype(f32) * f32(2.302585092994046)).astype(f32)
