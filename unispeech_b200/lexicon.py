"""Word lexicon for lexicon-constrained `ctc.ctc_beam_search`: a flashlight / fairseq lexicon file parsed on the host into a
word trie in device arrays (csrc/ctc_decode_lex.cu reads them; include/unispeech_b200.h, b200s_ctc_decode_lexicon, states the
semantics).

File format: one `WORD tok tok ...` per line, as fairseq's `librispeech_lexicon.lst` (`ABOUT A B O U T |`).  A trailing
word-boundary token is stripped; every other token must be a symbol of the model's dictionary (the first class with exactly
that symbol), and neither the blank (class `blank`) nor the boundary.  A word may have several spellings (several lines); a
spelling that several words share belongs to the first of them in file order.  Dropped spellings (unknown token, blank, a
boundary inside the word, no tokens left, or already taken) are counted in `dropped`.  A line without tokens raises
ValueError with its line number.

Device layout, nodes in BFS order with the children of a node contiguous and in class order (node 0 is the root, the empty
partial word):
  mask        int32 [nodes, ceil(V / 32)]  (uint32 bits) bit c: the node has a child by class c
  first_child int32 [nodes]                its child by c is first_child + the number of mask bits below c
  word        int32 [nodes]                -1: ends no word; -2: ends a word the LM does not know; else the LM word id (without
                                           an LM: the word's index in `words`)
  smear       fp32 [nodes]                 look-ahead: max over the words ending at or below the node of ln P(w | <s>) (w as
                                           <unk>, or 0 without <unk>, when the LM does not know it); 0 at the root, without an
                                           LM and with smearing="none"
Memory: nodes * (4 * ceil(V / 32) + 12) bytes; a lexicon has at most as many nodes as letters in all its spellings, plus one.
"""
from __future__ import annotations

from typing import Dict, List, Sequence, Tuple

import numpy as np
import torch

MAX_NODES = 1 << 30   # B200S_CTC_TRIE_MAX_NODES
SMEARING = ("max", "none")


def parse_lexicon(path, symbols: Sequence[str], word_boundary: int, blank: int = 0):
    """-> (words in first-appearance order, [(spelling as a tuple of class ids, word index)] in file order, dropped count)."""
    if not 0 <= word_boundary < len(symbols):
        raise ValueError(f"word_boundary={word_boundary} is not a class of the {len(symbols)} symbols")
    cls_of: Dict[str, int] = {}
    for c, s in enumerate(symbols):
        cls_of.setdefault(s, c)
    bsym = symbols[word_boundary]
    words: List[str] = []
    index: Dict[str, int] = {}
    taken: Dict[Tuple[int, ...], int] = {}
    spellings: List[Tuple[Tuple[int, ...], int]] = []
    dropped = 0
    with open(path, encoding="utf-8") as f:
        for lineno, line in enumerate(f, 1):
            parts = line.split()
            if not parts:
                continue
            if len(parts) < 2:
                raise ValueError(f"{path}:{lineno}: a lexicon line needs a word and its tokens, got {line.rstrip()!r}")
            word, toks = parts[0], parts[1:]
            if toks[-1] == bsym:
                toks = toks[:-1]
            ids = [cls_of.get(t, -1) for t in toks]
            if not ids or any(c < 0 or c == blank or c == word_boundary for c in ids):
                dropped += 1
                continue
            sp = tuple(ids)
            if sp in taken:
                dropped += 1
                continue
            if word not in index:
                index[word] = len(words)
                words.append(word)
            taken[sp] = index[word]
            spellings.append((sp, index[word]))
    return words, spellings, dropped


def build_trie(spellings, V: int):
    """-> (mask uint32 [N, W], first_child int32 [N], word index int32 [N] (-1 none), parent int32 [N], depth int32 [N]) with the
    nodes in BFS order, children in class order."""
    children: List[Dict[int, int]] = [{}]
    ends: List[int] = [-1]
    for sp, w in spellings:
        n = 0
        for c in sp:
            nxt = children[n].get(c)
            if nxt is None:
                nxt = len(children)
                children[n][c] = nxt
                children.append({})
                ends.append(-1)
            n = nxt
        ends[n] = w
    N = len(children)
    if N > MAX_NODES:
        raise ValueError(f"the lexicon's trie has {N} nodes, the limit is {MAX_NODES}")
    W = (V + 31) // 32
    order = [0]
    first_child = np.zeros(N, dtype=np.int32)
    parent = np.full(N, -1, dtype=np.int32)
    depth = np.zeros(N, dtype=np.int32)
    edge_p, edge_c = [], []
    head = 0
    while head < len(order):
        old = order[head]
        first_child[head] = len(order)
        for c in sorted(children[old]):
            ch = children[old][c]
            parent[len(order)] = head
            depth[len(order)] = depth[head] + 1
            order.append(ch)
            edge_p.append(head)
            edge_c.append(c)
        head += 1
    mask = np.zeros((N, W), dtype=np.uint32)
    if edge_p:
        ep, ec = np.asarray(edge_p, dtype=np.int64), np.asarray(edge_c, dtype=np.int64)
        np.bitwise_or.at(mask, (ep, ec >> 5), (np.uint32(1) << (ec & 31).astype(np.uint32)))
    word = np.asarray(ends, dtype=np.int32)[np.asarray(order, dtype=np.int64)]
    return mask, first_child, word, parent, depth


def trie_smear(word: np.ndarray, parent: np.ndarray, depth: np.ndarray, start_ln: np.ndarray, unk_ln) -> np.ndarray:
    """fp32 [N] look-ahead of every node: the max over the words ending at or below it of start_ln[word] (unk_ln, or 0 when it is
    None, for -2: a word the LM does not know); 0 at the root.  `word`, `parent`, `depth` as `build_trie` orders the nodes, with
    `word` holding LM word ids."""
    own = np.full(len(word), -np.inf, dtype=np.float32)
    ends = word != -1
    wid = word[ends]
    own[ends] = np.where(wid >= 0, start_ln[np.maximum(wid, 0)], np.float32(0.0) if unk_ln is None else unk_ln)
    for d in range(int(depth.max()), 0, -1):   # deepest first: a node's max is final before its parent reads it
        at = np.nonzero(depth == d)[0]
        np.maximum.at(own, parent[at], own[at])
    own[0] = 0.0
    return own


class Lexicon:
    """Device trie of a word lexicon for `ctc.ctc_beam_search(..., lexicon=)`.  `Lexicon.from_file(path, symbols, word_boundary,
    lm=None, smearing="max")`: `symbols[c]` is the string of class c (a fairseq letter dictionary), `word_boundary` the class
    that separates words (fairseq's "|"), `lm` the `ngram.NgramLM` the search will score with (its word ids and the
    look-ahead come from it; the search refuses any other LM)."""

    def __init__(self, words, V, word_boundary, blank, lm, smearing, mask, first_child, word, smear, dropped):
        self.words, self.V, self.word_boundary, self.blank, self.lm, self.smearing = words, V, word_boundary, blank, lm, smearing
        self.mask, self.first_child, self.word, self.smear, self.dropped = mask, first_child, word, smear, dropped

    @property
    def nodes(self) -> int:
        return self.first_child.numel()

    @property
    def nbytes(self) -> int:
        return self.nodes * (4 * ((self.V + 31) // 32) + 12)

    @classmethod
    def from_file(cls, path, symbols: Sequence[str], word_boundary: int, lm=None, smearing: str = "max", device=None,
                  blank: int = 0) -> "Lexicon":
        if smearing not in SMEARING:
            raise ValueError(f"smearing={smearing!r}: one of {SMEARING}")
        if lm is not None and lm.word_boundary != word_boundary:
            raise ValueError(f"the LM was built with word_boundary={lm.word_boundary}, the lexicon with {word_boundary}")
        if not 0 <= blank < len(symbols) or blank == word_boundary:
            raise ValueError(f"blank={blank} must be a class of the {len(symbols)} symbols other than word_boundary")
        words, spellings, dropped = parse_lexicon(path, symbols, word_boundary, blank)
        V = len(symbols)
        mask, first_child, widx, parent, depth = build_trie(spellings, V)
        N = len(first_child)
        ends = widx >= 0
        word = np.full(N, -1, dtype=np.int32)
        smear = np.zeros(N, dtype=np.float32)
        if lm is None:
            word[ends] = widx[ends]
        else:
            lm_id = np.asarray([lm.word_ids.get(w, -2) for w in words], dtype=np.int32)
            word[ends] = lm_id[widx[ends]]
            if smearing == "max":
                smear = trie_smear(word, parent, depth, lm.start_ln, np.float32(lm.start_ln[lm.unk]) if lm.has_unk else None)
        dev = torch.device(device) if device is not None else torch.device("cuda", torch.cuda.current_device())
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        return cls(words, V, word_boundary, blank, lm, smearing, t(mask.view(np.int32)), t(first_child), t(word), t(smear),
                   dropped)

    def check(self, V: int, lm, device, blank: int) -> None:
        """Raises ValueError unless this lexicon was built for V classes, `blank` and `lm`, and its arrays are intact on `device`."""
        if V != self.V:
            raise ValueError(f"the lexicon was built for V={self.V} classes, the logits have {V}")
        if blank != self.blank:
            raise ValueError(f"the lexicon was built for blank={self.blank}, the search has blank={blank}")
        if lm is not self.lm:
            raise ValueError("the lexicon was built for a different LM (pass the same NgramLM to Lexicon.from_file and the search)")
        if lm is not None and lm.word_boundary != self.word_boundary:
            raise ValueError(f"the LM's word_boundary={lm.word_boundary}, the lexicon's {self.word_boundary}")
        N, W = self.nodes, (self.V + 31) // 32
        for name, a, shape, dt in (("mask", self.mask, (N, W), torch.int32), ("first_child", self.first_child, (N,), torch.int32),
                                   ("word", self.word, (N,), torch.int32), ("smear", self.smear, (N,), torch.float32)):
            if tuple(a.shape) != shape or a.dtype != dt or a.device != device or not a.is_contiguous():
                raise ValueError(f"lexicon array {name}: {tuple(a.shape)} {a.dtype} on {a.device}, need contiguous {shape} {dt} "
                                 f"on {device}")
        if not 1 <= N <= MAX_NODES:
            raise ValueError(f"the lexicon's trie has {N} nodes, outside [1, {MAX_NODES}]")
