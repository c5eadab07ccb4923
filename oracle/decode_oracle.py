"""fp32 numpy restatement of CTC prefix beam search with word n-gram LM scoring (`unispeech_b200.ctc.ctc_beam_search`,
csrc/ctc_decode.cu), and an ARPA scorer.  This file is the definition of the semantics.

lp [T, V] fp32 log-probabilities (logit - lse); lae(a, b) = max + log1p(exp(-|a - b|)) in fp32 (-inf when both are).
Prefix hash: h' = splitmix64(h ^ (c + 1)) from h = 0 (the same function hashes spellings and n-grams).
Each beam: pb, pnb, lm, prefix hash, partial-word hash (0 when empty), last class (-1 for the empty prefix), word context.
Per frame, T_K = the beam_token non-blank classes of highest lp (ties to the smaller id):
  * stays, in beam rank order: pb' = lae(pb, pnb) + lp[blank], pnb' = pnb + lp[last] (-inf for the empty prefix);
  * extensions, by parent rank then class id, of every beam j by every c in T_K: contribution
    (c == last_j ? pb_j : lae(pb_j, pnb_j)) + lp[c] to pnb of prefix + c, merged into an existing entry by lae;
  * a boundary extension of a non-empty partial word adds lm_weight * lnP(word | ctx) + word_score (+ unk_score for an unknown
    spelling, whose LM term is 0 when the LM has no <unk>) to lm and pushes the word; an empty word scores nothing.  The partial
    word's class ids name an LM word only if they are that word's spelling (`spelling_table`: each character by the first
    single-character class with that symbol);
  * ranking score = lae(pb, pnb) + lm; sorted by (score desc, hash asc), the best `beam` kept.
At the end: a non-empty partial word is scored, then lm += lm_weight * lnP(</s> | ctx); score = lae(pb, pnb) + lm.
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np

F32 = np.float32
NEG_INF = F32(-np.inf)
M64 = (1 << 64) - 1
LN10 = F32(2.302585092994046)


def splitmix64(z: int) -> int:
    z = (z + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def hash_step(h: int, x: int) -> int:
    return splitmix64(h ^ ((x + 1) & M64))


def hash_seq(xs) -> int:
    h = 0
    for x in xs:
        h = hash_step(h, int(x))
    return h


def _mix_np(z: np.ndarray) -> np.ndarray:
    """splitmix64 over a uint64 array (wrapping arithmetic)."""
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        return z ^ (z >> np.uint64(31))


def lae(a, b):
    a, b = F32(a), F32(b)
    m = max(a, b)
    if m == NEG_INF:
        return NEG_INF
    return F32(m + F32(np.log1p(np.exp(F32(-abs(F32(a - b)))))))


class ArpaLM:
    """An ARPA file as dicts: `prob(word, ctx)` = ln P(word | ctx) with backoff, in the fp32 order the kernel uses."""

    def __init__(self, order: int, grams: List[Dict[Tuple[str, ...], Tuple[float, float]]]):
        self.order = order
        self.p = {}
        self.bo = {}
        for g in grams:
            for ws, (p, b) in g.items():
                self.p[ws] = F32(p)
                self.bo[ws] = F32(b)
        self.vocab = {w[0] for w in grams[0]}
        self.has_unk = "<unk>" in self.vocab

    @classmethod
    def from_file(cls, path):
        """Minimal ARPA reader of its own (well-formed files only): the n-gram sections after \\data\\, each line
        `log10 p  w_1 .. w_n  [log10 backoff]`."""
        grams: List[Dict[Tuple[str, ...], Tuple[float, float]]] = []
        n = 0
        with open(path, encoding="utf-8") as f:
            for line in f:
                line = line.strip()
                if line.endswith("-grams:") and line.startswith("\\"):
                    n = int(line[1:line.index("-")])
                    grams.append({})
                elif line == "\\end\\":
                    break
                elif n and line:
                    parts = line.split()
                    grams[n - 1][tuple(parts[1:n + 1])] = (float(parts[0]), float(parts[n + 1]) if len(parts) > n + 1 else 0.0)
        return cls(len(grams), grams)

    def log10(self, word: str, ctx: Sequence[str]) -> np.float32:
        """log10 P(word | ctx) by ARPA backoff (ctx oldest first), fp32: backoffs of the longer unmatched contexts from the
        longest down, then the matched n-gram's log10 p."""
        ctx = tuple(ctx)[-(self.order - 1):] if self.order > 1 else ()
        acc = F32(0.0)
        for L in range(len(ctx), -1, -1):
            c = ctx[len(ctx) - L:]
            if c + (word,) in self.p:
                return F32(acc + self.p[c + (word,)])
            if L >= 1 and c in self.bo:
                acc = F32(acc + self.bo[c])
        raise KeyError(word)

    def prob(self, word: str, ctx: Sequence[str]) -> np.float32:
        return F32(self.log10(word, ctx) * LN10)


def spelling_table(vocab, symbols, boundary) -> Dict[Tuple[int, ...], str]:
    """class-id sequence -> LM word.  Each character of a word is spelled by the FIRST class whose symbol is that single
    character (the boundary class excluded); a word with a character no such class has is left out, and so are <s>, </s> and
    <unk>.  A class sequence is a known word only if it is exactly such a spelling: a repeated symbol's later class spells
    nothing, and multi-character symbols spell nothing."""
    first: Dict[str, int] = {}
    for c, sym in enumerate(symbols):
        if len(sym) == 1 and c != boundary and sym not in first:
            first[sym] = c
    table = {}
    for w in vocab:
        if w not in ("<s>", "</s>", "<unk>") and all(ch in first for ch in w):
            table[tuple(first[ch] for ch in w)] = w
    return table


class _Scorer:
    def __init__(self, lm: ArpaLM, symbols, boundary, weight, word_score, unk_score):
        self.lm, self.symbols, self.boundary = lm, symbols, boundary
        self.weight, self.word_score, self.unk_score = F32(weight), F32(word_score), F32(unk_score)
        self.spell = spelling_table(lm.vocab, symbols, boundary)

    def word(self, chars: Tuple[int, ...], ctx: Tuple[str, ...]):
        """(LM term, new context) of ending the word spelled by class ids `chars`."""
        w = self.spell.get(tuple(chars))
        oov = w is None
        if oov:
            w = "<unk>"
        t = F32(0.0)
        if not oov or self.lm.has_unk:
            t = F32(self.weight * self.lm.prob(w, ctx))
        t = F32(t + self.word_score)
        if oov:
            t = F32(t + self.unk_score)
        return t, self.push(ctx, w)

    def push(self, ctx, w):
        n = self.lm.order - 1
        return (ctx + (w,))[-n:] if n > 0 else ()

    def finish(self, ctx):
        return F32(self.weight * self.lm.prob("</s>", ctx))


def beam_search(lp: np.ndarray, beam: int, nbest: int = 1, blank: int = 0, beam_token: Optional[int] = None,
                lm: Optional[ArpaLM] = None, symbols=None, word_boundary: int = -1, lm_weight: float = 0.0,
                word_score: float = 0.0, unk_score: float = 0.0):
    """lp fp32 [T, V].  Returns [(tokens list, score fp32)] best first, at most nbest (fewer when fewer prefixes exist)."""
    lp = np.asarray(lp, dtype=np.float32)
    T, V = lp.shape
    K = V - 1 if beam_token is None else beam_token
    sc = _Scorer(lm, symbols, word_boundary, lm_weight, word_score, unk_score) if lm is not None else None
    ctx0 = ("<s>",) if lm is not None and lm.order > 1 else ()
    # beam: dict(h, pb, pnb, lm, last, toks (tuple), chars (partial word class ids), ctx)
    beams = [dict(h=0, pb=F32(0.0), pnb=NEG_INF, lm=F32(0.0), last=-1, toks=(), chars=(), ctx=ctx0)]
    for t in range(T):
        row = lp[t]
        order = sorted((c for c in range(V) if c != blank), key=lambda c: (-row[c], c))
        top = np.asarray(sorted(order[:K]), dtype=np.int64)
        # stays, in beam rank order
        stays = []
        for bm in beams:
            pnb = F32(bm["pnb"] + row[bm["last"]]) if bm["last"] >= 0 else NEG_INF
            stays.append(dict(bm, pb=F32(lae(bm["pb"], bm["pnb"]) + row[blank]), pnb=pnb))
        where = {bm["h"]: i for i, bm in enumerate(stays)}
        st_h = np.asarray([bm["h"] for bm in stays], dtype=np.uint64)
        # extensions, by parent rank then class id (vectorised over the classes); one reaching a stay's prefix merges into it
        ext_h, ext_s, ext_j, ext_c = [], [], [], []
        for j, bm in enumerate(beams):
            base = lae(bm["pb"], bm["pnb"])
            h = _mix_np(np.uint64(bm["h"]) ^ (top + 1).astype(np.uint64))
            e = (np.where(top == bm["last"], bm["pb"], base).astype(np.float32) + row[top]).astype(np.float32)
            hit = np.isin(h, st_h)
            for k in np.nonzero(hit)[0]:
                st = stays[where[int(h[k])]]
                st["pnb"] = lae(st["pnb"], e[k])
            keep = ~hit
            lmv = np.full(int(keep.sum()), bm["lm"], dtype=np.float32)
            if sc is not None and bm["chars"]:
                kb = np.nonzero(top[keep] == word_boundary)[0]
                if len(kb):
                    lmv[kb] = F32(bm["lm"] + sc.word(bm["chars"], bm["ctx"])[0])
            ext_h.append(h[keep])
            ext_s.append((e[keep] + lmv).astype(np.float32))
            ext_j.append(np.full(int(keep.sum()), j))
            ext_c.append(top[keep])
        s_st = np.asarray([F32(lae(bm["pb"], bm["pnb"]) + bm["lm"]) for bm in stays], dtype=np.float32)
        all_h = np.concatenate([st_h] + ext_h)
        all_s = np.concatenate([s_st] + ext_s)
        all_j = np.concatenate([np.arange(len(stays))] + ext_j)
        all_c = np.concatenate([np.full(len(stays), -1)] + ext_c)
        pick = np.lexsort((all_h, -all_s))[:beam]
        nxt = []
        for q in pick:
            j, c = int(all_j[q]), int(all_c[q])
            if c < 0:
                nxt.append(stays[j])
                continue
            bm = beams[j]
            e = F32((bm["pb"] if c == bm["last"] else lae(bm["pb"], bm["pnb"])) + row[c])
            l, chars, ctx = bm["lm"], bm["chars"] + (c,), bm["ctx"]
            if sc is not None and c == word_boundary:
                chars = ()
                if bm["chars"]:
                    d, ctx = sc.word(bm["chars"], bm["ctx"])
                    l = F32(l + d)
            nxt.append(dict(h=int(all_h[q]), pb=NEG_INF, pnb=e, lm=l, last=c, toks=bm["toks"] + (c,), chars=chars, ctx=ctx))
        beams = nxt
    out = []
    for bm in beams:
        l = bm["lm"]
        if sc is not None:
            ctx = bm["ctx"]
            if bm["chars"]:
                d, ctx = sc.word(bm["chars"], ctx)
                l = F32(l + d)
            l = F32(l + sc.finish(ctx))
        out.append((list(bm["toks"]), F32(lae(bm["pb"], bm["pnb"]) + l), bm["h"]))
    out.sort(key=lambda x: (-x[1], x[2]))
    return [(tk, s) for tk, s, _ in out[:nbest]]


def ctc_log_likelihood(lp: np.ndarray, labels: Sequence[int], blank: int = 0) -> float:
    """Exact CTC ln P(labels | lp) by the forward algorithm in float64 (for brute-force checks)."""
    lp = np.asarray(lp, dtype=np.float64)
    ext = [blank]
    for c in labels:
        ext += [c, blank]
    L = len(ext)
    a = np.full(L, -np.inf)
    a[0] = lp[0, blank]
    if L > 1:
        a[1] = lp[0, ext[1]]
    for t in range(1, lp.shape[0]):
        n = np.full(L, -np.inf)
        for s in range(L):
            terms = [a[s]]
            if s >= 1:
                terms.append(a[s - 1])
            if s >= 2 and ext[s] != blank and ext[s] != ext[s - 2]:
                terms.append(a[s - 2])
            m = max(terms)
            n[s] = -np.inf if m == -np.inf else m + math.log(sum(math.exp(x - m) for x in terms)) + lp[t, ext[s]]
        a = n
    ends = [a[L - 1]] + ([a[L - 2]] if L > 1 else [])
    m = max(ends)
    return -math.inf if m == -math.inf else m + math.log(sum(math.exp(x - m) for x in ends))


def lm_score(labels: Sequence[int], lm: ArpaLM, symbols, word_boundary: int, lm_weight: float, word_score: float = 0.0,
             unk_score: float = 0.0) -> float:
    """LM part of a whole label sequence under the decoder's semantics (float64 sums of the same fp32 terms)."""
    sc = _Scorer(lm, symbols, word_boundary, lm_weight, word_score, unk_score)
    ctx = ("<s>",) if lm.order > 1 else ()
    total, chars = 0.0, ()
    for c in labels:
        if c == word_boundary:
            if chars:
                d, ctx = sc.word(chars, ctx)
                total += float(d)
            chars = ()
        else:
            chars += (c,)
    if chars:
        d, ctx = sc.word(chars, ctx)
        total += float(d)
    return total + float(sc.finish(ctx))


def write_random_arpa(path, words: Sequence[str], order: int, seed: int, ngrams_per_order: int, with_unk: bool = True):
    """A seeded random ARPA file over `words` (+ <s>, </s> and optionally <unk>): log10 p in [-3, -0.3], backoffs in [-1, 0]
    for every n-gram below the top order; each n-gram of order n >= 2 extends an (n-1)-gram of the file by one word."""
    rng = np.random.default_rng(seed)
    vocab = ["<s>", "</s>"] + (["<unk>"] if with_unk else []) + list(words)
    grams = [{(w,): None for w in vocab}]
    for n in range(2, order + 1):
        prev = list(grams[-1])
        g = {}
        for _ in range(ngrams_per_order * 4):
            if len(g) >= ngrams_per_order:
                break
            base = prev[int(rng.integers(len(prev)))]
            if base[-1] == "</s>":
                continue
            nxt = vocab[1 + int(rng.integers(len(vocab) - 1))]   # never <s> after the start
            g[base + (nxt,)] = None
        grams.append(g)
    lines = ["\\data\\"] + [f"ngram {n}={len(g)}" for n, g in enumerate(grams, 1)] + [""]
    for n, g in enumerate(grams, 1):
        lines.append(f"\\{n}-grams:")
        for ws in g:
            p = -99.0 if ws == ("<s>",) else float(np.round(rng.uniform(-3.0, -0.3), 4))
            ent = f"{p}\t{' '.join(ws)}"
            if n < order and ws[-1] != "</s>":
                ent += f"\t{float(np.round(rng.uniform(-1.0, 0.0), 4))}"
            lines.append(ent)
        lines.append("")
    lines.append("\\end\\")
    with open(path, "w", encoding="utf-8") as f:
        f.write("\n".join(lines) + "\n")


def random_words(letters: str, n: int, seed: int, max_len: int = 6) -> List[str]:
    """n distinct seeded words over `letters`."""
    if n > sum(len(letters) ** k for k in range(1, max_len + 1)):
        raise ValueError(f"fewer than {n} distinct words of at most {max_len} of {len(letters)} letters")
    rng = np.random.default_rng(seed)
    out = {}
    while len(out) < n:
        k = int(rng.integers(1, max_len + 1))
        out["".join(letters[int(i)] for i in rng.integers(0, len(letters), k))] = None
    return list(out)
