"""fp32 numpy restatement of lexicon-constrained CTC prefix beam search with word n-gram LM scoring and LM look-ahead
(`unispeech_b200.ctc.ctc_beam_search(..., lexicon=)`, csrc/ctc_decode_lex.cu).  This file is the definition of the semantics.

Everything of oracle/decode_oracle.py holds (lp, lae, prefix hash, stays, merges and their order, ranking ties, the backoff LM
term, fp32 order of operations), with these additions:
  * lexicon: each word has one or more spellings, sequences of non-blank classes other than the word boundary (`read_lexicon`:
    tokens by the first class with exactly that symbol, a trailing boundary token stripped, a spelling with an unknown token, the
    blank or a boundary dropped; the first word in file order keeps a spelling).  The spellings' prefixes are the trie's nodes,
    the empty prefix its root;
  * a beam's partial word (its node) is a function of its prefix;
  * extension of beam j by c in T_K: c != boundary only if partial_j + (c,) is a node (also the repeat from pb); c == boundary
    at the root (the empty word: scores nothing); c == boundary at a node that is a spelling of word w: lm += lm_weight *
    ln P(w | ctx) + word_score (+ unk_score when w is not an LM unigram, scored as <unk>, 0 without <unk>), the partial word
    empties and w (or <unk>) joins the context; without an LM only word_score; c == boundary anywhere else is not allowed.
    Every allowed extension is a candidate (no pruning beyond T_K); one reaching a stay's prefix is merged into it;
  * smear(n) = max over the words w spelled by n or by a longer node below it of ln P(w | <s>) (w as above), in the fp32 order
    of `ArpaLM.prob`; smear(root) = 0; 0 everywhere without an LM or with smearing="none";
  * ranking score = lae(pb, pnb) + (lm + lm_weight * smear(node)), each operation rounded to fp32; lm holds completed words;
  * end: a partial word that is a spelling is scored as at a boundary, then lm_weight * ln P(</s> | ctx); at the root only
    </s>; any other partial word drops the hypothesis.  The survivors are sorted by (score desc, hash asc).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence, Tuple

import numpy as np

from oracle.decode_oracle import F32, NEG_INF, ArpaLM, _mix_np, lae


def read_lexicon(path, symbols: Sequence[str], boundary: int, blank: int = 0) -> Dict[Tuple[int, ...], str]:
    """spelling (class ids) -> word, from a `WORD tok tok ...` file (well-formed lines only)."""
    first: Dict[str, int] = {}
    for c, s in enumerate(symbols):
        first.setdefault(s, c)
    out: Dict[Tuple[int, ...], str] = {}
    with open(path, encoding="utf-8") as f:
        for line in f:
            parts = line.split()
            if not parts:
                continue
            word, toks = parts[0], parts[1:]
            if toks and toks[-1] == symbols[boundary]:
                toks = toks[:-1]
            ids = tuple(first.get(t, -1) for t in toks)
            if ids and all(c >= 0 and c != blank and c != boundary for c in ids) and ids not in out:
                out[ids] = word
    return out


class _Lex:
    def __init__(self, spell: Dict[Tuple[int, ...], str], lm: Optional[ArpaLM], boundary, weight, word_score, unk_score,
                 smearing: str):
        self.spell, self.lm, self.boundary = spell, lm, boundary
        self.weight, self.word_score, self.unk_score = F32(weight), F32(word_score), F32(unk_score)
        self.children: Dict[Tuple[int, ...], set] = {(): set()}
        for sp in spell:
            for k in range(1, len(sp) + 1):
                self.children.setdefault(sp[:k - 1], set()).add(sp[k - 1])
                self.children.setdefault(sp[:k], set())
        self.smear_of: Dict[Tuple[int, ...], np.float32] = {}
        if lm is not None and smearing == "max":
            for sp, w in spell.items():
                v = self.start(w)
                for k in range(1, len(sp) + 1):
                    p = sp[:k]
                    if p not in self.smear_of or v > self.smear_of[p]:
                        self.smear_of[p] = v

    def start(self, w):
        """ln P(w | <s>), w as <unk> when the LM does not know it (0 without <unk>)."""
        if w in self.lm.vocab:
            return self.lm.prob(w, ("<s>",))
        return self.lm.prob("<unk>", ("<s>",)) if self.lm.has_unk else F32(0.0)

    def smear(self, node):
        return self.smear_of.get(node, F32(0.0)) if node else F32(0.0)

    def rank_lm(self, l, node):
        return F32(l + F32(self.weight * self.smear(node)))

    def allowed(self, node, top):
        """The classes of `top` (a set) that may extend the partial word `node`, in class order."""
        out = self.children[node] & top
        if self.boundary in top and (not node or node in self.spell):
            out = out | {self.boundary}
        return sorted(out)

    def word(self, node, ctx):
        """(LM part, new context) of ending the word spelled by `node`."""
        w = self.spell[node]
        if self.lm is None:
            return self.word_score, ctx
        oov = w not in self.lm.vocab
        if oov:
            w = "<unk>"
        t = F32(0.0)
        if not oov or self.lm.has_unk:
            t = F32(self.weight * self.lm.prob(w, ctx))
        t = F32(t + self.word_score)
        if oov:
            t = F32(t + self.unk_score)
        n = self.lm.order - 1
        return t, ((ctx + (w,))[-n:] if n > 0 else ())

    def finish(self, ctx):
        return F32(self.weight * self.lm.prob("</s>", ctx)) if self.lm is not None else F32(0.0)


def beam_search(lp: np.ndarray, beam: int, lexicon: Dict[Tuple[int, ...], str], word_boundary: int, nbest: int = 1,
                blank: int = 0, beam_token: Optional[int] = None, lm: Optional[ArpaLM] = None, lm_weight: float = 0.0,
                word_score: float = 0.0, unk_score: float = 0.0, smearing: str = "max"):
    """lp fp32 [T, V]; `lexicon` from `read_lexicon`.  Returns [(tokens list, score fp32)] best first, at most nbest (fewer when
    fewer hypotheses survive)."""
    lp = np.asarray(lp, dtype=np.float32)
    T, V = lp.shape
    K = V - 1 if beam_token is None else beam_token
    lx = _Lex(lexicon, lm, word_boundary, lm_weight, word_score, unk_score, smearing)
    ctx0 = ("<s>",) if lm is not None and lm.order > 1 else ()
    beams = [dict(h=0, pb=F32(0.0), pnb=NEG_INF, lm=F32(0.0), last=-1, toks=(), chars=(), ctx=ctx0)]
    for t in range(T):
        row = lp[t]
        order = sorted((c for c in range(V) if c != blank), key=lambda c: (-row[c], c))
        top = set(order[:K])
        stays = []
        for bm in beams:
            pnb = F32(bm["pnb"] + row[bm["last"]]) if bm["last"] >= 0 else NEG_INF
            stays.append(dict(bm, pb=F32(lae(bm["pb"], bm["pnb"]) + row[blank]), pnb=pnb))
        where = {bm["h"]: i for i, bm in enumerate(stays)}
        # allowed extensions, by parent rank then class id; one reaching a stay's prefix merges into it
        ext = []   # (hash, score, parent, class)
        for j, bm in enumerate(beams):
            cs = np.asarray(lx.allowed(bm["chars"], top), dtype=np.int64)
            if len(cs) == 0:
                continue
            base = lae(bm["pb"], bm["pnb"])
            hs = _mix_np(np.uint64(bm["h"]) ^ (cs + 1).astype(np.uint64))
            for c, h in zip(cs.tolist(), hs.tolist()):
                e = F32((bm["pb"] if c == bm["last"] else base) + row[c])
                if h in where:
                    st = stays[where[h]]
                    st["pnb"] = lae(st["pnb"], e)
                    continue
                if c == word_boundary:
                    l = bm["lm"]
                    if bm["chars"]:
                        l = F32(l + lx.word(bm["chars"], bm["ctx"])[0])
                    r = lx.rank_lm(l, ())
                else:
                    r = lx.rank_lm(bm["lm"], bm["chars"] + (c,))
                ext.append((h, F32(e + r), j, c))
        cand = [(bm["h"], F32(lae(bm["pb"], bm["pnb"]) + lx.rank_lm(bm["lm"], bm["chars"])), i, -1) for i, bm in enumerate(stays)]
        cand += ext
        cand.sort(key=lambda x: (-x[1], x[0]))
        nxt = []
        for h, _, j, c in cand[:beam]:
            if c < 0:
                nxt.append(stays[j])
                continue
            bm = beams[j]
            e = F32((bm["pb"] if c == bm["last"] else lae(bm["pb"], bm["pnb"])) + row[c])
            l, chars, ctx = bm["lm"], bm["chars"] + (c,), bm["ctx"]
            if c == word_boundary:
                chars = ()
                if bm["chars"]:
                    d, ctx = lx.word(bm["chars"], bm["ctx"])
                    l = F32(l + d)
            nxt.append(dict(h=h, pb=NEG_INF, pnb=e, lm=l, last=c, toks=bm["toks"] + (c,), chars=chars, ctx=ctx))
        beams = nxt
    out = []
    for bm in beams:
        chars, ctx, l = bm["chars"], bm["ctx"], bm["lm"]
        if chars and chars not in lexicon:
            continue
        if chars:
            d, ctx = lx.word(chars, ctx)
            l = F32(l + d)
        l = F32(l + lx.finish(ctx))
        out.append((list(bm["toks"]), F32(lae(bm["pb"], bm["pnb"]) + l), bm["h"]))
    out.sort(key=lambda x: (-x[1], x[2]))
    return [(tk, s) for tk, s, _ in out[:nbest]]


def lm_score(labels: Sequence[int], lexicon: Dict[Tuple[int, ...], str], word_boundary: int, lm: Optional[ArpaLM],
             lm_weight: float, word_score: float = 0.0, unk_score: float = 0.0) -> Optional[float]:
    """LM part of a whole label sequence (float64 sums of the same fp32 terms), or None when a word is not in the lexicon."""
    lx = _Lex(lexicon, lm, word_boundary, lm_weight, word_score, unk_score, "none")
    ctx = ("<s>",) if lm is not None and lm.order > 1 else ()
    total, chars = 0.0, ()
    for c in list(labels) + [word_boundary]:
        if c == word_boundary:
            if chars:
                if chars not in lexicon:
                    return None
                d, ctx = lx.word(chars, ctx)
                total += float(d)
            chars = ()
        else:
            chars += (c,)
    return total + float(lx.finish(ctx))
