"""Lexicon-constrained CTC beam search without a GPU: the lexicon reader, the trie arrays and the look-ahead against hand-built
values, and the numpy oracle (oracle/lexicon_oracle.py) against brute force over every label sequence."""
import itertools
import math

import numpy as np
import pytest

from oracle import decode_oracle as DO
from oracle import lexicon_oracle as LO
from unispeech_b200 import lexicon as LX
from unispeech_b200 import ngram

LN10 = math.log(10.0)
SYMBOLS = ["-", "|", "A", "B"]   # blank 0, word boundary 1

ARPA = """
\\data\\
ngram 1=6
ngram 2=2

\\1-grams:
-1.0\t<s>\t-0.5
-0.8\t</s>
-1.2\t<unk>
-0.6\tA\t-0.3
-0.7\tB
-0.9\tAB

\\2-grams:
-0.3\t<s> A
-0.4\tA B

\\end\\
"""

LEXICON = "A A |\nB B |\nAB A B |\nBA B A\n"


def _write(tmp_path, text, name):
    p = tmp_path / name
    p.write_text(text)
    return p


def test_parse(tmp_path):
    text = ("A A |\n"          # trailing boundary stripped
            "\n"
            "AB A B |\n"
            "AB A A B |\n"     # a second spelling of AB
            "AA A |\n"         # A's spelling: taken by A, dropped
            "AX A X |\n"       # unknown token
            "A|B A | B\n"      # boundary inside the word
            "A-B A - B\n"      # blank
            "BAR |\n"          # nothing left after the boundary
            "B B\n")           # no trailing boundary
    words, spellings, dropped = LX.parse_lexicon(_write(tmp_path, text, "lex.txt"), SYMBOLS, 1)
    assert words == ["A", "AB", "B"]
    assert spellings == [((2,), 0), ((2, 3), 1), ((2, 2, 3), 1), ((3,), 2)]
    assert dropped == 5
    ref = LO.read_lexicon(_write(tmp_path, text, "lex.txt"), SYMBOLS, 1)
    assert ref == {(2,): "A", (2, 3): "AB", (2, 2, 3): "AB", (3,): "B"}


def test_tokens_map_to_the_first_class_with_that_symbol(tmp_path):
    sym = ["-", "|", "A", "B", "A"]
    words, spellings, _ = LX.parse_lexicon(_write(tmp_path, "AB A B |\n", "lex.txt"), sym, 1)
    assert spellings == [((2, 3), 0)]


@pytest.mark.parametrize("line", ["WORD", "WORD\t"])
def test_malformed_line(tmp_path, line):
    with pytest.raises(ValueError, match=r"lex.txt:3: a lexicon line needs a word and its tokens"):
        LX.parse_lexicon(_write(tmp_path, f"A A |\nB B |\n{line}\n", "lex.txt"), SYMBOLS, 1)


def test_trie_arrays_against_hand_built(tmp_path):
    _, spellings, _ = LX.parse_lexicon(_write(tmp_path, LEXICON, "lex.txt"), SYMBOLS, 1)
    mask, first, word, parent, depth = LX.build_trie(spellings, len(SYMBOLS))
    # BFS: 0 root, 1 "A", 2 "B", 3 "AB", 4 "BA"
    assert mask.dtype == np.uint32 and mask.shape == (5, 1)
    assert mask[:, 0].tolist() == [0b1100, 0b1000, 0b0100, 0, 0]
    assert first[:3].tolist() == [1, 3, 4]
    assert word.tolist() == [-1, 0, 1, 2, 3]
    assert parent.tolist() == [-1, 0, 0, 1, 2] and depth.tolist() == [0, 1, 1, 2, 2]
    # a child is first_child + the mask bits below its class
    for n, sp in enumerate([(), (2,), (3,), (2, 3), (3, 2)]):
        for c in range(len(SYMBOLS)):
            if (mask[n, 0] >> c) & 1:
                ch = int(first[n]) + bin(int(mask[n, 0]) & ((1 << c) - 1)).count("1")
                assert [(), (2,), (3,), (2, 3), (3, 2)][ch] == sp + (c,)


def test_trie_spans_several_mask_words():
    V = 70
    spellings = [((65,), 0), ((3, 69), 1), ((3, 40), 2), ((3,), 3)]
    mask, first, word, _, _ = LX.build_trie(spellings, V)
    assert mask.shape == (5, 3)                              # root, "3", "65", "3 40", "3 69"
    assert mask[0].tolist() == [1 << 3, 0, 1 << 1]           # root: classes 3 and 65
    assert mask[1].tolist() == [0, 1 << 8, 1 << 5]           # "3": classes 40 and 69
    assert first[:2].tolist() == [1, 3] and word.tolist() == [-1, 3, 0, 2, 1]


def test_smear_against_hand_computed(tmp_path):
    order, grams = ngram.parse_arpa(_write(tmp_path, ARPA, "lm.arpa"))
    words = [w[0] for w in grams[0]]
    ids = {w: i for i, w in enumerate(words)}
    start = ngram.start_log_probs(order, grams, words)
    f32 = np.float32
    want = {"A": f32(-0.3), "B": f32(f32(-0.5) + f32(-0.7)), "AB": f32(f32(-0.5) + f32(-0.9)),
            "<unk>": f32(f32(-0.5) + f32(-1.2))}   # <s> A present; the others back off from <s>
    for w, v in want.items():
        assert start[ids[w]] == f32(v * f32(2.302585092994046)), w
    lm = DO.ArpaLM(order, grams)
    for w in want:
        assert start[ids[w]] == lm.prob(w, ("<s>",)), w   # the oracle's order of operations
    _, spellings, _ = LX.parse_lexicon(_write(tmp_path, LEXICON, "lex.txt"), SYMBOLS, 1)
    _, _, widx, parent, depth = LX.build_trie(spellings, len(SYMBOLS))
    lex_words = ["A", "B", "AB", "BA"]
    word = np.asarray([-1] + [ids.get(lex_words[i], -2) for i in widx[1:]], dtype=np.int32)
    s = LX.trie_smear(word, parent, depth, start, start[ids["<unk>"]])
    ln = {w: float(start[ids[w]]) for w in want}
    # root 0; "A": max(A, AB); "B": max(B, BA as <unk>); the leaves their own word
    assert s.tolist() == pytest.approx([0.0, ln["A"], ln["B"], ln["AB"], ln["<unk>"]], abs=0)
    s = LX.trie_smear(word, parent, depth, start, None)   # no <unk>: BA scores 0
    assert s.tolist() == pytest.approx([0.0, ln["A"], 0.0, ln["AB"], 0.0], abs=0)
    ref = LO._Lex(LO.read_lexicon(_write(tmp_path, LEXICON, "lex.txt"), SYMBOLS, 1), lm, 1, 1.0, 0.0, 0.0, "max")
    assert [ref.smear(n) for n in [(), (2,), (3,), (2, 3), (3, 2)]] == s.tolist()[:1] + [ln["A"], ln["B"], ln["AB"], ln["<unk>"]]


def test_lexicon_rejects_bad_arguments(tmp_path):
    p = _write(tmp_path, LEXICON, "lex.txt")
    with pytest.raises(ValueError, match="smearing"):
        LX.Lexicon.from_file(p, SYMBOLS, 1, smearing="logadd", device="cpu")
    with pytest.raises(ValueError, match="word_boundary=4"):
        LX.Lexicon.from_file(p, SYMBOLS, 4, device="cpu")
    lx = LX.Lexicon.from_file(p, SYMBOLS, 1, device="cpu")
    assert lx.nodes == 5 and lx.nbytes == 5 * 16 and lx.dropped == 0 and lx.words == ["A", "B", "AB", "BA"]
    assert lx.word.tolist() == [-1, 0, 1, 2, 3] and not lx.smear.any()


# ------------------------------------------------------------------------------------------------ oracle against brute force
def brute_force(lp, spell, lm, w, ws, us):
    """(best score, best labels), (second score, _) over every label sequence of at most T labels whose words are lexicon
    words: exact CTC likelihood (float64) + LM part."""
    T, V = lp.shape
    res = []
    for n in range(T + 1):
        for labels in itertools.product(range(1, V), repeat=n):
            if any(a == b for a, b in zip(labels, labels[1:])) and 2 * n - 1 > T:
                continue
            lm_part = LO.lm_score(labels, spell, 1, lm, w, ws, us)
            if lm_part is None:
                continue
            ll = DO.ctc_log_likelihood(lp, labels, blank=0)
            if ll > -math.inf:
                res.append((ll + lm_part, list(labels)))
    res.sort(key=lambda x: -x[0])
    return (res[0][0], res[0][1]), (res[1][0] if len(res) > 1 else -math.inf)


BRUTE = [  # (T, seed, with LM, lm_weight, word_score, unk_score)
    (4, 1, False, 0.0, 0.0, 0.0), (5, 2, False, 0.0, 0.5, 0.0), (6, 3, False, 0.0, -0.3, 0.0),
    (4, 4, True, 0.5, 0.0, 0.0), (5, 5, True, 1.0, 0.2, -1.0), (6, 6, True, 0.7, 0.0, -0.5), (6, 7, True, 2.0, 0.3, 0.0),
]


@pytest.mark.parametrize("smearing", ["none", "max"])
def test_oracle_against_brute_force(tmp_path, smearing):
    lm = DO.ArpaLM.from_file(_write(tmp_path, ARPA, "lm.arpa"))
    spell = LO.read_lexicon(_write(tmp_path, LEXICON, "lex.txt"), SYMBOLS, 1)
    for T, seed, with_lm, w, ws, us in BRUTE:
        rng = np.random.default_rng(seed)
        x = (rng.standard_normal((T, 4)) * 2.0).astype(np.float32)
        lp = (x - np.log(np.exp(x.astype(np.float64)).sum(-1, keepdims=True))).astype(np.float32)
        (best, y), second = brute_force(lp, spell, lm if with_lm else None, w, ws, us)
        got = LO.beam_search(lp, beam=128, lexicon=spell, word_boundary=1, lm=lm if with_lm else None, lm_weight=w,
                             word_score=ws, unk_score=us, smearing=smearing)[0]
        if best - second > 1e-3:
            assert got[0] == y, (T, seed)
        assert abs(float(got[1]) - best) <= 1e-4, (T, seed, got, best)
        for toks in [h[0] for h in LO.beam_search(lp, beam=128, nbest=8, lexicon=spell, word_boundary=1, smearing=smearing)]:
            assert LO.lm_score(toks, spell, 1, None, 0.0) is not None   # every word of every hypothesis is a lexicon word


def test_oracle_drops_hypotheses_inside_a_word():
    """The acoustics say "A" then blank, and AB is the only word: "A" is a node of the trie but no word, so that hypothesis is
    dropped at the end, and so is every other one that stops inside a word."""
    spell = {(2, 3): "AB"}
    lp = np.log(np.asarray([[0.05, 0.05, 0.85, 0.05], [0.85, 0.05, 0.05, 0.05]], dtype=np.float32)).astype(np.float32)
    out = LO.beam_search(lp, beam=16, nbest=16, lexicon=spell, word_boundary=1)
    toks = [t for t, _ in out]
    assert [2] not in toks and [] in toks and [2, 3] in toks
    assert all(LO.lm_score(t, spell, 1, None, 0.0) is not None for t in toks)
