"""CTC beam-search decoding without a GPU: the ARPA parser and backoff scoring against hand-computed values, malformed files and
the limits, word spelling, and the numpy oracle (oracle/decode_oracle.py) against brute force over every label sequence."""
import itertools
import math

import numpy as np
import pytest

from oracle import decode_oracle as DO
from unispeech_b200 import ngram

LN10 = math.log(10.0)

ARPA = """
\\data\\
ngram 1=6
ngram 2=4
ngram 3=1

\\1-grams:
-1.0\t<s>\t-0.5
-0.8\t</s>
-1.2\t<unk>
-0.6\tA\t-0.3
-0.7\tAA\t-0.2
-0.9\tAAA

\\2-grams:
-0.3\t<s> A\t-0.1
-0.4\tA AA
-0.2\tAA </s>
-0.5\tA </s>

\\3-grams:
-0.05\t<s> A AA

\\end\\
"""

SYMBOLS = ["<s>", "A", "|"]   # fairseq letter dictionary order: blank first, word boundary "|"


def _write(tmp_path, text, name="lm.arpa"):
    p = tmp_path / name
    p.write_text(text)
    return p


def test_arpa_parse_and_backoff(tmp_path):
    order, grams = ngram.parse_arpa(_write(tmp_path, ARPA))
    assert order == 3 and [len(g) for g in grams] == [6, 4, 1]
    assert grams[0][("<s>",)] == (-1.0, -0.5) and grams[0][("</s>",)] == (-0.8, 0.0)
    lm = DO.ArpaLM(order, grams)
    cases = [
        ("A", ("<s>",), -0.3),                       # bigram
        ("AA", ("<s>", "A"), -0.05),                 # trigram
        ("AAA", ("<s>", "A"), -0.1 - 0.3 - 0.9),     # bo(<s> A) + bo(A) + p(AAA)
        ("</s>", ("A", "AA"), -0.2),                 # no trigram, "A AA" has no backoff (0), bigram AA </s>
        ("AA", ("<s>",), -0.5 - 0.7),                # bo(<s>) + p(AA)
        ("<unk>", ("AAA",), -1.2),                   # AAA has no backoff entry
        ("A", ("<s>", "<s>", "AA"), -0.2 - 0.6),      # only the last order - 1 words count: bo(AA) + p(A)
    ]
    for w, ctx, want in cases:
        assert abs(float(lm.log10(w, ctx)) - want) < 1e-6, (w, ctx)
        assert abs(float(lm.prob(w, ctx)) - want * LN10) < 1e-5, (w, ctx)


@pytest.mark.parametrize("edit,match", [
    (lambda s: s.replace("\\end\\", ""), "expected \\\\end"),
    (lambda s: s.replace("ngram 2=4", "ngram 2=5"), "header says 5"),
    (lambda s: s.replace("-0.4\tA AA", "x\tA AA"), "bad number"),
    (lambda s: s.replace("-0.4\tA AA", "-0.4\tA AA -0.1 extra"), "needs log10 p"),
    (lambda s: s.replace("-0.8\t</s>\n", "").replace("ngram 1=6", "ngram 1=5").replace("-0.2\tAA </s>\n-0.5\tA </s>\n",
                                                                                      "-0.2\tAA A\n-0.5\tA A\n"),
     "</s> is not a unigram"),
    (lambda s: s.replace("-0.4\tA AA", "-0.4\tA B"), "not a unigram"),
    (lambda s: s.replace("-0.4\tA AA", "-0.4\tAA </s>"), "duplicate 2-gram"),
    (lambda s: s.replace("\\data\\", ""), "no \\\\data"),
    (lambda s: s.replace("ngram 2=4\n", ""), "orders 1..N"),
])
def test_malformed_arpa_raises(tmp_path, edit, match):
    with pytest.raises(ValueError, match=match):
        ngram.parse_arpa(_write(tmp_path, edit(ARPA)))


def test_order_above_five_raises(tmp_path):
    head = "\\data\\\n" + "".join(f"ngram {n}=1\n" for n in range(1, 7)) + "\n"
    body = "".join(f"\\{n}-grams:\n-0.1\t" + " ".join(["A"] * n) + "\n\n" for n in range(1, 7))
    with pytest.raises(ValueError, match="order 6 is above the supported 5"):
        ngram.parse_arpa(_write(tmp_path, head + body + "\\end\\\n"))


def test_unspellable_words_are_dropped_and_counted():
    words = ["<s>", "</s>", "<unk>", "A", "AB", "A-B", "C", "BA"]
    symbols = ["<s>", "<pad>", "</s>", "<unk>", "|", "A", "B", "A"]
    spelled, ids, dropped = ngram.spellings(words, symbols, word_boundary=4)
    assert spelled == [[5], [5, 6], [6, 5]] and ids == [3, 4, 7] and dropped == 2   # "A-B" and "C"; "A" is the first class 5
    # the boundary symbol never spells a character
    assert ngram.spellings(["|A"], ["<s>", "|", "A"], word_boundary=1) == ([], [], 1)


def test_oracle_spelling_rule_matches_the_table_builder():
    """The oracle states the spelling rule on its own; it agrees with the host table builder, including a repeated symbol (a
    later class with the same symbol spells no known word) and a multi-character symbol."""
    words = ["<s>", "</s>", "<unk>", "A", "AB", "A-B", "C", "BA"]
    symbols = ["<s>", "<pad>", "</s>", "<unk>", "|", "A", "B", "A"]
    spelled, ids, _ = ngram.spellings(words, symbols, word_boundary=4)
    table = DO.spelling_table(set(words), symbols, 4)
    assert table == {tuple(s): words[i] for s, i in zip(spelled, ids)}
    assert (7,) not in table and (5,) in table and (3,) not in table


def test_oracle_reader_equals_parser(tmp_path):
    order, grams = ngram.parse_arpa(_write(tmp_path, ARPA))
    lm = DO.ArpaLM.from_file(_write(tmp_path, ARPA))
    assert lm.order == order
    assert lm.p == {ws: np.float32(p) for g in grams for ws, (p, _) in g.items()}
    assert lm.bo == {ws: np.float32(b) for g in grams for ws, (_, b) in g.items()}


def test_hash_is_splitmix64_chain():
    # splitmix64 reference values (Vigna's generator, state += golden gamma, then the mix): seed 0 -> 0xE220A8397B1DCDAF
    assert DO.splitmix64(0) == 0xE220A8397B1DCDAF
    assert DO.hash_seq([]) == 0 and DO.hash_seq([0]) == DO.splitmix64(1)
    assert DO.hash_seq([3, 5]) == DO.splitmix64(DO.splitmix64(4) ^ 6)


def _lp(T, V, seed, scale=2.0):
    x = np.random.default_rng(seed).standard_normal((T, V)).astype(np.float32) * np.float32(scale)
    m = x.max(-1, keepdims=True)
    lse = (m + np.log(np.exp(x - m).sum(-1, keepdims=True))).astype(np.float32)
    return (x - lse).astype(np.float32)


def brute_force(lp, blank=0, lm=None, lm_weight=0.0, word_score=0.0, unk_score=0.0, boundary=2):
    """Every label sequence over the non-blank classes of length <= T: exact CTC log-likelihood + LM part, best two."""
    T, V = lp.shape
    labels = [c for c in range(V) if c != blank]
    scored = []
    for n in range(T + 1):
        for y in itertools.product(labels, repeat=n):
            ll = DO.ctc_log_likelihood(lp, y, blank)
            if ll == -math.inf:
                continue
            if lm is not None:
                ll += DO.lm_score(y, lm, SYMBOLS, boundary, lm_weight, word_score, unk_score)
            scored.append((ll, list(y)))
    scored.sort(key=lambda s: -s[0])
    return scored[0], scored[1]


BRUTE = [  # (T, seed, with LM, lm_weight, word_score, unk_score)
    (1, 0, False, 0, 0, 0), (2, 1, False, 0, 0, 0), (3, 2, False, 0, 0, 0), (4, 3, False, 0, 0, 0), (5, 4, False, 0, 0, 0),
    (6, 5, False, 0, 0, 0), (6, 6, False, 0, 0, 0), (6, 7, True, 0.8, 0.0, 0.0), (6, 8, True, 1.5, 0.3, -0.7),
    (5, 9, True, 0.5, -0.2, 0.4), (6, 10, True, 2.0, 1.0, -2.0), (4, 11, True, 1.0, 0.0, 0.0),
]


@pytest.fixture(scope="module")
def arpa_lm(tmp_path_factory):
    return DO.ArpaLM.from_file(_write(tmp_path_factory.mktemp("lm"), ARPA))


@pytest.mark.parametrize("case", range(len(BRUTE)))
def test_oracle_equals_brute_force(case, arpa_lm):
    """With beam 128 and two non-blank classes nothing is pruned for T <= 6 (at most 127 prefixes), so the oracle's best
    sequence and score are the exact argmax of CTC likelihood + LM part."""
    T, seed, with_lm, w, ws, us = BRUTE[case]
    lp = _lp(T, 3, seed)
    lm = arpa_lm if with_lm else None
    (best, y), (second, _) = brute_force(lp, lm=lm, lm_weight=w, word_score=ws, unk_score=us)
    got = DO.beam_search(lp, beam=128, nbest=2, lm=lm, symbols=SYMBOLS, word_boundary=2, lm_weight=w, word_score=ws,
                         unk_score=us)
    assert abs(float(got[0][1]) - best) <= 1e-5 * abs(best) + 1e-5
    if best - second > 1e-3:
        assert got[0][0] == y
    assert abs(float(got[1][1]) - second) <= 1e-5 * abs(second) + 1e-5


def test_oracle_prunes_to_the_beam_and_orders_ties_by_hash():
    lp = np.full((3, 4), np.float32(-math.log(4.0)), dtype=np.float32)   # every class equally likely: all ties
    got = DO.beam_search(lp, beam=4, nbest=4)
    assert len(got) == 4
    scores = [float(s) for _, s in got]
    assert scores == sorted(scores, reverse=True)
    hashes = [DO.hash_seq(t) for t, s in got if s == got[0][1]]
    assert hashes == sorted(hashes)
