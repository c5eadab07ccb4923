"""Lexicon-constrained CTC beam search (csrc/ctc_decode_lex.cu, `ctc_beam_search(..., lexicon=)`) on the GPU, against the numpy
oracle (oracle/lexicon_oracle.py) run on lp = float(logits) - lse built from the kernel's own lse, and against the lexicon-free
kernel where the two must agree.

As in test_ctc_decode_gpu, the oracle's numpy exp / log1p and CUDA's expf / log1pf can differ in the last bit, so bit equality
is not asserted against the oracle: top-1 tokens must agree wherever the oracle's top-1 / top-2 gap exceeds 1e-3 (and at least
95 % of utterances must qualify), and scores to 1e-5 |s| + 1e-3."""
import itertools

import numpy as np
import pytest
import torch

from oracle import decode_oracle as DO
from oracle import lexicon_oracle as LO
from unispeech_b200.lexicon import Lexicon
from unispeech_b200.ngram import NgramLM

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
LETTERS = "ETAONIHSRDLUMWCFGYPBVK'XJQZ"
SYMBOLS32 = ["<s>", "<pad>", "</s>", "<unk>", "|"] + list(LETTERS)   # fairseq's letter dictionary: 32 classes, "|" = 4


def _symbols(V):
    if V <= 5:
        return ["<s>", "|", "A", "B", "C"][:V]
    return (SYMBOLS32 + [f"<x{i}>" for i in range(V)])[:V]


def _boundary(V):
    return 1 if V == 5 else 4


def _alphabet(V):
    """Classes lexicon words are spelled with: letters, and for V >= 300 also classes far into the upper mask words."""
    if V == 5:
        return [2, 3, 4]
    out = list(range(5, 17))
    if V >= 300:
        out += [int(c) for c in np.linspace(40, V - 1, 12).astype(int)]
    return out


def _write_lexicon(path, V, n, seed, max_len=6):
    """n seeded random words (distinct spellings, a few with a second spelling) in the fairseq format, named by their symbols
    joined with '_'; returns the names."""
    sym, alpha = _symbols(V), _alphabet(V)
    rng = np.random.default_rng(seed)
    seen, lines, names = set(), [], []
    while len(names) < n:
        k = int(rng.integers(1, max_len + 1))
        sp = tuple(alpha[int(i)] for i in rng.integers(0, len(alpha), k))
        if sp in seen:
            continue
        seen.add(sp)
        name = "_".join(sym[c] for c in sp)
        names.append(name)
        lines.append(f"{name} {' '.join(sym[c] for c in sp)} |")
        if rng.random() < 0.05:   # a second spelling: the first one with its last class doubled
            sp2 = sp + sp[-1:]
            if sp2 not in seen:
                seen.add(sp2)
                lines.append(f"{name} {' '.join(sym[c] for c in sp2)}")
    path.write_text("\n".join(lines) + "\n")
    return names


def _distinct_logits(T, B, V, seed, dev, scale):
    """Rows view of bf16 logits whose V values are distinct within every frame."""
    g = torch.Generator().manual_seed(seed)
    bits = (torch.randn(B * T, V, generator=g) * scale).to(BF).view(torch.int16).numpy().copy()
    for row in bits:
        while True:
            vals = row.view(np.uint16).astype(np.int64)
            order = np.argsort(vals, kind="stable")
            dup = np.nonzero(np.diff(vals[order]) == 0)[0]
            if len(dup) == 0:
                break
            row[order[dup + 1]] += 1
    buf = torch.zeros(B * T, V + 13, dtype=BF)
    buf[:, :V] = torch.from_numpy(bits).view(BF)
    buf = buf.to(dev)
    return buf[:, :V].reshape(B, T, V).transpose(0, 1), buf


def _lp(logits, il):
    from unispeech_b200 import ops
    T, B, V = logits.shape
    lse = torch.zeros(B, T, dtype=torch.float32, device=logits.device)
    ops.ctc_stats(logits, logits.stride(0), logits.stride(1), torch.as_tensor(il).to(logits.device).int(), B, T, V, lse, None)
    return (logits.float().transpose(0, 1) - lse[..., None]).cpu().numpy()


def _decode(logits, il, **kw):
    from unispeech_b200.ctc import ctc_beam_search
    return ctc_beam_search(logits, torch.as_tensor(il).to(logits.device), **kw)


def _rows(hyp):
    tokens, lengths, scores = (t.cpu() for t in hyp)
    return [[(tokens[b, n, :int(lengths[b, n])].tolist(), float(scores[b, n])) for n in range(tokens.shape[1])]
            for b in range(tokens.shape[0])]


def _same(a, b):
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def _words_ok(tokens, spell, boundary):
    words, cur = [], ()
    for c in list(tokens) + [boundary]:
        if c == boundary:
            if cur:
                words.append(cur)
            cur = ()
        else:
            cur += (c,)
    return all(w in spell for w in words)


LEX_SIZES = {5: 10, 32: 20000, 300: 2000, 1024: 500}


@pytest.fixture(scope="module")
def setups(tmp_path_factory, cuda_device):
    """Per V: a lexicon, a 3-gram and an order-5 LM whose words are partly lexicon words and partly not."""
    d = tmp_path_factory.mktemp("lex")
    out = {}
    for V in (5, 32, 300, 1024):
        sym, wb = _symbols(V), _boundary(V)
        lex = d / f"v{V}.lex"
        names = _write_lexicon(lex, V, LEX_SIZES[V], seed=V, max_len=3 if V == 5 else 6)
        rng = np.random.default_rng(V + 1)
        short = [w for w in names if w.count("_") < 2] or names
        lm_words = list(rng.choice(short, size=min(len(short), 40), replace=False)) + ["NOTALEXICONWORD", "ZZZ"]
        lms = {}
        for order, per in ((3, 150), (5, 1500)):
            if order == 5 and V not in (5, 32):
                continue
            p = d / f"v{V}_o{order}.arpa"
            words = lm_words if order == 3 else lm_words[:6]
            DO.write_random_arpa(p, words, order=order, seed=V + order, ngrams_per_order=per)
            lms[order] = (NgramLM.from_arpa(p, sym, wb), DO.ArpaLM.from_file(p))
        out[V] = dict(sym=sym, wb=wb, path=lex, spell=LO.read_lexicon(lex, sym, wb), lms=lms)
    return out


def _lexicon(st, lm, smearing):
    return Lexicon.from_file(st["path"], st["sym"], st["wb"], lm=lm, smearing=smearing)


def test_against_oracle(cuda_device, setups):
    """V in {5, 32, 300, 1024} x beam in {1, 8, 32, 128} x (no LM, 3-gram) x smearing (none, max), ragged, plus an order-5 LM
    for V in {5, 32} at beams 8 and 32."""
    total = qualified = 0
    cases = [(V, beam, order, sm) for V in (5, 32, 300, 1024) for beam in (1, 8, 32, 128) for order in (0, 3)
             for sm in ("none", "max")]
    cases += [(V, beam, 5, sm) for V in (5, 32) for beam in (8, 32) for sm in ("none", "max")]
    for V, beam, order, sm in cases:
        st = setups[V]
        lm_dev, lm_host = st["lms"][order] if order else (None, None)
        lex = _lexicon(st, lm_dev, sm)
        B = 4
        Tmax = int(np.clip(60000 // (V * beam), 6, 40))
        seed = V * 1000 + beam * 10 + order + (sm == "max")
        rng = np.random.default_rng(seed)
        il = [int(x) for x in rng.integers(1, Tmax + 1, B)]
        il[0] = Tmax
        logits, _ = _distinct_logits(Tmax, B, V, seed, cuda_device, scale=2.0 if V <= 32 else 4.0)
        lp = _lp(logits, il)
        kw = dict(lm_weight=0.7, word_score=0.4, unk_score=-1.5) if order else dict(word_score=0.4)
        got = _rows(_decode(logits, il, beam_size=beam, nbest=1, lm=lm_dev, lexicon=lex, **kw))
        for b in range(B):
            ref = LO.beam_search(lp[b, :il[b]], beam=beam, nbest=2, lexicon=st["spell"], word_boundary=st["wb"], lm=lm_host,
                                 smearing=sm, **kw)
            total += 1
            if not ref:
                assert got[b][0] == ([], float("-inf")), (V, beam, order, sm, b)
                qualified += 1
                continue
            s_ref = float(ref[0][1])
            assert abs(got[b][0][1] - s_ref) <= 1e-5 * abs(s_ref) + 1e-3, (V, beam, order, sm, b, got[b][0], ref[0])
            if len(ref) == 1 or float(ref[0][1]) - float(ref[1][1]) > 1e-3:
                qualified += 1
                assert got[b][0][0] == ref[0][0], (V, beam, order, sm, b)
    assert total >= 200 and qualified >= 0.95 * total, (total, qualified)


def test_beam_size_token_and_nbest_against_oracle(cuda_device, setups):
    st = setups[32]
    lm_dev, lm_host = st["lms"][3]
    lex = _lexicon(st, lm_dev, "max")
    logits, _ = _distinct_logits(30, 4, 32, 77, cuda_device, 2.0)
    il = [30, 25, 12, 1]
    lp = _lp(logits, il)
    kw = dict(lm_weight=0.5, word_score=0.2, unk_score=-1.0)
    got = _rows(_decode(logits, il, beam_size=16, nbest=4, beam_size_token=5, lm=lm_dev, lexicon=lex, **kw))
    for b in range(4):
        ref = LO.beam_search(lp[b, :il[b]], beam=16, nbest=5, beam_token=5, lexicon=st["spell"], word_boundary=4, lm=lm_host, **kw)
        for n in range(min(4, len(ref))):
            assert abs(got[b][n][1] - float(ref[n][1])) <= 1e-5 * abs(float(ref[n][1])) + 1e-3
            if all(abs(float(ref[n][1]) - float(ref[m][1])) > 1e-3 for m in range(len(ref)) if m != n):
                assert got[b][n][0] == ref[n][0], (b, n)
        for n in range(len(ref), 4):
            assert got[b][n] == ([], float("-inf"))


def test_every_word_is_a_lexicon_word(cuda_device, setups):
    st = setups[32]
    lm_dev = st["lms"][3][0]
    g = torch.Generator().manual_seed(3)
    logits = (torch.randn(300, 6, 32, generator=g) * 3.0).to(BF).to(cuda_device)
    il = [300, 250, 200, 150, 100, 7]
    for lm, sm in ((None, "max"), (lm_dev, "none"), (lm_dev, "max")):
        lex = _lexicon(st, lm, sm)
        rows = _rows(_decode(logits, il, beam_size=32, nbest=8, lm=lm, lexicon=lex, lm_weight=0.5, word_score=0.3))
        n_words = 0
        for per in rows:
            for toks, s in per:
                if s == float("-inf"):
                    assert toks == []
                    continue
                assert _words_ok(toks, st["spell"], 4), toks
                n_words += sum(1 for c in toks if c == 4) + 1
        assert n_words > 100


def _all_spellings_lexicon(path, T):
    letters = ["A", "B", "C"]
    lines = []
    for k in range(1, T + 1):
        for sp in itertools.product(letters, repeat=k):
            lines.append(f"{''.join(sp)} {' '.join(sp)} |")
    path.write_text("\n".join(lines) + "\n")


def test_reduces_to_the_lexicon_free_decoder(cuda_device, tmp_path):
    """A lexicon of every spelling of length <= T over the letters, each named by its letters, without look-ahead: every
    non-empty partial word is a word and the LM's unknown spellings score as <unk> in both modes, so the result must be the
    lexicon-free decoder's."""
    sym = ["-", "|", "A", "B", "C"]
    T = 8
    _all_spellings_lexicon(tmp_path / "all.lex", T)
    arpa = tmp_path / "abc.arpa"
    DO.write_random_arpa(arpa, DO.random_words("ABC", 25, seed=4, max_len=3), order=3, seed=5, ngrams_per_order=120)
    lm = NgramLM.from_arpa(arpa, sym, 1)
    lex_lm = Lexicon.from_file(tmp_path / "all.lex", sym, 1, lm=lm, smearing="none")
    lex_free = Lexicon.from_file(tmp_path / "all.lex", sym, 1, smearing="none")
    total = qualified = 0
    for beam in (1, 4, 8, 32, 128):
        for with_lm in (False, True):
            B = 8
            seed = beam * 2 + with_lm
            logits, _ = _distinct_logits(T, B, 5, seed, cuda_device, 2.0)
            il = [int(x) for x in np.random.default_rng(seed).integers(1, T + 1, B)]
            kw = dict(lm=lm, lm_weight=0.8, word_score=0.3, unk_score=-1.0) if with_lm else {}
            nb = min(2, beam)
            want = _rows(_decode(logits, il, beam_size=beam, nbest=nb, **kw))
            got = _rows(_decode(logits, il, beam_size=beam, nbest=nb, lexicon=lex_lm if with_lm else lex_free, **kw))
            for b in range(B):
                total += 1
                s = want[b][0][1]
                assert abs(got[b][0][1] - s) <= 1e-5 * abs(s) + 1e-3, (beam, with_lm, b, got[b], want[b])
                if nb == 1 or want[b][1][1] == float("-inf") or s - want[b][1][1] > 1e-3:
                    qualified += 1
                    assert got[b][0][0] == want[b][0][0], (beam, with_lm, b)
    assert qualified >= 0.95 * total, (total, qualified)


def test_lexicon_picks_the_word_over_a_misspelling(cuda_device, tmp_path):
    """K is slightly ahead of C on frame 1: the lexicon-free best is "KAT", which no lexicon word spells; the lexicon of CAT,
    AT, TACK gives "CAT"."""
    sym = ["<s>", "|", "C", "K", "A", "T"]
    rows = [[0, -9, -9, -9, -9, -9], [0, -9, 4.8, 5.0, -9, -9], [0, -9, -9, -9, 6, -9], [0, -9, -9, -9, -9, 6],
            [4, -9, -9, -9, -9, -9]]
    x = torch.tensor(rows, dtype=torch.float32)[:, None, :].to(BF).to(cuda_device)
    (tmp_path / "l.lex").write_text("CAT C A T |\nAT A T |\nTACK T A C K |\n")
    lex = Lexicon.from_file(tmp_path / "l.lex", sym, 1)
    from unispeech_b200.ctc import hypotheses_to_words
    assert hypotheses_to_words(_decode(x, [5], beam_size=8), sym, 1)[0][0] == ["KAT"]
    h = _decode(x, [5], beam_size=8, lexicon=lex)
    assert hypotheses_to_words(h, sym, 1)[0][0] == ["CAT"]
    ref = LO.beam_search(_lp(x, [5])[0], beam=8, lexicon=LO.read_lexicon(tmp_path / "l.lex", sym, 1), word_boundary=1)[0]
    assert h.tokens[0, 0, :int(h.lengths[0, 0])].tolist() == ref[0] and abs(float(h.scores[0, 0]) - float(ref[1])) < 1e-4


def test_padded_frames_are_never_read(cuda_device, setups):
    st = setups[32]
    lm = st["lms"][3][0]
    lex = _lexicon(st, lm, "max")
    T, B = 120, 4
    logits, buf = _distinct_logits(T, B, 32, 31, cuda_device, 2.0)
    il = [120, 77, 30, 0]
    kw = dict(beam_size=16, nbest=3, lm=lm, lexicon=lex, lm_weight=0.5)
    clean = [t.clone() for t in _decode(logits, il, **kw)]
    rows = buf.view(B, T, -1)
    for b in range(B):
        rows[b, il[b]:] = float("nan")
    _same(_decode(logits, il, **kw), clean)
    assert int(clean[1][3, 0]) == 0


def test_row_view_equals_contiguous_copy(cuda_device, setups):
    st = setups[32]
    lex = _lexicon(st, None, "max")
    logits, _ = _distinct_logits(90, 3, 32, 41, cuda_device, 2.0)
    il = [90, 60, 45]
    _same(_decode(logits, il, beam_size=32, nbest=2, lexicon=lex), _decode(logits.contiguous(), il, beam_size=32, nbest=2,
                                                                               lexicon=lex))


def test_deterministic_and_batch_independent(cuda_device, setups):
    st = setups[32]
    lm = st["lms"][3][0]
    lex = _lexicon(st, lm, "max")
    T, B = 150, 5
    logits, _ = _distinct_logits(T, B, 32, 51, cuda_device, 2.0)
    il = torch.tensor([150, 99, 150, 12, 140], dtype=torch.int32)
    kw = dict(beam_size=32, nbest=2, lm=lm, lexicon=lex, lm_weight=0.8, word_score=0.2)
    a = [t.cpu() for t in _decode(logits, il, **kw)]
    _same(a, [t.cpu() for t in _decode(logits, il, **kw)])
    for u in range(B):
        n = int(il[u])
        one = [t.cpu()[0] for t in _decode(logits[:n, u:u + 1], il[u:u + 1], **kw)]
        assert torch.equal(one[0][:, :n], a[0][u][:, :n]) and torch.equal(one[1], a[1][u])
        assert torch.equal(one[2].view(torch.int32), a[2][u].view(torch.int32))


def test_cuda_graph_replay_matches_eager(cuda_device, setups):
    from unispeech_b200.ctc import ctc_beam_search
    dev = cuda_device
    st = setups[32]
    lm = st["lms"][3][0]
    kw = dict(beam_size=16, nbest=2, lm=lm, lexicon=_lexicon(st, lm, "max"), lm_weight=0.5)
    logits, _ = _distinct_logits(100, 3, 32, 61, dev, 2.0)
    il = torch.tensor([100, 80, 64], dtype=torch.int32, device=dev)
    eager = [t.clone() for t in ctc_beam_search(logits, il, **kw)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ctc_beam_search(logits, il, **kw)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = ctc_beam_search(logits, il, **kw)
    for t in out:
        t.fill_(7)
    g.replay()
    torch.cuda.synchronize()
    _same(out, eager)
    logits.copy_(_distinct_logits(100, 3, 32, 62, dev, 2.0)[0])
    g.replay()
    torch.cuda.synchronize()
    _same(out, ctc_beam_search(logits, il, **kw))


def test_errors_before_any_launch(cuda_device, setups):
    from unispeech_b200 import ops
    dev = cuda_device
    st = setups[32]
    lm = st["lms"][3][0]
    lex = _lexicon(st, lm, "max")
    logits, _ = _distinct_logits(20, 2, 32, 71, dev, 2.0)
    il = torch.full((2,), 20, dtype=torch.int32, device=dev)
    with pytest.raises(ValueError, match="different LM"):
        _decode(logits, il, lexicon=lex)
    with pytest.raises(ValueError, match="different LM"):
        _decode(logits, il, lexicon=_lexicon(st, None, "max"), lm=lm)
    with pytest.raises(ValueError, match="V=32 classes, the logits have 31"):
        _decode(logits[..., :31], il, lexicon=_lexicon(st, None, "max"))
    with pytest.raises(ValueError, match="blank=0, the search has blank=2"):
        _decode(logits, il, lexicon=_lexicon(st, None, "max"), blank=2)
    with pytest.raises(ValueError, match="word_boundary"):
        Lexicon.from_file(st["path"], st["sym"], 5, lm=lm)
    bad = _lexicon(st, None, "max")
    bad.word = bad.word[:-1]
    with pytest.raises(ValueError, match="lexicon array word"):
        _decode(logits, il, lexicon=bad)
    bad = _lexicon(st, None, "max")
    bad.mask = bad.mask.to(torch.int64)
    with pytest.raises(ValueError, match="lexicon array mask"):
        _decode(logits, il, lexicon=bad)
    lx = _lexicon(st, None, "max")
    with pytest.raises(RuntimeError, match=r"beam=129 outside \[1, 128\]"):
        _decode(logits, il, beam_size=129, lexicon=lx)
    with pytest.raises(RuntimeError, match=r"nbest=9 outside \[1, beam=8\]"):
        _decode(logits, il, beam_size=8, nbest=9, lexicon=lx)
    with pytest.raises(RuntimeError, match=r"beam_token=32 outside"):
        _decode(logits, il, beam_size_token=32, lexicon=lx)
    B, T = 2, 20
    lse = torch.zeros(B, T, device=dev)
    out = (torch.empty(B, 1, T, dtype=torch.int32, device=dev), torch.empty(B, 1, dtype=torch.int32, device=dev),
           torch.empty(B, 1, device=dev))
    ws = torch.empty(ops.ctc_decode_workspace_bytes(B, T, 8), dtype=torch.uint8, device=dev)
    with pytest.raises(RuntimeError, match="word_boundary=0 must be a class"):
        ops.ctc_decode_lexicon(logits, logits.stride(0), logits.stride(1), lse, il, B, T, 32, 0, 8, 1, 31, 0, None, 0.0, 0.0,
                               0.0, lx, ws, *out)
    small = torch.empty(ops.ctc_decode_workspace_bytes(B, T, 8) - 1, dtype=torch.uint8, device=dev)
    with pytest.raises(RuntimeError, match="workspace of"):
        ops.ctc_decode_lexicon(logits, logits.stride(0), logits.stride(1), lse, il, B, T, 32, 0, 8, 1, 31, 4, None, 0.0, 0.0,
                               0.0, lx, small, *out)
    torch.cuda.synchronize()
