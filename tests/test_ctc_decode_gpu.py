"""CTC beam-search decoding (csrc/ctc_decode.cu, unispeech_b200.ctc.ctc_beam_search) on the GPU, against brute force and the
numpy oracle (oracle/decode_oracle.py) run on lp = float(logits) - lse built from the kernel's own lse (b200s_ctc_stats).

The oracle uses numpy's fp32 exp / log1p and the kernel CUDA's expf / log1pf; they can differ in the last bit, so where two
prefixes are within an ulp of each other at the beam cutoff the two can keep different ones.  Bit equality is therefore not
asserted against the oracle: top-1 tokens must agree wherever the oracle's top-1 / top-2 gap exceeds 1e-3 (and at least 95 % of
utterances must qualify), and scores to 1e-5 |s| + 1e-3."""
import numpy as np
import pytest
import torch

from oracle import decode_oracle as DO
from unispeech_b200.ngram import NgramLM

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
LETTERS = "ETAONIHSRDLUMWCFGYPBVK'XJQZ"
SYMBOLS32 = ["<s>", "<pad>", "</s>", "<unk>", "|"] + list(LETTERS)   # fairseq's letter dictionary: 32 classes, "|" = 4


def _symbols(V):
    if V <= 5:
        return ["<s>", "|", "A", "B", "C"][:V]
    return (SYMBOLS32 + [f"<x{i}>" for i in range(V)])[:V]   # classes past the letters are multi-character: never spelled


def _logits(T, B, V, seed, dev, scale=3.0, layout="rows"):
    g = torch.Generator().manual_seed(seed)
    Vp = V + 13 if layout == "rows" else V
    buf = (torch.randn(B * T, Vp, generator=g) * scale).to(BF).to(dev)
    if layout == "rows":
        return buf[:, :V].reshape(B, T, V).transpose(0, 1), buf
    return buf.reshape(B, T, V).transpose(0, 1).contiguous(), buf


def _distinct_logits(T, B, V, seed, dev, scale):
    """Rows view of bf16 logits whose V values are distinct within every frame (a repeated bf16 value is moved to the next
    representable one), so that bf16 rounding does not make different hypotheses tie exactly."""
    g = torch.Generator().manual_seed(seed)
    bits = (torch.randn(B * T, V, generator=g) * scale).to(BF).view(torch.int16).numpy().copy()
    for row in bits:
        while True:
            vals = row.view(np.uint16).astype(np.int64)
            order = np.argsort(vals, kind="stable")
            dup = np.nonzero(np.diff(vals[order]) == 0)[0]
            if len(dup) == 0:
                break
            row[order[dup + 1]] += 1   # the next bf16 value away from zero
    buf = torch.zeros(B * T, V + 13, dtype=BF)
    buf[:, :V] = torch.from_numpy(bits).view(BF)
    buf = buf.to(dev)
    return buf[:, :V].reshape(B, T, V).transpose(0, 1)


def _lp(logits, il):
    from unispeech_b200 import ops
    T, B, V = logits.shape
    lse = torch.zeros(B, T, dtype=torch.float32, device=logits.device)
    ops.ctc_stats(logits, logits.stride(0), logits.stride(1), torch.as_tensor(il).to(logits.device).int(), B, T, V, lse, None)
    return (logits.float().transpose(0, 1) - lse[..., None]).cpu().numpy()   # [B, T, V]


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


@pytest.fixture(scope="module")
def small_lm(tmp_path_factory, cuda_device):
    from test_ctc_decode_cpu import ARPA, SYMBOLS
    p = tmp_path_factory.mktemp("lm") / "small.arpa"
    p.write_text(ARPA)
    return NgramLM.from_arpa(p, SYMBOLS, 2), DO.ArpaLM.from_file(p)


def test_brute_force_cases(cuda_device, small_lm):
    from test_ctc_decode_cpu import BRUTE, SYMBOLS, brute_force
    lm_dev, lm_host = small_lm
    for T, seed, with_lm, w, ws, us in BRUTE:
        logits, _ = _logits(T, 1, 3, seed, cuda_device, scale=2.0)
        lp = _lp(logits, [T])[0]
        (best, y), (second, _) = brute_force(lp, lm=lm_host if with_lm else None, lm_weight=w, word_score=ws, unk_score=us)
        got = _rows(_decode(logits, [T], beam_size=128, nbest=1, lm=lm_dev if with_lm else None, lm_weight=w, word_score=ws,
                            unk_score=us))[0][0]
        if best - second > 1e-3:
            assert got[0] == y, (T, seed)
        assert abs(got[1] - best) <= 1e-4, (T, seed, got, best)


@pytest.fixture(scope="module")
def letter_lms(tmp_path_factory, cuda_device):
    """A random 3-gram LM per vocabulary size, over words spelled from the letters that vocabulary has."""
    d = tmp_path_factory.mktemp("lms")
    out = {}
    for V in (5, 32, 300, 1024):
        sym = _symbols(V)
        letters = "ABC" if V == 5 else LETTERS[:12]
        p = d / f"v{V}.arpa"
        DO.write_random_arpa(p, DO.random_words(letters, 30 if V == 5 else 60, seed=V, max_len=3), order=3, seed=V + 1, ngrams_per_order=120)
        out[V] = (NgramLM.from_arpa(p, sym, 1 if V == 5 else 4), DO.ArpaLM.from_file(p), sym, 1 if V == 5 else 4)
    return out


def test_against_oracle(cuda_device, letter_lms, tmp_path_factory):
    """At least 200 seeded utterances over V in {5, 32, 300, 1024}, beam in {1, 8, 32, 128}, with and without the LM, ragged,
    plus 28 with an order-5 LM (the longest context the kernel keeps).
    The logits of a frame are distinct: with V >= 300 bf16 values repeat within a frame, and two hypotheses that differ only in
    two classes of equal logit tie exactly (the tie goes to the smaller hash in both, but it would not count as qualifying)."""
    total = qualified = 0
    for V in (5, 32, 300, 1024):
        for beam in (1, 8, 32, 128):
            for with_lm in (False, True):
                B = 7
                Tmax = int(np.clip(60000 // (V * beam), 6, 40))
                seed = V * 1000 + beam * 10 + with_lm
                rng = np.random.default_rng(seed)
                il = [int(x) for x in rng.integers(1, Tmax + 1, B)]
                il[0] = Tmax
                logits = _distinct_logits(Tmax, B, V, seed, cuda_device, scale=2.0 if V <= 32 else 4.0)
                lp = _lp(logits, il)
                lm_dev, lm_host, sym, wb = letter_lms[V]
                kw = dict(lm_weight=0.7, word_score=0.4, unk_score=-1.5) if with_lm else {}
                got = _rows(_decode(logits, il, beam_size=beam, nbest=1, lm=lm_dev if with_lm else None, **kw))
                for b in range(B):
                    ref = DO.beam_search(lp[b, :il[b]], beam=beam, nbest=2, lm=lm_host if with_lm else None, symbols=sym,
                                         word_boundary=wb, **kw)
                    total += 1
                    s_ref = float(ref[0][1])
                    assert abs(got[b][0][1] - s_ref) <= 1e-5 * abs(s_ref) + 1e-3, (V, beam, with_lm, b, got[b][0], ref[0])
                    if len(ref) == 1 or float(ref[0][1]) - float(ref[1][1]) > 1e-3:
                        qualified += 1
                        assert got[b][0][0] == ref[0][0], (V, beam, with_lm, b)
    # an order-5 LM over six short words, dense enough that four-word contexts occur and back off from 5-grams
    d = tmp_path_factory.mktemp("lm5")
    for V in (5, 32):
        sym, wb = _symbols(V), 1 if V == 5 else 4
        p = d / f"o5_v{V}.arpa"
        DO.write_random_arpa(p, DO.random_words("ABC" if V == 5 else LETTERS[:4], 6, seed=V + 5, max_len=2), order=5, seed=V + 6,
                             ngrams_per_order=1500)
        lm_dev, lm_host = NgramLM.from_arpa(p, sym, wb), DO.ArpaLM.from_file(p)
        assert lm_dev.order == 5
        for beam in (8, 32):
            B, T = 7, 40
            seed = V * 7 + beam
            logits = _distinct_logits(T, B, V, seed, cuda_device, scale=2.0)
            il = [40, 40, 33, 27, 40, 15, 38]
            lp = _lp(logits, il)
            kw = dict(lm_weight=0.7, word_score=0.4, unk_score=-1.5)
            got = _rows(_decode(logits, il, beam_size=beam, nbest=1, lm=lm_dev, **kw))
            for b in range(B):
                ref = DO.beam_search(lp[b, :il[b]], beam=beam, nbest=2, lm=lm_host, symbols=sym, word_boundary=wb, **kw)
                total += 1
                s_ref = float(ref[0][1])
                assert abs(got[b][0][1] - s_ref) <= 1e-5 * abs(s_ref) + 1e-3, (V, beam, "order 5", b, got[b][0], ref[0])
                if len(ref) == 1 or float(ref[0][1]) - float(ref[1][1]) > 1e-3:
                    qualified += 1
                    assert got[b][0][0] == ref[0][0], (V, beam, "order 5", b)
    assert total >= 200 and qualified >= 0.95 * total, (total, qualified)


def test_beam_size_token_and_nbest_against_oracle(cuda_device):
    V, T, B = 32, 30, 4
    logits, _ = _logits(T, B, V, 77, cuda_device)
    il = [30, 25, 12, 1]
    lp = _lp(logits, il)
    got = _rows(_decode(logits, il, beam_size=16, nbest=4, beam_size_token=5))
    for b in range(B):
        ref = DO.beam_search(lp[b, :il[b]], beam=16, nbest=5, beam_token=5)
        for n in range(min(4, len(ref))):
            assert abs(got[b][n][1] - float(ref[n][1])) <= 1e-5 * abs(float(ref[n][1])) + 1e-3
            gap_ok = all(abs(float(ref[n][1]) - float(ref[m][1])) > 1e-3 for m in range(len(ref)) if m != n)
            if gap_ok:
                assert got[b][n][0] == ref[n][0], (b, n)


def test_peaky_logits_equal_greedy(cuda_device):
    from unispeech_b200.ctc import ctc_beam_search, greedy_collapse
    T, B, V = 200, 3, 32
    g = torch.Generator().manual_seed(5)
    x = torch.randn(T, B, V, generator=g)
    lead = torch.randint(0, V, (T, B), generator=g)
    lead[::3] = 0   # plenty of blanks
    x.scatter_(2, lead[..., None], x.max(-1, keepdim=True).values + 10.0)
    logits = x.to(BF).to(cuda_device)
    il = torch.tensor([200, 150, 7], dtype=torch.int32)
    hyp = ctc_beam_search(logits, il.to(cuda_device), beam_size=8)
    want = greedy_collapse(lead.t().int(), il.tolist(), blank=0)
    for b in range(B):
        assert hyp.tokens[b, 0, :int(hyp.lengths[b, 0])].tolist() == want[b]
        assert (hyp.tokens[b, 0, int(hyp.lengths[b, 0]):] == -1).all()


LM_CASE = """
\\data\\
ngram 1=5
ngram 2=3

\\1-grams:
-99\t<s>\t-0.2
-1.0\t</s>
-4.0\t<unk>\t0
-0.5\tCAT\t-0.1
-0.7\tAT\t-0.1

\\2-grams:
-0.3\t<s> CAT
-0.4\tCAT </s>
-0.6\t<s> AT

\\end\\
"""
LM_SYMBOLS = ["<s>", "|", "C", "K", "A", "T"]


def _cat_logits(dev):
    """K slightly ahead of C on frame 1, then A and T: acoustics prefer "KAT" (not in the LM) over "CAT" by 0.2 nats."""
    rows = [[0, -9, -9, -9, -9, -9], [0, -9, 4.8, 5.0, -9, -9], [0, -9, -9, -9, 6, -9], [0, -9, -9, -9, -9, 6],
            [4, -9, -9, -9, -9, -9]]
    return torch.tensor(rows, dtype=torch.float32)[:, None, :].to(BF).to(dev)


def test_lm_semantics(cuda_device, tmp_path):
    from unispeech_b200.ctc import hypotheses_to_words
    dev = cuda_device
    p = tmp_path / "cat.arpa"
    p.write_text(LM_CASE)
    lm = NgramLM.from_arpa(p, LM_SYMBOLS, 1)
    assert lm.dropped == 0 and lm.has_unk
    x = _cat_logits(dev)
    il = [5]

    def words(**kw):
        h = _decode(x, il, beam_size=8, nbest=1, lm=lm, **kw)
        return hypotheses_to_words(h, LM_SYMBOLS, 1)[0][0], float(h.scores[0, 0])

    assert words(lm_weight=0.0)[0] == ["KAT"]
    assert words(lm_weight=0.5)[0] == ["CAT"]
    # unk_score alone (no LM weight) also moves it: KAT is <unk>, CAT is a word
    assert words(lm_weight=0.0, unk_score=-1.0)[0] == ["CAT"]
    # word_score: one word, so the score moves by exactly word_score
    (w0, s0), (w1, s1) = words(lm_weight=0.5), words(lm_weight=0.5, word_score=1.0)
    assert w0 == w1 == ["CAT"] and abs((s1 - s0) - 1.0) < 1e-5
    # </s>: the same LM with P(</s> | CAT) lower by 0.5 (log10) lowers the score by 0.5 ln 10 * lm_weight
    p2 = tmp_path / "cat2.arpa"
    p2.write_text(LM_CASE.replace("-0.4\tCAT </s>", "-0.9\tCAT </s>"))
    lm2 = NgramLM.from_arpa(p2, LM_SYMBOLS, 1)
    s2 = float(_decode(x, il, beam_size=8, lm=lm2, lm_weight=0.5).scores[0, 0])
    assert abs((s0 - s2) - 0.5 * np.log(10) * 0.5) < 1e-4
    # all of it equals the oracle
    lp = _lp(x, il)[0]
    host = DO.ArpaLM.from_file(p)
    for kw in (dict(lm_weight=0.5), dict(lm_weight=0.5, word_score=1.0), dict(lm_weight=0.0, unk_score=-1.0)):
        ref = DO.beam_search(lp, beam=8, lm=host, symbols=LM_SYMBOLS, word_boundary=1, **kw)[0]
        h = _decode(x, il, beam_size=8, lm=lm, **kw)
        assert h.tokens[0, 0, :int(h.lengths[0, 0])].tolist() == ref[0]
        assert abs(float(h.scores[0, 0]) - float(ref[1])) < 1e-4


def test_repeated_symbol_spells_no_known_word(cuda_device, tmp_path):
    """Classes 3 and 5 are both "A": a word is spelled by the first class with each character, so C-(class 5)-T is not the
    LM word CAT but <unk>, in the kernel as in the oracle."""
    sym = ["<s>", "|", "C", "A", "T", "A"]
    p = tmp_path / "cat.arpa"
    p.write_text(LM_CASE)
    lm = NgramLM.from_arpa(p, sym, 1)
    rows = [[0, -9, 6, -9, -9, -9], [0, -9, -9, 0, -9, 8], [0, -9, -9, -9, 6, -9], [4, -9, -9, -9, -9, -9]]
    x = torch.tensor(rows, dtype=torch.float32)[:, None, :].to(BF).to(cuda_device)
    lp = _lp(x, [4])[0]
    host = DO.ArpaLM.from_file(p)
    scores = []
    for kw in (dict(lm_weight=0.0), dict(lm_weight=0.0, unk_score=-1.0), dict(lm_weight=0.5, unk_score=-1.0)):
        h = _decode(x, [4], beam_size=8, lm=lm, **kw)
        ref = DO.beam_search(lp, beam=8, lm=host, symbols=sym, word_boundary=1, **kw)[0]
        assert h.tokens[0, 0, :int(h.lengths[0, 0])].tolist() == ref[0] == [2, 5, 4]
        assert abs(float(h.scores[0, 0]) - float(ref[1])) < 1e-4
        scores.append(float(h.scores[0, 0]))
    assert abs((scores[0] - scores[1]) - 1.0) < 1e-5   # scored as <unk>


def test_lm_without_unk_scores_unk_score_alone(cuda_device, tmp_path):
    text = LM_CASE.replace("-4.0\t<unk>\t0\n", "").replace("ngram 1=5", "ngram 1=4")
    p = tmp_path / "nounk.arpa"
    p.write_text(text)
    lm = NgramLM.from_arpa(p, LM_SYMBOLS, 1)
    assert not lm.has_unk
    x = _cat_logits(cuda_device)
    lp = _lp(x, [5])[0]
    host = DO.ArpaLM.from_file(p)
    for kw in (dict(lm_weight=1.0), dict(lm_weight=1.0, unk_score=-0.1), dict(lm_weight=1.0, unk_score=3.0)):
        ref = DO.beam_search(lp, beam=8, nbest=2, lm=host, symbols=LM_SYMBOLS, word_boundary=1, **kw)
        h = _decode(x, [5], beam_size=8, nbest=2, lm=lm, **kw)
        assert h.tokens[0, 0, :int(h.lengths[0, 0])].tolist() == ref[0][0]
        for n in range(2):
            assert abs(float(h.scores[0, n]) - float(ref[n][1])) < 1e-4


def test_padded_frames_are_never_read(cuda_device, letter_lms):
    V, T, B = 32, 120, 4
    logits, buf = _logits(T, B, V, 31, cuda_device)
    il = [120, 77, 30, 0]
    lm = letter_lms[32][0]
    clean = [t.clone() for t in _decode(logits, il, beam_size=16, nbest=3, lm=lm, lm_weight=0.5)]
    rows = buf.view(B, T, -1)
    for b in range(B):
        rows[b, il[b]:] = float("nan")
    poisoned = _decode(logits, il, beam_size=16, nbest=3, lm=lm, lm_weight=0.5)
    _same(poisoned, clean)
    assert int(clean[1][3, 0]) == 0   # no frames: the empty hypothesis


def test_row_view_equals_contiguous_copy(cuda_device):
    logits, _ = _logits(90, 3, 32, 41, cuda_device)
    il = [90, 60, 45]
    _same(_decode(logits, il, beam_size=32, nbest=2), _decode(logits.contiguous(), il, beam_size=32, nbest=2))


def test_deterministic_and_batch_independent(cuda_device, letter_lms):
    V, T, B = 32, 150, 5
    logits, _ = _logits(T, B, V, 51, cuda_device)
    il = torch.tensor([150, 99, 150, 12, 140], dtype=torch.int32)
    lm = letter_lms[32][0]
    kw = dict(beam_size=32, nbest=2, lm=lm, lm_weight=0.8, word_score=0.2)
    a = [t.cpu() for t in _decode(logits, il, **kw)]
    b = [t.cpu() for t in _decode(logits, il, **kw)]
    _same(a, b)
    for u in range(B):
        n = int(il[u])
        one = [t.cpu()[0] for t in _decode(logits[:n, u:u + 1], il[u:u + 1], **kw)]
        assert torch.equal(one[0][:, :n], a[0][u][:, :n]) and torch.equal(one[1], a[1][u])
        assert torch.equal(one[2].view(torch.int32), a[2][u].view(torch.int32))


def test_cuda_graph_replay_matches_eager(cuda_device, letter_lms):
    from unispeech_b200.ctc import ctc_beam_search
    dev = cuda_device
    logits, _ = _logits(100, 3, 32, 61, dev)
    il = torch.tensor([100, 80, 64], dtype=torch.int32, device=dev)
    kw = dict(beam_size=16, nbest=2, lm=letter_lms[32][0], lm_weight=0.5)
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
    logits.copy_(_logits(100, 3, 32, 62, dev)[0])
    g.replay()
    torch.cuda.synchronize()
    _same(out, ctc_beam_search(logits, il, **kw))


def test_errors_before_any_launch(cuda_device):
    from unispeech_b200 import ops
    from unispeech_b200.ctc import ctc_beam_search
    dev = cuda_device
    T, B, V = 20, 2, 16
    logits, _ = _logits(T, B, V, 71, dev)
    il = torch.full((B,), T, dtype=torch.int32, device=dev)
    with pytest.raises(RuntimeError, match=r"beam=0 outside \[1, 128\]"):
        ctc_beam_search(logits, il, beam_size=0)
    with pytest.raises(RuntimeError, match=r"beam=129 outside \[1, 128\]"):
        ctc_beam_search(logits, il, beam_size=129)
    with pytest.raises(RuntimeError, match=r"nbest=9 outside \[1, beam=8\]"):
        ctc_beam_search(logits, il, beam_size=8, nbest=9)
    with pytest.raises(RuntimeError, match=r"blank=16 outside \[0, V=16\)"):
        ctc_beam_search(logits, il, blank=16)
    with pytest.raises(RuntimeError, match=r"beam_token=16 outside"):
        ctc_beam_search(logits, il, beam_size_token=16)
    big = torch.zeros(T, B, 1025, dtype=BF, device=dev)
    lse = torch.zeros(B, T, device=dev)
    out = (torch.empty(B, 1, T, dtype=torch.int32, device=dev), torch.empty(B, 1, dtype=torch.int32, device=dev),
           torch.empty(B, 1, device=dev))
    ws = torch.empty(ops.ctc_decode_workspace_bytes(B, T, 8), dtype=torch.uint8, device=dev)
    with pytest.raises(RuntimeError, match=r"V=1025 outside \[2, 1024\]"):
        ops.ctc_decode(big, big.stride(0), big.stride(1), lse, il, B, T, 1025, 0, 8, 1, 1024, -1, None, 0.0, 0.0, 0.0, ws, *out)
    small = torch.empty(ops.ctc_decode_workspace_bytes(B, T, 8) - 1, dtype=torch.uint8, device=dev)
    with pytest.raises(RuntimeError, match="workspace of"):
        ops.ctc_decode(logits, logits.stride(0), logits.stride(1), lse, il, B, T, V, 0, 8, 1, V - 1, -1, None, 0.0, 0.0, 0.0,
                       small, *out)
    with pytest.raises(ValueError, match="bf16"):
        ctc_beam_search(logits.float(), il)
    torch.cuda.synchronize()


def test_table_build_reports_collisions(cuda_device):
    """The build kernel never resolves a repeated key silently: the same sequence twice is reported as a collision."""
    from unispeech_b200 import ops
    dev = cuda_device
    seqs = torch.tensor([[1, 2, -1], [3, -1, -1], [1, 2, -1]], dtype=torch.int32, device=dev)
    v = torch.zeros(3, dtype=torch.int32, device=dev)
    keys = torch.zeros(8, dtype=torch.int64, device=dev)
    vals = torch.zeros(8, 2, dtype=torch.int32, device=dev)
    status = torch.zeros(1, dtype=torch.int32, device=dev)
    ops.ctc_lm_table_build(seqs, 3, 3, v, v, keys, vals, status)
    assert int(status.item()) == 1
    assert sorted(int(k) & ((1 << 64) - 1) for k in keys.cpu() if int(k) != 0) == sorted([DO.hash_seq([1, 2]), DO.hash_seq([3])])
