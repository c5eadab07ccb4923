"""CTC forced alignment (csrc/ctc_align.cu, unispeech_b200.ctc.forced_align / token_spans) on the GPU.

Paths and frame scores are compared bit for bit with torchaudio.functional.forced_align on the CPU, run per utterance on
lp = float(logits) - lse built from the kernel's own lse (b200s_ctc_stats), and the score with the fp32 oracle
(oracle/align_oracle.py) on the same lp."""
import numpy as np
import pytest
import torch

from oracle import align_oracle as AO
from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu
TA = pytest.importorskip("torchaudio.functional")

BF = torch.bfloat16


def _logits(T, B, V, seed, dev, layout="rows", quant=None, scale=3.0):
    """bf16 logits T x B x V: "rows" = the view of a [B*T, Vp] buffer (Vp > V), as the fine-tuning wrappers return it.
    `quant`: round to multiples of it first, which makes exact ties in the recursion common."""
    g = torch.Generator().manual_seed(seed)
    Vp = V + 13 if layout == "rows" else V
    x = torch.randn(B * T, Vp, generator=g) * scale
    if quant is not None:
        x = torch.round(x / quant) * quant
    buf = x.to(BF).to(dev)
    if layout == "rows":
        return buf[:, :V].reshape(B, T, V).transpose(0, 1), buf
    return buf.reshape(B, T, V).transpose(0, 1).contiguous(), buf


def _targets(B, S, V, seed, blank=0, repeat_p=0.1):
    g = np.random.default_rng(seed)
    out = np.zeros((B, S), dtype=np.int64)
    for b in range(B):
        for i in range(S):
            if i > 0 and g.random() < repeat_p:
                out[b, i] = out[b, i - 1]
            else:
                c = int(g.integers(0, V - 1))
                out[b, i] = c + (c >= blank)
    return torch.from_numpy(out)


def _lse(logits, il):
    from unispeech_b200 import ops
    T, B, V = logits.shape
    lse = torch.zeros(B, T, dtype=torch.float32, device=logits.device)
    ops.ctc_stats(logits, logits.stride(0), logits.stride(1), il.to(logits.device).int(), B, T, V, lse, None)
    return lse


def _reference(logits, il, targets, tl, blank=0):
    """Per utterance: torchaudio's CPU forced_align and the oracle's score on lp built from the kernel's lse; infeasible
    utterances get the batch semantics (-1 / 0 / -inf)."""
    T, B, V = logits.shape
    lse = _lse(logits, torch.as_tensor(il)).cpu()
    x = logits.float().cpu()
    labels = torch.full((B, T), -1, dtype=torch.int32)
    fs = torch.zeros(B, T)
    score = torch.full((B,), float("-inf"))
    Smax = targets.shape[1]
    for b in range(B):
        n, s = min(max(int(il[b]), 0), T), int(tl[b])
        if s < 0 or s > Smax:
            continue
        tg = [int(c) for c in targets[b, :s]]
        if not AO.feasible(n, tg, V, blank):
            continue
        if n == 0:
            score[b] = 0.0
            continue
        lp = x[:n, b] - lse[b, :n, None]
        if s == 0:
            labels[b, :n] = blank
            fs[b, :n] = lp[:, blank]
        else:
            p, sc = TA.forced_align(lp[None], torch.tensor([tg], dtype=torch.int32), blank=blank)
            labels[b, :n], fs[b, :n] = p[0], sc[0]
        score[b] = float(AO.viterbi(lp.numpy(), tg, blank)[2])
    return labels, fs, score


def _check(got, want, il):
    labels, fs, score = (t.cpu() for t in got)
    wl, wf, ws = want
    assert torch.equal(labels, wl), (labels != wl).nonzero()[:5]
    assert torch.equal(fs.view(torch.int32), wf.view(torch.int32))
    assert torch.equal(score.view(torch.int32), ws.view(torch.int32)), (score, ws)
    # the score is the sum of the frame scores in another order: |error| <= n * 2^-24 * sum |fs| (sequential fp32 bound)
    for b in range(labels.shape[0]):
        if torch.isfinite(score[b]):
            n = int(il[b])
            s64 = fs[b, :n].double()
            assert abs(float(score[b]) - float(s64.sum())) <= max(n, 1) * 2.0 ** -24 * float(s64.abs().sum()) + 1e-30


def _align(logits, il, targets, tl, blank=0):
    from unispeech_b200.ctc import forced_align
    dev = logits.device
    return forced_align(logits, torch.as_tensor(il).to(dev), targets.to(dev), torch.as_tensor(tl).to(dev), blank=blank)


def _ragged(il, targets, tl, T, dev, V=32, seed=0, quant=None, blank=0):
    logits, _ = _logits(T, len(il), V, seed, dev, quant=quant)
    il, tl = torch.tensor(il, dtype=torch.int32), torch.tensor(tl, dtype=torch.int32)
    got = _align(logits, il, targets, tl, blank)
    want = _reference(logits, il, targets, tl, blank)
    _check(got, want, il)
    return got, want


def test_finetuning_shape_and_valid_paths(cuda_device):
    """B = 8, T = 999, V = 32, about 0.3 labels per frame; decoding each path with greedy_collapse gives the target back."""
    from unispeech_b200.ctc import greedy_collapse
    B, T, V, S = 8, 999, 32, 300
    targets = _targets(B, S, V, seed=1)
    tl = [300, 290, 250, 300, 120, 1, 299, 200]
    il = [999, 999, 900, 999, 500, 3, 998, 999]
    (labels, _, score), _ = _ragged(il, targets, tl, T, cuda_device, V, seed=2)
    hyps = greedy_collapse(labels.cpu(), il, blank=0)
    for b in range(B):
        assert hyps[b] == targets[b, :tl[b]].tolist()
        assert torch.isfinite(score[b])


def test_ragged_lengths_one_two_minimum_and_full(cuda_device):
    T, V = 64, 12
    targets = torch.tensor([[3, 0, 0, 0, 0, 0], [4, 0, 0, 0, 0, 0], [5, 5, 6, 6, 6, 7], [1, 2, 3, 4, 5, 6],
                            [2, 2, 2, 0, 0, 0], [0, 0, 0, 0, 0, 0]])
    tl = [1, 1, 6, 6, 3, 0]
    il = [1, 2, 9, 64, 5, 1]            # 9 = 6 labels + 3 repeats; 5 = 3 labels + 2 repeats
    _ragged(il, targets, tl, T, cuda_device, V, seed=3)


@pytest.mark.parametrize("quant", [1.0, 2.0])
def test_coarse_bf16_logits_with_many_ties(cuda_device, quant):
    B, T, V, S = 6, 300, 8, 60
    targets = _targets(B, S, V, seed=4, repeat_p=0.3)
    tl = [60, 60, 30, 10, 59, 1]
    il = [300, 150, 299, 40, 120, 300]
    _ragged(il, targets, tl, T, cuda_device, V, seed=5, quant=quant)


@pytest.mark.parametrize("S", [1, 511, 512, 4095, 4096, 8191])
def test_transcript_lengths_up_to_the_limit(cuda_device, S):
    """S = 511 is the loss kernels' limit, 512 the first past it; 4095 / 4096 and 8191 straddle the per-thread run widths."""
    from unispeech_b200.ctc import MAX_ALIGN_TARGET
    assert MAX_ALIGN_TARGET == 8191
    B, V = 2, 40
    targets = _targets(B, S, V, seed=S)
    need = [n for n in (AO.min_frames(targets[b].tolist()) for b in range(B))]
    T = need[0] + S // 2 + 3
    il = [T, max(need[1], 1)]
    _ragged(il, targets, [S, S], T, cuda_device, V, seed=S + 1)


def test_long_form(cuda_device):
    """One 10-minute utterance (T = 30 000 frames) with 4 000 labels."""
    T, V, S = 30000, 48, 4000
    targets = _targets(1, S, V, seed=9)
    (labels, _, _), _ = _ragged([T], targets, [S], T, cuda_device, V, seed=10)
    from unispeech_b200.ctc import greedy_collapse
    assert greedy_collapse(labels.cpu(), [T])[0] == targets[0].tolist()


def test_infeasible_utterances_leave_the_others_alone(cuda_device):
    dev = cuda_device
    T, V, blank = 40, 10, 3
    targets = torch.tensor([[1, 2, 4, 5], [1, 1, 1, 1], [1, 2, 3, 4], [1, 10, 2, 4], [1, -2, 2, 4], [5, 6, 7, 8],
                            [5, 6, 7, 8], [7, 7, 8, 9]])
    tl = [4, 4, 4, 4, 4, 5, -1, 4]
    il = [40, 6, 40, 40, 40, 40, 40, 30]   # [1,1,1,1] needs 7 frames; blank label; label >= V; label < 0; tl > Smax; tl < 0
    logits, _ = _logits(T, len(il), V, 11, dev)
    il_t, tl_t = torch.tensor(il, dtype=torch.int32), torch.tensor(tl, dtype=torch.int32)
    labels, fs, score = (t.cpu() for t in _align(logits, il_t, targets, tl_t, blank))
    _check((labels, fs, score), _reference(logits, il_t, targets, tl_t, blank), il_t)
    for b in range(1, 7):
        assert (labels[b] == -1).all() and (fs[b] == 0).all() and score[b] == float("-inf"), b
    for b in (0, 7):
        alone = _align(logits[:, b:b + 1], il_t[b:b + 1], targets[b:b + 1], tl_t[b:b + 1], blank)
        assert torch.equal(alone[0].cpu()[0], labels[b]) and torch.equal(alone[1].cpu()[0].view(torch.int32), fs[b].view(torch.int32))
        assert torch.equal(alone[2].cpu()[0].view(torch.int32), score[b].view(torch.int32))


def test_rows_layout_with_nan_padding_is_never_read(cuda_device):
    """The T x B x V view of a [B*T, Vp] buffer, Vp > V: padded frames and the columns past V hold NaN."""
    dev = cuda_device
    B, T, V, S = 4, 200, 30, 40
    logits, buf = _logits(T, B, V, 12, dev)
    il = [200, 150, 81, 97]
    rows = buf.view(B, T, -1)
    rows[:, :, V:] = float("nan")
    for b in range(B):
        rows[b, il[b]:] = float("nan")
    targets = _targets(B, S, V, seed=13)
    il_t, tl_t = torch.tensor(il, dtype=torch.int32), torch.tensor([40, 40, 40, 40], dtype=torch.int32)
    got = _align(logits, il_t, targets, tl_t)
    _check(got, _reference(logits, il_t, targets, tl_t), il_t)
    assert torch.isfinite(got[1]).all() and torch.isfinite(got[2]).all()


def test_limits_fail_before_any_launch(cuda_device):
    from unispeech_b200 import ops
    from unispeech_b200.ctc import forced_align
    dev = cuda_device
    T, B, V = 20, 2, 16
    logits, _ = _logits(T, B, V, 14, dev)
    il = torch.full((B,), T, dtype=torch.int32, device=dev)
    with pytest.raises(RuntimeError, match=r"Smax=8192 outside \[0, 8191\]"):
        forced_align(logits, il, torch.ones(B, 8192, dtype=torch.int32, device=dev), torch.ones(B, dtype=torch.int32, device=dev))
    with pytest.raises(RuntimeError, match=r"blank=16 outside \[0, V=16\)"):
        forced_align(logits, il, torch.ones(B, 3, dtype=torch.int32, device=dev), torch.ones(B, dtype=torch.int32, device=dev),
                     blank=16)
    big = torch.zeros(T, B, 1025, dtype=BF, device=dev)
    lse = torch.zeros(B, T, device=dev)
    ws = torch.empty(ops.ctc_align_workspace_bytes(B, T, 3), dtype=torch.uint8, device=dev)
    out = (torch.empty(B, T, dtype=torch.int32, device=dev), torch.empty(B, T, device=dev), torch.empty(B, device=dev))
    with pytest.raises(RuntimeError, match=r"V=1025 outside \[1, 1024\]"):
        ops.ctc_align(big, big.stride(0), big.stride(1), lse, il, torch.ones(B, 3, dtype=torch.int32, device=dev), 3,
                      torch.ones(B, dtype=torch.int32, device=dev), B, T, 1025, 0, ws, *out)
    with pytest.raises(ValueError, match="bf16"):
        forced_align(logits.float(), il, torch.ones(B, 3, dtype=torch.int32, device=dev), torch.ones(B, dtype=torch.int32, device=dev))
    with pytest.raises(ValueError, match="unit stride"):
        forced_align(logits.transpose(1, 2).contiguous().transpose(1, 2), il, torch.ones(B, 3, dtype=torch.int32, device=dev),
                     torch.ones(B, dtype=torch.int32, device=dev))
    torch.cuda.synchronize()


def test_deterministic_and_batch_independent(cuda_device):
    dev = cuda_device
    B, T, V, S = 5, 400, 32, 100
    logits, _ = _logits(T, B, V, 15, dev, quant=1.0)
    targets = _targets(B, S, V, seed=16)
    il = torch.tensor([400, 321, 400, 250, 399], dtype=torch.int32)
    tl = torch.tensor([100, 90, 50, 100, 1], dtype=torch.int32)
    a = [t.cpu() for t in _align(logits, il, targets, tl)]
    b = [t.cpu() for t in _align(logits, il, targets, tl)]
    for x, y in zip(a, b):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    for u in range(B):
        one = [t.cpu()[0] for t in _align(logits[:, u:u + 1], il[u:u + 1], targets[u:u + 1], tl[u:u + 1])]
        for x, y in zip(one, a):
            assert torch.equal(x.view(torch.int32), y[u].view(torch.int32)), u


def test_cuda_graph_replay_matches_eager(cuda_device):
    from unispeech_b200.ctc import forced_align
    dev = cuda_device
    B, T, V, S = 3, 300, 32, 80
    logits, _ = _logits(T, B, V, 17, dev)
    targets = _targets(B, S, V, seed=18).to(dev).int()
    il = torch.tensor([300, 280, 200], dtype=torch.int32, device=dev)
    tl = torch.tensor([80, 70, 60], dtype=torch.int32, device=dev)
    eager = [t.clone() for t in forced_align(logits, il, targets, tl)]
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        forced_align(logits, il, targets, tl)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        out = forced_align(logits, il, targets, tl)
    for _ in range(2):
        for t in out:
            t.fill_(7)
        g.replay()
        torch.cuda.synchronize()
        for x, y in zip(out, eager):
            assert torch.equal(x.view(torch.int32), y.view(torch.int32))
    # new inputs in the captured buffers are picked up
    logits.copy_(_logits(T, B, V, 19, dev)[0])
    g.replay()
    torch.cuda.synchronize()
    fresh = forced_align(logits, il, targets, tl)
    for x, y in zip(out, fresh):
        assert torch.equal(x.view(torch.int32), y.view(torch.int32))


def test_wav2vec_ctc_end_to_end(cuda_device):
    """waveform -> Wav2VecCtc (eval) -> get_logits -> forced_align -> token_spans, against torchaudio on the same logits."""
    from unispeech_b200.ctc import Wav2VecCtc, forced_align, token_spans
    from unispeech_b200.wav2vec2 import Wav2Vec2Config, Wav2Vec2Model
    dev = cuda_device
    V, B = 32, 2
    cfg = O.tiny_config(pre_ln=True, encoder_embed_dim=256, encoder_attention_heads=4, relative_position_embedding=False,
                        gru_rel_pos=False)
    m = Wav2Vec2Model(Wav2Vec2Config(vars(cfg)))
    assert not m.load_state_dict(O.deterministic_state_dict(cfg), strict=False).unexpected_keys
    torch.manual_seed(0)
    model = Wav2VecCtc.build_model(m, V).to(dev).eval()
    wav, pmask = O.deterministic_waveform(B, 32000, seed=6, lengths=[32000, 24000])
    with torch.no_grad():
        out = model(source=wav.to(dev), padding_mask=pmask)
    logits = model.get_logits(out)
    il = (~out["padding_mask"]).sum(1).int()
    targets = _targets(B, 12, V, seed=20)
    tl = torch.tensor([12, 9], dtype=torch.int32)
    labels, fs, score = forced_align(logits, il, targets.to(dev), tl.to(dev))
    spans = token_spans(labels, fs, il.tolist())
    want = _reference(logits, il.cpu(), targets, tl)
    _check((labels, fs, score), want, il.cpu())
    for b in range(B):
        n = int(il[b])
        ref = TA.merge_tokens(want[0][b, :n], want[1][b, :n])
        assert [tuple(s) for s in spans[b]] == [(s.token, s.start, s.end, s.score) for s in ref]
        assert [s.token for s in spans[b]] == targets[b, :int(tl[b])].tolist()
