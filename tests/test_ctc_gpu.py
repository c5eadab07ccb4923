"""CTC kernels (csrc/ctc.cu) and the CTC fine-tuning surface (unispeech_b200/ctc.py) on the GPU.

Op level: b200s_ctc_stats / _alpha / _beta_grad called directly with every output pre-filled with NaN, against the float64 oracle
(oracle/ctc_oracle.py) evaluated on the SAME bf16 logits; the oracle's gradient comes from torch.autograd through its alpha
recursion, not from the alpha-beta closed form the kernel uses.  Then the autograd wrapper's reductions, and end to end:
HubertCtc / Wav2VecCtc through CtcCriterion against the same model driven by F.log_softmax + F.ctc_loss, best-path decoding, and
the fine-tuning step captured in a CUDA graph."""
import itertools
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import ctc_oracle as CO
from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
EPS32, EPS_BF = 2.0 ** -24, 2.0 ** -8   # half an fp32 ulp; one bf16 ulp (relative)


# ------------------------------------------------------------------------------------------------------------------ helpers
def _logits(T, B, V, layout, seed, dev, scale=2.0):
    """bf16 logits T x B x V: "rows" = the strided view of a [B*T, Vp] buffer (what the fine-tuning wrappers return),
    "contig" = a plain contiguous tensor."""
    g = torch.Generator().manual_seed(seed)
    if layout == "rows":
        Vp = (V + 63) // 64 * 64
        buf = (torch.randn(B * T, Vp, generator=g) * scale).to(BF).to(dev)
        return buf[:, :V].reshape(B, T, V).transpose(0, 1)
    return (torch.randn(T, B, V, generator=g) * scale).to(BF).to(dev)


def _need(targets, tl):
    """Shortest feasible input length per utterance: the labels plus one blank per repeated label."""
    out = []
    for row, n in zip(targets.tolist(), tl):
        out.append(n + sum(1 for i in range(1, n) if row[i] == row[i - 1]))
    return out


def _run(logits, il, targets, tl, blank=0, zero_infinity=False, up=None):
    """The three kernels with NaN-filled outputs.  Returns a dict of device results."""
    from unispeech_b200 import ops
    dev = logits.device
    T, B, V = logits.shape
    fs, bs = logits.stride(0), logits.stride(1)
    Smax = targets.shape[1]
    i32 = lambda v: torch.as_tensor(v, dtype=torch.int32).to(dev).contiguous()  # noqa: E731
    il_d, tg_d, tl_d = i32(il), i32(targets), i32(tl)
    lse = torch.full((B, T), float("nan"), device=dev)
    am = torch.full((B, T), -7, dtype=torch.int32, device=dev)
    la = torch.full((B, T, 2 * Smax + 1), float("nan"), device=dev)
    nll = torch.full((B,), float("nan"), device=dev)
    tot = torch.zeros(1, dtype=torch.float64, device=dev)
    ops.ctc_stats(logits, fs, bs, il_d, B, T, V, lse, am)
    ops.ctc_alpha(logits, fs, bs, lse, il_d, tg_d, Smax, tl_d, B, T, V, blank, zero_infinity, la, nll, tot)
    if bs == T * fs:
        gbuf = torch.full((B * T, fs), float("nan"), dtype=BF, device=dev)
        g, vpad = gbuf[:, :V].reshape(B, T, V).transpose(0, 1), fs
    else:
        gbuf = g = torch.full((T, B, V), float("nan"), dtype=BF, device=dev)
        vpad = V
    up_d = torch.ones(B, device=dev) if up is None else torch.as_tensor(up, dtype=torch.float32).to(dev)
    ops.ctc_beta_grad(logits, fs, bs, lse, il_d, tg_d, Smax, tl_d, B, T, V, blank, la, nll, up_d, g, g.stride(0), g.stride(1), vpad)
    torch.cuda.synchronize()
    return {"lse": lse, "argmax": am, "nll": nll, "total": tot, "grad": g, "gbuf": gbuf, "up": up_d}


def _reference(logits, il, targets, tl, blank, up):
    """float64 oracle on the bf16 logits (padded frames zeroed: the oracle multiplies them by zero, the kernel never reads them)."""
    T, B, V = logits.shape
    x = logits.detach().float().cpu().double()
    valid = torch.arange(T)[:, None] < torch.as_tensor(il)[None, :]
    x = torch.where(valid[:, :, None], x, torch.zeros_like(x)).requires_grad_(True)
    nll = CO.ctc_nll(x, il, targets, tl, blank)
    finite = torch.isfinite(nll)
    if finite.any():
        (nll[finite] * up.cpu().double()[finite]).sum().backward()
    grad = x.grad if x.grad is not None else torch.zeros_like(x)
    return x.detach(), nll.detach(), grad, valid


def _check(logits, il, targets, tl, blank=0, zero_infinity=False, up=None, expect_finite=None):
    T, B, V = logits.shape
    res = _run(logits, il, targets, tl, blank, zero_infinity, up)
    x, nll_ref, g_ref, valid = _reference(logits, il, targets, tl, blank, res["up"])
    # ---- row statistics: fp32 online log-sum-exp of V exactly representable inputs; the first class holding the maximum
    lse, am = res["lse"].cpu().double().t(), res["argmax"].cpu().t()
    lse_ref = torch.logsumexp(x, -1)
    assert (lse - lse_ref)[valid].abs().max().item() <= 16 * EPS32 * max(1.0, lse_ref[valid].abs().max().item())
    first = torch.where(x == x.max(-1, keepdim=True).values, torch.arange(V), torch.tensor(V)).min(-1).values
    assert torch.equal(am[valid].long(), first[valid])
    assert torch.isnan(res["lse"].cpu().t()[~valid]).all() and (am[~valid] == -7).all()   # padded frames: untouched
    # ---- nll: every frame rounds alpha (of magnitude up to |nll|) to fp32 once, and the roundings of the T frames are
    # independent: 4 sqrt(T) half-ulps of |nll| is ~10 standard deviations of that walk; + the final log-add-exp
    nll = res["nll"].cpu().double()
    finite = torch.isfinite(nll_ref)
    if expect_finite is not None:
        assert finite.tolist() == expect_finite
    assert torch.equal(torch.isfinite(nll), finite) and (nll[~finite] == float("inf")).all()
    tol = (4 * math.sqrt(T) + 8) * EPS32 * nll_ref[finite].abs().clamp(min=1.0)
    assert ((nll - nll_ref)[finite].abs() <= tol).all(), ((nll - nll_ref)[finite].abs().max().item(), tol.max().item())
    want_total = nll[finite].sum() if (zero_infinity or bool(finite.all())) else torch.tensor(float("inf"), dtype=torch.float64)
    got_total = res["total"].cpu()[0]
    assert got_total == want_total or abs(got_total - want_total) <= 1e-12 * abs(want_total)   # fp64 sum of B fp32 values
    # ---- gradient
    g = res["grad"].cpu().double()
    gbuf = res["gbuf"].cpu().float()
    assert torch.isfinite(gbuf).all()                                # every element written, nothing read from padding
    assert g[~valid].abs().sum().item() == 0                         # padded frames: exactly zero
    if gbuf.dim() == 2:
        assert gbuf[:, V:].abs().sum().item() == 0                   # padding columns V..Vp: exactly zero
    assert g[:, ~finite].abs().sum().item() == 0                     # infeasible utterance: whole gradient zero
    up_h = res["up"].cpu().double()
    # one bf16 rounding of the result, + the error of gamma = exp(alpha + beta - lp + nll): its exponent carries the same
    # rounding walk as nll (gamma <= 1, so a relative error of gamma is an absolute one), + fast-math exp of the two terms (1e-5)
    fp32_term = ((4 * math.sqrt(T) + 8) * EPS32 * nll_ref.abs().clamp(min=1.0) + 1e-5) * up_h.abs()
    fp32_term = torch.where(finite, fp32_term, torch.zeros_like(fp32_term))
    bound = EPS_BF * g_ref.abs() + fp32_term[None, :, None]
    err = (g - g_ref).abs()
    assert (err <= bound).all(), (err.max().item(), (err - bound).max().item())
    # every valid frame's row sums to ~0 (softmax and the occupancies both sum to 1): V bf16 roundings of entries <= row max
    rows = g.sum(-1).abs()
    row_tol = V * EPS_BF * g.abs().max(-1).values + 2 * fp32_term[None, :]
    assert (rows[valid] <= row_tol[valid]).all(), (rows[valid] - row_tol[valid]).max().item()
    return res, nll_ref


def _targets(B, S, V, blank, seed, lens):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, V - 1, (B, max(S, 1)), generator=g)
    t = t + (t >= blank).long()   # every class but the blank
    return t, list(lens)


# ------------------------------------------------------------------------------------------------------------------ shipped shapes
@pytest.mark.parametrize("T", [499, 999, 1499])
def test_letter_vocabulary_at_utterance_lengths(cuda_device, T):
    """V = 32 (letter dictionary), B = 8, targets up to about T / 3 labels, ragged input lengths, the wrappers' strided layout;
    per-utterance upstream gradients; two runs bit-identical."""
    B, V = 8, 32
    S = T // 3
    tl = [S, S // 2, S - 7, 40, 1, S // 3, S - 1, 0]
    targets, tl = _targets(B, S, V, 0, T, tl)
    need = _need(targets, tl)
    g = torch.Generator().manual_seed(T + 1)
    il = [max(n, int(v)) for n, v in zip(need, torch.randint(T // 2, T + 1, (B,), generator=g))]
    il[0] = T
    logits = _logits(T, B, V, "rows", T + 2, cuda_device)
    up = [1.0, 0.5, 2.0, 1.0, -1.0, 0.25, 1.0, 3.0]
    res, _ = _check(logits, il, targets, tl, up=up, expect_finite=[True] * B)
    again = _run(logits, il, targets, tl, up=up)
    assert torch.equal(res["nll"], again["nll"]) and torch.equal(res["gbuf"], again["gbuf"])


# ------------------------------------------------------------------------------------------------------------------ edges
@pytest.mark.parametrize("V,layout", [(33, "rows"), (33, "contig"), (504, "rows"), (1024, "rows"), (1024, "contig"), (32, "contig")])
def test_vocabulary_sizes_and_layouts(cuda_device, V, layout):
    T, B = 70, 3
    targets, tl = _targets(B, 20, V, 0, V, [20, 11, 3])
    _check(_logits(T, B, V, layout, V + 5, cuda_device), [70, 52, 9], targets, tl, up=[1.0, 2.0, 0.5])


def test_single_class_vocabulary(cuda_device):
    """V = 1: only the blank exists; the empty target has probability 1 (nll 0, zero gradient), any label is infeasible."""
    targets = torch.zeros(2, 1, dtype=torch.long)
    res, _ = _check(_logits(12, 2, 1, "rows", 3, cuda_device), [12, 7], targets, [0, 0], expect_finite=[True, True])
    assert res["nll"].abs().max().item() == 0 and res["grad"].float().abs().max().item() == 0


@pytest.mark.parametrize("layout", ["rows", "contig"])
def test_batch_of_one(cuda_device, layout):
    targets, tl = _targets(1, 30, 32, 0, 9, [30])
    _check(_logits(120, 1, 32, layout, 10, cuda_device), [120], targets, tl)


def test_empty_single_and_repeated_targets(cuda_device):
    """target_len = 0 (all-blank path), one label, and all labels equal (a blank is forced between every pair)."""
    T, B, V = 64, 4, 32
    targets = torch.full((B, 16), 5, dtype=torch.long)
    targets[3] = torch.arange(16) % 3 + 1
    _check(_logits(T, B, V, "rows", 21, cuda_device), [64, 64, 40, 64], targets, [0, 1, 16, 16], expect_finite=[True] * 4)


@pytest.mark.parametrize("zero_infinity", [False, True])
def test_minimum_feasible_length_and_one_below(cuda_device, zero_infinity):
    """Labels (3, 3, 4, 4, 4, 7) need 6 + 3 = 9 frames: exactly 9 is feasible, 8 is not (nll = +inf, gradient zero, left out of the
    sum with zero_infinity); a label outside [0, V) and a target length above Smax are reported the same way."""
    T, B, V = 12, 4, 16
    targets = torch.tensor([[3, 3, 4, 4, 4, 7]] * 4)
    bad = targets.clone()
    bad[2, 1] = V
    res, _ = _check(_logits(T, B, V, "rows", 31, cuda_device), [9, 8, 12, 12], targets, [6, 6, 6, 6], zero_infinity=zero_infinity,
                    expect_finite=[True, False, True, True])
    res = _run(_logits(T, B, V, "rows", 31, cuda_device), [9, 8, 12, 12], bad, [6, 6, 6, 7], zero_infinity=zero_infinity)
    assert torch.isfinite(res["nll"]).tolist() == [True, False, False, False]
    assert res["grad"][:, 1:].float().abs().sum().item() == 0 and torch.isfinite(res["gbuf"].float()).all()
    assert bool(torch.isfinite(res["total"])[0]) == zero_infinity


@pytest.mark.parametrize("layout", ["rows", "contig"])
def test_padded_frames_are_never_read(cuda_device, layout):
    """The row GEMMs skip every utterance's padded tail, so those logits may hold anything: NaN there must not reach the loss, and
    the gradient there is exactly zero."""
    T, B, V = 90, 4, 32
    il = [90, 61, 33, 5]
    logits = _logits(T, B, V, layout, 41, cuda_device)
    valid = (torch.arange(T)[:, None] < torch.tensor(il)[None, :]).to(cuda_device)
    logits.masked_fill_(~valid[:, :, None], float("nan"))
    targets, tl = _targets(B, 12, V, 0, 42, [12, 12, 8, 2])
    _check(logits, il, targets, tl, expect_finite=[True] * 4)


def test_nonzero_blank(cuda_device):
    T, B, V = 80, 3, 32
    for blank in (31, 7):
        targets, tl = _targets(B, 15, V, blank, 50 + blank, [15, 9, 0])
        assert not (targets == blank).any()
        _check(_logits(T, B, V, "rows", 51, cuda_device), [80, 66, 30], targets, tl, blank=blank)


def test_target_length_bound(cuda_device):
    """Smax = 511 (2 * 511 + 1 = 1023 positions, one thread each) runs; 512 fails with an error, nothing is truncated."""
    from unispeech_b200.ctc import MAX_TARGET, ctc_loss
    assert MAX_TARGET == 511
    T, B, V = 1100, 2, 32
    targets, tl = _targets(B, 511, V, 0, 61, [511, 300])
    il = [T, max(_need(targets, tl)[1], 700)]
    assert _need(targets, tl)[0] <= T
    logits = _logits(T, B, V, "rows", 62, cuda_device)
    _check(logits, il, targets, tl, expect_finite=[True, True])
    with pytest.raises(RuntimeError, match="Smax=512"):
        ctc_loss(logits, torch.tensor(il), torch.ones(B, 512, dtype=torch.long), torch.tensor([5, 5]))
    with pytest.raises(RuntimeError, match="V=1025"):
        ctc_loss(_logits(4, 1, 1025, "contig", 1, cuda_device), torch.tensor([4]), torch.ones(1, 2, dtype=torch.long), torch.tensor([2]))


# ------------------------------------------------------------------------------------------------------------------ autograd wrapper
@pytest.mark.parametrize("layout", ["rows", "contig"])
def test_ctc_loss_reductions_and_gradient_layout(cuda_device, layout):
    """ctc_loss(): "sum" / "mean" / "none" against F.ctc_loss's definitions on the oracle's nll; zero_infinity; the gradient arrives
    with the strides of the logits."""
    from unispeech_b200.ctc import ctc_loss
    dev = cuda_device
    T, B, V = 50, 4, 32
    targets, tl = _targets(B, 10, V, 0, 71, [10, 4, 10, 0])
    il = [50, 3, 44, 20]   # utterance 1 is infeasible
    logits = _logits(T, B, V, layout, 72, dev)
    up = torch.ones(B)
    _, nll_ref, g_ref, _ = _reference(logits, il, targets, tl, 0, up)
    finite = torch.isfinite(nll_ref)
    assert finite.tolist() == [True, False, True, True]
    args = (torch.tensor(il).to(dev), targets.to(dev), torch.tensor(tl).to(dev))
    none = ctc_loss(logits, *args, reduction="none").cpu().double()
    assert torch.equal(torch.isfinite(none), finite)
    assert torch.isinf(ctc_loss(logits, *args, reduction="sum"))
    x = logits.detach().requires_grad_(True)
    produced = []
    x.register_hook(lambda g: produced.append((g.stride(), g.dtype)))   # the gradient as the Function hands it to autograd
    s = ctc_loss(x, *args, reduction="sum", zero_infinity=True)
    want = nll_ref[finite].sum()
    assert abs(float(s.detach()) - float(want)) <= 1e-4 * float(want)   # fp32 nll of T = 50 frames, fp64 sum rounded to fp32 once
    s.backward()
    assert produced == [(x.stride(), BF)]
    err = (x.grad.cpu().double() - g_ref).abs()
    assert (err <= EPS_BF * g_ref.abs() + 1e-3).all(), err.max().item()   # the bounds of _check, rounded up
    mean = ctc_loss(logits, *args, reduction="mean", zero_infinity=True)
    z = torch.where(finite, nll_ref, torch.zeros_like(nll_ref))
    want = (z / torch.tensor(tl).clamp(min=1).double()).mean()
    assert abs(float(mean) - float(want)) <= 1e-4 * float(want)
    zn = ctc_loss(logits, *args, reduction="none", zero_infinity=True).cpu()
    assert zn[1].item() == 0 and torch.isfinite(zn).all()


# ------------------------------------------------------------------------------------------------------------------ end to end
def _tiny_ctc_model(kind, dev, V=32):
    from unispeech_b200.ctc import HubertCtc, Wav2VecCtc
    from unispeech_b200.wav2vec2 import Wav2Vec2Config, Wav2Vec2Model
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    w2v = kind == "wav2vec"
    cfg = O.tiny_config(pre_ln=w2v, encoder_embed_dim=256, encoder_attention_heads=4, relative_position_embedding=not w2v,
                        gru_rel_pos=not w2v)
    sd = O.deterministic_state_dict(cfg)
    if w2v:
        m, Model = Wav2Vec2Model(Wav2Vec2Config(vars(cfg))), Wav2VecCtc
    else:
        m, Model = WavLM(WavLMConfig(vars(cfg))), HubertCtc
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys
    torch.manual_seed(0)
    return Model.build_model(m, V, apply_mask=True).to(dev), cfg


def _sample(B, L, lengths, V, dev, seed=0):
    wav, pmask = O.deterministic_waveform(B, L, seed=6, lengths=lengths)
    pad, eos, S = 1, 2, 9
    g = torch.Generator().manual_seed(seed)
    target = torch.full((B, S + 2), pad, dtype=torch.long)
    for b in range(B):
        n = S - 3 * b
        target[b, :n] = torch.randint(3, V, (n,), generator=g)
        target[b, n] = eos
    return {"net_input": {"source": wav.to(dev), "padding_mask": pmask}, "target": target, "id": torch.arange(B)}


@pytest.mark.parametrize("kind", ["hubert", "wav2vec"])
def test_training_step_matches_aten_ctc_on_the_same_model(cuda_device, kind):
    """One training step of a tiny HubertCtc / Wav2VecCtc through CtcCriterion against the same model, same masks, driven by
    F.log_softmax + F.ctc_loss(reduction="sum") on `encoder_out`: both hand `proj`'s backward a gradient rounded to bf16 once, so
    the parameter gradients agree to the library's bf16 bounds (DESIGN.md section 1: cosine > 0.999, norm within 2 %)."""
    from unispeech_b200.ctc import CtcCriterion, prepare_targets
    dev = cuda_device
    V, B, L = 32, 2, 16000
    model, cfg = _tiny_ctc_model(kind, dev, V)
    model.train()
    enc, m = model.w2v_encoder, model.w2v_encoder.w2v_model
    sample = _sample(B, L, [16000, 12000], V, dev)
    crit = CtcCriterion()
    names = ["mask_emb", "post_extract_proj.weight", "encoder.layers.0.fc1.weight"]
    params = dict(m.named_parameters())

    np.random.seed(123)
    loss, sample_size, log = crit(model, sample)
    assert loss.is_cuda and log["loss"].is_cuda and int(sample_size) == 9 + 6 and int(log["ntokens"]) == 15 and log["nsentences"] == 2
    assert "hypotheses" not in log
    loss.backward()
    torch.cuda.synchronize()
    got = {k: params[k].grad.detach().clone() for k in names}
    got["proj.weight"] = enc.proj.weight.grad.detach().clone()
    m.zero_grad_buffer()
    enc.proj.weight.grad = enc.proj.bias.grad = None

    np.random.seed(123)
    out = model(**sample["net_input"])
    tg, tl = prepare_targets(sample["target"], 1, 2)
    in_len = (~out["padding_mask"]).sum(1)
    ref = F.ctc_loss(F.log_softmax(out["encoder_out"].float(), -1), tg.long().to(dev), in_len, tl.long().to(dev), blank=0,
                     reduction="sum")
    ref.backward()
    torch.cuda.synchronize()
    # both read the same bf16 logits; fp32 recursions on both sides
    assert abs(float(loss) - float(ref)) <= 1e-4 * abs(float(ref)), (float(loss), float(ref))
    want = {k: params[k].grad for k in names}
    want["proj.weight"] = enc.proj.weight.grad
    for k in got:
        a, b = got[k].double().flatten(), want[k].double().flatten()
        cos = float((a * b).sum() / (a.norm() * b.norm()))
        rel = abs(float(a.norm() / b.norm()) - 1.0)
        assert cos > 0.999 and rel < 0.02, (k, cos, rel)


@pytest.mark.parametrize("kind", ["hubert", "wav2vec"])
def test_eval_returns_the_best_path(cuda_device, kind):
    from unispeech_b200.ctc import CtcCriterion
    dev = cuda_device
    V, B, L = 32, 2, 16000
    model, cfg = _tiny_ctc_model(kind, dev, V)
    model.eval()
    sample = _sample(B, L, [16000, 12000], V, dev)
    with torch.no_grad():
        loss, _, log = CtcCriterion()(model, sample)
        out = model(**sample["net_input"])
    assert torch.isfinite(loss)
    y = out["encoder_out"].float().cpu()                       # T x B x V
    in_len = (~out["padding_mask"]).sum(1).tolist()
    lp = model.get_normalized_probs(out, log_probs=True)
    assert lp.dtype == torch.float32 and torch.allclose(lp.exp().sum(-1), torch.ones_like(lp[..., 0]), atol=1e-5)
    want = []
    for b in range(B):
        yb = y[:in_len[b], b]
        first = torch.where(yb == yb.max(-1, keepdim=True).values, torch.arange(V), torch.tensor(V)).min(-1).values.tolist()
        want.append([c for c, _ in itertools.groupby(first) if c != 0])
    assert log["hypotheses"] == want
    assert any(len(h) > 0 for h in want)


def test_finetuning_step_captures_in_a_cuda_graph(cuda_device):
    """Fixed-length batch, masks injected as data: encoder -> final_dropout / proj -> ctc_loss -> backward captured once and
    replayed; every replay equals the eager step with the same mask (nothing in the CTC path synchronises or allocates outside
    the graph's pool)."""
    from unispeech_b200.ctc import ctc_loss
    from unispeech_b200.graphed import GraphedForwardBackward
    dev = cuda_device
    V, B, L = 32, 2, 16000
    model, cfg = _tiny_ctc_model("hubert", dev, V)
    model.train()
    enc, m = model.w2v_encoder, model.w2v_encoder.w2v_model
    T = O.num_frames(L, cfg)
    wav, _ = O.deterministic_waveform(B, L, seed=3)
    wav_host = wav.float().pin_memory()
    targets, tl = _targets(B, 10, V, 0, 5, [10, 6])
    il_d = torch.full((B,), T, dtype=torch.int32, device=dev)
    tg_d, tl_d = targets.to(dev).int(), torch.tensor(tl, dtype=torch.int32, device=dev)

    def loss_fn(x):
        for p in enc.proj.parameters():
            if p.grad is not None:
                p.grad.zero_()
        return ctc_loss(enc._tail(x, True), il_d, tg_d, tl_d, reduction="sum")

    g = GraphedForwardBackward(m, loss_fn, B, L, dev).capture()
    np.random.seed(11)
    masks = []
    for step in range(3):
        loss = g.step(wav_host)
        torch.cuda.synchronize()
        mask = g.mask_host.clone()
        masks.append(mask)
        got_loss, got, got_proj = float(loss), m.grad_buffer().detach().clone(), enc.proj.weight.grad.detach().clone()
        m.zero_grad_buffer()
        m._engine.prepared_version = None
        x, _ = m.extract_features(wav.to(dev), padding_mask=None, mask=True, mask_indices=mask)
        ref = loss_fn(x)
        ref.backward()
        torch.cuda.synchronize()
        want, want_proj = m.grad_buffer().detach().clone(), enc.proj.weight.grad.detach().clone()
        # the tolerances of test_graph_gpu.py: the same kernels, fp32 atomics of the encoder's backward in another order
        assert abs(got_loss - float(ref)) <= 2e-3 * max(1.0, abs(float(ref))), (step, got_loss, float(ref))
        scale = want.abs().max().item()
        assert (got - want).abs().max().item() <= 2e-2 * scale, (step, (got - want).abs().max().item(), scale)
        assert (got_proj - want_proj).abs().max().item() <= 2e-2 * want_proj.abs().max().item()
    assert not torch.equal(masks[0], masks[1])
