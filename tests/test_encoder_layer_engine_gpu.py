"""Op-level tests of the encoder layer around its attention, as the engine wires it (Engine.layer_forward / layer_backward):
the LayerNorms (gate-fused, stand-alone, D = 1920), the gru_rel_pos gate, the four projections with their fused epilogues
(bias + residual, bias + GELU storing gelu', gelu' x aux with column sums, two residuals), the weight and bias gradients, the
gate backward, the dropout sites and the ragged-batch rules, at the shipped widths.

Teacher-forced: every forward stage is checked against float64 applied to the kernel's own saved bf16 input (`st`), and every
backward step against float64 applied to the operands the engine handed to the kernel (recorded by wrapping `ops`), so no
bound has to absorb an earlier step's roundings.  The attention itself is only checked to be the kernel called directly on
the saved operands (its numerics are test_encoder_layer_gpu.py's).  Bounds are per element, built from a magnitude reference
(the same computation on absolute values, or the sum of squared terms for long fp32 sums, `acc_tol`), never from max|ref|.
Every buffer the engine allocates with torch.empty starts as NaN, and every parameter gradient starts at BASE.  Parameters are
re-drawn so that every term matters: weights N(0, 1/K), non-zero biases, LayerNorm affine terms 1 +- 0.2 / +-0.1, non-trivial
grep_linear / grep_a.  Ragged batches are checked at valid frames, at the exact values promised for padded frames, and for
parameter gradients that do not depend on the output gradient at padded frames."""
import pytest
import torch

import unispeech_b200.engine as engine_mod
from oracle.wavlm_oracle import HashDropout
from test_conv_stem_gpu import BASE, EPS32, acc_tol, bf16_bound, dgelu64, gelu64, ln_fwd_parts, term_tol, ulp_bf16
from test_encoder_layer_gpu import _summary, check, report  # noqa: F401  (_summary: the module-end table of worst ratios)
from unispeech_b200 import dropout as DR
from unispeech_b200 import ops
from unispeech_b200 import workloads as W

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
GELU_ABS = 2.0 ** -21  # gelu' from the erfc approximation (ptx.cuh gelu_half_erfc): absolute error below 2^-21;
#                        gelu = x - |x| h with the same h: below 2^-21 |x|


# ------------------------------------------------------------------------------------------------------------- models
_MODELS = {}


def model(name, layers, p_drop, dev):
    """The shipped configuration with `layers` encoder layers, parameters re-drawn so that every term of the layer matters."""
    key = (name, layers, p_drop)
    if key not in _MODELS:
        from unispeech_b200.wavlm import WavLM, WavLMConfig
        cfg, _, _ = W.model_config(name)
        cfg = dict(cfg, encoder_layers=layers, dropout=p_drop, activation_dropout=p_drop, attention_dropout=0.0, dropout_input=0.0,
                   encoder_layerdrop=0.0)
        torch.manual_seed(1000 + 7 * layers + int(100 * p_drop) + sum(map(ord, name)))
        m = WavLM(WavLMConfig(cfg))
        with torch.no_grad():
            for lyr in m.encoder.layers:
                a = lyr.self_attn
                for lin in (a.q_proj, a.k_proj, a.v_proj, a.out_proj, lyr.fc1, lyr.fc2):
                    lin.weight.normal_(0.0, lin.weight.shape[1] ** -0.5)
                    lin.bias.normal_(0.0, 0.5)
                for ln in (lyr.self_attn_layer_norm, lyr.final_layer_norm):
                    ln.weight.normal_(1.0, 0.2)
                    ln.bias.normal_(0.0, 0.1)
                if getattr(a, "grep_linear", None) is not None:
                    a.grep_linear.weight.normal_(0.0, 0.3)
                    a.grep_linear.bias.normal_(0.0, 0.5)
                    a.grep_a.uniform_(0.5, 1.5)
                if getattr(a, "relative_attention_bias", None) is not None:
                    a.relative_attention_bias.weight.normal_(0.0, 0.5)
        m.dropout_seed = 12345
        _MODELS[key] = m.to(dev).train()
    return _MODELS[key]


class _NanEmpty:
    """Stands in for `torch` inside the engine: floating tensors from `empty` start as NaN, so an element no kernel writes
    fails the test.  Everything else is torch."""

    def __init__(self, t):
        self._t = t

    def __getattr__(self, name):
        return getattr(self._t, name)

    def empty(self, *shape, **kw):
        out = self._t.empty(*shape, **kw)
        if out.is_floating_point():
            out.fill_(float("nan"))
        return out


def record(monkeypatch, log):
    """Copies of the operands the engine hands to the backward kernels, in call order per op."""
    def wrap(name, before, after):
        orig = getattr(ops, name)

        def f(*a, **kw):
            b = before(*a, **kw)
            orig(*a, **kw)
            log.setdefault(name, []).append((b, after(*a, **kw)))
        monkeypatch.setattr(ops, name, f)

    cl = lambda t: None if t is None else t.clone()
    wrap("gemm_rows", lambda *a, **kw: a[0].clone(), lambda *a, **kw: a[8].clone())
    wrap("gemm_wgrad", lambda *a, **kw: (a[0].clone(), a[3]), lambda *a, **kw: None)
    wrap("layer_norm_bwd", lambda *a, **kw: (a[0].clone(), cl(a[10])), lambda *a, **kw: a[13].clone())
    wrap("colsum", lambda *a, **kw: a[0].clone(), lambda *a, **kw: None)
    wrap("gate_bwd", lambda *a, **kw: a[9].clone(), lambda *a, **kw: a[10].clone())
    wrap("dropout_rows", lambda *a, **kw: a[0].clone(), lambda *a, **kw: a[6].clone())
    wrap("attn_bwd_fused", lambda *a, **kw: [cl(t) for t in a[:7]] + [cl(a[11])],
         lambda *a, **kw: (a[9].clone(), cl(a[10]), cl(a[11])))


# ------------------------------------------------------------------------------------------------------------- references
def sum_tol(sq, n):
    """Bound on the fp32 error of a sum over n frames (weight and bias gradients, the LayerNorm and gate parameter gradients)
    whose squared terms sum to `sq`: 128 EPS32 sqrt(n sq), half of acc_tol.  Those sums run as stream-K pieces, 64-row
    blocks and per-tile atomics in any order; their errors are independent roundings of partial sums that stay within a few
    sqrt(sq), so the total is a few EPS32 sqrt(n sq).  The worst seen over every case here is 2^-18.5 sqrt(n sq) (d qkv
    weight, base 16 x 749): this bound keeps a margin near 3.  A tile, block or row summed twice or not at all moves a sum
    by whole terms, sqrt(rows / n) of its size, far above the bound.  The column sums (bias gradients, d beta, d grep_linear
    .bias) realise much less than the weight gradients (one fp32 add per 32 or 64 rows before the atomics) and sit between
    2^-9 and 2^-7 of this bound; it is kept because any order of the atomics may occur."""
    return 0.5 * acc_tol(sq, n)


def mm_ref(a, w, bias=None, res=()):
    """a w^T [+ bias] [+ residuals] in float64, and the fp32 error bound of the GEMM epilogue that computes it: the K-long
    fp32 accumulation (acc_tol) plus a few roundings of the bias / residual adds."""
    ref = a @ w.t()
    tol = acc_tol((a * a) @ (w * w).t(), a.shape[1])
    extra = 0.0
    if bias is not None:
        ref = ref + bias
        extra = extra + bias.abs()
    for r in res:
        ref = ref + r
        extra = extra + r.abs()
    return ref, tol + 4 * EPS32 * (ref.abs() + extra)


def ln_err(x, mean, r):
    """Bound on the error of the kernel's fp32 xh = (x - mean) rstd: the subtraction and the product (a few EPS32 of
    r (|x| + |mean|)), the stored mean (2^-18 of mean |x|) and the relative error of the stored rstd."""
    ym = x.abs().mean(1, keepdim=True)
    xh = (x - mean) * r
    return r * (4 * EPS32 * (x.abs() + mean.abs()) + 2.0 ** -18 * ym) + xh.abs() * (2.0 ** -18 + 16 * EPS32 * ym * r)


def check_ln_fwd(rep, tag, x, ln, y_k, mean_k, rstd_k):
    g, b = ln.weight.detach().double(), ln.bias.detach().double()
    mean, r, xh, z = ln_fwd_parts(x, g, b)
    ym = x.abs().mean(1)
    D = x.shape[1]
    # mean: fp32 sums of D / 32 exact bf16 values per lane, a 5-level shuffle tree (and up to 8 warps), times 1 / D; a
    # recursive sum of n terms is off by at most (n - 1) EPS32 of the sum of |terms|
    tm = (D / 32 + 8) * EPS32 * ym
    check(rep, "ln mean", tag, mean_k, mean[:, 0], tm)
    # rstd: the two-pass variance is a sum of squares (every term >= 0): (x - mean) and its square round once each, the sum
    # as above, the 1 / D scaling and the eps add once more, so var is within (D / 32 + 12) EPS32 relative; rsqrtf (2 ulp)
    # adds 2^-22 and halves the rest.  The mean's error enters the variance only squared: (tm r)^2.  (eps = 1e-6 instead of
    # 1e-5 moves rstd by 4.5e-6 / var relative: 2x this bound or more at var <= 1.4 for D <= 1024, and the DC regime has rows
    # with var < 0.1.)
    rr = r[:, 0]
    check(rep, "ln rstd", tag, rstd_k, rr, rr * (0.5 * (D / 32 + 12) * EPS32 + 2.0 ** -22 + (tm * rr) ** 2))
    # y = xh gamma + beta: the error of xh times |gamma|, two fp32 roundings, one bf16 store
    check(rep, "ln y", tag, y_k, z, bf16_bound(z, g.abs() * ln_err(x, mean, r) + 2 * EPS32 * (xh.abs() * g.abs() + b.abs())))


def gate_parts(y, w, b, a, H):
    """gru_rel_pos gate of rows y [R, D] (float64): the gate [R, H], the two sigmoids and the error bound of the kernel's
    fp32 sigmoid arguments: weight rows pre-summed in fp32 (3 adds), a 64-long dot product as 2 or 8 fmas per lane and a 3-
    or 5-level shuffle tree, the bias add: at most 16 roundings, 16 EPS32 of the sum of |terms|."""
    R, D = y.shape
    q = y.view(R, H, D // H)
    s = (q @ w.t() + b).view(R, H, 2, 4).sum(-1)
    ga, gb = torch.sigmoid(s[..., 0]), torch.sigmoid(s[..., 1])
    aa = a.view(1, H)
    gate = ga * (gb * aa - 1.0) + 2.0
    wa, wb = w.abs()[:4].sum(0), w.abs()[4:].sum(0)
    es = 16 * EPS32 * (q.abs() @ wa + b[:4].abs().sum() + q.abs() @ wb + b[4:].abs().sum())
    return gate, ga, gb, es


def check_gate(rep, tag, y, attn, H, gate_k):
    """gate_k: [R, H] kernel gate of rows y (float64 of the bf16 tensor the kernel read)."""
    w, b, a = (t.detach().double() for t in (attn.grep_linear.weight, attn.grep_linear.bias, attn.grep_a))
    gate, ga, gb, es = gate_parts(y, w, b, a, H)
    # sigmoid' <= 1/4 of the argument errors, |d gate / d ga| <= |a| + 1, |d gate / d gb| <= |a|; __expf and the divide
    # a few 2^-22 of each sigmoid
    A = a.view(1, H).abs()
    # (this worst case of the dot product stays far from what a 64-term sum of random-sign terms realises, so the family sits
    # near 2^-7 of its bound; a gate from the wrong grep_* or the wrong input row is off by O(1): the post-LN hand-off built
    # from the producing layer's grep_* fails here)
    check(rep, "gate", tag, gate_k, gate, (A + 1.0) * (0.25 * es + 2.0 ** -20) * 2)


def rows_of(t, idx):
    """[B, T, ...] -> rows idx of the flattened [B*T, ...] as float64."""
    return t.reshape(-1, *t.shape[2:])[idx].double()


def gate_rows(gate, idx):
    B, H, T = gate.shape
    return gate.permute(0, 2, 1).reshape(B * T, H)[idx].double()


def keep_mask(drop, idx_layer, which, R, N, p, dev):
    k = HashDropout(drop.seed).keep_rows(HashDropout.layer_site(idx_layer, which), R, N, p)
    return torch.from_numpy(k).to(dev)


def bits_equal(a, b):
    if a is None or b is None:
        return a is None and b is None
    it = {BF: torch.int16, F32: torch.int32}[a.dtype]
    return torch.equal(a.view(it), b.view(it))


# ------------------------------------------------------------------------------------------------------------- one case
def run_case(dev, monkeypatch, name, layers, B, T, lengths, regime, p_drop):
    m = model(name, layers, p_drop, dev)
    cfg = m.cfg
    D, Fd, H = cfg.encoder_embed_dim, cfg.encoder_ffn_embed_dim, cfg.encoder_attention_heads
    hd = D // H
    pre_ln = cfg.layer_norm_first
    tag0 = f"{name} B{B} T{T}{' ragged' if lengths else ''} {regime}{' drop' if p_drop else ''}"
    eng = m._begin(dev)
    d = eng.active_drop()
    assert (d is not None) == (p_drop > 0)
    g = torch.Generator().manual_seed(B * 1009 + T)
    x = torch.randn(B, T, D, generator=g)
    if regime == "dc":  # a residual stream with a per-row DC offset and scale (the growing pre-LN residual of WavLM-Large)
        sc = torch.exp(torch.empty(B, T, 1).uniform_(-2.3, 4.6, generator=g))  # 0.1 .. 100: variances 0.01 .. 10^4
        x = x * sc + torch.empty(B, T, 1).uniform_(-100.0, 100.0, generator=g)
    x = x.to(BF).to(dev)
    if regime == "wide":  # fc1 pre-activations over +-6 and beyond: GELU and GELU' across their whole curve
        saved = [lyr.fc1.weight.detach().clone() for lyr in m.encoder.layers]
        with torch.no_grad():
            for lyr in m.encoder.layers:
                lyr.fc1.weight.mul_(3.0)
        eng.prepare()
    try:
        _run(dev, monkeypatch, m, eng, cfg, D, Fd, H, hd, pre_ln, tag0, d, x, B, T, lengths)
    finally:
        if regime == "wide":
            with torch.no_grad():  # (copied back: mul_(3) then div_(3) is not exact in fp32)
                for lyr, w0 in zip(m.encoder.layers, saved):
                    lyr.fc1.weight.copy_(w0)


def _run(dev, monkeypatch, m, eng, cfg, D, Fd, H, hd, pre_ln, tag0, d, x, B, T, lengths):
    rep = {}
    layers = len(m.encoder.layers)
    p_h = d.p if d is not None else 0.0
    p_act = d.p_act if d is not None else 0.0
    lens = lengths if lengths is not None else (T,) * B
    vm = torch.arange(T)[None, :] < torch.tensor(lens)[:, None]  # [B, T] valid frames
    idx = vm.flatten().nonzero()[:, 0].to(dev)
    pidx = (~vm).flatten().nonzero()[:, 0].to(dev)
    R = int(idx.numel())
    rag = pad = None
    if lengths is not None:
        rag = torch.tensor(lens, dtype=torch.int32, device=dev)
        pad = (~vm).to(torch.uint8).contiguous().to(dev)
    tab = None
    if cfg.relative_position_embedding:
        tab = m.encoder._make_bias_state(T, dev)["tab"]
    scale = hd ** -0.5

    # ---- the engine's bf16 operands are bf16(master), bit for bit
    for li, lyr in enumerate(m.encoder.layers):
        a, w = lyr.self_attn, eng.lw[li]
        qkv_m = torch.cat([a.q_proj.weight, a.k_proj.weight, a.v_proj.weight], 0).detach()
        for key, master in (("qkv", qkv_m), ("o", a.out_proj.weight), ("w1", lyr.fc1.weight), ("w2", lyr.fc2.weight)):
            want = master.detach().to(BF)
            assert bits_equal(w[key], want), f"{tag0}: layer {li} operand {key}"
            assert bits_equal(w[key + "T"], want.t().contiguous()), f"{tag0}: layer {li} operand {key}T"

    # ---- forward, every buffer the engine allocates starting as NaN
    monkeypatch.setattr(engine_mod, "torch", _NanEmpty(torch))
    eng._pending_gate = None
    sts, h = [], x
    for li in range(layers):
        h, st = eng.layer_forward(li, h, pad, tab, True, rag=rag)
        sts.append((h, st))
    eng._pending_gate = None
    monkeypatch.undo()
    torch.cuda.synchronize()

    pad_fail = []
    for li, (out, st) in enumerate(sts):
        tag = f"{tag0} layer {li}"
        lyr = m.encoder.layers[li]
        a = lyr.self_attn
        w = {k: eng.lw[li][k].double() for k in ("qkv", "o", "w1", "w2")}
        xin = rows_of(st["x"], idx)
        if pre_ln:
            check_ln_fwd(rep, tag + " LN1", xin, lyr.self_attn_layer_norm, rows_of(st["xn"], idx), st["mean1"][idx], st["rstd1"][idx])
        attn_in = st["xn"] if pre_ln else st["x"]
        ain = rows_of(attn_in, idx)
        if st["gate"] is not None:
            check_gate(rep, tag, ain, a, H, gate_rows(st["gate"], idx))
        # qkv = xn Wqkv^T + b
        ref, tol = mm_ref(ain, w["qkv"], eng.lw[li]["bqkv"].double())
        check(rep, "qkv", tag, rows_of(st["qkv"], idx), ref, bf16_bound(ref, tol))
        # attention: the kernel called directly on the saved operands (scale, head width, gate, table and key mask wiring)
        ao2 = torch.full_like(st["ao"], float("nan"))
        lse2 = torch.full_like(st["lse"], float("nan"))
        ops.attn_fwd(st["qkv"], st["gate"], tab, pad, ao2, lse2, B, T, H, scale, head_dim=hd)
        torch.cuda.synchronize()
        assert bits_equal(st["ao"], ao2) and bits_equal(st["lse"], lse2), f"{tag}: attention output is not the direct call's"
        # y1 = x + dropout1(ao Wo^T + bo)
        ao = rows_of(st["ao"], idx)
        if p_h > 0:
            keep = keep_mask(d, li, DR.L_DROPOUT1, B * T, D, p_h, dev)[idx].double() / (1.0 - p_h)
            gref, gtol = mm_ref(ao, w["o"], a.out_proj.bias.detach().double())
            # the GEMM stores bf16, the dropout kernel scales it and adds the residual in fp32, one more bf16 store
            ref = xin + keep * gref
            tol = bf16_bound(ref, keep * bf16_bound(gref, gtol) + 2 * EPS32 * (xin.abs() + (keep * gref).abs()))
        else:
            ref, tol = mm_ref(ao, w["o"], a.out_proj.bias.detach().double(), (xin,))
            tol = bf16_bound(ref, tol)
        check(rep, "y1 (out_proj + residual)", tag, rows_of(st["y1"], idx), ref, tol)
        y1 = rows_of(st["y1"], idx)
        if pre_ln:
            check_ln_fwd(rep, tag + " LN2", y1, lyr.final_layer_norm, rows_of(st["ffn_in"], idx), st["mean2"][idx], st["rstd2"][idx])
        else:
            check_ln_fwd(rep, tag + " LN1", y1, lyr.self_attn_layer_norm, rows_of(st["x1"], idx), st["mean1"][idx], st["rstd1"][idx])
        # hg = gelu(z), hp = gelu'(z), z = ffn_in W1^T + b1, the activation-dropout mask folded into both
        ffn = rows_of(st["ffn_in"], idx)
        z, zt = mm_ref(ffn, w["w1"], lyr.fc1.bias.detach().double())
        kz = 1.0
        if p_act > 0:
            kz = keep_mask(d, li, DR.L_ACTIVATION, B * T, Fd, p_act, dev)[idx].double() / (1.0 - p_act)
        ghg, ghp = gelu64(z), dgelu64(z)
        # |gelu'| <= 1.13 and |gelu''| <= 0.8 carry the argument's error; the erfc approximation adds GELU_ABS (times |z| for gelu)
        thg = bf16_bound(ghg, 1.13 * zt + GELU_ABS * z.abs())
        thp = bf16_bound(ghp, 0.8 * zt + GELU_ABS)
        if p_act > 0:  # stored bf16, then scaled by keep / (1 - p) and stored again
            thg, thp = bf16_bound(kz * ghg, kz * thg), bf16_bound(kz * ghp, kz * thp)
        check(rep, "hg = gelu(z)", tag, rows_of(st["hg"], idx), kz * ghg, thg)
        check(rep, "hp = gelu'(z)", tag, rows_of(st["hp"], idx), kz * ghp, thp)
        # y2 = x1 + dropout3(hg W2^T + b2)
        hg = rows_of(st["hg"], idx)
        x1 = rows_of(st["x1"], idx)
        if p_h > 0:
            keep = keep_mask(d, li, DR.L_DROPOUT3, B * T, D, p_h, dev)[idx].double() / (1.0 - p_h)
            gref, gtol = mm_ref(hg, w["w2"], lyr.fc2.bias.detach().double())
            ref = x1 + keep * gref
            tol = bf16_bound(ref, keep * bf16_bound(gref, gtol) + 2 * EPS32 * (x1.abs() + (keep * gref).abs()))
        else:
            ref, tol = mm_ref(hg, w["w2"], lyr.fc2.bias.detach().double(), (x1,))
            tol = bf16_bound(ref, tol)
        check(rep, "y2 (fc2 + residual)", tag, rows_of(st["y2"], idx), ref, tol)
        if not pre_ln:
            y2 = rows_of(st["y2"], idx)
            check_ln_fwd(rep, tag + " final LN", y2, lyr.final_layer_norm, rows_of(out, idx), st["mean2"][idx], st["rstd2"][idx])
            if li + 1 < layers and cfg.gru_rel_pos and tab is not None:
                # the next layer's gate is built from ITS grep_* on this layer's stored output
                nst = sts[li + 1][1]
                check_gate(rep, tag + " hand-off", rows_of(out, idx), m.encoder.layers[li + 1].self_attn, H,
                           gate_rows(nst["gate"], idx))
        # ---- padded frames: the exact values the ragged kernels promise (asserted after the backward checks)
        if rag is not None:
            pz = [("y1n" if pre_ln else "x1", st["ffn_in"] if pre_ln else st["x1"])]
            if pre_ln:  # (post-LN: the ragged final LayerNorm backward already zeroes dz2 at padded frames)
                pz += [("xn", st["xn"]), ("hg", st["hg"]), ("hp", st["hp"])]
            else:
                pz.append(("out", out))
            for nm, t in pz:
                if not bool((t.reshape(B * T, -1)[pidx] == 0).all()):
                    pad_fail.append(f"{tag}: {nm} at padded frames is not zero")
            for nm in ("mean1", "rstd1", "mean2", "rstd2"):
                if not bool((st[nm][pidx] == 0).all()):
                    pad_fail.append(f"{tag}: {nm} at padded frames is not zero")
            fused = pre_ln and st["gate"] is not None or (not pre_ln and li > 0 and st["gate"] is not None
                                                           and D in (256, 512, 768, 1024))
            if fused and not bool((gate_rows(st["gate"], pidx) == 1).all()):
                pad_fail.append(f"{tag}: gate at padded frames is not 1")

    # ---- backward, recording what each kernel is handed
    gdout = torch.Generator().manual_seed(B * 7 + T)
    dout = torch.randn(B, T, D, generator=gdout)
    if rag is not None:
        dout[~vm] = 1000.0 * torch.randn(int((~vm).sum()), D, generator=gdout)  # large, finite: must not reach any gradient
    dout = dout.to(BF).to(dev)
    params = [p for p in m.encoder.layers.parameters()]
    dtab = torch.zeros(H, 2 * T - 1, dtype=F32, device=dev) if tab is not None else None

    def backward(dy):
        m.zero_grad_buffer()
        for p in params:
            eng.g(p).fill_(BASE)
        if dtab is not None:
            dtab.fill_(BASE)
        for li in reversed(range(layers)):
            dy = eng.layer_backward(li, sts[li][1], dy, dtab)
        return dy

    logs = []
    monkeypatch.setattr(engine_mod, "torch", _NanEmpty(torch))
    dy = dout
    m.zero_grad_buffer()
    for p in params:
        eng.g(p).fill_(BASE)
    if dtab is not None:
        dtab.fill_(BASE)
    for li in reversed(range(layers)):
        log = {}
        record(monkeypatch, log)
        dy_in = dy
        dy = eng.layer_backward(li, sts[li][1], dy, dtab)
        logs.append((li, dy_in, dy, log))
        monkeypatch.undo()
        monkeypatch.setattr(engine_mod, "torch", _NanEmpty(torch))
    monkeypatch.undo()
    torch.cuda.synchronize()
    # ---- ragged: parameter gradients and valid rows of dx do not depend on dout at padded frames
    if rag is not None:
        flat1 = m.grad_buffer().clone()
        grads = {id(p): eng.g(p).double() - BASE for p in params}
        dt1 = dtab.clone() if dtab is not None else None
        dx1 = logs[-1][2].clone()
        d0 = dout.clone()
        d0[~vm.to(dev)] = 0
        dx0 = backward(d0)
        torch.cuda.synchronize()
        # equal but for the order of the fp32 atomic adds (column sums, d tab, the attention's dQ), which changes from call to
        # call and can flip a bf16 rounding of dQ that then enters every gradient below it: 2^-12 of the value plus 2^-6 of the
        # parameter's rms gradient.  dout at a padded frame is 1000x that of a valid frame: reaching a gradient through a
        # single row, it moves it by tens of rms.
        # (q / k / v are one fused gradient: d k_proj.bias alone is rounding noise, softmax being shift-invariant over keys)
        def same(a_, b_, rms):
            return bool(((a_ - b_).abs() <= 2.0 ** -12 * b_.abs() + 2.0 ** -6 * rms).all())

        def before(p):
            return flat1[eng.flat.offsets[id(p)]:eng.flat.offsets[id(p)] + p.numel()].view_as(p).double()

        def rms(n, p):
            if "_proj." in n and "out_proj" not in n:
                sa = m.encoder.layers[int(n.split(".")[0])].self_attn
                kind = n.rsplit(".", 1)[1]
                return torch.cat([before(getattr(sa, q).get_parameter(kind)).flatten() for q in ("q_proj", "k_proj", "v_proj")]
                                 ).pow(2).mean().sqrt()
            return before(p).pow(2).mean().sqrt()
        bad = [n for n, p in m.encoder.layers.named_parameters() if not same(eng.g(p).double(), before(p), rms(n, p))]
        assert not bad, f"{tag0}: gradients depend on dout at padded frames: {bad}"
        if dt1 is not None:
            assert same(dtab.double(), dt1.double(), dt1.double().pow(2).mean().sqrt()), f"{tag0}: d tab depends on dout at padded frames"
        dxa, dxb = dx0.reshape(B * T, D)[idx].double(), dx1.reshape(B * T, D)[idx].double()
        # (dx sits below every dQ of the stack: 2^-4 of its rms, still far below one padded frame's 1000x dout)
        assert bool(((dxa - dxb).abs() <= 2.0 ** -8 * dxb.abs() + 2.0 ** -4 * dxb.pow(2).mean().sqrt()).all()), \
            f"{tag0}: dx depends on dout at padded frames"
    if rag is None:
        grads = {id(p): eng.g(p).double() - BASE for p in params}
    for li, dy_in, dx, log in logs:
        check_layer_bwd(rep, f"{tag0} layer {li}", m, eng, li, sts[li][1], dy_in, dx, log, grads, idx, pidx, B, T, H, hd, D, Fd,
                        pre_ln, d, tab, pad, scale, R, layers)

    assert not pad_fail, pad_fail
    report("layer", tag0, rep)


def check_ln_bwd(rep, tag, x, ln, dy, dres, dx_k, R):
    """LayerNorm backward of rows x (float64 of the saved bf16 input) with the recorded dy [+ dres]; returns the references
    and bounds of d gamma / d beta."""
    g, b = ln.weight.detach().double(), ln.bias.detach().double()
    xx = x.clone().requires_grad_(True)
    gg, bb = g.clone().requires_grad_(True), b.clone().requires_grad_(True)
    mean, r, xh, z = ln_fwd_parts(xx, gg, bb)
    dx, dgm, dbt = torch.autograd.grad(z, (xx, gg, bb), dy)
    mean, r, xh = mean.detach(), r.detach(), xh.detach()
    ex = ln_err(x, mean, r)
    dxh = dy.abs() * g.abs()
    xa = xh.abs()
    # fp32 arithmetic with the stored mean / rstd: 2^-16 of the terms of dx = r (dxh - mean(dxh) - xh mean(dxh xh)); the
    # error of xh enters the third term twice
    mag = r * (dxh + dxh.mean(1, keepdim=True) + xa * (dxh * xa).mean(1, keepdim=True))
    tx = 2.0 ** -16 * mag + r * (ex * (dxh * xa).mean(1, keepdim=True) + xa * (dxh * ex).mean(1, keepdim=True))
    if dres is not None:
        dx = dx + dres
        tx = tx + 2 * EPS32 * dres.abs()
    check(rep, "ln bwd dx", tag, dx_k, dx, bf16_bound(dx, tx))
    q_g, q_b = ((dy * xh) ** 2).sum(0), (dy * dy).sum(0)
    # (d gamma sits near 2^-8 of this bound: term_tol and the worst-case error of xh, ex, dominate it)
    tg = sum_tol(q_g, R) + term_tol(q_g, R) + (dy.abs() * ex).sum(0) + 2 * EPS32 * BASE
    tb = sum_tol(q_b, R) + 2 * EPS32 * BASE
    return dgm, tg, dbt, tb


def colsum_ref(t, R):
    """Column sum over rows of a stored bf16 tensor (float64 rows [R, N]) and its fp32 long-sum bound."""
    return t.sum(0), sum_tol((t * t).sum(0), R) + 2 * EPS32 * BASE


def check_layer_bwd(rep, tag, m, eng, li, st, dout, dx_k, log, grads, idx, pidx, B, T, H, hd, D, Fd, pre_ln, d, tab, pad, scale,
                    R, layers):
    lyr = m.encoder.layers[li]
    a = lyr.self_attn
    w = {k: eng.lw[li][k].double() for k in ("qkv", "o", "w1", "w2")}
    p_h = d.p if d is not None else 0.0
    V = lambda t: rows_of(t, idx)
    G = lambda p: grads[id(p)]
    rows, wgr, lnb = log["gemm_rows"], log["gemm_wgrad"], log.get("layer_norm_bwd", [])
    drops, cols = log.get("dropout_rows", []), log.get("colsum", [])
    assert len(rows) == 4 and len(wgr) == 4 and len(lnb) == 2, f"{tag}: unexpected launch sequence"

    def through_dropout(dy_rows, got, which):
        keep = keep_mask(d, li, which, B * T, D, p_h, dev=idx.device)[idx].double() / (1.0 - p_h)
        ref = dy_rows * keep
        check(rep, "dropout bwd", tag, V(got), ref, bf16_bound(ref, EPS32 * ref.abs()))

    # ---- FFN block
    if pre_ln:
        dy2 = V(dout)
        dz2_t = wgr[0][0][0]
        if p_h > 0:
            assert torch.equal(drops[0][0], dout)
            through_dropout(dy2, drops[0][1], DR.L_DROPOUT3)
        assert torch.equal(dz2_t, drops[0][1] if p_h > 0 else dout), f"{tag}: fc2 weight gradient is not fed dz2"
        ref, tol = colsum_ref(V(cols[0][0]), R)
        check(rep, "d fc2.bias (colsum)", tag, G(lyr.fc2.bias), ref, tol)
    else:
        dy_in, _ = lnb[0][0]
        assert torch.equal(dy_in, dout)
        dgm, tg, dbt, tb = check_ln_bwd(rep, tag + " final LN", V(st["y2"]), lyr.final_layer_norm, V(dout), None, V(lnb[0][1]), R)
        check(rep, "d ln.weight", tag, G(lyr.final_layer_norm.weight), dgm, tg)
        check(rep, "d ln.bias", tag, G(lyr.final_layer_norm.bias), dbt, tb)
        dy2_t = lnb[0][1]
        dz2_t = dy2_t
        if p_h > 0:
            through_dropout(V(dy2_t), drops[0][1], DR.L_DROPOUT3)
            dz2_t = drops[0][1]
            ref, tol = colsum_ref(V(cols[0][0]), R)
            assert torch.equal(cols[0][0], dz2_t)
        else:  # taken inside the LayerNorm backward: the column sum of its stored output
            ref, tol = colsum_ref(V(dy2_t), R)
        check(rep, "d fc2.bias (colsum)", tag, G(lyr.fc2.bias), ref, tol)
        dy2 = V(dy2_t)
    dz2 = V(dz2_t)
    # weight gradients: sums over the valid frames only
    assert torch.equal(wgr[0][0][0], dz2_t) and wgr[0][0][1] is st["hg"], f"{tag}: fc2 weight gradient operands"
    hg = V(st["hg"])
    check(rep, "d fc2.weight", tag, G(lyr.fc2.weight), dz2.t() @ hg, sum_tol((dz2 * dz2).t() @ (hg * hg), R) + 2 * EPS32 * BASE)
    # dhp = (dz2 W2) * hp, bf16; the fp32 accumulation's error is scaled by |hp|
    assert torch.equal(rows[0][0], dz2_t)
    hp = V(st["hp"])
    acc, at = mm_ref(dz2, w["w2"].t())
    ref = acc * hp
    check(rep, "dhp (dgelu=2 epilogue)", tag, V(rows[0][1]), ref, bf16_bound(ref, at * hp.abs() + EPS32 * ref.abs()))
    dhp_t = rows[0][1]
    dhp = V(dhp_t)
    ref, tol = colsum_ref(dhp, R)
    check(rep, "d fc1.bias (epilogue colsum)", tag, G(lyr.fc1.bias), ref, tol)
    assert torch.equal(wgr[1][0][0], dhp_t) and wgr[1][0][1] is st["ffn_in"], f"{tag}: fc1 weight gradient operands"
    ffn = V(st["ffn_in"])
    check(rep, "d fc1.weight", tag, G(lyr.fc1.weight), dhp.t() @ ffn, sum_tol((dhp * dhp).t() @ (ffn * ffn), R) + 2 * EPS32 * BASE)
    assert torch.equal(rows[1][0], dhp_t)
    if pre_ln:
        ref, tol = mm_ref(dhp, w["w1"].t())
        check(rep, "dffn_in", tag, V(rows[1][1]), ref, bf16_bound(ref, tol))
        dy_in, dres = lnb[0][0]
        assert torch.equal(dy_in, rows[1][1]) and torch.equal(dres, dout), f"{tag}: final LN backward operands"
        dgm, tg, dbt, tb = check_ln_bwd(rep, tag + " LN2", V(st["x1"]), lyr.final_layer_norm, V(dy_in), dy2, V(lnb[0][1]), R)
        check(rep, "d ln.weight", tag, G(lyr.final_layer_norm.weight), dgm, tg)
        check(rep, "d ln.bias", tag, G(lyr.final_layer_norm.bias), dbt, tb)
        dy1_t = lnb[0][1]
    else:
        ref, tol = mm_ref(dhp, w["w1"].t(), res=(dy2,))
        check(rep, "dx1 (+ res1 = dy2)", tag, V(rows[1][1]), ref, bf16_bound(ref, tol))
        dy_in, dres = lnb[1][0]
        assert torch.equal(dy_in, rows[1][1]) and dres is None
        dgm, tg, dbt, tb = check_ln_bwd(rep, tag + " LN1", V(st["y1"]), lyr.self_attn_layer_norm, V(dy_in), None, V(lnb[1][1]), R)
        check(rep, "d ln.weight", tag, G(lyr.self_attn_layer_norm.weight), dgm, tg)
        check(rep, "d ln.bias", tag, G(lyr.self_attn_layer_norm.bias), dbt, tb)
        dy1_t = lnb[1][1]
    dz1_t = dy1_t
    if p_h > 0:
        through_dropout(V(dy1_t), drops[1][1], DR.L_DROPOUT1)
        dz1_t = drops[1][1]
        assert torch.equal(cols[1][0], dz1_t)
        ref, tol = colsum_ref(V(dz1_t), R)
    else:
        ref, tol = colsum_ref(V(dy1_t), R)
    check(rep, "d out_proj.bias", tag, G(a.out_proj.bias), ref, tol)
    dz1 = V(dz1_t)
    # ---- attention block
    assert torch.equal(wgr[2][0][0], dz1_t) and wgr[2][0][1] is st["ao"], f"{tag}: out_proj weight gradient operands"
    ao = V(st["ao"])
    check(rep, "d out_proj.weight", tag, G(a.out_proj.weight), dz1.t() @ ao, sum_tol((dz1 * dz1).t() @ (ao * ao), R) + 2 * EPS32 * BASE)
    assert torch.equal(rows[2][0], dz1_t)
    ref, tol = mm_ref(dz1, w["o"].t())
    check(rep, "dao", tag, V(rows[2][1]), ref, bf16_bound(ref, tol))
    # attention backward: the kernel called directly on the recorded operands.  dK / dV are bit-equal; dQ, d gate and d tab
    # are fp32 atomic sums whose order differs from call to call: one bf16 ulp of dQ plus 2^-8 of the mean |dQ| of its head
    # (a sum that cancels to near zero moves by the rounding of its large terms); for the fp32 sums 2^-16 relative plus 2^-13
    # of the mean |d gate| of the head (|d tab| of the head).  The spread changes from call to call; these sit near 2^-7 of
    # their bounds, which are kept wide enough for any order of the atomics and still 2^-13 of the head's typical value
    (ins, outs), = log["attn_bwd_fused"]
    qkv, ao_, dao_, gate, tab_, pad_, lse, dtab_before = ins
    assert torch.equal(dao_, rows[2][1]) and qkv is not st["qkv"] and torch.equal(qkv, st["qkv"])
    dqkv2 = torch.full_like(outs[0], float("nan"))
    dgate2 = torch.full_like(outs[1], float("nan")) if outs[1] is not None else None
    dtab2 = dtab_before.clone() if dtab_before is not None else None
    ops.attn_bwd_fused(qkv, ao_, dao_, gate, tab_, pad_, lse, torch.empty(B, H, T, dtype=F32, device=qkv.device),
                       torch.zeros(B, T, D, dtype=F32, device=qkv.device), dqkv2, dgate2, dtab2, B, T, H, scale, head_dim=hd)
    torch.cuda.synchronize()
    assert bits_equal(outs[0][..., D:], dqkv2[..., D:]), f"{tag}: attention dK / dV are not the direct call's"
    dq_k, dq_d = outs[0][..., :D].reshape(B * T, D)[idx].double(), dqkv2[..., :D].reshape(B * T, D)[idx].double()
    assert_rel = lambda got, want, tol, what: check(rep, what, tag, got, want, tol)
    dq_mag = dq_d.abs().view(-1, H, hd).mean(-1, keepdim=True).expand(-1, H, hd).reshape(-1, D)
    assert_rel(dq_k, dq_d, ulp_bf16(dq_d) + 2.0 ** -8 * dq_mag, "attn bwd dQ vs direct")
    if dgate2 is not None:
        gk, gd = gate_rows(outs[1], idx), gate_rows(dgate2, idx)
        assert_rel(gk, gd, 2.0 ** -16 * (gk.abs() + gd.abs()) + 2.0 ** -13 * gd.abs().mean(0, keepdim=True),
                   "attn bwd dgate vs direct")
        assert_rel(outs[2], dtab2, 2.0 ** -16 * (outs[2].abs() + dtab2.abs()) + 2.0 ** -13 * dtab2.abs().mean(1, keepdim=True),
                   "attn bwd dtab vs direct")
    dqkv_t = outs[0]
    dqkv = V(dqkv_t)
    ref, tol = colsum_ref(dqkv, R)
    gb = torch.cat([G(a.q_proj.bias), G(a.k_proj.bias), G(a.v_proj.bias)])
    check(rep, "d qkv bias (colsum)", tag, gb, ref, tol)
    attn_in = st["xn"] if pre_ln else st["x"]
    ain = V(attn_in)
    dxg = None
    if gate is not None:
        (dgate_in, dxg_t), = log["gate_bwd"]
        assert torch.equal(dgate_in, outs[1])
        check_gate_bwd(rep, tag, ain, a, H, gate_rows(dgate_in, idx), V(dxg_t), G, R)
        dxg = V(dxg_t)
    assert torch.equal(wgr[3][0][0], dqkv_t) and wgr[3][0][1] is attn_in, f"{tag}: qkv weight gradient operands"
    gw = torch.cat([G(a.q_proj.weight), G(a.k_proj.weight), G(a.v_proj.weight)])
    check(rep, "d qkv weight", tag, gw, dqkv.t() @ ain, sum_tol((dqkv * dqkv).t() @ (ain * ain), R) + 2 * EPS32 * BASE)
    assert torch.equal(rows[3][0], dqkv_t)
    res = (dxg,) if dxg is not None else ()
    if pre_ln:
        ref, tol = mm_ref(dqkv, w["qkv"].t(), res=res)
        check(rep, "dxn (+ res1 = dxg)", tag, V(rows[3][1]), ref, bf16_bound(ref, tol))
        dy_in, dres = lnb[1][0]
        assert torch.equal(dy_in, rows[3][1]) and torch.equal(dres, dy1_t)
        dgm, tg, dbt, tb = check_ln_bwd(rep, tag + " LN1", V(st["x"]), lyr.self_attn_layer_norm, V(dy_in), V(dy1_t), V(lnb[1][1]), R)
        check(rep, "d ln.weight", tag, G(lyr.self_attn_layer_norm.weight), dgm, tg)
        check(rep, "d ln.bias", tag, G(lyr.self_attn_layer_norm.bias), dbt, tb)
        assert torch.equal(lnb[1][1], dx_k)
    else:
        ref, tol = mm_ref(dqkv, w["qkv"].t(), res=(V(dy1_t),) + res)
        check(rep, "dx (+ res1 = dy1, res2 = dxg)", tag, V(dx_k), ref, bf16_bound(ref, tol))
    if pidx.numel():
        assert bool((dx_k.reshape(B * T, D)[pidx] == 0).all()), f"{tag}: dx at padded frames is not zero"


def check_gate_bwd(rep, tag, y, attn, H, dg, dxg_k, G, R):
    """Gate backward from the recorded d gate [R, H] at rows y; returns the float64 reference of dxg."""
    w, b, a = (t.detach().double() for t in (attn.grep_linear.weight, attn.grep_linear.bias, attn.grep_a))
    leaves = [t.clone().requires_grad_(True) for t in (y, w, b, a)]
    gate, ga, gb, es = gate_parts(*leaves, H)
    dy, dw, db, da = torch.autograd.grad(gate, leaves, dg)
    ga, gb, es = ga.detach(), gb.detach(), es.detach()
    A = a.view(1, H).abs()
    R_, D = y.shape
    hd = D // H
    # error of the kernel's d sa / d sb: the sigmoids' (1/4 of the argument error plus __expf) through derivatives <= |a| + 1
    dds = 2 * dg.abs() * (A + 1.0) * (0.25 * es + 2.0 ** -20)  # [R, H]
    wa, wb = w[:4].sum(0).abs(), w[4:].sum(0).abs()
    dsa = (dg * (gb * a.view(1, H) - 1.0) * ga * (1 - ga)).abs()
    dsb = (dg * ga * a.view(1, H) * gb * (1 - gb)).abs()
    tdx = (dds[..., None] * (wa + wb) + 2.0 ** -22 * (dsa[..., None] * wa + dsb[..., None] * wb)).reshape(R_, D)
    check(rep, "dxg (gate bwd)", tag, dxg_k, dy, bf16_bound(dy, tdx))
    yq = y.view(R_, H, hd)
    dsa_s = (dg * (gb * a.view(1, H) - 1.0) * ga * (1 - ga))
    sq = ((dsa_s[..., None] * yq) ** 2).sum((0, 1))
    # (d grep_linear and its bias sit far below their bounds: the propagated worst-case sigmoid-argument error dds
    # dominates them, as it does the gate forward's)
    tw = sum_tol(sq, R * H) + (dds[..., None] * yq.abs()).sum((0, 1)) + 2 * EPS32 * BASE
    # rows 0-3 (and 4-7) of d grep_linear.weight are the same sum (each row is held to it: the kernel's atomics add in any order)
    gwk = G(attn.grep_linear.weight)
    dsb_s = dg * ga * a.view(1, H) * gb * (1 - gb)
    sqb = ((dsb_s[..., None] * yq) ** 2).sum((0, 1))
    twb = sum_tol(sqb, R * H) + (dds[..., None] * yq.abs()).sum((0, 1)) + 2 * EPS32 * BASE
    check(rep, "d grep_linear.weight", tag, gwk, dw, torch.cat([tw.expand(4, hd), twb.expand(4, hd)]))
    tb = torch.stack([sum_tol((dsa_s ** 2).sum(), R * H), sum_tol((dsb_s ** 2).sum(), R * H)]) + dds.sum() + 2 * EPS32 * BASE
    check(rep, "d grep_linear.bias", tag, G(attn.grep_linear.bias), db, tb.repeat_interleave(4))
    t_a = sum_tol(((dg * ga * gb) ** 2).sum(0), R) + (dg.abs() * (0.5 * es + 2.0 ** -20)).sum(0) + 2 * EPS32 * BASE
    check(rep, "d grep_a", tag, G(attn.grep_a).view(H), da.view(H), t_a)
    return dy


# ------------------------------------------------------------------------------------------------------------- cases
# (model, layers, B, T, valid lengths or None, input regime, dropout).  Post-LN models run two layers: the second layer's
# gate is left behind by the first layer's final LayerNorm (the hand-off) on base, computed by gate_fwd on tiny (D = 128).
SHIPPED = [("base", 2, 16, 749, None), ("base", 2, 4, 749, (749, 300, 129, 1)), ("large", 1, 8, 999, None),
           ("large", 1, 4, 1499, (1499, 501, 129, 1)), ("xlsr1b", 1, 8, 999, None), ("xlsr1b", 1, 4, 999, (999, 640, 129, 1)),
           ("xlsr2b", 1, 8, 999, None), ("tiny", 2, 4, 99, None)]
# tile edges: T around the 128-row tiles and the 64-row weight-gradient blocks, valid lengths at 64k and 128k + 1
EDGES = [(n, 2 if n == "base" else 1, 2, T, None) for n in ("base", "large") for T in (1, 127, 128, 129, 255, 257)] + \
        [(n, 2 if n == "base" else 1, 4, 257, (257, 192, 129, 64)) for n in ("base", "large")]
CASES = [c + ("normal", 0.0) for c in SHIPPED + EDGES] + \
        [(n, 2 if n == "base" else 1, 2, 300, None, rg, 0.0) for n in ("base", "large") for rg in ("dc", "wide")] + \
        [("base", 2, 2, 300, None, "normal", 0.1), ("large", 1, 2, 300, (300, 129), "normal", 0.1)]


def _id(c):
    n, L, B, T, lens, rg, p = c
    return f"{n}-B{B}-T{T}{'-ragged' if lens else ''}-{rg}{'-drop' if p else ''}"


@pytest.mark.parametrize("name,layers,B,T,lengths,regime,p_drop", CASES, ids=[_id(c) for c in CASES])
def test_layer_engine(cuda_device, monkeypatch, name, layers, B, T, lengths, regime, p_drop):
    run_case(cuda_device, monkeypatch, name, layers, B, T, lengths, regime, p_drop)
