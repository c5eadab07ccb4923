"""Op-level tests of the stages between the waveform and the first encoder layer: conv layer 0 (csrc/conv0.cu, conv0_gn.cu),
conv layers 1-6 as the engine wires them (Engine.conv_forward / conv_backward over the overlapping-row GEMMs) and the pos_conv
stem (Engine.posconv_forward / posconv_backward, posconv_prep / posconv_unprep).

Every reference is computed in float64 on the GPU from the same bf16 / fp32 tensors the kernel reads, and every reference
gradient comes from torch.autograd on a plain float64 restatement of the reference module (Conv1d without bias, GroupNorm(C, C)
or LayerNorm(C), exact-erf GELU; weight_norm(dim=2) grouped Conv1d with padding 64 minus the last frame, GELU, residual, post-LN
encoder.layer_norm).  References are built per utterance (and per frame chunk) to bound memory.

The engine tests are teacher-forced: each layer is checked against the float64 layer applied to the kernel's own bf16 input,
and the backward chain runs at the kernel's saved activations.  The kernel rounds every inter-layer gradient to bf16, so
gradient bounds come from a magnitude reference (the same chain on absolute values = sum of |terms| per element), never from
max|dW|, and the probe gradients (non-zero at one frame per utterance) make an error at an utterance or tile edge the whole
signal.  Outputs are pre-filled with NaN and `+=` outputs (all parameter gradients) start non-zero.  EPS32 = 2^-24 is the fp32
unit roundoff; each tolerance is written next to its reason."""
import math
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from unispeech_b200 import ops
from unispeech_b200 import workloads as W

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
EPS32 = 2.0 ** -24
SR = 16000
K0, S0 = 10, 5  # conv layer 0: kernel 10, stride 5
GOLDEN = Path(__file__).resolve().parent / "golden"


# ------------------------------------------------------------------------------------------------------------- helpers
def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp at |x| (the ulp of the smallest normal below it)."""
    a = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def bf16_bound(ref: torch.Tensor, delta) -> torch.Tensor:
    """Bound on |bf16(v) - ref| when the kernel's fp32 value v is within `delta` of ref: half an ulp at |ref| + delta, plus delta."""
    delta = torch.as_tensor(delta, dtype=F64, device=ref.device)
    return ulp_bf16(ref.abs() + delta) * 0.5 + delta


def nan_like(shape, dtype, dev):
    return torch.full(shape, float("nan"), dtype=dtype, device=dev)


def assert_close(got, ref, tol, what):
    """|got - ref| <= tol elementwise (tol a tensor or a number); NaN anywhere fails."""
    got, ref = got.double(), ref.double()
    tol = torch.as_tensor(tol, dtype=F64, device=ref.device).expand_as(ref)
    bad = ~((got - ref).abs() <= tol)
    if bad.any():
        i = int(bad.flatten().nonzero()[0])
        raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements out of bounds; first at flat index {i}: "
                             f"got {got.flatten()[i].item()!r}, want {ref.flatten()[i].item()!r}, tol {tol.flatten()[i].item():.3g}")


def gelu64(z):
    return F.gelu(z)  # exact erf form (approximate="none")


def dgelu64(z):
    return 0.5 * (1.0 + torch.erf(z * 0.5 ** 0.5)) + z * torch.exp(-0.5 * z * z) / math.sqrt(2.0 * math.pi)


def speech(B: int, L: int, dev, zero_last=True) -> torch.Tensor:
    """B rows of real speech (the 5 recordings of the golden file, pcm / 32768 at gains 1, 0.5, 2), zero tails, and optionally
    an all-zero last row (GroupNorm variance 0: rstd = 1/sqrt(1e-5))."""
    z = np.load(GOLDEN / "vox_real_large2l.npz")
    pcm, lengths = z["pcm"].astype(np.float32) / 32768.0, z["lengths"]
    wav = torch.zeros(B, L)
    for b in range(B):
        u = b % 5
        n = int(min(lengths[u], L))
        wav[b, :n] = torch.from_numpy(pcm[u, :n]) * (1.0, 0.5, 2.0)[(b // 5) % 3]
    if zero_last and B > 1:
        wav[-1] = 0.0
    return wav.to(dev)


def make_wav(kind: str, B: int, L: int, seed: int, dev) -> torch.Tensor:
    g = torch.Generator().manual_seed(seed)
    if kind == "speech":
        return speech(B, L, dev)
    if kind == "noise":
        return torch.randn(B, L, generator=g).to(dev)
    if kind.startswith("dc"):  # DC offset of growing size on weak noise: E[conv]^2 >> Var[conv] for GroupNorm
        return (float(kind[2:]) + 0.01 * torch.randn(B, L, generator=g)).to(dev)
    raise ValueError(kind)


ACC = 2.0 ** -16


def acc_tol(sq, n):
    """Bound on the fp32 error of a long sum (a weight-gradient GEMM over frames, a column sum) of n terms whose squares sum
    to `sq`.  A worst-case bound (n EPS32 sum |t|) grows n / sqrt(n) times faster than the sum of n random-sign terms and is
    vacuous at 10^4-10^5 frames; the rounding errors of the partial sums are independent, and the partial sums stay within a
    few sqrt(sum t^2), so their total is a small multiple of EPS32 sqrt(n sum t^2).  ACC = 256 EPS32 leaves a wide margin."""
    return ACC * (n * sq).sqrt()


TERM = 2.0 ** -15


def term_tol(sq, n):
    """Allowance for fp32 arithmetic inside each term of a sum the kernel recomputes (LayerNorm with its stored fp32
    statistics, gelu' from its erfc approximation): 2^-15 of each |term|, and sum |t| <= sqrt(n sum t^2)."""
    return TERM * (n * sq).sqrt()


def record(monkeypatch, log):
    """Copies of the operands the engine hands to the backward ops: the kernels' own intermediate gradients.  Each backward
    step is then checked from the kernel's own input (teacher-forced), so no step's bound has to cover the roundings of the
    steps before it."""
    def wrap(name, before=None, after=None):
        orig = getattr(ops, name)

        def f(*a, **kw):
            if before is not None:
                log.setdefault(name + ".in", []).append(before(*a, **kw))
            orig(*a, **kw)
            if after is not None:
                log.setdefault(name + ".out", []).append(after(*a, **kw))
        monkeypatch.setattr(ops, name, f)

    def rows(t, bs, rs, nb, nr, N):
        return torch.as_strided(t, (nb, nr, N), (bs, rs, 1)).clone()
    wrap("gemm_wgrad", before=lambda *a, **kw: rows(a[0], a[1], a[2], a[7], a[6], a[8]))
    wrap("layer_norm_bwd", before=lambda *a, **kw: rows(a[0], a[1], a[2], a[20], a[19], a[21]),
         after=lambda *a, **kw: rows(a[13], a[14], a[15], a[20], a[19], a[21]))
    wrap("conv0_bwd", before=lambda *a, **kw: rows(a[15], a[16], a[4], a[2], a[3], a[4]),
         after=lambda *a, **kw: None if kw.get("dconv_ws") is None else rows(kw["dconv_ws"], kw["ws_bs"], a[4], a[2], a[3], a[4]))
    wrap("posconv_wgrad", before=lambda *a, **kw: rows(a[0], a[1], a[2], a[6], a[5], a[7]), after=lambda *a, **kw: a[10].clone())


# ------------------------------------------------------------------------------------------------- conv layer 0 reference
def conv0_ref(x, T, w, gamma, beta, ln, da=None, da_mag=None):
    """Layer 0 of one utterance in float64: x [L], w [C, k], gamma / beta [C].  With `da` ([T, C], the gradient at the GELU
    output) also the autograd gradients of w / gamma / beta and their magnitude references (`da_mag` >= |da|, default |da|)."""
    dim = 1 if ln else 0  # LayerNorm: over channels per frame; GroupNorm(C, C): over frames per channel
    X = x.unfold(0, K0, S0)[:T]  # [T, k]: x[s t + j]
    want = da is not None
    w_, g_, b_ = (p.detach().clone().requires_grad_(want) for p in (w, gamma, beta))
    conv = X @ w_.t()
    mean = conv.mean(dim, keepdim=True)
    var = ((conv - mean) ** 2).mean(dim, keepdim=True)
    r = (var + 1e-5).rsqrt()
    xh = (conv - mean) * r
    z = xh * g_ + b_
    out = gelu64(z)
    cmag = X.abs() @ w.abs().t()  # sum_j |w_j x_j|
    res = dict(out=out.detach(), mean=mean.detach(), rstd=r.detach(), S1=conv.detach().sum(0), S2=(conv.detach() ** 2).sum(0),
               S1mag=cmag.sum(0), S2mag=(cmag ** 2).sum(0), fmag=cmag.mean(1),
               zmag=gamma.abs() * r.detach() * (cmag + mean.detach().abs()) + beta.abs())
    if want:
        res["dw"], res["dgamma"], res["dbeta"], res["dconv"] = torch.autograd.grad(out, (w_, g_, b_, conv), da)
        with torch.no_grad():
            dam = da.abs() if da_mag is None else da_mag
            xh, z = xh.detach(), z.detach()
            dz = dam * dgelu64(z).abs()
            dxh = dz * gamma.abs()
            dconv = r.detach() * (dxh + dxh.mean(dim, keepdim=True) + xh.abs() * (dxh * xh.abs()).mean(dim, keepdim=True))
            res["Mdw"] = dconv.t() @ X.abs()
            res["Mdconv"] = dconv
            res["Qdgamma"] = ((dz * xh.abs()) ** 2).sum(0)  # sums of squared terms (long-sum bounds, acc_tol)
            res["Qdbeta"] = (dz ** 2).sum(0)
            res["Mdgamma"] = (dz * xh.abs()).sum(0)
            # the fp32 xh itself is off by a few EPS32 of the terms it is formed from (it is not 0 when conv == mean)
            ex = r.detach() * (cmag + mean.detach().abs())
            if ln:  # and |xh| times the stored per-frame rstd's error (16 EPS32 fmag rstd, see check_conv0_fwd), in 2^-16 units
                ex = ex + xh.abs() * 2.0 ** -4 * cmag.mean(1, keepdim=True) * r.detach()
            # gelu' from the Abramowitz-Stegun 7.1.26 erfc approximation: absolute error below 2^-21 (2^-5 in these units)
            res["Mdgamma_x"] = (dz * ex + dam * xh.abs() * 2.0 ** -5).sum(0)
            res["Mdbeta"] = dz.sum(0)
            # ... and moves gelu'(gamma xh + beta) by |gamma| |gelu''| (<= 0.8) times that error
            res["Mdbeta_x"] = (dam * (gamma.abs() * ex + 2.0 ** -5)).sum(0)
    return res


def conv0_kernel_fwd(wav, C, ln, w, gamma, beta):
    B, L_ = wav.shape
    T = (L_ - K0) // S0 + 1
    Tp = T + (T & 1)
    dev = wav.device
    out = nan_like((B, Tp, C), BF, dev)
    stats = None if ln else nan_like((B * C * 2 + B * 128,), F64, dev)
    fmean = nan_like((B, T), F32, dev) if ln else None
    frstd = nan_like((B, T), F32, dev) if ln else None
    ops.conv0_fwd(wav, L_, B, T, C, K0, S0, w, gamma, beta, 1 if ln else 0, stats, fmean, frstd, out, Tp * C)
    return dict(T=T, Tp=Tp, out=out, stats=stats, fmean=fmean, frstd=frstd)


def check_conv0_fwd(k, wav, w, gamma, beta, ln, refs):
    """Kernel layer-0 forward (dict of conv0_kernel_fwd) against the per-utterance references."""
    T = k["T"]
    for b, r in enumerate(refs):
        # fp32 conv (10 FMAs) and normalisation (GroupNorm folded into the taps: a*w, beta - a*mean) are exact to a few
        # EPS32 of the magnitudes involved (zmag); 2^-16 also covers an fp32-accurate mean / rstd.  GELU' <= 1.13.
        assert_close(k["out"][b, :T], r["out"], bf16_bound(r["out"], 1.13 * 2.0 ** -16 * r["zmag"]), f"out[{b}]")
        if ln:
            # per-frame mean over C fp32 values (C/32 per lane, 5-level shuffle tree) of conv values exact to a few EPS32 of
            # sum_j |w_j x_j|; two-pass variance: its error is a few EPS32 * fmag * sigma, i.e. a relative rstd error of
            # 16 EPS32 * fmag * rstd at most, plus rsqrtf (2 ulp)
            assert_close(k["fmean"][b], r["mean"][:, 0], 2.0 ** -18 * r["fmag"], f"fmean[{b}]")
            rs = r["rstd"][:, 0]
            assert_close(k["frstd"][b], rs, rs * (2.0 ** -20 + 16 * EPS32 * r["fmag"] * rs), f"frstd[{b}]")
    if not ln:
        B, C = wav.shape[0], w.shape[0]
        st = k["stats"][:B * C * 2].view(B, C, 2)
        # autocorrelation partials: fp32 products and sums over n_f frames per thread, a 32-lane fp32 shuffle sum, then fp64;
        # S2 = sum_jj' w_j w_j' A[j, j'] so its error is bounded by (n_f + 8) EPS32 sum_t (sum_j |w_j x_j|)^2
        gx = max(1, min((T + 2047) // 2048, 64))
        nf = (T + 256 * gx - 1) // (256 * gx)
        for b, r in enumerate(refs):
            assert_close(st[b, :, 0], r["S1"], (nf + 8) * EPS32 * r["S1mag"] + 1e-300, f"stats sum conv [{b}]")
            assert_close(st[b, :, 1], r["S2"], (nf + 8) * EPS32 * r["S2mag"] + 1e-300, f"stats sum conv^2 [{b}]")


def conv0_params(C, seed, dev):
    g = torch.Generator().manual_seed(seed)
    w = torch.randn(C, 1, K0, generator=g) * (2.0 / K0) ** 0.5  # kaiming_normal_, as the model initialises it
    gamma = 1.0 + 0.2 * torch.randn(C, generator=g)
    beta = 0.1 * torch.randn(C, generator=g)
    return w.to(dev), gamma.to(dev), beta.to(dev)


# Shipped geometry: Base 16 x 15 s (GroupNorm), Large 8 x 20 s (LayerNorm), tiny 4 x 2 s at 64 channels; DC offsets; and the
# launch-geometry edges: B = 1 / 4 / 8 / 16 (8 * SMs / B chunks), T0 = 1 (L = 10), 79 (L = 400), 50 (< one 64-frame tile),
# 1000 (not a multiple of the tile, (L - 10) % 5 = 4).
CONV0_CASES = [
    ("gn", 512, 16, 15 * SR, "speech"), ("ln", 512, 8, 20 * SR, "speech"), ("gn", 512, 16, 15 * SR, "noise"),
    ("gn", 64, 4, 2 * SR, "noise"), ("ln", 64, 4, 2 * SR, "noise"),
    ("gn", 512, 4, 15 * SR, "dc0.05"), ("gn", 512, 4, 15 * SR, "dc0.3"), ("gn", 512, 4, 15 * SR, "dc1"),
    ("ln", 512, 4, 15 * SR, "dc0.3"), ("gn", 64, 4, 2 * SR, "dc0.3"),
] + [(mode, C, B, L, "noise") for mode in ("gn", "ln") for (C, B, L) in
     ((512, 1, 10), (512, 8, 400), (512, 4, 255), (512, 16, 5004), (64, 1, 10), (64, 8, 400), (64, 16, 5004))]


@pytest.mark.parametrize("mode,C,B,L,kind", CONV0_CASES, ids=[f"{m}-C{c}-B{b}-L{l}-{k}" for m, c, b, l, k in CONV0_CASES])
def test_conv0(cuda_device, mode, C, B, L, kind):
    dev = cuda_device
    ln = mode == "ln"
    seed = C + B + L % 9973
    wav = make_wav(kind, B, L, seed, dev)
    w, gamma, beta = conv0_params(C, seed, dev)
    k = conv0_kernel_fwd(wav, C, ln, w, gamma, beta)
    T, Tp = k["T"], k["Tp"]
    g = torch.Generator().manual_seed(seed + 1)
    da = torch.randn(B, T, C, generator=g).to(dev).to(BF)
    dap = torch.zeros(B, Tp, C, dtype=BF, device=dev)
    dap[:, :T] = da
    refs = [conv0_ref(wav[b].double(), T, w.double().view(C, K0), gamma.double(), beta.double(), ln, da=da[b].double())
            for b in range(B)]
    torch.cuda.synchronize()
    check_conv0_fwd(k, wav, w, gamma, beta, ln, refs)
    ref = {n: sum(r[n] for r in refs) for n in ("dw", "dgamma", "dbeta", "Mdw", "Mdgamma", "Mdgamma_x", "Mdbeta", "Mdbeta_x")}

    def run_bwd(variant):
        # += outputs start at their own magnitude (exactly representable offsets, far below the bounds after subtraction)
        base = {n: ref["M" + n].float().clamp_min(1.0) for n in ("dw", "dgamma", "dbeta")}
        dw, dg, db = base["dw"].clone().view(C, 1, K0), base["dgamma"].clone(), base["dbeta"].clone()
        bstats = nan_like((B, C, 12), F32, dev)
        ws = None
        dain = dap
        if variant == "ws":
            ws = nan_like((B, Tp, C), BF, dev)
        elif variant == "alias":  # as the engine calls it: the incoming gradient buffer doubles as the workspace
            dain = dap.clone()
            ws = dain
        ops.conv0_bwd(wav, L, B, T, C, K0, S0, w, gamma, beta, 1 if ln else 0, k["stats"], bstats, k["fmean"], k["frstd"],
                      dain, Tp * C, dw, dg, db, dconv_ws=ws, ws_bs=Tp * C)
        torch.cuda.synchronize()
        # fp32 per-frame arithmetic and fp32 partial sums (chunks of <= 1024 frames, then atomics): 2^-12 of the sum of
        # |terms|.  The two-pass LayerNorm backward stores d(conv) as bf16 (unit roundoff 2^-8) before the weight-gradient pass.
        rel_dw = 2.0 ** -12 + (2.0 ** -8 if ws is not None else 0.0)
        assert_close(dw.view(C, K0).double() - base["dw"].double(), ref["dw"], rel_dw * ref["Mdw"], f"dw ({variant})")
        assert_close(dg.double() - base["dgamma"].double(), ref["dgamma"], 2.0 ** -12 * ref["Mdgamma"] + 2.0 ** -16 * ref["Mdgamma_x"],
                     f"dgamma ({variant})")
        assert_close(db.double() - base["dbeta"].double(), ref["dbeta"], 2.0 ** -12 * ref["Mdbeta"] + 2.0 ** -16 * ref["Mdbeta_x"],
                     f"dbeta ({variant})")

    for variant in (("ws", "alias", "none") if ln else ("gn",)):
        run_bwd(variant)


def test_conv0_gn_300s(cuda_device):
    """300 s in one utterance: the autocorrelation grid is at its 64-block cap (about 59 frames per thread).  Checks the
    GroupNorm sums and a strided sample of output frames (the full float64 output would be 3.9 GB)."""
    dev = cuda_device
    C, L = 512, 300 * SR
    T = (L - K0) // S0 + 1
    z = np.load(GOLDEN / "vox_real_large2l.npz")
    pcm = np.concatenate([z["pcm"][u, :z["lengths"][u]] for u in range(5)]).astype(np.float32) / 32768.0
    wav = torch.from_numpy(np.resize(pcm, L)).view(1, L).to(dev)
    w, gamma, beta = conv0_params(C, 300, dev)
    k = conv0_kernel_fwd(wav, C, False, w, gamma, beta)
    torch.cuda.synchronize()
    x = wav[0].double()
    w64 = w.double().view(C, K0)
    S1 = torch.zeros(C, dtype=F64, device=dev)
    S2, S1m, S2m = torch.zeros_like(S1), torch.zeros_like(S1), torch.zeros_like(S1)
    for t0 in range(0, T, 1 << 16):
        X = x[t0 * S0:].unfold(0, K0, S0)[:min(T - t0, 1 << 16)]
        c, cm = X @ w64.t(), X.abs() @ w64.abs().t()
        S1 += c.sum(0); S2 += (c * c).sum(0); S1m += cm.sum(0); S2m += (cm * cm).sum(0)
    st = k["stats"][:C * 2].view(C, 2)
    nf = (T + 256 * 64 - 1) // (256 * 64)
    assert nf >= 58
    assert_close(st[:, 0], S1, (nf + 8) * EPS32 * S1m, "stats sum conv")
    assert_close(st[:, 1], S2, (nf + 8) * EPS32 * S2m, "stats sum conv^2")
    mean = S1 / T
    r = (S2 / T - mean * mean + 1e-5).rsqrt()
    ts = torch.cat([torch.arange(0, T, 997), torch.arange(T - 3, T)]).to(dev)
    X = x.unfold(0, K0, S0)[ts]
    c, cm = X @ w64.t(), X.abs() @ w64.abs().t()
    ref = gelu64((c - mean) * r * gamma.double() + beta.double())
    zmag = gamma.double().abs() * r * (cm + mean.abs()) + beta.double().abs()
    assert_close(k["out"][0, ts], ref, bf16_bound(ref, 1.13 * 2.0 ** -16 * zmag), "out (strided frames)")


# ------------------------------------------------------------------------------------------------- models through the engine
_MODELS = {}


def model(name, dev):
    """The shipped configuration with one encoder layer (the pos_conv stem's gate-fused LayerNorm needs a consumer layer), with
    non-trivial normalisation affine terms, pos_conv bias and weight_g."""
    if name not in _MODELS:
        from unispeech_b200.wavlm import WavLM, WavLMConfig
        cfg, B, secs = W.model_config(name)
        torch.manual_seed({"base": 11, "large": 12, "tiny": 13}[name])
        m = WavLM(WavLMConfig(dict(cfg, encoder_layers=1)))
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, (torch.nn.LayerNorm, torch.nn.GroupNorm)):
                    mod.weight.normal_(1.0, 0.2)
                    mod.bias.normal_(0.0, 0.1)
            pc = m.encoder.pos_conv[0]
            pc.bias.normal_(0.0, 0.1)
            pc.weight_g.mul_(torch.rand_like(pc.weight_g) + 0.5)
        _MODELS[name] = (m.to(dev).eval(), B, secs)
    return _MODELS[name]


def conv_rows(a, w, k, s, T):
    """Conv1d without bias on channels-last rows: a [T_in, Cin], w [Cout, Cin, k] -> [T, Cout] (float64)."""
    X = a.unfold(0, k, s)[:T]  # [T, Cin, k]
    return X.reshape(T, -1) @ w.reshape(w.shape[0], -1).t()


def receptive_rows(last, convs, T):
    """Rows of each conv layer's output that frames [0, last) of the final layer read (the receptive field, from the
    definition: frames [0, V) of layer l + 1 read rows [0, s (V - 1) + k) of layer l), clamped to the layer's frame count."""
    V = [0] * len(convs)
    V[-1] = min(last, T[-1])
    for l in range(len(convs) - 2, -1, -1):
        _, k, s = convs[l + 1]
        V[l] = min(s * (V[l + 1] - 1) + k, T[l]) if V[l + 1] > 0 else 0
    return V


def ln_fwd_parts(y, gamma, beta):
    mean = y.mean(1, keepdim=True)
    r = (((y - mean) ** 2).mean(1, keepdim=True) + 1e-5).rsqrt()
    xh = (y - mean) * r
    return mean, r, xh, xh * gamma + beta


def ln_bwd_mag(dA_mag, r, xh, z, gamma):
    """Magnitude of the LayerNorm(+GELU) backward per element, and of its gamma / beta gradients (sums over frames)."""
    dz = dA_mag * dgelu64(z).abs()
    dxh = dz * gamma.abs()
    dy = r * (dxh + dxh.mean(1, keepdim=True) + xh.abs() * (dxh * xh.abs()).mean(1, keepdim=True))
    return dy, (dz * xh.abs()).sum(0), dz.sum(0)


def conv_params(m):
    """[(name, parameter)] of the conv stack: seven weights and the normalisation affine terms."""
    out = []
    for i, blk in enumerate(m.feature_extractor.conv_layers):
        out.append((f"w{i}", blk[0].weight))
        if isinstance(blk[2], torch.nn.GroupNorm):
            out += [(f"gamma{i}", blk[2].weight), (f"beta{i}", blk[2].bias)]
        elif isinstance(blk[2], torch.nn.Sequential):
            out += [(f"gamma{i}", blk[2][1].weight), (f"beta{i}", blk[2][1].bias)]
    return out


CONV_STACK_CASES = [("base", False), ("large", False), ("tiny", False), ("base", True), ("large", True)]
BASE = 2.0 ** -20  # += outputs start here: exact, non-zero, and far below every bound once subtracted


def convT_rows(dY, w, k, s, T_in):
    """Input gradient of conv_rows (autograd of the forward restatement): dY [T, Cout] -> [T_in, Cin]."""
    a = torch.zeros(T_in, w.shape[1], dtype=F64, device=dY.device, requires_grad=True)
    (da,) = torch.autograd.grad(conv_rows(a, w, k, s, dY.shape[0]), (a,), dY)
    return da


def wgrad_rows(a, dY, w_shape, k, s):
    """Weight gradient of conv_rows (autograd): sum over frames of dY (x) the input windows."""
    w = torch.zeros(w_shape, dtype=F64, device=dY.device, requires_grad=True)
    (dw,) = torch.autograd.grad(conv_rows(a, w, k, s, dY.shape[0]), (w,), dY)
    return dw


def nonzero_rows(t):
    return int((t != 0).any(-1).sum())


@pytest.mark.parametrize("name,ragged", CONV_STACK_CASES, ids=[f"{n}-{'ragged' if r else 'full'}" for n, r in CONV_STACK_CASES])
def test_conv_stack(cuda_device, monkeypatch, name, ragged):
    dev = cuda_device
    m, B, secs = model(name, dev)
    convs = m.conv_cfg
    n = len(convs)
    ln = m.cfg.extractor_mode == "layer_norm"
    C = convs[0][0]
    L_ = secs * SR
    wav = speech(B, L_, dev) if name != "tiny" else make_wav("noise", B, L_, 3, dev)
    eng = m._begin(dev)
    T = [L_]
    for (_, k, s) in convs:
        T.append((T[-1] - k) // s + 1)
    T = T[1:]
    T6 = T[-1]
    if ragged:
        # one full-length utterance, one with a single valid frame, and ends at both parities of the final frame count.  (With
        # this stack V_l = 2 V_{l+1} (k = 2) or 2 V_{l+1} + 1 (k = 3) and never reaches T_l, so every utterance's tail has
        # the same parity in a given layer: each phase GEMM sees one tail phase per layer.)
        lasts = [T6, T6 - 1, 1, T6 // 2, T6 // 2 + 1, 100, 101, 2, 3, 37, T6 - 2, 64, 65, 127, 128, T6][:B]
    else:
        lasts = [T6] * B
    V = [receptive_rows(l, convs, T) for l in lasts]  # V[b][layer]
    st = eng.conv_forward(wav, True, torch.tensor(lasts, dtype=torch.int32) if ragged else None)
    torch.cuda.synchronize()
    Wb = {i: m.feature_extractor.conv_layers[i][0].weight.detach().to(BF).double() for i in range(1, n)}  # the GEMM operands
    norms = {i: (m.feature_extractor.conv_layers[i][2][1] if ln else None) for i in range(n)}

    # ---- forward, teacher-forced: layer i on the kernel's own bf16 input a[i-1].  A full batch checks every row [0, T_i)
    # (rows beyond the last frame's receptive field included: the GEMM's M tail); a ragged one the rows [0, V_i) valid
    # frames read, since the GEMMs zero-fill whole tiles beyond them.
    for i in range(1, n):
        _, k, s = convs[i]
        for b in range(B):
            v = V[b][i] if ragged else T[i]
            if v == 0:
                continue
            a_prev = st["a"][i - 1][b, :T[i - 1]].double()
            y = conv_rows(a_prev, Wb[i], k, s, T[i])[:v]
            # fp32 accumulation of k * C <= 1536 bf16 products: at most K EPS32 <= 2^-12 of sum |w a|
            mag = conv_rows(a_prev.abs(), Wb[i].abs(), k, s, T[i])[:v]
            if ln:
                assert_close(st["y"][i][b, :v], y, bf16_bound(y, 2.0 ** -12 * mag), f"y{i}[{b}]")
                yk = st["y"][i][b, :v].double()
                nm = norms[i]
                mean, r, xh, z = ln_fwd_parts(yk, nm.weight.double(), nm.bias.double())
                ym = yk.abs().mean(1)
                # fp32 LayerNorm over C values of the stored bf16 y: mean to 2^-18 of mean |y|, rstd to 2^-18 relative plus
                # the variance's sensitivity to the mean's error
                mk = st["mean"][i].view(B, T[i])[b, :v]
                rk = st["rstd"][i].view(B, T[i])[b, :v]
                assert_close(mk, mean[:, 0], 2.0 ** -18 * ym, f"mean{i}[{b}]")
                assert_close(rk, r[:, 0], r[:, 0] * (2.0 ** -18 + 16 * EPS32 * ym * r[:, 0]), f"rstd{i}[{b}]")
                ref = gelu64(z)
                # fp32 LayerNorm + GELU of exact bf16 inputs: a few EPS32 of |gamma xh| + |beta|, plus the rstd error above
                zm = (xh.abs() * nm.weight.double().abs() + nm.bias.double().abs())
                assert_close(st["a"][i][b, :v], ref, bf16_bound(ref, 2.0 ** -16 * zm), f"a{i}[{b}]")
            else:
                ref = gelu64(y)
                assert_close(st["a"][i][b, :v], ref, bf16_bound(ref, 1.13 * 2.0 ** -12 * mag), f"a{i}[{b}]")
                # the stored y is gelu'(conv output) (epilogue gelu = 2); gelu'' <= 0.8
                assert_close(st["y"][i][b, :v], dgelu64(y), bf16_bound(dgelu64(y), 0.8 * 2.0 ** -12 * mag), f"gelu'{i}[{b}]")

    # ---- backward, teacher-forced step by step from the kernel's own intermediate gradients, for several probes
    g = torch.Generator().manual_seed(7)
    probes = ["dense", "first", "last"] + (["boundary"] if ragged else [])
    params = dict(conv_params(m))
    Tp6 = st["a"][-1].shape[1]
    w0 = m.feature_extractor.conv_layers[0][0].weight.detach().double().view(C, K0)
    nm0 = m.feature_extractor.conv_layers[0][2]
    nm0 = nm0[1] if ln else nm0
    for probe in probes:
        dfeat = torch.zeros(B, Tp6, C, dtype=BF, device=dev)
        full = torch.randn(B, T6, C, generator=g).to(BF).to(dev)
        for b in range(B):
            v = V[b][-1]
            sel = {"dense": slice(0, v), "first": slice(0, 1), "last": slice(v - 1, v), "boundary": slice(max(0, v - 3), v)}[probe]
            dfeat[b, sel] = full[b, sel]
        log = {}
        record(monkeypatch, log)
        m.zero_grad_buffer()
        for p in params.values():
            eng.g(p).fill_(BASE)
        eng.conv_backward(st, dfeat)
        torch.cuda.synchronize()
        monkeypatch.undo()

        def grad(nm_):
            return eng.g(params[nm_]).double() - BASE

        dY = dict(zip(range(n - 1, 0, -1), log["gemm_wgrad.in"]))  # kernel d(conv output) of layers n-1 .. 1
        dA0 = log["conv0_bwd.in"][0]  # kernel gradient at layer 0's output
        assert len(dY) == n - 1 and all(dY[i].shape == (B, T[i], C) for i in dY)
        if ln:
            dA = dict(zip(range(n - 1, 0, -1), log["layer_norm_bwd.in"]))
            assert torch.equal(dA[n - 1], dfeat[:, :T6]) and all(torch.equal(o, dY[i]) for i, o in
                                                                  zip(range(n - 1, 0, -1), log["layer_norm_bwd.out"]))
        for i in range(n - 1, 0, -1):
            _, k, s = convs[i]
            # d(conv output) of layer i from the gradient at its output
            if ln:
                nm = norms[i]
                dgm_ref = torch.zeros(C, dtype=F64, device=dev); dbt_ref = torch.zeros_like(dgm_ref)
                qg = torch.zeros_like(dgm_ref); qb = torch.zeros_like(dgm_ref)
                xg = torch.zeros_like(dgm_ref); xb = torch.zeros_like(dgm_ref)
                for b in range(B):
                    yk = st["y"][i][b, :T[i]].double().requires_grad_(True)
                    gm, bt = nm.weight.detach().double().requires_grad_(True), nm.bias.detach().double().requires_grad_(True)
                    mean, r, xh, z = ln_fwd_parts(yk, gm, bt)
                    dA_b = dA[i][b].double()
                    ref, dgm, dbt = torch.autograd.grad(gelu64(z), (yk, gm, bt), dA_b)
                    dz = (dA_b * dgelu64(z.detach())).abs()
                    Mdy, _, _ = ln_bwd_mag(dA_b.abs(), r.detach(), xh.detach(), z.detach(), nm.weight.double())
                    # fp32 LayerNorm backward over C channels (kernel mean / rstd within 2^-18): 2^-16 of the terms
                    assert_close(dY[i][b], ref, bf16_bound(ref, 2.0 ** -16 * Mdy), f"{probe}: dY{i}[{b}] (LayerNorm backward)")
                    dgm_ref += dgm; dbt_ref += dbt
                    qg += ((dz * xh.detach().abs()) ** 2).sum(0); qb += (dz ** 2).sum(0)
                    # the fp32 xh is off by a few EPS32 of r (|y| + |mean|) in absolute terms (large relative to xh near 0),
                    # plus |xh| times the stored rstd's error (the forward bound above, large for near-constant rows); it
                    # enters dgamma directly and dbeta through gelu' (|gelu''| <= 0.8)
                    rd, ya = r.detach(), yk.detach().abs()
                    ex = 2.0 ** -16 * rd * (ya + mean.detach().abs()) + xh.detach().abs() * (
                        2.0 ** -18 + 16 * EPS32 * ya.mean(1, keepdim=True) * rd)
                    # gelu' comes from the Abramowitz-Stegun 7.1.26 erfc approximation (absolute error 1.5e-7 < 2^-21 for erf)
                    xg += (dz * ex + dA_b.abs() * xh.detach().abs() * 2.0 ** -21).sum(0)
                    xb += (dA_b.abs() * (nm.weight.double().abs() * ex + 2.0 ** -21)).sum(0)
                nr = sum(nonzero_rows(dA[i][b]) for b in range(B))
                assert_close(grad(f"gamma{i}"), dgm_ref, acc_tol(qg, nr) + term_tol(qg, nr) + xg + 2 * EPS32 * BASE, f"{probe}: dgamma{i}")
                assert_close(grad(f"beta{i}"), dbt_ref, acc_tol(qb, nr) + term_tol(qb, nr) + xb + 2 * EPS32 * BASE, f"{probe}: dbeta{i}")
            elif i == n - 1:
                # dY = bf16(dfeat * gelu') with gelu' the stored bf16: the fp32 product is exact, one rounding
                ref = dfeat[:, :T6].double() * st["y"][i][:, :T6].double()
                assert_close(dY[i], ref, bf16_bound(ref, 0.0), f"{probe}: dY{i} (dgelu)")
            # weight gradient of layer i from the kernel's dY_i and a_{i-1}
            dw_ref = torch.zeros(C, C, k, dtype=F64, device=dev)
            sq = torch.zeros_like(dw_ref)
            for b in range(B):
                a_prev = st["a"][i - 1][b, :T[i - 1]].double()
                d = dY[i][b].double()
                dw_ref += wgrad_rows(a_prev, d, dw_ref.shape, k, s)
                sq += wgrad_rows(a_prev * a_prev, d * d, dw_ref.shape, k, s)
            nr = sum(nonzero_rows(dY[i][b]) for b in range(B))
            assert_close(grad(f"w{i}"), dw_ref, acc_tol(sq, nr) + 2 * EPS32 * BASE, f"{probe}: dw{i}")
            # gradient at layer i-1's output (phase GEMMs over the stride, GroupNorm mode with the fused dgelu epilogue)
            for b in range(B):
                d = dY[i][b].double()
                ref = convT_rows(d, Wb[i], k, s, T[i - 1])
                # fp32 accumulation of at most 2 * C <= 1024 products: K EPS32 = 2^-14 of sum |terms|
                mag = convT_rows(d.abs(), Wb[i].abs(), k, s, T[i - 1])
                if i - 1 == 0:
                    got, what = dA0[b], "dA0"
                elif ln:
                    got, what = dA[i - 1][b], f"dA{i - 1}"
                else:
                    gp = st["y"][i - 1][b, :T[i - 1]].double()
                    ref, mag, got, what = ref * gp, mag * gp.abs(), dY[i - 1][b], f"dY{i - 1} (fused dgelu)"
                assert_close(got, ref, bf16_bound(ref, 2.0 ** -14 * mag), f"{probe}: {what}[{b}]")
        # ---- layer 0 from the kernel's gradient at its output
        dw0 = torch.zeros(C, K0, dtype=F64, device=dev)
        M = {key: 0.0 for key in ("dw", "dgamma", "dbeta", "Mdw", "Mdgamma", "Mdgamma_x", "Mdbeta", "Mdbeta_x", "Qdgamma", "Qdbeta",
                                  "sq")}
        for b in range(B):
            r0 = conv0_ref(wav[b].double(), T[0], w0, nm0.weight.detach().double(), nm0.bias.detach().double(), ln,
                           da=dA0[b].double())
            for key in M:
                if key in r0:
                    M[key] = M[key] + r0[key]
            if ln:
                dconv_k = log["conv0_bwd.out"][0][b]
                # fp32 LayerNorm backward over C channels (kernel fmean / frstd), stored as bf16
                assert_close(dconv_k, r0["dconv"], bf16_bound(r0["dconv"], 2.0 ** -16 * r0["Mdconv"]), f"{probe}: dconv0[{b}]")
                X = wav[b].double().unfold(0, K0, S0)[:T[0]]
                dw0 += dconv_k.double().t() @ X
                M["sq"] = M["sq"] + (dconv_k.double() ** 2).t() @ (X * X)
        nr0 = sum(nonzero_rows(dA0[b]) for b in range(B))
        if ln:
            # pass B: fp32 sum over frames of the stored d(conv) times the waveform; pass A: dgamma / dbeta in fp32
            assert_close(grad("w0").view(C, K0), dw0, acc_tol(M["sq"], nr0) + 2 * EPS32 * BASE, f"{probe}: dw0")
            assert_close(grad("gamma0"), M["dgamma"], acc_tol(M["Qdgamma"], nr0) + term_tol(M["Qdgamma"], nr0) + 2.0 ** -16 * M["Mdgamma_x"]
                         + 2 * EPS32 * BASE, f"{probe}: dgamma0")
            assert_close(grad("beta0"), M["dbeta"], acc_tol(M["Qdbeta"], nr0) + term_tol(M["Qdbeta"], nr0) + 2.0 ** -16 * M["Mdbeta_x"]
                         + 2 * EPS32 * BASE, f"{probe}: dbeta0")
        else:
            # GroupNorm single-pass backward: fp32 per-frame arithmetic and chunk sums, as in test_conv0
            assert_close(grad("w0").view(C, K0), M["dw"], 2.0 ** -12 * M["Mdw"] + 2 * EPS32 * BASE, f"{probe}: dw0")
            assert_close(grad("gamma0"), M["dgamma"], 2.0 ** -12 * M["Mdgamma"] + 2.0 ** -16 * M["Mdgamma_x"] + 2 * EPS32 * BASE,
                         f"{probe}: dgamma0")
            assert_close(grad("beta0"), M["dbeta"], 2.0 ** -12 * M["Mdbeta"] + 2.0 ** -16 * M["Mdbeta_x"] + 2 * EPS32 * BASE,
                         f"{probe}: dbeta0")


# ------------------------------------------------------------------------------------------------- pos_conv stem
def weight_norm64(v, g):
    """nn.utils.weight_norm(dim=2): w = g * v / ||v||, the norm over the two leading dims, per tap."""
    return g * v / v.norm(2, dim=(0, 1), keepdim=True)


def posconv_rows(xrows, w, G, n):
    """Grouped Conv1d (128 taps) of one utterance's zero-padded rows: xrows [n + taps - 1, D] -> [n, D] (float64); output
    frame t reads rows t .. t + 127, i.e. padding 64 with SamePad's last frame dropped."""
    D, Cg, taps = w.shape
    X = xrows.unfold(0, taps, 1)[:n].reshape(n, G, Cg * taps).transpose(0, 1)  # [G, n, Cg*taps] (ci major, j minor)
    Wg = w.reshape(G, Cg, Cg * taps)  # [G, co, ci*taps]
    return torch.bmm(X, Wg.transpose(1, 2)).transpose(0, 1).reshape(n, D)


def kernel_taps(eng, D, G, taps):
    """The bf16 forward taps the kernel reads, in the reference Conv1d layout [D, Cg, taps] (float64)."""
    Cg = D // G
    return eng.pc_fwd[:, :Cg, :, :Cg].permute(0, 1, 3, 2).reshape(D, Cg, taps).double()


POSCONV_CASES = [("base", 16, 749), ("base", 16, 1499), ("base", 16, 1), ("base", 16, 63), ("base", 1, 64), ("base", 8, 65),
                 ("base", 16, 128), ("base", 1, 14999), ("large", 8, 999), ("large", 8, 1), ("large", 1, 127),
                 ("large", 8, 129), ("large", 1, 999), ("large", 8, 64)]


def test_posconv_prep(cuda_device):
    """posconv_prep at the shipped widths: D = 768 (Cg = 48, the 64-wide tile holds zero columns) and 1024 (Cg = 64)."""
    dev = cuda_device
    for name in ("base", "large"):
        m, _, _ = model(name, dev)
        eng = m._begin(dev)
        torch.cuda.synchronize()
        pc = m.encoder.pos_conv[0]
        G, taps = m.cfg.conv_pos_groups, m.cfg.conv_pos
        D = m.cfg.encoder_embed_dim
        Cg = D // G
        w = weight_norm64(pc.weight_v.detach().double(), pc.weight_g.detach().double())  # [D, Cg, taps]
        ref_f = w.view(G, Cg, Cg, taps).permute(0, 1, 3, 2)  # [g, co, j, ci]
        # fp32 g * v * rsqrtf(norm^2) (a few ulp) rounded to bf16
        assert_close(eng.pc_fwd[:, :Cg, :, :Cg], ref_f, bf16_bound(ref_f, 2.0 ** -20 * ref_f.abs()), f"{name} forward taps")
        assert (eng.pc_fwd[:, Cg:] == 0).all() and (eng.pc_fwd[:, :, :, Cg:] == 0).all(), f"{name} forward taps: padding"
        # the input-gradient taps are the same values flipped and transposed: pc_dg[g, ci, j', co] = pc_fwd[g, co, taps-1-j', ci]
        assert torch.equal(eng.pc_dg, eng.pc_fwd.flip(2).permute(0, 3, 2, 1)), f"{name} input-gradient taps"


@pytest.mark.parametrize("name,B,T", POSCONV_CASES, ids=[f"{n}-B{b}-T{t}" for n, b, t in POSCONV_CASES])
def test_posconv_stem(cuda_device, monkeypatch, name, B, T):
    dev = cuda_device
    m, _, _ = model(name, dev)
    eng = m._begin(dev)
    cfg = m.cfg
    D, G, taps, half = cfg.encoder_embed_dim, cfg.conv_pos_groups, cfg.conv_pos, cfg.conv_pos // 2
    Cg = D // G
    K = Cg * taps  # products per output element of the tap GEMMs
    post_ln = not cfg.layer_norm_first
    pc, eln = m.encoder.pos_conv[0], m.encoder.layer_norm
    g = torch.Generator().manual_seed(B * 100003 + T)
    x = torch.randn(B, T, D, generator=g).to(BF).to(dev)
    xpad = torch.zeros(B, T + taps, D, dtype=BF, device=dev)
    xpad[:, half:half + T] = x
    out, st = eng.posconv_forward(xpad, T, True)
    eng._pending_gate = None
    torch.cuda.synchronize()
    wk = kernel_taps(eng, D, G, taps)  # checked against the float64 weight norm by test_posconv_prep
    bias64 = pc.bias.detach().double()
    gam, bet = eln.weight.detach().double(), eln.bias.detach().double()
    CH = 1024  # output frames per reference chunk (the unfolded window is CH x D x 128 float64)
    dx0 = torch.randn(B, T, D, generator=g).to(BF).to(dev)

    # ---- forward
    for b in range(B):
        xr = xpad[b].double()
        for t0 in range(0, T, CH):
            n = min(CH, T - t0)
            rows = xr[t0:t0 + n + taps - 1]
            conv = posconv_rows(rows, wk, G, n) + bias64
            # fp32 accumulation of K products of the kernel's own bf16 taps and inputs, plus the bias
            tc = acc_tol(posconv_rows(rows * rows, wk * wk, G, n), K) + 4 * EPS32 * bias64.abs()
            ref_xs = x[b, t0:t0 + n].double() + gelu64(conv)
            assert_close(st["xs"][b, t0:t0 + n], ref_xs, bf16_bound(ref_xs, 1.13 * tc + 2 * EPS32 * ref_xs.abs()), f"xs[{b}]")
            gp = dgelu64(conv)
            assert_close(st["pre"][b, t0:t0 + n], gp, bf16_bound(gp, 0.8 * tc), f"gelu'[{b}]")
        if post_ln:  # post-LN encoder.layer_norm on the kernel's own xs (teacher-forced)
            xs_k = st["xs"][b].double()
            mean, r, xh, z = ln_fwd_parts(xs_k, gam, bet)
            assert_close(out[b], z, bf16_bound(z, 2.0 ** -16 * (xh.abs() * gam.abs() + bet.abs())), f"x0[{b}]")
            ym = xs_k.abs().mean(1)
            assert_close(st["mean"].view(B, T)[b], mean[:, 0], 2.0 ** -18 * ym, f"mean[{b}]")
            rr = r[:, 0]
            assert_close(st["rstd"].view(B, T)[b], rr, rr * (2.0 ** -18 + 16 * EPS32 * ym * rr), f"rstd[{b}]")

    # ---- kernel backward, recording its intermediate gradients
    log = {}
    record(monkeypatch, log)
    m.zero_grad_buffer()
    pnames = {"bias": pc.bias, "weight_v": pc.weight_v, "weight_g": pc.weight_g}
    if post_ln:
        pnames.update({"ln.weight": eln.weight, "ln.bias": eln.bias})
    for p in pnames.values():
        eng.g(p).fill_(BASE)
    dxm = eng.posconv_backward(st, dx0, T)
    torch.cuda.synchronize()
    monkeypatch.undo()

    def grad(nm_):
        return eng.g(pnames[nm_]).double() - BASE

    dpre_k = log["posconv_wgrad.in"][0]  # [B, T, D] bf16
    dwp_k = log["posconv_wgrad.out"][0]  # [G, Cg, taps, 64] fp32
    dxs_k = log["layer_norm_bwd.out"][0] if post_ln else dx0
    nrows = B * T
    # ---- post-LN backward from dx0 at the kernel's xs
    if post_ln:
        dgm_ref = torch.zeros_like(gam); dbt_ref = torch.zeros_like(gam); qg = torch.zeros_like(gam); qb = torch.zeros_like(gam)
        xg = torch.zeros_like(gam)
        for b in range(B):
            xs_ = st["xs"][b].double().requires_grad_(True)
            gm_, bt_ = gam.clone().requires_grad_(True), bet.clone().requires_grad_(True)
            mean, r, xh, z = ln_fwd_parts(xs_, gm_, bt_)
            d0 = dx0[b].double()
            ref, dg_, db_ = torch.autograd.grad(z, (xs_, gm_, bt_), d0)
            dxh = d0.abs() * gam.abs()
            xha = xh.detach().abs()
            Mdxs = r.detach() * (dxh + dxh.mean(1, keepdim=True) + xha * (dxh * xha).mean(1, keepdim=True))
            assert_close(dxs_k[b], ref, bf16_bound(ref, 2.0 ** -16 * Mdxs), f"dxs[{b}] (LayerNorm backward)")
            dgm_ref += dg_; dbt_ref += db_
            qg += ((d0 * xha) ** 2).sum(0); qb += (d0 ** 2).sum(0)
            # the fp32 xh's absolute error and the stored rstd's error (see test_conv_stack)
            rd, xa = r.detach(), xs_.detach().abs()
            xg += (d0.abs() * (2.0 ** -16 * rd * (xa + mean.detach().abs())
                               + xha * (2.0 ** -18 + 16 * EPS32 * xa.mean(1, keepdim=True) * rd))).sum(0)
        assert_close(grad("ln.weight"), dgm_ref, acc_tol(qg, nrows) + term_tol(qg, nrows) + xg + 2 * EPS32 * BASE, "d ln.weight")
        assert_close(grad("ln.bias"), dbt_ref, acc_tol(qb, nrows) + term_tol(qb, nrows) + 2 * EPS32 * BASE, "d ln.bias")
    # ---- dpre = bf16(dxs * gelu'), both bf16: the fp32 product is exact, one rounding
    ref = dxs_k.double() * st["pre"].double()
    assert_close(dpre_k, ref, bf16_bound(ref, 0.0), "dpre (dgelu)")
    dp = dpre_k.double()
    assert_close(grad("bias"), dp.sum((0, 1)), acc_tol((dp * dp).sum((0, 1)), nrows) + 2 * EPS32 * BASE, "d bias")
    # ---- tap weight gradient (posconv_wgrad) and input gradient (posconv_gemm on the flipped taps) from the kernel's dpre
    dw = torch.zeros(D, Cg, taps, dtype=F64, device=dev)
    sqw = torch.zeros_like(dw)
    for b in range(B):
        xr = xpad[b].double()
        dx_conv = torch.zeros(T + taps, D, dtype=F64, device=dev)
        sqx = torch.zeros_like(dx_conv)
        for t0 in range(0, T, CH):
            n = min(CH, T - t0)
            rows = xr[t0:t0 + n + taps - 1].clone().requires_grad_(True)
            w_ = wk.clone().requires_grad_(True)
            d = dp[b, t0:t0 + n]
            d_rows, d_w = torch.autograd.grad(posconv_rows(rows, w_, G, n), (rows, w_), d)
            dx_conv[t0:t0 + n + taps - 1] += d_rows
            dw += d_w
            rows2 = (xr[t0:t0 + n + taps - 1] ** 2).requires_grad_(True)
            w2 = (wk * wk).requires_grad_(True)
            s_rows, s_w = torch.autograd.grad(posconv_rows(rows2, w2, G, n), (rows2, w2), d * d)
            sqx[t0:t0 + n + taps - 1] += s_rows
            sqw += s_w
        branch = dx_conv[half:half + T]
        tb = acc_tol(sqx[half:half + T], K)
        # dxm = bf16(dxs + conv branch): check the conv branch on its own (the residual is the kernel's own dxs, exact)
        ref_dxm = dxs_k[b].double() + branch
        assert_close(dxm[b].double() - dxs_k[b].double(), branch, bf16_bound(ref_dxm, tb), f"dxm - dxs (conv branch)[{b}]")
    ref_dwp = dw.view(G, Cg, Cg, taps).permute(0, 1, 3, 2)  # [g, co, j, ci]
    tol_w = acc_tol(sqw, nrows)
    assert_close(dwp_k[:, :, :, :Cg], ref_dwp, tol_w.view(G, Cg, Cg, taps).permute(0, 1, 3, 2), "d taps (posconv_wgrad)")
    # ---- weight-norm backward (posconv_unprep) from the kernel's own tap gradient
    v64, g64 = pc.weight_v.detach().double(), pc.weight_g.detach().double()
    dwk = dwp_k[:, :, :, :Cg].double().permute(0, 1, 3, 2).reshape(D, Cg, taps)
    v_, g_ = v64.clone().requires_grad_(True), g64.clone().requires_grad_(True)
    dv, dgw = torch.autograd.grad(weight_norm64(v_, g_), (v_, g_), dwk)
    nrm = v64.norm(2, dim=(0, 1), keepdim=True)
    dot = (dwk * v64).sum((0, 1), keepdim=True)
    # fp32 tap reductions (norm^2 and dot(dw, v), fp32 per thread then fp64) and fp32 arithmetic of both terms
    tdot = acc_tol(((dwk * v64) ** 2).sum((0, 1), keepdim=True), D * Cg) + 2.0 ** -18 * dot.abs()
    tdv = 2.0 ** -18 * (g64.abs() / nrm * dwk.abs() + g64.abs() * dot.abs() / nrm ** 3 * v64.abs()) \
        + g64.abs() / nrm ** 3 * v64.abs() * tdot
    assert_close(grad("weight_v"), dv, tdv + 2 * EPS32 * BASE, "d weight_v")
    assert_close(grad("weight_g"), dgw, tdot / nrm + 2 * EPS32 * BASE, "d weight_g")
