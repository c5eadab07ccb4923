"""Op-level tests of the pre-training loss-head kernels: the masked-prediction head (csrc/nce.cu), the contrastive heads and the
Gumbel quantizer (csrc/sat.cu) and the feature-penalty pair of csrc/rowops.cu.

Every reference is computed in float64 from the same bf16 / fp32 tensors the kernel reads, so only the kernel's arithmetic is
under test (the oracle's cosine similarity alone runs in fp32, and the bounds allow for it), and every reference gradient
comes from torch.autograd on that reference, never from the kernel's closed form.
The sizes are the shipped ones (final_dim 256 / 768, 504 classes, 100 negatives, 2 x 320 latent codes) and the edges of each
kernel's thread mapping.  Outputs are pre-filled with NaN and `+=` outputs with non-zero values, so an element left unwritten
or an accumulation that overwrites shows.  Each tolerance is written next to its reason; EPS32 = 2^-24 is the fp32 unit
roundoff."""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wavlm_oracle as O
from unispeech_b200 import dropout as DR
from unispeech_b200 import ops

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
F64 = torch.float64
EPS32 = 2.0 ** -24
SITE_GUMBEL = 0x7F000003  # noise site of the wav2vec 2.0 quantizer (unispeech_b200/wav2vec2.py)


# ------------------------------------------------------------------------------------------------------------- helpers
def f32(v: float) -> float:
    """The value a float argument has once it crosses the C ABI as a float32."""
    return float(np.float32(v))


def ulp_bf16(x: torch.Tensor) -> torch.Tensor:
    """One bf16 ulp at |x| (the ulp of the smallest normal below it)."""
    a = x.abs().clamp_min(2.0 ** -126)
    return torch.exp2(torch.floor(torch.log2(a)) - 7)


def bits(t: torch.Tensor) -> torch.Tensor:
    """Bit pattern of a tensor, for bit-exact comparisons (NaN == NaN)."""
    t = t.contiguous()
    return t.view({2: torch.int16, 4: torch.int32, 8: torch.int64}[t.element_size()])


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


def first_argmax(x: torch.Tensor) -> torch.Tensor:
    """Index of the first maximum along the last dim (torch.max's rule, stated explicitly rather than relied on)."""
    mx = x.max(-1, keepdim=True).values
    ar = torch.arange(x.shape[-1], device=x.device).expand_as(x)
    return torch.where(x == mx, ar, x.shape[-1]).min(-1).values


def sms() -> int:
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------------- masked-prediction head
@pytest.mark.parametrize("Dp", [64, 256, 768])
@pytest.mark.parametrize("C", [1, 37, 504, 1024])
def test_nce_prep(cuda_device, C, Dp):
    dev = cuda_device
    Cpad = (C + 63) // 64 * 64
    g = torch.Generator().manual_seed(C * 7 + Dp)
    E = torch.randn(C, Dp, generator=g) * torch.exp2(torch.randint(-6, 7, (C, 1), generator=g).float())
    if C > 1:
        E[C // 2] = 0.0  # the norm clamps at 1e-8: en row 0, invn = 1e8
    E = E.to(dev)
    en, en_t, invn = nan_like((Cpad, Dp), BF, dev), nan_like((Dp, Cpad), BF, dev), nan_like((C,), torch.float32, dev)
    ops.nce_prep(E, C, Cpad, Dp, en, en_t, invn)
    torch.cuda.synchronize()
    nrm = E.double().norm(dim=1, keepdim=True).clamp_min(1e-8)
    ref = E.double() / nrm
    # fp32 quotient (a few EPS32 relative) rounded to bf16: within one bf16 ulp
    assert_close(en[:C], ref, ulp_bf16(ref), "en")
    assert (en[C:].float() == 0).all(), "padded rows of en must be exactly 0"
    assert torch.equal(bits(en_t), bits(en.t())), "en_t must be en transposed, bit for bit"
    # sum of squares over Dp / 32 terms per lane + a 5-level shuffle tree, sqrt, reciprocal
    assert_close(invn, 1.0 / nrm.squeeze(1), 1e-6 / nrm.squeeze(1), "invn")


def _nce_ce_inputs(S, C, Dp, seed, dev):
    """proj (second half of an [S, 2 Dp] untied projection), zraw on a coarse bf16 grid with its target column set to tie the
    best other class (rows s % 4 == 0), to be the unique maximum (1), to sit below the maximum (2) or as drawn (3)."""
    Cpad = (C + 63) // 64 * 64
    g = torch.Generator().manual_seed(seed)
    proj_full = torch.randn(S, 2 * Dp, generator=g).to(BF)
    k = torch.randint(-24, 25, (S, Cpad), generator=g).double()
    t = torch.randint(0, C, (S,), generator=g)
    t[0] = 0
    if S > 1:
        t[1] = C - 1
    rows = torch.arange(S)
    if C > 1:
        others = k[:, :C].clone()
        others[rows, t] = -math.inf
        mo = others.max(1).values
        mode = rows % 4
        k[rows, t] = torch.where(mode == 0, mo, torch.where(mode == 1, mo + 1, torch.where(mode == 2, mo - 1, k[rows, t])))
    k[:, C:] = 100.0  # padded columns of the GEMM output: the kernel must ignore them
    zraw = (k * 0.25).to(BF)
    return proj_full.to(dev), zraw.to(dev), t.to(torch.int32).to(dev), Cpad


def _nce_ce_reference(proj, zraw, t, C, temp, w):
    """fp64: z = zraw / |proj| / temp; the [S, C+1] logits of compute_nce (positive first, -inf at the target's own column);
    summed weighted cross entropy; G = d loss / d zraw (at fixed |proj|) by autograd."""
    S = proj.shape[0]
    rows = torch.arange(S, device=proj.device)
    nrm = proj.double().norm(dim=1).clamp_min(1e-8)
    zr = zraw[:, :C].double().requires_grad_(True)
    z = zr / nrm[:, None] / temp
    tl = t.long()
    onehot = F.one_hot(tl, C).bool()
    L = torch.cat([z[rows, tl][:, None], z.masked_fill(onehot, -math.inf)], dim=1)
    ce = F.cross_entropy(L, torch.zeros(S, dtype=torch.long, device=proj.device), reduction="none")
    (w * ce).sum().backward()
    G = zr.grad
    z = z.detach()
    L = L.detach()
    correct = int(((L.argmax(1) == 0) & ~(L.argmin(1) == 0)).sum())
    p = torch.softmax(z, 1)
    return dict(nrm=nrm, z=z, ce=ce.detach(), G=G, p=p, onehot=onehot, rvec=(G * z * temp).sum(1), correct=correct)


@pytest.mark.parametrize("C", [1, 37, 504, 1000])
@pytest.mark.parametrize("S", [1, 7, 3000])
def test_nce_ce(cuda_device, S, C):
    dev = cuda_device
    Dp = 768 if C == 1000 else 256
    temp, w = f32(0.1), f32(0.7)
    proj_full, zraw, t, Cpad = _nce_ce_inputs(S, C, Dp, S * 131 + C, dev)
    proj = proj_full[:, Dp:]
    G, pn, rvec = nan_like((S, Cpad), BF, dev), nan_like((S,), torch.float32, dev), nan_like((S,), torch.float32, dev)
    loss = torch.full((1,), 1.25, dtype=F64, device=dev)
    correct = torch.full((1,), 3, dtype=torch.int32, device=dev)
    ops.nce_ce(proj, 2 * Dp, Dp, zraw, Cpad, t, S, C, Cpad, temp, w, G, Cpad, pn, rvec, loss, correct)
    torch.cuda.synchronize()
    R = _nce_ce_reference(proj, zraw, t, C, temp, w)
    z, p = R["z"], R["p"]
    zmax = z.max(1).values
    zt = z[torch.arange(S, device=dev), t.long()]
    # Relative error of every fp32 logit and softmax value: |proj| over Dp / 32 products per lane + shuffles, the scale
    # inv / temp, __expf (2 ulp) and the C-term sum and its reciprocal.
    rel = (Dp / 32 + C / 32 + 32) * EPS32
    # loss: per row w (lse - z_t) with __logf's absolute error (2^-21.4) and the relative error above on |lse| + |z_t|
    tol_loss = (abs(w) * (2.0 ** -21 + rel * (1 + zmax.abs() + zt.abs()))).sum().item()
    assert abs(loss.item() - 1.25 - R["ce"].sum().item() * w) <= tol_loss, (loss.item() - 1.25, R["ce"].sum().item() * w, tol_loss)
    assert_close(pn, 1.0 / R["nrm"], (Dp / 32 + 8) * EPS32 / R["nrm"], "pn")
    # G: one bf16 ulp on the bf16 output plus the fp32 error of p, scaled by w / (|proj| temp)
    zs = 1.0 / (R["nrm"] * temp)
    gscale = abs(w) * zs[:, None] * (p + R["onehot"].double())
    assert_close(G[:, :C], R["G"], ulp_bf16(R["G"]) + gscale * rel, "G")
    assert (G[:, C:].float() == 0).all(), "padded columns of G must be exactly 0 (NaN there poisons the G En GEMM)"
    # rvec = sum_c G_sc cos_sc: the error of each fp32 term plus the fp32 sum over C / 32 terms per lane and the shuffles
    cos = z * temp
    tol_r = (2 * rel + (C / 32 + 8) * EPS32) * (R["G"] * cos).abs().sum(1) + 1e-30
    assert_close(rvec, R["rvec"], tol_r, "rvec")
    # compute_correct on the [S, C+1] layout is exact: z is a positive multiple of the bf16 zraw, so order and ties survive
    assert correct.item() - 3 == R["correct"], (correct.item() - 3, R["correct"])
    if C > 1 and S > 4:
        mode = torch.arange(S, device=dev) % 4
        assert 0 < R["correct"] < S and bool(((mode == 0) & (zt == zmax)).any())
    # correct = NULL: same results, nothing counted
    G2 = nan_like((S, Cpad), BF, dev)
    pn2, rvec2 = nan_like((S,), torch.float32, dev), nan_like((S,), torch.float32, dev)
    loss2 = torch.zeros(1, dtype=F64, device=dev)
    ops.nce_ce(proj, 2 * Dp, Dp, zraw, Cpad, t, S, C, Cpad, temp, w, G2, Cpad, pn2, rvec2, loss2, None)
    torch.cuda.synchronize()
    assert torch.equal(bits(G2), bits(G)) and torch.equal(bits(pn2), bits(pn)) and torch.equal(bits(rvec2), bits(rvec))
    assert abs(loss2.item() - (loss.item() - 1.25)) <= tol_loss


@pytest.mark.parametrize("S,Dp", [(1, 64), (37, 256), (3000, 768)])
def test_nce_dproj(cuda_device, S, Dp):
    dev = cuda_device
    g = torch.Generator().manual_seed(S + Dp)
    dstore = torch.randn(S, 2 * Dp + 16, generator=g).to(BF).to(dev)
    pstore = torch.randn(S, 3 * Dp, generator=g).to(BF).to(dev)
    pn = (torch.rand(S, generator=g) * 0.15 + 0.05).to(dev)
    rvec = (torch.randn(S, generator=g) * 3).to(dev)
    d, p = dstore[:, 8:8 + Dp], pstore[:, Dp:2 * Dp]
    before = dstore.clone()
    a, b = d.double(), p.double()
    k = (rvec.double() * pn.double())[:, None]
    ref = a - k * b
    ops.nce_dproj(d, dstore.stride(0), p, pstore.stride(0), S, Dp, pn, rvec)
    torch.cuda.synchronize()
    # one bf16 ulp on the bf16 output plus fp32 rounding of rvec pn and of the fma
    assert_close(d, ref, ulp_bf16(ref) + 4 * EPS32 * (a.abs() + (k * b).abs()), "dproj")
    assert torch.equal(bits(dstore[:, :8]), bits(before[:, :8])) and torch.equal(bits(dstore[:, 8 + Dp:]), bits(before[:, 8 + Dp:]))


def _dlabel_reference(dEn, E):
    """d E of E -> E / max(|E|, 1e-8) under the upstream gradient dEn, by fp64 autograd."""
    Er = E.double().requires_grad_(True)
    (Er / Er.norm(dim=1, keepdim=True).clamp_min(1e-8)).backward(dEn.double())
    return Er.grad


@pytest.mark.parametrize("C,Dp", [(1, 64), (504, 256), (1000, 768)])
def test_nce_dlabel(cuda_device, C, Dp):
    dev = cuda_device
    g = torch.Generator().manual_seed(C + Dp)
    E = (torch.randn(C, Dp, generator=g) * torch.exp2(torch.randint(-4, 5, (C, 1), generator=g).float())).to(dev)
    nrm = E.double().norm(dim=1, keepdim=True)
    En = E.double() / nrm
    # d En with a large component along En: the projection term of the backward carries weight
    dEn = (torch.randn(C, Dp, generator=g).to(dev).double() + 4 * torch.randn(C, 1, generator=g).to(dev).double() * En).float()
    invn = (1.0 / nrm.squeeze(1)).float()
    init = torch.randn(C, Dp, generator=g).to(dev)
    dE = init.clone()
    ops.nce_dlabel(dEn, E, invn, C, Dp, dE)
    torch.cuda.synchronize()
    ref = init.double() + _dlabel_reference(dEn, E)
    inv = 1.0 / nrm
    dot = (dEn.double() * En).sum(1, keepdim=True)
    # fp32 dot over Dp / 32 products per lane + shuffles, fp32 rounding of invn and of each output term, and the += rounding
    err_dot = (Dp / 32 + 8) * EPS32 * (dEn.double() * En).abs().sum(1, keepdim=True)
    tol = inv * (8 * EPS32 * (dEn.double().abs() + dot.abs() * En.abs()) + err_dot * En.abs()) + 2 * EPS32 * (ref.abs() + init.double().abs())
    assert_close(dE, ref, tol, "d label_embs")


def test_nce_head_derivation(cuda_device):
    """The hand-derived decomposition itself: nce_prep -> zraw = proj En^T -> nce_ce -> d proj = G En - rvec pn proj (nce_dproj)
    and d En = G^T proj -> d E (nce_dlabel), against fp64 autograd of compute_nce + summed cross entropy.  The three GEMMs run
    in fp64 and are rounded where the library's GEMMs round (bf16 outputs for zraw and G En, fp32 for G^T proj)."""
    dev = cuda_device
    S, C, Dp, temp, w = 3000, 504, 256, f32(0.1), f32(0.5)
    Cpad = (C + 63) // 64 * 64
    g = torch.Generator().manual_seed(11)
    E = torch.randn(C, Dp, generator=g).to(dev)
    t = torch.randint(0, C, (S,), generator=g).to(dev)
    # trained-like projections: each leans towards its target's embedding, so the positive's cosine is large (about 0.4)
    En64 = E.double() / E.double().norm(dim=1, keepdim=True)
    proj = (7.0 * En64[t] * math.sqrt(Dp) / 16 + torch.randn(S, Dp, generator=g).to(dev).double()).to(BF)
    en, en_t, invn = nan_like((Cpad, Dp), BF, dev), nan_like((Dp, Cpad), BF, dev), nan_like((C,), torch.float32, dev)
    ops.nce_prep(E, C, Cpad, Dp, en, en_t, invn)
    zraw = (proj.double() @ en.double().t()).to(BF)
    G = nan_like((S, Cpad), BF, dev)
    pn, rvec = nan_like((S,), torch.float32, dev), nan_like((S,), torch.float32, dev)
    loss = torch.zeros(1, dtype=F64, device=dev)
    ops.nce_ce(proj, Dp, Dp, zraw, Cpad, t.to(torch.int32), S, C, Cpad, temp, w, G, Cpad, pn, rvec, loss, None)
    dproj = (G.double() @ en.double()).to(BF)
    ops.nce_dproj(dproj, Dp, proj, Dp, S, Dp, pn, rvec)
    d_en = (G.double().t() @ proj.double()).float()
    dE = torch.zeros(C, Dp, device=dev)
    ops.nce_dlabel(d_en, E, invn, C, Dp, dE)
    torch.cuda.synchronize()

    pr = proj.double().requires_grad_(True)
    Er = E.double().requires_grad_(True)
    ref_loss = 0.0
    for s0 in range(0, S, 500):
        s1 = min(S, s0 + 500)
        logits = O.compute_nce(pr[s0:s1], Er[t[s0:s1]], Er.unsqueeze(1).expand(-1, s1 - s0, -1), temp)
        part = w * F.cross_entropy(logits, torch.zeros(s1 - s0, dtype=torch.long, device=dev), reduction="sum")
        part.backward()
        ref_loss += part.item()
    # zraw, En, G and G En are each rounded to bf16 (2^-9 relative per element); four independent roundings stay well
    # inside 1 % of the gradient's norm, while a missing term of the decomposition moves it by tens of percent
    assert abs(loss.item() - ref_loss) <= 2e-3 * abs(ref_loss), (loss.item(), ref_loss)
    for name, got, ref in (("d proj", dproj, pr.grad), ("d label_embs", dE, Er.grad)):
        assert torch.isfinite(got.float()).all(), name
        err = (got.double() - ref).norm() / ref.norm()
        assert err < 1e-2, (name, err.item())


@pytest.mark.parametrize("S,D", [(1, 8), (37, 768), (30000, 264)])
def test_gather_rows(cuda_device, S, D):
    dev = cuda_device
    R = max(S // 3, 5)
    g = torch.Generator().manual_seed(S + D)
    x = torch.randn(R, D + 24, generator=g).to(BF).to(dev)
    idx = torch.randint(0, R, (S,), generator=g).to(torch.int32).to(dev)
    out = nan_like((S, D + 8), BF, dev)
    ops.gather_rows(x, D + 24, idx, S, D, out, D + 8)
    torch.cuda.synchronize()
    assert torch.equal(bits(out[:, :D]), bits(x[idx.long(), :D]))
    assert torch.isnan(out[:, D:].float()).all(), "columns beyond D must be untouched"
    if S == 30000:
        assert S * (D // 8) > 16 * sms() * 256  # more row vectors than the grid-stride loop's grid


@pytest.mark.parametrize("S,D", [(1, 8), (37, 768), (30000, 264)])
def test_scatter_add_rows(cuda_device, S, D):
    dev = cuda_device
    R = S + 1000
    g = torch.Generator().manual_seed(S * 3 + D)
    src = torch.randn(S, D + 8, generator=g).to(BF).to(dev)
    dx = (torch.randn(R, D + 16, generator=g) * 4).to(BF).to(dev)
    idx = torch.randperm(R, generator=g)[:S].to(torch.int32).to(dev)  # the rows of one call are distinct
    want = dx.cpu()
    il = idx.long().cpu()
    want[il, :D] = (want[il, :D].float() + src[:, :D].float().cpu()).to(BF)  # bf16(float(dx) + float(src)), host rounding
    ops.scatter_add_rows(src, D + 8, idx, S, D, dx, D + 16)
    torch.cuda.synchronize()
    assert torch.equal(bits(dx.cpu()), bits(want))


def test_gather_scatter_zero_rows(cuda_device):
    dev = cuda_device
    x = torch.randn(4, 16, device=dev).to(BF)
    idx = torch.zeros(1, dtype=torch.int32, device=dev)
    out = nan_like((1, 16), BF, dev)
    before = x.clone()
    ops.gather_rows(x, 16, idx, 0, 16, out, 16)
    ops.scatter_add_rows(out, 16, idx, 0, 16, x, 16)
    torch.cuda.synchronize()
    assert torch.isnan(out.float()).all() and torch.equal(bits(x), bits(before))


# ------------------------------------------------------------------------------------------------------ contrastive heads
def _contrastive_inputs(S, N, Dp, shared, seed, dev, aligned_pos=False):
    """proj / y as bf16 rows in buffers with row stride Dp + 12, built around a shared direction with a random sign per row,
    so every cosine sits near +-0.5 (no logit within 1e-4 of 0); idx [N, S] in [0, S), same [N, S] random flags."""
    g = torch.Generator().manual_seed(seed)
    m = torch.randn(Dp, generator=g)
    m = m / m.norm() * math.sqrt(Dp)

    def rows():
        sign = torch.randint(0, 2, (S, 1), generator=g).float() * 2 - 1
        return sign * m + torch.randn(S, Dp, generator=g)

    rs = Dp + 12
    pbuf = torch.zeros(S, rs, dtype=BF)
    pbuf[:, :Dp] = rows().to(BF)
    if shared:
        ybuf = pbuf
    else:
        ybuf = torch.zeros(S, rs, dtype=BF)
        yv = rows()
        if aligned_pos:  # even frames: the positive leans towards the projection (the frame is usually predicted right)
            yv[::2] = pbuf[::2, :Dp].float() * 1.5 + yv[::2] * 0.5
        ybuf[:, :Dp] = yv.to(BF)
    idx = torch.randint(0, S, (N, S), generator=g).to(torch.int32)
    same = (torch.rand(N, S, generator=g) < 0.3).to(torch.uint8)
    pbuf = pbuf.to(dev)
    ybuf = pbuf if shared else ybuf.to(dev)
    return pbuf, ybuf, rs, idx.to(dev), same.to(dev)


def _ref_logits(kind, proj, y, idx, temp):
    """[S, N+1] logits from the oracle (sat: compute_nce with replace_inf=False; w2v: compute_preds), chunked over frames;
    differentiable in proj / y when they require grad.  The oracle takes the cosine in fp32 and returns it as fp64; all
    that follows (loss, autograd) is fp64."""
    S, Dp = proj.shape
    N = idx.shape[0]
    step = max(1, (1 << 24) // max(1, (N + 1) * Dp))
    out = []
    for s0 in range(0, S, step):
        s1 = min(S, s0 + step)
        inst = y[idx[:, s0:s1].long()]  # [N, n, Dp]
        if kind == "sat":
            out.append(O.sat_compute_nce(proj[s0:s1], y[s0:s1], inst, temp, replace_inf=False))
        else:
            out.append(O.w2v_compute_preds(proj[s0:s1], y[s0:s1], inst, temp).transpose(0, 1))
    return torch.cat(out, 0)


def _ref_loss(kind, L, same):
    """sat: mean BCE-with-logits (targets [1, same]); w2v: summed cross entropy with the positive at 0."""
    S = L.shape[0]
    if kind == "sat":
        T = torch.cat([torch.ones(S, 1, dtype=F64, device=L.device), same.t().double()], 1)
        return F.binary_cross_entropy_with_logits(L, T, reduction="sum") / L.numel(), T
    return F.cross_entropy(L, torch.zeros(S, dtype=torch.long, device=L.device), reduction="sum"), None


def _run_fwd(kind, proj, y, rs, idx, same, S, N, Dp, temp, dev):
    gbuf = nan_like((S, N + 1), torch.float32, dev)
    loss = torch.full((1,), 0.5, dtype=F64, device=dev)
    stats = torch.tensor([7, 11], dtype=torch.int32, device=dev)
    if kind == "sat":
        ops.sat_nce_fwd(proj, rs, y, rs, idx if N else None, same if N else None, S, N, Dp, temp, gbuf, loss, stats)
    else:
        ops.w2v_nce_fwd(proj, rs, y, rs, idx if N else None, S, N, Dp, temp, gbuf, loss, stats)
    torch.cuda.synchronize()
    return gbuf, loss.item() - 0.5, (stats[0].item() - 7, stats[1].item() - 11)


def _check_fwd(kind, L, same, gbuf, loss, stats, Dp, temp):
    S, K = L.shape
    N = K - 1
    Lr = L.clone().requires_grad_(True)
    lref, T = _ref_loss(kind, Lr, same)
    lref.backward()
    gref = Lr.grad
    finite = torch.isfinite(L)
    Lf = torch.where(finite, L, torch.zeros_like(L))
    # fp32 logit: dot and norms over Dp / 32 products per lane + shuffles (sum |p_i y_i| <= |p||y|), the quotient, / temp.
    # The oracle's cosine is itself evaluated in fp32 (torch.cosine_similarity on .float() inputs): the same bound again.
    ez = 2 * (3 * (Dp / 32 + 8) * EPS32 / temp + 4 * EPS32 * Lf.abs())
    if kind == "sat":
        scale = 1.0 / (S * K)
        bce = F.binary_cross_entropy_with_logits(L, T, reduction="none")
        # per logit |d BCE / dz| <= 1, log1pf / __expf, and the fp32 sum of a frame's N+1 terms
        tol_loss = scale * (ez + 2.0 ** -21 + (N + 8) * EPS32 * (bce + Lf.abs())).sum().item()
        # sigmoid' <= 1/4, plus __expf, the quotient and the fp32 1 / (S (N+1))
        tol_g = scale * (ez / 4 + 8 * EPS32)
        assert stats[1] == S + int(same.sum()), stats
        amb = L.abs() < 1e-4
        ref_acc = int(((L >= 0) == (T > 0.5)).sum())
    else:
        p = torch.softmax(L, 1)
        ezr = ez.max(1, keepdim=True).values
        # per frame lse - z_0: two logit errors, __logf (2^-21.4), __expf and the fp32 sum over N+1 terms
        tol_loss = (2 * ezr.squeeze(1) + 2.0 ** -20 + (N / 32 + 8) * EPS32 * (1 + Lf.abs().max(1).values)).sum().item()
        tol_g = p * (2 * ezr + (N / 32 + 16) * EPS32) + 2 * EPS32
        assert stats[1] == S, stats
        z0 = L[:, :1]
        others = L[:, 1:]
        near = lambda v: ((z0 - v).abs() < 1e-4) & torch.isfinite(v)  # noqa: E731
        amb = near(others.max(1, keepdim=True).values) | near(others.min(1, keepdim=True).values) if N else torch.zeros(S, 1, dtype=torch.bool, device=L.device)
        ref_acc = int(((L.argmax(1) == 0) & ~(L.argmin(1) == 0)).sum())
        assert (gbuf[~finite] == 0).all(), "a masked negative must get g = 0"
    assert abs(loss - lref.item()) <= tol_loss, (kind, loss, lref.item(), tol_loss)
    assert_close(gbuf, gref, tol_g, f"{kind} g")
    n_amb = int(amb.sum())
    assert n_amb <= 1 + amb.numel() // 10000, f"{n_amb} ambiguous logits: the inputs should keep them near zero"
    assert abs(stats[0] - ref_acc) <= n_amb, (kind, stats[0], ref_acc, n_amb)
    return gref


FWD_SIZES = [(64, 0, 1), (64, 1, 5), (260, 8, 5), (260, 100, 4000), (768, 100, 4000), (1024, 1, 4000), (1024, 100, 5),
             (768, 8, 1), (64, 100, 4000), (1024, 0, 4000)]


@pytest.mark.parametrize("shared", [False, True], ids=["proj_y", "proj_is_y"])
@pytest.mark.parametrize("Dp,N,S", FWD_SIZES)
@pytest.mark.parametrize("kind", ["sat", "w2v"])
def test_contrastive_fwd(cuda_device, kind, Dp, N, S, shared):
    dev = cuda_device
    temp = f32(0.1)
    pbuf, ybuf, rs, idx, same = _contrastive_inputs(S, N, Dp, shared, Dp * 7 + N * 3 + S, dev, aligned_pos=(kind == "w2v"))
    gbuf, loss, stats = _run_fwd(kind, pbuf, ybuf, rs, idx, same, S, N, Dp, temp, dev)
    L = _ref_logits(kind, pbuf[:, :Dp].double(), ybuf[:, :Dp].double(), idx, temp)
    _check_fwd(kind, L, same, gbuf, loss, stats, Dp, temp)
    if kind == "w2v" and N == 0:
        assert stats[0] == 0, "a frame without negatives is never counted correct"


def test_w2v_negatives_equal_to_positive(cuda_device):
    """wav2vec 2.0 masks a negative that equals the positive in every element with -inf (duplicated quantized targets)."""
    dev = cuda_device
    S, N, Dp, temp = 64, 8, 256, f32(0.1)
    pbuf, ybuf, rs, idx, same = _contrastive_inputs(S, N, Dp, False, 5, dev, aligned_pos=True)
    ybuf[10] = ybuf[0]           # row 10 duplicates frame 0's positive
    ybuf[11] = ybuf[1]
    ybuf[11, 17] += 4.0          # row 11 differs from frame 1's positive in one element only
    idx[:, 0] = torch.tensor([0, 10] * (N // 2), dtype=torch.int32, device=dev)  # every negative of frame 0 equals its positive
    idx[0, 1] = 11
    idx[1, 1] = 10
    gbuf, loss, stats = _run_fwd("w2v", pbuf, ybuf, rs, idx, same, S, N, Dp, temp, dev)
    L = _ref_logits("w2v", pbuf[:, :Dp].double(), ybuf[:, :Dp].double(), idx, temp)
    assert torch.isinf(L[0, 1:]).all() and torch.isfinite(L[1, 1:2]).all()
    _check_fwd("w2v", L, same, gbuf, loss, stats, Dp, temp)
    assert (gbuf[0] == 0).all(), "frame 0: every negative masked, so the softmax is one-hot on the positive"
    assert gbuf[1, 1].item() > 0, "a negative that differs in one element is not masked"
    # frame 0 alone: loss exactly 0, counted correct
    g1, loss1, stats1 = _run_fwd("w2v", pbuf, ybuf, rs, idx[:, :1].contiguous(), same, 1, N, Dp, temp, dev)
    assert loss1 == 0.0 and stats1 == (1, 1) and (g1 == 0).all()


BWD_CASES = [("sat", False, 260, 8, 300), ("sat", True, 260, 8, 300), ("w2v", False, 260, 8, 300),
             ("sat", False, 768, 100, 2000), ("sat", True, 768, 100, 2000), ("w2v", False, 768, 100, 2000)]


@pytest.mark.parametrize("kind,shared,Dp,N,S", BWD_CASES)
def test_sat_nce_bwd(cuda_device, kind, shared, Dp, N, S):
    dev = cuda_device
    temp, up = f32(0.1), f32(0.37)
    pbuf, ybuf, rs, idx, same = _contrastive_inputs(S, N, Dp, shared, Dp + N + S, dev, aligned_pos=(kind == "w2v"))
    idx[:, 1::7] = idx[:, 0::7][:, :idx[:, 1::7].shape[1]]  # frames that share their whole set of negatives
    gbuf, _, _ = _run_fwd(kind, pbuf, ybuf, rs, idx, same, S, N, Dp, temp, dev)
    pr = pbuf[:, :Dp].double().requires_grad_(True)
    yr = pr if shared else ybuf[:, :Dp].double().requires_grad_(True)
    L = _ref_logits(kind, pr, yr, idx, temp)
    loss, _ = _ref_loss(kind, L, same)
    (up * loss).backward()
    # non-zero accumulators on the scale of the gradients they receive
    g = torch.Generator().manual_seed(S)
    init_p = (torch.randn(S, Dp, generator=g).to(dev) * pr.grad.abs().mean()).float()
    init_y = init_p if shared else (torch.randn(S, Dp, generator=g).to(dev) * yr.grad.abs().mean()).float()
    dacc_p = init_p.clone()
    dacc_y = dacc_p if shared else init_y.clone()
    upstream = torch.full((1,), up, device=dev)
    ops.sat_nce_bwd(pbuf, rs, ybuf, rs, idx, S, N, Dp, temp, gbuf, upstream, dacc_p, dacc_y)
    torch.cuda.synchronize()
    # vector reductions per row: one from its own frame's d proj, one per (frame, logit) that reads it as y
    n_y = 1 + torch.bincount(idx.long().flatten(), minlength=S).double()[:, None]
    # The forward's g also has an absolute error floor (fp32 p - 1 for wav2vec, the rounded 1 / (S (N+1)) for SAT): up to
    # 8 EPS32 of its scale per logit, times |d cos / d x_i| <= 2 / |x| and up / temp, over the logits that reach the row.
    g_floor = 8 * EPS32 * (1.0 if kind == "w2v" else 1.0 / (S * (N + 1))) * 2 * up / temp
    floor_p = (N + 1) * g_floor / pr.detach().norm(dim=1, keepdim=True)
    floor_y = n_y * g_floor / yr.detach().norm(dim=1, keepdim=True)
    refs = [("d proj and d y (one buffer)", dacc_p, init_p, pr.grad, n_y + 1, floor_p + floor_y)] if shared else \
        [("d proj", dacc_p, init_p, pr.grad, 1.0, floor_p), ("d y", dacc_y, init_y, yr.grad, n_y, floor_y)]
    for name, got, init, ref, n_red, floor in refs:
        want = init.double() + ref
        # per logit the forward's g carries ~1e-5 of its scale (its own bound), summed over a row's N+1 logits, plus fp32
        # dot products: 2e-4 of the row's largest gradient; and one fp32 rounding of the running sum per reduction
        rowmax = ref.abs().max(1, keepdim=True).values
        tol = 2e-4 * rowmax + floor + (n_red + 1) * EPS32 * (init.double().abs() + rowmax * n_red)
        assert_close(got, want, tol, f"{kind} {name}")


@pytest.mark.parametrize("rows,N", [(3, 4), (7, 1020), (20000, 260)])
def test_f32_to_bf16_rows(cuda_device, rows, N):
    dev = cuda_device
    g = torch.Generator().manual_seed(rows + N)
    src_rs, dst_rs = N + 8, N + 4
    x = torch.randn(rows, src_rs, generator=g) * torch.exp2(torch.randint(-140, 126, (rows, src_rs), generator=g).float())
    xb = x.numpy().view(np.uint32)
    sel = torch.randint(0, 6, (rows, src_rs), generator=g).numpy()
    hi = torch.randint(0, 1 << 16, (rows, src_rs), generator=g).numpy().astype(np.uint32) << np.uint32(16)  # any bf16, even or odd
    xb = np.where(sel == 0, hi | np.uint32(0x8000), xb)   # exactly halfway: round to nearest even
    xb = np.where(sel == 1, hi | np.uint32(0x8001), xb)   # just above halfway
    xb = np.where(sel == 2, hi | np.uint32(0x7FFF), xb)   # just below halfway
    x = torch.from_numpy(xb.astype(np.uint32).view(np.float32).copy())
    x[0, :4] = torch.tensor([3.4028235e38, -1e-45, 0.0, -0.0])  # largest finite (rounds to inf), smallest subnormal, zeros
    x = torch.where(torch.isfinite(x), x, torch.zeros_like(x))
    src = x.to(dev)
    dst = nan_like((rows, dst_rs), BF, dev)
    ops.f32_to_bf16_rows(src, src_rs, dst, dst_rs, rows, N)
    torch.cuda.synchronize()
    assert torch.equal(bits(dst[:, :N].cpu()), bits(x[:, :N].to(BF)))  # torch's host conversion: round to nearest even
    assert torch.isnan(dst[:, N:].float()).all(), "columns beyond N must be untouched"
    if rows == 20000:
        assert rows * N // 4 > 16 * sms() * 256


# --------------------------------------------------------------------------------------------------------- Gumbel quantizer
def _vq_inputs(S, G, V, dv, seed, dev, coarse=True):
    g = torch.Generator().manual_seed(seed)
    GV = G * V
    if coarse:  # a coarse bf16 grid: exact ties for the row maximum are common
        lg = torch.randint(-6, 7, (S, GV + 8), generator=g).float() * 0.5
    else:
        lg = torch.randn(S, GV + 8, generator=g) * 2
    logits = lg.to(BF).to(dev)
    vars_ = torch.randn(GV, dv, generator=g).to(dev)
    return logits, vars_


def _run_vq_hard(logits, vars_, S, G, V, dv, gumbel, key, dev):
    GV = G * V
    codes = torch.full((S * G,), -7, dtype=torch.int32, device=dev)
    q = nan_like((S, G * dv + 8), BF, dev)
    counts = torch.full((GV,), 2.0, device=dev)
    probs = torch.full((GV,), 0.5, device=dev)
    ops.vq_hard(logits, GV + 8, vars_, S, G, V, dv, codes, q, G * dv + 8, counts, probs, gumbel=gumbel, key=key)
    torch.cuda.synchronize()
    return codes.view(S, G), q, counts, probs


def _check_vq_stats(lg, counts, probs, S, G, V):
    """counts: noise-free first-index arg-max counts, exact; probs: summed softmax with fp32 atomics."""
    carg = first_argmax(lg)
    want_counts = 2.0 + F.one_hot(carg, V).double().sum(0).view(-1)
    assert torch.equal(counts.double(), want_counts), "counts"
    want_probs = 0.5 + torch.softmax(lg, -1).sum(0).view(-1)
    # fp32 sums of up to S terms (block shared memory, then global atomics) and __expf / the reciprocal sum per term
    assert_close(probs, want_probs, (S + 16) * EPS32 * want_probs + 2.0 ** -20 * want_probs, "probs")


def _vq_S(G, factor):
    """Enough frames that every warp of the capped grid handles `factor` or more (frame, group) items."""
    return -(-factor * 8 * 2 * sms() // G) + 5


@pytest.mark.parametrize("dv", [128, 40])
@pytest.mark.parametrize("G,V", [(2, 320), (3, 37), (1, 8), (4, 3000)])
def test_vq_hard_eval(cuda_device, G, V, dv):
    dev = cuda_device
    S = _vq_S(G, 3)
    logits, vars_ = _vq_inputs(S, G, V, dv, G * V + dv, dev)
    codes, q, counts, probs = _run_vq_hard(logits, vars_, S, G, V, dv, False, (0, 0), dev)
    lg = logits[:, :G * V].double().view(S, G, V)
    ref = first_argmax(lg)
    assert (lg == lg.max(-1, keepdim=True).values).sum(-1).gt(1).float().mean() > 0.2, "the inputs should have many ties"
    assert torch.equal(codes.long(), ref), "codes: first-index arg-max"
    rowsel = (torch.arange(G, device=dev) * V)[None, :] + ref
    want_q = vars_[rowsel.view(-1)].cpu().to(BF).view(S, G * dv)
    assert torch.equal(bits(q[:, :G * dv].contiguous().cpu()), bits(want_q)), "q = bf16(vars[g V + code])"
    assert torch.isnan(q[:, G * dv:].float()).all()
    _check_vq_stats(lg, counts, probs, S, G, V)


def _noise(seed, S, G, V, dev):
    return O.gumbel_noise(seed, SITE_GUMBEL, S * G * V).to(dev).double().view(S, G, V)


@pytest.mark.parametrize("G,V", [(2, 320), (3, 37)])
def test_vq_hard_training(cuda_device, G, V):
    dev = cuda_device
    S, dv, seed = _vq_S(G, 3), 128, 5
    logits, vars_ = _vq_inputs(S, G, V, dv, 77 + V, dev, coarse=False)
    key = DR.site_key(seed, SITE_GUMBEL)
    codes, q, counts, probs = _run_vq_hard(logits, vars_, S, G, V, dv, True, key, dev)
    lg = logits[:, :G * V].double().view(S, G, V)
    y = lg + _noise(seed, S, G, V, dev)
    ref = y.argmax(-1)
    top2 = y.topk(2, -1).values
    amb = (top2[..., 0] - top2[..., 1]) < 1e-3  # the fp32 noise cannot decide these: excluded
    assert int(amb.sum()) <= 0.005 * amb.numel(), int(amb.sum())
    ok = ~amb
    assert torch.equal(codes.long()[ok], ref[ok]), f"{int((codes.long() != ref)[ok].sum())} codes differ"
    rowsel = (torch.arange(G, device=dev) * V)[None, :] + codes.long()
    want_q = vars_[rowsel.view(-1)].cpu().to(BF).view(S, G, dv)
    assert torch.equal(bits(q[:, :G * dv].contiguous().cpu().view(S, G, dv)), bits(want_q))
    _check_vq_stats(lg, counts, probs, S, G, V)  # the logged statistics ignore the noise


def _logits_bwd_reference(lg, c, h, noise, tau):
    """fp64 autograd of sum(c . mean_s softmax(logits)) + sum(h . softmax((logits + noise) / tau)), and the error scale of each
    element: softmax x (|weight| + the softmax-weighted sum of |weight|), the sizes of the terms the kernel adds and subtracts."""
    S, G, V = lg.shape
    lr = lg.clone().requires_grad_(True)
    loss = lr.sum() * 0.0
    mag = torch.zeros_like(lg)
    if c is not None:
        cc = c.double().view(G, V)
        p = torch.softmax(lr, -1)
        loss = loss + (cc * p.mean(0)).sum()
        p = p.detach()
        mag += p * (cc.abs() + (cc.abs() * p).sum(-1, keepdim=True)) / S
    if h is not None:
        hh = h.double().view(S, G, V)
        ys = torch.softmax((lr + noise) / tau, -1)
        loss = loss + (hh * ys).sum()
        ys = ys.detach()
        mag += ys * (hh.abs() + (hh.abs() * ys).sum(-1, keepdim=True)) / tau
    loss.backward()
    return lr.grad, mag


def _run_logits_bwd(logits, S, G, V, c, h, tau, key, dev):
    GV = G * V
    out = nan_like((S, GV + 16), BF, dev)
    ops.vq_logits_bwd(logits, GV + 8, S, G, V, c, h, GV + 8 if h is not None else 0, tau, key, out, GV + 16)
    torch.cuda.synchronize()
    assert torch.isnan(out[:, GV:].float()).all(), "columns beyond G V must be untouched"
    return out[:, :GV].view(S, G, V)


def _check_logits_bwd(got, ref, mag, what):
    # bf16 output: one ulp; fp32 softmax statistics (__expf, sums over V / 32 terms per lane, the reciprocal), the
    # (x + noise) / tau argument rounded in fp32 (|arg| up to ~40: 2.4e-6 relative in the softmax) and the fp32 noise itself:
    # 2^-16 of the terms the gradient is the difference of
    assert_close(got, ref, ulp_bf16(ref) + 2.0 ** -16 * mag, what)


@pytest.mark.parametrize("tau", [2.0, 0.5])
@pytest.mark.parametrize("mode", ["c", "h", "both", "neither"])
def test_vq_logits_bwd(cuda_device, mode, tau):
    dev = cuda_device
    G, V, seed = 2, 320, 9
    S = -(-5 * 8 * 8 * sms() // (2 * G))  # 2.5 (frame, group) items per warp of the capped grid
    logits, _ = _vq_inputs(S, G, V, 8, 123, dev, coarse=False)
    g = torch.Generator().manual_seed(4)
    c = torch.randn(G * V, generator=g).to(dev) if mode in ("c", "both") else None
    hbuf = (torch.randn(S, G * V + 8, generator=g) * 0.1).to(BF).to(dev) if mode in ("h", "both") else None
    key = DR.site_key(seed, SITE_GUMBEL)
    got = _run_logits_bwd(logits, S, G, V, c, hbuf, tau, key, dev)
    if mode == "neither":
        assert (got.float() == 0).all()
        return
    lg = logits[:, :G * V].double().view(S, G, V)
    h = hbuf[:, :G * V] if hbuf is not None else None
    ref, mag = _logits_bwd_reference(lg, c, h, _noise(seed, S, G, V, dev), f32(tau))
    _check_logits_bwd(got, ref, mag, f"d logits ({mode}, tau {tau})")


def _extreme_seed(n):
    """A seed whose Gumbel counters 0..n-1 include u >= 1 - 2^-22 (float32 u, as the kernel forms it), and those counters."""
    for seed in range(256):
        k0, k1 = DR.site_key(seed, SITE_GUMBEL)
        b = O._drop_bits(np.uint64(k0), np.uint64(k1), np.arange(n, dtype=np.uint64))
        u = (b.astype(np.float32) + np.float32(0.5)) * np.float32(2.3283064365386963e-10)
        hit = np.nonzero(u >= np.float32(1.0 - 2.0 ** -22))[0]
        if hit.size:
            return seed, hit
    raise AssertionError("no seed in range")


def test_gumbel_extremes(cuda_device):
    """Counters whose uniform sits within 2^-22 of 1: -log u is then about as small as __logf's absolute error, so an
    approximate logarithm can turn the noise there into +inf or NaN, or misplace it.  The reference noise is about 15-17, so
    those codes are almost surely picked; the straight-through gradient must stay finite and match the reference."""
    dev = cuda_device
    S, G, V, dv, tau = 4096, 2, 320, 128, 2.0
    seed, hit = _extreme_seed(S * G * V)
    logits, vars_ = _vq_inputs(S, G, V, dv, 31, dev, coarse=False)
    key = DR.site_key(seed, SITE_GUMBEL)
    codes, _, _, _ = _run_vq_hard(logits, vars_, S, G, V, dv, True, key, dev)
    lg = logits[:, :G * V].double().view(S, G, V)
    noise = _noise(seed, S, G, V, dev)
    ref = (lg + noise).argmax(-1).view(-1)
    w = torch.from_numpy(hit // V).to(dev)
    assert (noise.view(-1)[torch.from_numpy(hit).to(dev)] > 14).all()
    assert torch.equal(codes.view(-1)[w].long(), ref[w]), (hit, codes.view(-1)[w], ref[w])
    g = torch.Generator().manual_seed(6)
    c = torch.randn(G * V, generator=g).to(dev)
    hbuf = (torch.randn(S, G * V + 8, generator=g) * 0.1).to(BF).to(dev)
    got = _run_logits_bwd(logits, S, G, V, c, hbuf, tau, key, dev)
    assert torch.isfinite(got.float()).all(), "d logits must be finite everywhere"
    ref_d, mag = _logits_bwd_reference(lg, c, hbuf[:, :G * V], noise, tau)
    _check_logits_bwd(got, ref_d, mag, "d logits at the noise extremes")


@pytest.mark.parametrize("S,G,V,dv", [(3000, 3, 37, 40), (4000, 2, 320, 128)])
def test_vq_dvars(cuda_device, S, G, V, dv):
    dev = cuda_device
    g = torch.Generator().manual_seed(S + V)
    codes = torch.randint(0, V, (S, G), generator=g)
    codes[:, 1] = 5  # one group whose frames all share one code: S atomics on the same row
    dq = torch.randn(S, G * dv + 8, generator=g).to(BF).to(dev)
    init = torch.randn(G * V, dv, generator=g).to(dev)
    dvars = init.clone()
    codes = codes.to(torch.int32).to(dev)
    ops.vq_dvars(dq, G * dv + 8, codes, S, G, V, dv, dvars)
    torch.cuda.synchronize()
    rowsel = ((torch.arange(G, device=dev) * V)[None, :] + codes.long()).view(-1)
    src = dq[:, :G * dv].double().reshape(S * G, dv)
    want = init.double().index_add_(0, rowsel, src)
    mag = init.double().abs().index_add_(0, rowsel, src.abs())
    n = torch.zeros(G * V, dtype=F64, device=dev).index_add_(0, rowsel, torch.ones(S * G, dtype=F64, device=dev))
    # fp32 atomics in any order: at most (terms + 1) roundings of the running sum
    assert_close(dvars, want, (n[:, None] + 2) * EPS32 * mag, "dvars")


# -------------------------------------------------------------------------------------------------------- feature penalty
@pytest.mark.parametrize("B,Tp,T,C", [(3, 50, 37, 264), (4, 1600, 1499, 768)])
def test_sumsq_rows(cuda_device, B, Tp, T, C):
    dev = cuda_device
    g = torch.Generator().manual_seed(T)
    x = torch.randn(B, Tp, C + 8, generator=g).to(BF)
    x[:, T:] = 1e4  # rows past T must not be read
    x = x.to(dev)
    out = torch.full((1,), 12.5, dtype=F64, device=dev)
    ops.sumsq_rows(x, Tp * (C + 8), C + 8, T, B, C, out)
    torch.cuda.synchronize()
    ss = (x[:, :T, :C].double() ** 2).sum().item()
    vecs = B * T * C // 8
    iters = -(-vecs // (min(-(-vecs // 256), 8 * sms()) * 256))
    # each thread sums 8 products per vector in fp32, then fp64 across threads
    tol = (8 * iters + 16) * EPS32 * ss
    assert abs(out.item() - 12.5 - ss) <= tol, (out.item() - 12.5, ss, tol)


@pytest.mark.parametrize("pen", [None, 0.8])
@pytest.mark.parametrize("scale", [0.1, 1.0])
def test_grad_multiply(cuda_device, scale, pen):
    dev = cuda_device
    B, Tp, T, C, pen_mul = 3, 40, 33, 264, 0.5
    g = torch.Generator().manual_seed(int(scale * 10) + (pen is not None))
    gst = torch.randn(B, Tp, C + 8, generator=g).to(BF).to(dev)
    xst = torch.randn(B, Tp + 3, C + 16, generator=g).to(BF).to(dev)
    before = gst.clone()
    pen_t = torch.full((1,), pen, device=dev) if pen is not None else None
    ops.grad_multiply(gst, Tp * (C + 8), C + 8, xst, (Tp + 3) * (C + 16), C + 16, T, B, C, scale, pen_t, pen_mul)
    torch.cuda.synchronize()
    a, b = before[:, :T, :C].double(), xst[:, :T, :C].double()
    coef = f32(pen) * f32(pen_mul) if pen is not None else 0.0
    ref = f32(scale) * (a + coef * b)
    # one bf16 ulp on the bf16 output plus fp32 rounding of the coefficient, the fma and the scaling
    assert_close(gst[:, :T, :C], ref, ulp_bf16(ref) + 4 * EPS32 * f32(scale) * (a.abs() + abs(coef) * b.abs()), "grad_multiply")
    assert torch.equal(bits(gst[:, T:]), bits(before[:, T:])) and torch.equal(bits(gst[:, :, C:]), bits(before[:, :, C:]))
