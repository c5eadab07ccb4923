"""Op-level tests of the encoder layer's attention: the gated relative-position attention kernels (csrc/attn_fwd.cu,
attn_bwd2.cu) through every entry point, at the shipped shapes and at tile edges, in four input regimes.

Every reference is computed in float64 on the GPU from the same bf16 / fp32 tensors the kernel reads; reference gradients come
from torch.autograd on a plain float64 restatement.  Bounds are per element and built from a magnitude reference (the same
computation on absolute values), never from max|ref|, so an error confined to a few rows, columns or diagonals is the whole
signal.  Outputs are pre-filled with NaN and `+=` outputs start at BASE.  Each tolerance is written next to its reason; the
worst err / bound of every check family is printed per case and summarised at the end of the module (run with -s).

Attention, in the natural-log domain (the kernels work in log2 and fold log2(e) into the scale):
  s_ij = scale q_i.k_j + gate_i tab[j - i + T - 1]   (-inf at padded keys),  P = softmax_j(s),  O = (P o keep / (1-p)) V
  dS = P o (dP - Delta),  dP = keep / (1-p) o dO V^T,  Delta_i = sum_d dO_id O_id
  dQ = scale dS K,  dK = scale dS^T Q,  dV = (P o keep / (1-p))^T dO,  d gate_i = sum_j dS_ij tab[j-i],
  d tab[d] = sum_i gate_i dS_{i,i+d}.
Where the kernels round (attn_fwd.cu, attn_bwd2.cu): P is rounded to bf16 as the A operand of P V (the row sum l is the fp32
sum of the unrounded exponentials) and of dV += P^T dO; dS is staged in bf16 for dK = dS^T Q and dQ = dS K; gate * dS is
staged in bf16 for the d tab diagonal sums; d gate is summed from the fp32 dS.  Delta is computed from the STORED bf16 O, which
differs from the exact O by the forward's own rounding: that difference enters dS as P_ij (Delta_stored - Delta_exact)_i and is
carried as its own term (E below), computed from the kernel's stored O."""
import math

import pytest
import torch

from test_attn_hd80_gpu import unpack_mask
from test_conv_stem_gpu import BASE, assert_close, bf16_bound, nan_like
from unispeech_b200 import ops
from unispeech_b200.engine import relative_positions_bucket_lut

pytestmark = pytest.mark.gpu

BF = torch.bfloat16
F32 = torch.float32
F64 = torch.float64
EPS32 = 2.0 ** -24
LOG2E = 1.0 / math.log(2.0)
# A bf16-rounded operand (P, dS, gate * dS): its unit roundoff 2^-8, plus 2^-12 for the second-order terms (fp32 errors of the
# value before it is rounded, and of the sums it enters), which stay below 2^-12 at T <= 4096 (derived at each use)
RND = 2.0 ** -8 + 2.0 ** -12


# ------------------------------------------------------------------------------------------------------------- reporting
_WORST = {}  # check family -> (worst err / bound, case)


def check(rep, fam, where, got, ref, tol):
    """assert_close, and the worst err / bound over the elements with a non-zero bound into rep[fam]."""
    g, r = got.double(), ref.double()
    t = torch.as_tensor(tol, dtype=F64, device=r.device).expand_as(r)
    pos = t > 0
    ratio = ((g - r).abs()[pos] / t[pos]).max().item() if bool(pos.any()) else 0.0
    rep[fam] = max(rep.get(fam, 0.0), ratio)
    assert_close(got, ref, tol, f"{where}: {fam}")


def report(prefix, case, rep):
    print(f"\n{prefix} {case}: " + ", ".join(f"{k} {v:.3f}" for k, v in sorted(rep.items())))
    for k, v in rep.items():
        if v >= _WORST.get(f"{prefix} {k}", (-1.0, ""))[0]:
            _WORST[f"{prefix} {k}"] = (v, case)


@pytest.fixture(scope="module", autouse=True)
def _summary():
    yield
    if _WORST:
        print("\nworst err / bound per check family:")
        for k in sorted(_WORST):
            print(f"  {k:<28} {_WORST[k][0]:.3f}   ({_WORST[k][1]})")


# ------------------------------------------------------------------------------------------------- attention reference
_TOEPLITZ = {}


def toeplitz_index(T, dev):
    """[T, T] index j - i + T - 1 of the bias table (the bias of query i and key j)."""
    if T not in _TOEPLITZ:
        i = torch.arange(T, device=dev)
        _TOEPLITZ[T] = (i[None, :] - i[:, None] + T - 1).contiguous()
    return _TOEPLITZ[T]


def attn_ref(q, k, v, scale, g, tab, kpad, dO, keep=None, p=0.0):
    """One utterance, all heads, float64: q / k / v [H, T, hd], g [H, T], tab [H, 2T-1] (or None), kpad bool [T] (or None),
    dO [H, T, hd], keep bool [H, T, T] (or None).  Values, autograd gradients and the magnitude references of the bounds."""
    H, T, hd = q.shape
    leaves = [t.detach().clone().requires_grad_(True) for t in (q, k, v)]
    if tab is not None:
        leaves += [g.detach().clone().requires_grad_(True), tab.detach().clone().requires_grad_(True)]
    s = scale * leaves[0] @ leaves[1].transpose(1, 2)
    idx = toeplitz_index(T, q.device)
    if tab is not None:
        s = s + leaves[3][:, :, None] * leaves[4][:, idx]
    if kpad is not None:
        s = s.masked_fill(kpad[None, None, :], float("-inf"))
    lse = torch.logsumexp(s, -1)
    P = torch.exp(s - lse[..., None])
    Pd = P * keep / (1.0 - p) if keep is not None else P
    O = Pd @ leaves[2]
    grads = torch.autograd.grad(O, leaves, dO)
    with torch.no_grad():
        P, Pd, O, s = P.detach(), Pd.detach(), O.detach(), s.detach()
        r = dict(O=O, lse2=lse.detach() * LOG2E, P=P, Pd=Pd, dq=grads[0], dk=grads[1], dv=grads[2])
        if tab is not None:
            r["dgate"], r["dtab"] = grads[3], grads[4]
            r["bias_abs"] = tab.abs()[:, idx]
        r["Mout"] = Pd @ v.abs()                          # sum_j P_ij |v_j|
        kd = keep / (1.0 - p) if keep is not None else 1.0
        dP = (dO @ v.transpose(1, 2)) * kd
        A = (dO.abs() @ v.abs().transpose(1, 2)) * kd    # magnitude of dP (its fp32 accumulation error)
        M = P * (dP.abs() + (P * dP.abs()).sum(-1, keepdim=True))
        Fm = P * (A + (P * A).sum(-1, keepdim=True))
        r["M"], r["F"] = M, Fm
        r["Delta"] = (dO * O).sum(-1)                    # exact: sum_j P_ij dP_ij
        # score range of each row for the lse bound: max_j |scale q.k| + |gate tab| over valid keys, plus |lse|
        sm = scale * (q.abs() @ k.abs().transpose(1, 2))
        if tab is not None:
            sm = sm + g.abs()[:, :, None] * r["bias_abs"]
        if kpad is not None:
            sm = sm.masked_fill(kpad[None, None, :], 0.0)
        r["R2"] = sm.amax(-1) * LOG2E + r["lse2"].abs()
    return r


def check_attn_utt(rep, tag, r, got, q, k, g, tab, dO, kpad, valid_q, scale, T):
    """Kernel outputs of one utterance (`got`: out / lse / delta / dq / dk / dv [/ dgate], heads first) against attn_ref.
    Returns the d tab reference of the utterance and its bound before the diagonal sums ([H, T, T] each), or None."""
    # out: bf16(P) has relative error below 2^-8 (bf16 unit roundoff; the row sum is of the unrounded fp32 exponentials).
    # The second-order terms stay below 2^-12: P's relative error before the rounding (lse and the exponent argument, 2^-14 at
    # most), ex2.approx (2^-22), the fp32 accumulation of at most T / 16 k16 steps (2^-16 at T = 4096) and the 1 / l scaling.
    # delta = RND sum_j P_ij |v_j|.  A one-ulp fault on P (truncation instead of rounding) reaches 2^-7 and is not covered.
    vq = valid_q[None, :, None]
    ref_o = torch.where(vq, r["O"], 0.0)
    check(rep, "out", tag, torch.where(vq, got["out"].double(), 0.0), ref_o, bf16_bound(ref_o, RND * r["Mout"]))
    # lse (log2): m + log2(l) with l the fp32 sum of T/4 exponentials per thread then 4 (relative error <= (T/4 + 8) EPS32,
    # plus 2^-21 for ex2.approx); the exponent arguments and the final add round at the score range R (2^-20 R: 16 ulps)
    tl = LOG2E * ((T / 4 + 8) * EPS32 + 2.0 ** -21) + 2.0 ** -20 * r["R2"]
    vr = valid_q[None, :].expand_as(r["lse2"])
    check(rep, "lse", tag, got["lse"].double()[vr], r["lse2"][vr], tl[vr])
    # delta = rowsum(dO o O_stored): products of two bf16 are exact in fp32, a sum of hd of them is within hd EPS32 <= 2^-17
    # of sum |dO O|
    Ost = got["out"].double()
    d_st = (dO * Ost).sum(-1)
    d_mag = (dO.abs() * Ost.abs()).sum(-1)
    check(rep, "delta", tag, got["delta"], d_st, 2.0 ** -17 * d_mag)
    # The backward reads Delta of the STORED O, not the exact one: dS_ij = P_ij (dP_ij - Delta_stored_i).  Its difference from
    # autograd's dS is P_ij c_i with c = Delta_stored - Delta_exact, a first-order term known exactly here, so the reference
    # gradients are autograd's minus that term's contribution (teacher-forced on the kernel's own O, like every other input).
    Pc = r["P"] * (d_st - r["Delta"])[..., None]
    ref_dq = r["dq"] - scale * Pc @ k
    ref_dk = r["dk"] - scale * Pc.transpose(1, 2) @ q
    # what is left: the bf16 staging of dS (below 2^-8 of |dS| <= M); second order, below 2^-12 M together: P's relative
    # error (2^-14 at most: lse and the exponent argument) and the fp32 sums of dQ / dK (T / 16 k16 steps, <= 2^-16 at
    # T = 4096); the fp32 dP of hd exact products (2^-18 A: 2^-16 F leaves a factor of four); the fp32 Delta (2^-17 d_mag
    # above) times P.  Each of them also passes through the staging: a factor 1 + 2^-8, inside the margins.
    E = r["P"] * (2.0 ** -17 * d_mag)[..., None]
    G = RND * r["M"] + 2.0 ** -16 * r["F"] + E
    check(rep, "dq", tag, got["dq"], ref_dq, bf16_bound(ref_dq, scale * G @ k.abs()))
    check(rep, "dk", tag, got["dk"], ref_dk, bf16_bound(ref_dk, scale * G.transpose(1, 2) @ q.abs()))
    # dV = bf16(P)^T dO: below 2^-8 of P, plus P's own 2^-14 and the fp32 sum (second order, below 2^-12): RND P^T |dO|
    check(rep, "dv", tag, got["dv"], r["dv"], bf16_bound(r["dv"], RND * r["Pd"].transpose(1, 2) @ dO.abs()))
    if kpad is not None:  # header contract: dK and dV of padded keys are exactly zero
        assert (got["dk"][:, kpad] == 0).all() and (got["dv"][:, kpad] == 0).all(), f"{tag}: dK / dV of padded keys"
    if "dgate" not in got:
        return None
    bias = tab[:, toeplitz_index(T, tab.device)]
    # d gate sums the fp32 dS (no bf16 staging) over at most 2 + 3 + 8 + T/128 partial sums (2^-18 at T = 4096); P's relative
    # error is ln 2 times the lse error bounded above (below 2^-13.5 at T = 4096, with the exponent argument's rounding):
    # 2^-13 M covers both
    Gg = 2.0 ** -13 * r["M"] + 2.0 ** -16 * r["F"] + E
    check(rep, "dgate", tag, got["dgate"], r["dgate"] - (Pc * bias).sum(-1), (Gg * r["bias_abs"]).sum(-1))
    # d tab: gate * dS staged in bf16 (2^-8) then fp32 diagonal sums (16 per task, then T / 128 blocks): |gate| G per element
    return g[:, :, None] * (-Pc), g.abs()[:, :, None] * G


def diag_sum(X):
    """[H, T, T] -> [H, 2T - 1]: sums along the diagonals j - i (the adjoint of the Toeplitz gather)."""
    H, T, _ = X.shape
    out = torch.zeros(H, 2 * T - 1, dtype=X.dtype, device=X.device)
    return out.index_add_(1, toeplitz_index(T, X.device).flatten(), X.reshape(H, T * T))


# ------------------------------------------------------------------------------------------------- attention inputs
def grep_gate(x, H, seed, dev):
    """gate [B, H, T] of gru_rel_pos (WavLM/modules.py:523-533) in float64 from x [B, T, H*64] and random grep_linear /
    grep_a (grep_a != 1): gate = ga (gb a - 1) + 2, (ga, gb) = sigmoid of the sums of the first / last 4 outputs."""
    gen = torch.Generator().manual_seed(seed)
    w = (0.15 * torch.randn(8, 64, generator=gen)).double().to(dev)
    b = (0.3 * torch.randn(8, generator=gen)).double().to(dev)
    a = (0.6 + 1.2 * torch.rand(H, generator=gen)).double().to(dev)
    B, T, _ = x.shape
    u = x.double().view(B, T, H, 64) @ w.t() + b
    ga, gb = torch.sigmoid(u[..., :4].sum(-1)), torch.sigmoid(u[..., 4:].sum(-1))
    return (ga * (gb * a - 1.0) + 2.0).permute(0, 2, 1).contiguous().float()


def shipped_tab(T, H, seed, dev):
    """tab as the model builds it (wavlm.py _make_bias_state): bucket LUT and a relative_attention_bias embedding through
    b200s_relpos_table_fwd, which is a plain gather (checked bit for bit)."""
    gen = torch.Generator().manual_seed(seed)
    emb = (1.5 * torch.randn(320, H, generator=gen)).to(dev)
    lut = relative_positions_bucket_lut(T, 320, 800).to(dev)
    tab = torch.full((H, 2 * T - 1), float("nan"), dtype=F32, device=dev)
    ops.relpos_table_fwd(emb, lut, 2 * T - 1, H, tab)
    assert torch.equal(tab, emb[lut.long()].t()), "relpos_table_fwd"
    return tab


LATE = ((3, 72.0), (77, 79.0), (100, 90.0))  # (query row, log2 units above the first key tile's maximum)


def late_key(T):
    """The key of the second tile that carries the late maximum."""
    return 128 + (T - 128) // 2


def attn_inputs(dev, B, T, H, hd, bias, lengths, regime, seed):
    """qkv, gate, tab, pad, dO, scale.  Regimes: diffuse (random), shipped (model-built table, grep gate), peaked (q x 16: rows
    nearly one-hot), late (one key of the second tile lifts rows of LATE 72, 79 and 90 log2 units above the first tile's
    maximum, on both sides of the 2^80 row-sum re-base of attn_fwd.cu)."""
    gen = torch.Generator().manual_seed(seed)
    D = H * hd
    scale = hd ** -0.5
    qkv = torch.randn(B, T, 3 * D, generator=gen)
    if regime == "peaked":
        qkv[..., :D] *= 16.0  # exact in bf16
    gate = tab = None
    if bias:
        if regime == "shipped":
            x = torch.randn(B, T, D, generator=gen).to(BF).to(dev)
            gate = grep_gate(x, H, seed, dev)
            tab = shipped_tab(T, H, seed, dev)
        else:
            gate = (0.2 + 2.0 * torch.rand(B, H, T, generator=gen)).to(dev)
            tab = torch.randn(H, 2 * T - 1, generator=gen).to(dev)
    qkv = qkv.to(BF).to(dev)
    if regime == "late":
        assert T > 128
        jl = late_key(T)
        qh = qkv[..., :D].view(B, T, H, hd)
        kh = qkv[..., D:2 * D].view(B, T, H, hd)
        kh[..., 0] = 0.0          # column 0 of k is zero except at jl, so q[:, 0] moves only the scores of key jl
        kh[:, jl] = 0.0
        kh[:, jl, :, 0] = 8.0
        for i, off in LATE:
            if i >= T:
                continue
            for b in range(B):
                for h in range(H):
                    s = scale * (qh[b, i, h].double() @ kh[b, :128, h].double().t())
                    bias_i = 0.0
                    if bias:
                        s = s + gate[b, h, i].double() * tab[h, torch.arange(128, device=dev) - i + T - 1].double()
                        bias_i = float(gate[b, h, i]) * float(tab[h, jl - i + T - 1])
                    target = float(s.max()) + off / LOG2E  # natural-log units
                    qh[b, i, h, 0] = (target - bias_i) / (scale * 8.0)
                    # q is rounded to bf16 (about 0.2 log2 units at these values): the realised offset stays within 0.5 of
                    # its target, so the 79 row's sum stays below 2^80 (no re-base) and the 90 row's reaches it.  Whether
                    # the kernel re-bases is not observable from outside; its output and lse are checked either way.
                    got_off = (float(qh[b, i, h, 0]) * scale * 8.0 + bias_i - float(s.max())) * LOG2E
                    assert abs(got_off - off) < 0.5, (i, off, got_off)
    pad = None
    if lengths is not None:
        pad = torch.zeros(B, T, dtype=torch.uint8, device=dev)
        for b, n in enumerate(lengths):
            pad[b, n:] = 1
    dO = torch.randn(B, T, D, generator=gen).to(BF).to(dev)
    if pad is not None:
        dO[pad.bool()] = 0  # padded query frames carry no gradient in the model
    return qkv, gate, tab, pad, dO, scale


def run_attn(dev, B, T, H, hd, qkv, gate, tab, pad, dO, scale, p=0.0, key=(0, 0), entry="fused"):
    """Forward (attn_fwd, or attn_fwd_dropout when p > 0) and backward through `entry` ('fused': attn_bwd_fused[_dropout],
    'plain': attn_bwd) with NaN-filled outputs, d tab starting at BASE and a zero dQ workspace."""
    D = H * hd
    k = dict(out=nan_like((B, T, D), BF, dev), lse=nan_like((B, H, T), F32, dev))
    if p > 0:
        k["words"] = torch.full((ops.attn_dropout_mask_words(B, T, H),), -1, dtype=torch.int32, device=dev)
        ops.attn_fwd_dropout(qkv, gate, tab, pad, k["out"], k["lse"], B, T, H, scale, p, key, k["words"], head_dim=hd)
    else:
        ops.attn_fwd(qkv, gate, tab, pad, k["out"], k["lse"], B, T, H, scale, head_dim=hd)
    k["delta"] = nan_like((B, H, T), F32, dev)
    k["dqkv"] = nan_like((B, T, 3 * D), BF, dev)
    k["dgate"] = nan_like((B, H, T), F32, dev) if tab is not None else None  # written, not accumulated: NaN must go
    k["dtab"] = torch.full((H, 2 * T - 1), BASE, dtype=F32, device=dev) if tab is not None else None
    if entry == "plain":
        ops.attn_bwd(qkv, k["out"], dO, gate, tab, pad, k["lse"], k["delta"], k["dqkv"], k["dgate"], k["dtab"], B, T, H, scale,
                     head_dim=hd)
    else:
        k["dq_acc"] = torch.zeros(B, T, D, dtype=F32, device=dev)
        if p > 0:
            ops.attn_bwd_fused_dropout(qkv, k["out"], dO, gate, tab, pad, k["lse"], k["delta"], k["dq_acc"], k["dqkv"],
                                       k["dgate"], k["dtab"], B, T, H, scale, p, k["words"], head_dim=hd)
        else:
            ops.attn_bwd_fused(qkv, k["out"], dO, gate, tab, pad, k["lse"], k["delta"], k["dq_acc"], k["dqkv"], k["dgate"],
                               k["dtab"], B, T, H, scale, head_dim=hd)
    torch.cuda.synchronize()
    return k


def heads(t, b, H, hd, part=0):
    """[B, T, n D] bf16 -> float64 [H, T, hd] of utterance b, column block `part` (q / k / v of qkv: 0 / 1 / 2)."""
    T = t.shape[1]
    D = H * hd
    return t[b, :, part * D:(part + 1) * D].double().view(T, H, hd).transpose(0, 1)


def check_attn(rep, tag, dev, B, T, H, hd, qkv, gate, tab, pad, dO, scale, k, keep=None, p=0.0):
    """Every kernel output of run_attn against the float64 reference, utterance by utterance; the header contracts."""
    D = H * hd
    assert torch.isfinite(k["out"].float()).all(), f"{tag}: out (rows of padded queries are unspecified but finite)"
    if "dq_acc" in k:
        assert (k["dq_acc"] == 0).all(), f"{tag}: the dQ workspace is zero on return"
    dtab_ref = torch.zeros(H, 2 * T - 1, dtype=F64, device=dev) if tab is not None else None
    dtab_tol = torch.zeros_like(dtab_ref) if tab is not None else None
    for b in range(B):
        q, kk, v = heads(qkv, b, H, hd, 0), heads(qkv, b, H, hd, 1), heads(qkv, b, H, hd, 2)
        kpad = pad[b].bool() if pad is not None else None
        valid_q = ~kpad if kpad is not None else torch.ones(T, dtype=torch.bool, device=dev)
        if kpad is not None:
            # fully padded 128-row query blocks: lse = +inf (the backward skips them), zero output rows
            n_valid = int(valid_q.sum())
            dead = torch.zeros(T, dtype=torch.bool, device=dev)
            for q0 in range(0, T, 128):
                if not valid_q[q0:q0 + 128].any():
                    dead[q0:q0 + 128] = True
            if dead.any():
                assert torch.isinf(k["lse"][b][:, dead]).all() and (k["lse"][b][:, dead] > 0).all(), f"{tag}: lse of padded blocks"
                assert (k["out"][b, dead] == 0).all(), f"{tag}: out of padded blocks"
            assert n_valid >= 1
        g = gate[b].double() if gate is not None else None
        dOb = heads(dO, b, H, hd, 0)
        r = attn_ref(q, kk, v, scale, g, tab.double() if tab is not None else None, kpad, dOb,
                     keep[b].double() if keep is not None else None, p)
        got = dict(out=heads(k["out"], b, H, hd, 0), lse=k["lse"][b], delta=k["delta"][b], dq=heads(k["dqkv"], b, H, hd, 0),
                   dk=heads(k["dqkv"], b, H, hd, 1), dv=heads(k["dqkv"], b, H, hd, 2))
        if tab is not None:
            got["dgate"] = k["dgate"][b]
        tb = tab.double() if tab is not None else None
        res = check_attn_utt(rep, f"{tag}[{b}]", r, got, q, kk, g, tb, dOb, kpad, valid_q, scale, T)
        if tab is not None:
            dtab_ref += r["dtab"] + diag_sum(res[0])
            dtab_tol += diag_sum(res[1])
        del r
    if tab is not None:
        check(rep, "dtab", tag, k["dtab"].double() - BASE, dtab_ref, dtab_tol + 2 * EPS32 * BASE)


def attn_case(rep, tag, dev, B, T, H, hd, bias, lengths, regime, p=0.0, entries=("fused", "plain")):
    seed = (B * 1009 + T * 17 + H + hd + (len(lengths) if lengths else 0)) * 31 + len(regime)
    qkv, gate, tab, pad, dO, scale = attn_inputs(dev, B, T, H, hd, bias, lengths, regime, seed)
    if p > 0:
        key = (0x9E3779B9 ^ T, 0x85EBCA6B ^ B)
        k = run_attn(dev, B, T, H, hd, qkv, gate, tab, pad, dO, scale, p, key)
        # keep bits from the kernel's own mask words (compared bit for bit with the hash in test_attn_hd80_gpu /
        # test_dropout_gpu): teacher-forced here
        keep = unpack_mask(k["words"], B, T, H).to(dev)
        check_attn(rep, f"{tag} dropout", dev, B, T, H, hd, qkv, gate, tab, pad, dO, scale, k, keep, p)
        return
    for entry in entries:
        k = run_attn(dev, B, T, H, hd, qkv, gate, tab, pad, dO, scale, entry=entry)
        check_attn(rep, f"{tag} {entry}", dev, B, T, H, hd, qkv, gate, tab, pad, dO, scale, k)


# name, B, T, H, head width, bias, lengths (None: no padding).  The shipped shapes: WavLM Base 16 x 15 s, Large 8 x 20 s, a
# ragged Large batch (one utterance of one frame, one a single row into its second tile), XLS-R 1B (head width 80, no bias).
SHIPPED = [("base", 16, 749, 12, 64, True, None), ("large", 8, 999, 16, 64, True, None),
           ("large-ragged", 4, 1499, 16, 64, True, (1499, 501, 129, 1)), ("xlsr1b", 8, 999, 16, 80, False, None),
           ("xlsr1b-ragged", 4, 999, 16, 80, False, (999, 640, 129, 1))]
SHIPPED_CASES = [(c, rg) for c in SHIPPED for rg in (("diffuse", "shipped") if c[5] else ("diffuse",))]


@pytest.mark.parametrize("case,regime", SHIPPED_CASES, ids=[f"{c[0]}-{rg}" for c, rg in SHIPPED_CASES])
def test_attn_shipped(cuda_device, case, regime):
    name, B, T, H, hd, bias, lengths = case
    rep = {}
    attn_case(rep, name, cuda_device, B, T, H, hd, bias, lengths, regime, entries=("fused",))
    report("attn", f"{name} {regime}", rep)


# Tile edges (128 queries / keys per tile; 64-query tiles in the head-width-80 backward).  At T = 300 the second consumer
# warpgroup's rows of the last query tile all lie beyond T.  The second utterance is padded to about half its length (in the
# late regime to just past the late key), so the larger T also have a fully padded query block.
EDGE_T = (1, 63, 64, 65, 127, 128, 129, 255, 256, 257, 300)
EDGE_CASES = ([(T, 64, rg) for T in EDGE_T for rg in ("diffuse", "shipped", "peaked") + (("late",) if T > 128 else ())]
              + [(T, 80, rg) for T in EDGE_T for rg in ("diffuse",) + (("peaked", "late") if T > 128 else ())])


@pytest.mark.parametrize("T,hd,regime", EDGE_CASES, ids=[f"T{T}-hd{hd}-{rg}" for T, hd, rg in EDGE_CASES])
def test_attn_edges(cuda_device, T, hd, regime):
    rep = {}
    # the late maximum needs its key and rows valid in both utterances: the second one ends just after the late key
    n2 = late_key(T) + 1 if regime == "late" else (T + 1) // 2
    attn_case(rep, f"T{T}", cuda_device, 2, T, 2, hd, hd == 64, (T, n2), regime)
    report("attn", f"edge T={T} hd={hd} {regime}", rep)


@pytest.mark.parametrize("regime", ["diffuse", "late"])
def test_attn_t4096(cuda_device, regime):
    """T = 4096 with the bias and a ragged tail: 32 key tiles of bias window and d tab blocks."""
    rep = {}
    attn_case(rep, "T4096", cuda_device, 2, 4096, 1, 64, True, (4096, 4000), regime)
    report("attn", f"T=4096 {regime}", rep)


DROP_CASES = [(2, 300, 2, 64, True, (300, 200)), (2, 749, 3, 64, True, None), (2, 257, 2, 80, False, (257, 129))]


@pytest.mark.parametrize("B,T,H,hd,bias,lengths", DROP_CASES, ids=[f"B{c[0]}-T{c[1]}-hd{c[3]}" for c in DROP_CASES])
def test_attn_dropout(cuda_device, B, T, H, hd, bias, lengths):
    rep = {}
    attn_case(rep, f"T{T}", cuda_device, B, T, H, hd, bias, lengths, "diffuse", p=0.1)
    report("attn", f"dropout T={T} hd={hd}", rep)
