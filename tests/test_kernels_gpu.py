"""GPU parity tests of the memory-bound kernels, parameter preparation and attention against plain PyTorch fp32
references of the same op (op-level; whole-model parity against the oracle lives in test_model_gpu.py)."""
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def bf(t):
    return t.to(torch.bfloat16)


@pytest.mark.parametrize("D", [64, 128, 512, 768, 1024])
@pytest.mark.parametrize("gelu", [False, True])
def test_layer_norm_fwd_bwd(cuda_device, D, gelu):
    from unispeech_b200 import ops
    torch.manual_seed(D)
    B, T = 3, 37
    dev = cuda_device
    x = bf(torch.randn(B, T, D, device=dev) * 2 + 0.5)
    gamma = torch.rand(D, device=dev) + 0.5
    beta = torch.randn(D, device=dev) * 0.1
    y = torch.empty_like(x)
    mean = torch.empty(B * T, device=dev)
    rstd = torch.empty(B * T, device=dev)
    ops.layer_norm_fwd(x, T * D, D, gamma, beta, y, T * D, D, mean, rstd, T, B, D, gelu)
    xr = x.float().requires_grad_(True)
    gr = gamma.clone().requires_grad_(True)
    br = beta.clone().requires_grad_(True)
    ref = F.layer_norm(xr, (D,), gr, br, 1e-5)
    if gelu:
        ref = F.gelu(ref)
    torch.cuda.synchronize()
    assert (y.float() - ref).abs().max().item() < 0.04
    dy = bf(torch.randn(B, T, D, device=dev))
    dres = bf(torch.randn(B, T, D, device=dev))
    ref.backward(dy.float())
    dx = torch.empty_like(x)
    dgamma = torch.zeros(D, device=dev)
    dbeta = torch.zeros(D, device=dev)
    cs = torch.zeros(D, device=dev)
    ops.layer_norm_bwd(dy, T * D, D, x, T * D, D, mean, rstd, gamma, beta, dres, T * D, D, dx, T * D, D, dgamma, dbeta,
                       cs, T, B, D, gelu)
    torch.cuda.synchronize()
    assert (dx.float() - (xr.grad + dres.float())).abs().max().item() < 0.06
    assert (dgamma - gr.grad).abs().max().item() < 0.02 * max(1.0, gr.grad.abs().max().item())
    assert (dbeta - br.grad).abs().max().item() < 0.02 * max(1.0, br.grad.abs().max().item())
    assert (cs - dx.float().sum((0, 1))).abs().max().item() < 0.05


def test_colsum_dgelu_mask(cuda_device):
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(0)
    B, T, N = 2, 75, 200
    x = bf(torch.randn(B, T, N, device=dev))
    out = torch.zeros(N, device=dev)
    ops.colsum(x, T * N, N, T, B, N, out)
    torch.cuda.synchronize()
    assert (out - x.float().sum((0, 1))).abs().max().item() < 1e-2
    pre = bf(torch.randn(B, T, N, device=dev))
    Tp = T + 10
    dst = torch.zeros(B, Tp, N, device=dev, dtype=torch.bfloat16)
    cs = torch.zeros(N, device=dev)
    ops.dgelu_mul(x, T * N, N, pre, T * N, N, dst[:, 3:], Tp * N, N, T, B, N, cs)
    torch.cuda.synchronize()
    pr = pre.float().requires_grad_(True)
    g = torch.autograd.grad(F.gelu(pr).sum(), pr)[0]
    ref = x.float() * g
    assert (dst[:, 3:3 + T].float() - ref).abs().max().item() < 0.03
    assert dst[:, :3].abs().max().item() == 0 and dst[:, 3 + T:].abs().max().item() == 0
    assert (cs - dst.float().sum((0, 1))).abs().max().item() < 1e-2
    # frame masking
    D = 128
    y = bf(torch.randn(B, T, D, device=dev))
    y0 = y.clone()
    mask = (torch.rand(B, T, device=dev) > 0.5).to(torch.uint8)
    pad = (torch.rand(B, T, device=dev) > 0.8).to(torch.uint8)
    emb = torch.rand(D, device=dev)
    ops.frame_mask_fwd(y, T * D, D, T, B, D, mask, pad, emb)
    torch.cuda.synchronize()
    ref = torch.where(mask.bool().unsqueeze(-1), bf(emb).expand(B, T, D), y0)
    ref = ref.masked_fill(pad.bool().unsqueeze(-1), 0)
    assert torch.equal(y, ref)
    dy = bf(torch.randn(B, T, D, device=dev))
    dy0 = dy.clone()
    demb = torch.zeros(D, device=dev)
    ops.frame_mask_bwd(dy, T * D, D, T, B, D, mask, pad, demb)
    torch.cuda.synchronize()
    sel = mask.bool() & ~pad.bool()
    assert (demb - dy0.float()[sel].sum(0)).abs().max().item() < 1e-2
    keep = ~(mask.bool() | pad.bool())
    assert torch.equal(dy[keep], dy0[keep]) and dy[~keep].abs().max().item() == 0


@pytest.mark.parametrize("H", [4, 12, 16])
def test_layer_norm_gate_fwd(cuda_device, H):
    """LayerNorm fused with the gate of the consuming attention == layer_norm_fwd followed by gate_fwd on the stored output."""
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(100 + H)
    B, T, D = 3, 77, H * 64
    x = bf(torch.randn(B, T, D, device=dev) * 2 + 0.3)
    gamma, beta = torch.rand(D, device=dev) + 0.5, torch.randn(D, device=dev) * 0.1
    gw = torch.randn(8, 64, device=dev) * 0.2
    gb = torch.randn(8, device=dev) * 0.1
    ga = torch.rand(1, H, 1, 1, device=dev) + 0.5
    y1, y2 = torch.empty_like(x), torch.empty_like(x)
    m1, r1, m2, r2 = (torch.empty(B * T, device=dev) for _ in range(4))
    g1, g2 = torch.empty(B, H, T, device=dev), torch.empty(B, H, T, device=dev)
    ops.layer_norm_fwd(x, T * D, D, gamma, beta, y1, T * D, D, m1, r1, T, B, D)
    ops.gate_fwd(y1, T * D, D, T, B, H, gw, gb, ga, g1)
    ops.layer_norm_gate_fwd(x, T * D, D, gamma, beta, y2, T * D, D, m2, r2, T, B, D, gw, gb, ga, H, g2)
    torch.cuda.synchronize()
    ref = F.layer_norm(x.float(), (D,), gamma, beta)
    assert (y1.float() - ref).abs().max().item() < 0.03
    # (at the wide widths the fused kernel spreads a row over the block: its reduction order differs from the warp-per-row
    # kernel's, so the statistics agree to fp32 rounding and y to one bf16 step, not bit for bit)
    assert (m1 - m2).abs().max().item() < 1e-5 and (r1 - r2).abs().max().item() < 1e-4 * r1.abs().max().item()
    assert (y1.float() - y2.float()).abs().max().item() <= 0.0625
    # the gate must be that of the STORED y of the same kernel: recompute it from y2 with the stand-alone gate kernel
    ops.gate_fwd(y2, T * D, D, T, B, H, gw, gb, ga, g1)
    torch.cuda.synchronize()
    assert (g1 - g2).abs().max().item() < 1e-5


@pytest.mark.parametrize("H", [2, 12, 16])
def test_gate_fwd_bwd(cuda_device, H):
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(H)
    B, T, D = 2, 45, H * 64
    x = bf(torch.randn(B, T, D, device=dev))
    gw = torch.randn(8, 64, device=dev) * 0.2
    gb = torch.randn(8, device=dev) * 0.1
    ga = torch.rand(1, H, 1, 1, device=dev) + 0.5
    gate = torch.empty(B, H, T, device=dev)
    ops.gate_fwd(x, T * D, D, T, B, H, gw, gb, ga, gate)
    xr = x.float().requires_grad_(True)
    gwr, gbr, gar = gw.clone().requires_grad_(True), gb.clone().requires_grad_(True), ga.clone().requires_grad_(True)
    q = xr.view(B, T, H, 64).permute(0, 2, 1, 3)
    g = torch.sigmoid(F.linear(q, gwr, gbr).view(B, H, T, 2, 4).sum(-1))
    a, b_ = g.chunk(2, dim=-1)
    ref = (a * (b_ * gar - 1.0) + 2.0).squeeze(-1)
    torch.cuda.synchronize()
    assert (gate - ref).abs().max().item() < 1e-4
    dgate = torch.randn(B, H, T, device=dev)
    ref.backward(dgate)
    dxg = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    dgw, dgb, dga = torch.zeros_like(gw), torch.zeros_like(gb), torch.zeros(H, device=dev)
    ops.gate_bwd(x, T * D, D, T, B, H, gw, gb, ga, dgate, dxg, T * D, D, dgw, dgb, dga)
    torch.cuda.synchronize()
    assert (dxg.float() - xr.grad).abs().max().item() < 0.02
    assert (dgw - gwr.grad).abs().max().item() < 1e-3 * max(1, gwr.grad.abs().max().item())
    assert (dgb - gbr.grad).abs().max().item() < 1e-3 * max(1, gbr.grad.abs().max().item())
    assert (dga - gar.grad.view(-1)).abs().max().item() < 1e-3 * max(1, gar.grad.abs().max().item())


@pytest.mark.parametrize("Cc,mode", [(64, 0), (64, 1), (512, 0), (512, 1)])
def test_conv0_fwd_bwd(cuda_device, Cc, mode):
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(Cc + mode)
    B, L_, k, s = 2, 4003, 10, 5
    T = (L_ - k) // s + 1
    wav = torch.randn(B, L_, device=dev)
    wav[1, 3000:] = 0
    w = torch.randn(Cc, 1, k, device=dev) * 0.5
    gamma = torch.rand(Cc, device=dev) + 0.5
    beta = torch.randn(Cc, device=dev) * 0.1
    Tp = T + (T % 2)
    out = torch.zeros(B, Tp, Cc, device=dev, dtype=torch.bfloat16)
    stats = torch.zeros(B * Cc * 2 + B * 128, device=dev, dtype=torch.float64)
    fmean = torch.zeros(B, T, device=dev)
    frstd = torch.zeros(B, T, device=dev)
    ops.conv0_fwd(wav, L_, B, T, Cc, k, s, w, gamma, beta, mode, stats, fmean, frstd, out, Tp * Cc)
    wr, gr, br = w.clone().requires_grad_(True), gamma.clone().requires_grad_(True), beta.clone().requires_grad_(True)
    c = F.conv1d(wav.unsqueeze(1), wr, stride=s)
    if mode == 0:
        n = F.group_norm(c, Cc, gr, br, 1e-5)
    else:
        n = F.layer_norm(c.transpose(1, 2), (Cc,), gr, br, 1e-5).transpose(1, 2)
    ref = F.gelu(n).transpose(1, 2)  # [B,T,C]
    torch.cuda.synchronize()
    assert (out[:, :T].float() - ref).abs().max().item() < 0.03
    da = bf(torch.randn(B, T, Cc, device=dev))
    ref.backward(da.float())
    dap = torch.zeros(B, Tp, Cc, device=dev, dtype=torch.bfloat16)
    dap[:, :T] = da
    dw, dg, db = torch.zeros_like(w), torch.zeros_like(gamma), torch.zeros_like(beta)
    bstats = torch.zeros(B, Cc, 12, device=dev)
    ops.conv0_bwd(wav, L_, B, T, Cc, k, s, w, gamma, beta, mode, stats, bstats, fmean, frstd, dap, Tp * Cc, dw, dg, db)
    torch.cuda.synchronize()
    for got, want, name in ((dw, wr.grad, "dw"), (dg, gr.grad, "dgamma"), (db, br.grad, "dbeta")):
        err = (got - want).abs().max().item()
        assert err < 5e-3 * max(1.0, want.abs().max().item()), (name, err, want.abs().max().item())
    if mode == 1:
        # two-pass variant with a dconv workspace: separate buffer, then aliasing the incoming gradient (as the engine does)
        for ws in (torch.zeros_like(dap), dap):
            dw2, dg2, db2 = torch.zeros_like(w), torch.zeros_like(gamma), torch.zeros_like(beta)
            ops.conv0_bwd(wav, L_, B, T, Cc, k, s, w, gamma, beta, mode, stats, bstats, fmean, frstd, dap, Tp * Cc, dw2, dg2, db2,
                          dconv_ws=ws, ws_bs=Tp * Cc)
            torch.cuda.synchronize()
            for got, want, name in ((dw2, wr.grad, "dw"), (dg2, gr.grad, "dgamma"), (db2, br.grad, "dbeta")):
                err = (got - want).abs().max().item()
                assert err < 8e-3 * max(1.0, want.abs().max().item()), (name, err, want.abs().max().item())


def test_prep_kernels(cuda_device):
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(0)
    N, K = 70, 100
    w = torch.randn(N, K, device=dev)
    d = torch.zeros(N + 5, K + 3, device=dev, dtype=torch.bfloat16)
    dT = torch.zeros(K, N + 7, device=dev, dtype=torch.bfloat16)
    ops.prep_linear(w, N, K, 0.5, d, K + 3, dT, N + 7)
    torch.cuda.synchronize()
    assert torch.equal(d[:N, :K], bf(w * 0.5)) and torch.equal(dT[:, :N], bf(w * 0.5).t())
    Co, Ci, k, s = 16, 24, 3, 2
    cw = torch.randn(Co, Ci, k, device=dev)
    f = torch.empty(Co, k * Ci, device=dev, dtype=torch.bfloat16)
    ops.prep_conv_fwd(cw, Co, Ci, k, f)
    torch.cuda.synchronize()
    assert torch.equal(f, bf(cw.permute(0, 2, 1).reshape(Co, k * Ci)))
    e = torch.empty(Ci, 2 * Co, device=dev, dtype=torch.bfloat16)
    o = torch.empty(Ci, Co, device=dev, dtype=torch.bfloat16)
    ops.prep_conv_dgrad(cw, Co, Ci, k, s, 0, e)
    ops.prep_conv_dgrad(cw, Co, Ci, k, s, 1, o)
    torch.cuda.synchronize()
    assert torch.equal(e[:, :Co], bf(cw[:, :, 2].t())) and torch.equal(e[:, Co:], bf(cw[:, :, 0].t()))
    assert torch.equal(o, bf(cw[:, :, 1].t()))
    dwk = torch.randn(Co, k * Ci, device=dev)
    dw = torch.ones(Co, Ci, k, device=dev)
    ops.unprep_conv_wgrad(dwk, Co, Ci, k, dw)
    torch.cuda.synchronize()
    assert torch.allclose(dw, 1 + dwk.view(Co, k, Ci).permute(0, 2, 1))
    # pos_conv weight norm
    D, G, taps = 128, 16, 128
    Cg = D // G
    v = torch.randn(D, Cg, taps, device=dev)
    g = torch.rand(1, 1, taps, device=dev) + 0.5
    norm2 = torch.zeros(2 * taps, device=dev)   # fp64[taps]
    wf = torch.empty(G, 64, taps, 64, device=dev, dtype=torch.bfloat16)
    wd = torch.empty_like(wf)
    ops.posconv_prep(v, g, D, G, taps, norm2, wf, wd)
    torch.cuda.synchronize()
    vr, gr = v.clone().requires_grad_(True), g.clone().requires_grad_(True)
    wn = gr * vr / vr.norm(2, dim=(0, 1), keepdim=True)
    ref_f = wn.view(G, Cg, Cg, taps).permute(0, 1, 3, 2)  # [g, co, j, ci]
    assert (wf[:, :Cg, :, :Cg].float() - ref_f).abs().max().item() < 0.02
    assert wf[:, Cg:].abs().max().item() == 0 and wf[:, :, :, Cg:].abs().max().item() == 0
    ref_d = wn.view(G, Cg, Cg, taps).flip(-1).permute(0, 2, 3, 1)  # [g, ci, j', co]
    assert (wd[:, :Cg, :, :Cg].float() - ref_d).abs().max().item() < 0.02
    dwp = torch.zeros(G, Cg, taps, 64, device=dev)
    dwn = torch.randn(D, Cg, taps, device=dev)
    dwp[:, :, :, :Cg] = dwn.view(G, Cg, Cg, taps).permute(0, 1, 3, 2)
    wn.backward(dwn)
    dv, dg = torch.zeros_like(v), torch.zeros_like(g)
    work = torch.zeros(4 * taps, device=dev)   # fp64[2 * taps]
    ops.posconv_unprep(v, g, dwp, D, G, taps, work, dv, dg)
    torch.cuda.synchronize()
    assert (dv - vr.grad).abs().max().item() < 1e-3 * max(1, vr.grad.abs().max().item())
    assert (dg - gr.grad).abs().max().item() < 1e-3 * max(1, gr.grad.abs().max().item())
    # relative position table
    H, T = 3, 50
    emb = torch.randn(320, H, device=dev)
    lut = torch.randint(0, 320, (2 * T - 1,), device=dev, dtype=torch.int32)
    tab = torch.empty(H, 2 * T - 1, device=dev)
    ops.relpos_table_fwd(emb, lut, 2 * T - 1, H, tab)
    torch.cuda.synchronize()
    assert torch.equal(tab, emb[lut.long()].t())
    dtab = torch.randn(H, 2 * T - 1, device=dev)
    demb = torch.zeros_like(emb)
    ops.relpos_table_bwd(dtab, lut, 2 * T - 1, H, demb)
    torch.cuda.synchronize()
    ref = torch.zeros_like(emb).index_add_(0, lut.long(), dtab.t().contiguous())
    assert (demb - ref).abs().max().item() < 1e-4


def _attn_ref(qkv, gate, tab, pad, B, T, H, scale):
    D = H * 64
    q, k, v = qkv.float().split(D, dim=-1)
    q = q.view(B, T, H, 64).transpose(1, 2)
    k = k.view(B, T, H, 64).transpose(1, 2)
    v = v.view(B, T, H, 64).transpose(1, 2)
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    if tab is not None:
        i = torch.arange(T, device=qkv.device)[:, None]
        j = torch.arange(T, device=qkv.device)[None, :]
        bias = tab[:, (j - i) + T - 1]  # [H,T,T]
        g = gate if gate is not None else torch.ones(B, H, T, device=qkv.device)
        s = s + g.unsqueeze(-1) * bias.unsqueeze(0)
    if pad is not None:
        s = s.masked_fill(pad.bool()[:, None, None, :], float("-inf"))
    p = torch.softmax(s, dim=-1)
    o = torch.matmul(p, v).transpose(1, 2).reshape(B, T, D)
    return o


@pytest.mark.parametrize("B,T,H,bias,padded", [(2, 100, 2, True, True), (1, 128, 2, True, False), (2, 333, 3, True, True),
                                               (1, 749, 12, True, False), (2, 257, 2, False, True), (1, 1499, 2, True, True),
                                               (2, 3072, 1, True, True)])
def test_attn_fwd(cuda_device, B, T, H, bias, padded):
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(T)
    D = H * 64
    qkv = bf(torch.randn(B, T, 3 * D, device=dev))
    gate = (torch.rand(B, H, T, device=dev) * 2 + 0.2) if bias else None
    tab = torch.randn(H, 2 * T - 1, device=dev) if bias else None
    pad = None
    if padded:
        pad = torch.zeros(B, T, device=dev, dtype=torch.uint8)
        pad[0, T - T // 3:] = 1
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    ops.attn_fwd(qkv, gate, tab, pad, out, lse, B, T, H, 0.125)
    torch.cuda.synchronize()
    ref = _attn_ref(qkv, gate, tab, pad, B, T, H, 0.125)
    assert torch.isfinite(out.float()).all()
    d = (out.float() - ref).abs()
    if padded:  # rows of padded QUERY frames are unspecified-but-finite (zeros where a whole 128-row block is padded): the
        d = d[pad == 0]  # reference's values there never reach a valid frame (padded keys are masked)
    err = d.max().item()
    assert err < 0.03, err


def test_attn_fwd_rebase(cuda_device):
    """Scores in later key tiles far above the first tile's maximum: the single-pass softmax must re-base (fast-path guard)."""
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(5)
    B, T, H = 2, 520, 2
    D = H * 64
    qkv = torch.randn(B, T, 3 * D, device=dev)
    qkv[:, 200:, D:2 * D] *= 30.0   # keys of the later tiles -> logits up to ~ +-100 nats
    qkv[0, 300:330, D:2 * D] *= 4.0
    qkv = bf(qkv)
    gate = torch.rand(B, H, T, device=dev) * 2 + 0.2
    tab = torch.randn(H, 2 * T - 1, device=dev)
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    ops.attn_fwd(qkv, gate, tab, None, out, lse, B, T, H, 0.125)
    torch.cuda.synchronize()
    ref = _attn_ref(qkv, gate, tab, None, B, T, H, 0.125)
    assert torch.isfinite(out.float()).all() and torch.isfinite(lse).all()
    assert (out.float() - ref).abs().max().item() < 0.05


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("B,T,H,bias,padded", [(2, 100, 2, True, True), (1, 128, 2, True, False), (2, 333, 3, True, True),
                                               (1, 520, 4, True, False), (2, 257, 2, False, True), (1, 749, 3, True, False),
                                               (2, 1499, 1, True, True)])
def test_attn_bwd(cuda_device, B, T, H, bias, padded, fused):
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(T + 1)
    D = H * 64
    qkv = bf(torch.randn(B, T, 3 * D, device=dev))
    gate = (torch.rand(B, H, T, device=dev) * 2 + 0.2) if bias else None
    tab = torch.randn(H, 2 * T - 1, device=dev) if bias else None
    pad = None
    if padded:
        pad = torch.zeros(B, T, device=dev, dtype=torch.uint8)
        pad[0, T - T // 3:] = 1
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    ops.attn_fwd(qkv, gate, tab, pad, out, lse, B, T, H, 0.125)
    dout = bf(torch.randn(B, T, D, device=dev))
    if padded:  # padded query frames carry no gradient in the model (the loss never reads them); their forward values are unspecified
        dout[pad.bool()] = 0
    delta = torch.empty(B, H, T, device=dev)
    dqkv = torch.zeros(B, T, 3 * D, device=dev, dtype=torch.bfloat16)
    dgate = torch.zeros(B, H, T, device=dev) if bias else None
    dtab = torch.zeros(H, 2 * T - 1, device=dev) if bias else None
    if fused:
        dq_acc = torch.zeros(B, T, D, device=dev)
        if bias:
            dgate.fill_(7.0)  # the fused path must overwrite, not accumulate into, d gate
        ops.attn_bwd_fused(qkv, out, dout, gate, tab, pad, lse, delta, dq_acc, dqkv, dgate, dtab, B, T, H, 0.125)
        torch.cuda.synchronize()
        assert dq_acc.abs().max().item() == 0.0  # workspace handed back clean
    else:
        ops.attn_bwd(qkv, out, dout, gate, tab, pad, lse, delta, dqkv, dgate, dtab, B, T, H, 0.125)
    torch.cuda.synchronize()
    qr = qkv.float().requires_grad_(True)
    gr = gate.clone().requires_grad_(True) if bias else None
    tr = tab.clone().requires_grad_(True) if bias else None
    ref = _attn_ref(qr, gr, tr, pad, B, T, H, 0.125)
    ref.backward(dout.float())
    assert torch.isfinite(dqkv.float()).all()
    scale_ref = qr.grad.abs().max().item()
    err = (dqkv.float() - qr.grad).abs().max().item()
    assert err < 0.03 * max(1.0, scale_ref), (err, scale_ref)
    if bias:
        e1 = (dgate - gr.grad).abs().max().item()
        assert e1 < 0.03 * max(1.0, gr.grad.abs().max().item()), e1
        e2 = (dtab - tr.grad).abs().max().item()
        assert e2 < 0.03 * max(1.0, tr.grad.abs().max().item()), (e2, tr.grad.abs().max().item())


def test_attn_bwd_long_sequence(cuda_device):
    """The longest utterance the bias path takes (T = 3072 frames, about 61 s), ragged: b200s_attn_bwd (the entry point used beyond
    the fused API's T <= 2048) against autograd of the reference."""
    test_attn_bwd(cuda_device, 2, 3072, 1, True, True, False)


def test_prep_linear_batched_shapes(cuda_device):
    """One launch, several nn.Linear masters (aligned and ragged shapes): bf16 copy and bf16 transpose, bit exact."""
    import struct
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(3)
    shapes = [(70, 100), (64, 64), (130, 36), (1, 5), (256, 768), (192, 64), (66, 130)]
    recs, tiles, keep = [], 0, []
    for N, K in shapes:
        src = torch.randn(N, K, device=dev)
        dst = torch.full((N, K), 9.0, device=dev, dtype=torch.bfloat16)
        dstT = torch.full((K, N), 9.0, device=dev, dtype=torch.bfloat16)
        tk = (K + 63) // 64
        recs.append(struct.pack("<QQQqqiiii", src.data_ptr(), dst.data_ptr(), dstT.data_ptr(), K, N, N, K, tiles, tk))
        tiles += ((N + 63) // 64) * tk
        keep.append((src, dst, dstT))
    descs = torch.frombuffer(bytearray(b"".join(recs)), dtype=torch.uint8).to(dev)
    ops.prep_linear_batched(descs, len(recs), tiles)
    torch.cuda.synchronize()
    for (N, K), (src, dst, dstT) in zip(shapes, keep):
        want = src.to(torch.bfloat16)
        assert torch.equal(dst, want), (N, K)
        assert torch.equal(dstT, want.t().contiguous()), (N, K)


@pytest.mark.parametrize("D,gelu", [(128, False), (512, True), (1024, False)])
def test_ragged_row_kernels(cuda_device, D, gelu):
    """`valid` forms (BASELINE configs[4]): rows below valid[b] are bit-identical to the dense kernels, padded rows come out as
    zeros, and the parameter-gradient sums equal the dense sums of a gradient that is zero on the padded rows."""
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(7 + D)
    B, T = 3, 61
    valid = torch.tensor([61, 17, 0], dtype=torch.int32, device=dev)
    live = (torch.arange(T, device=dev)[None, :] < valid[:, None])            # [B, T]
    x = bf(torch.randn(B, T, D, device=dev) * 1.5 + 0.2)
    gamma, beta = torch.rand(D, device=dev) + 0.5, torch.randn(D, device=dev) * 0.1
    y0, y1 = torch.empty_like(x), torch.full_like(x, float("nan"))
    m0, r0, m1, r1 = (torch.full((B * T,), float("nan"), device=dev) for _ in range(4))
    ops.layer_norm_fwd(x, T * D, D, gamma, beta, y0, T * D, D, m0, r0, T, B, D, gelu)
    ops.layer_norm_fwd(x, T * D, D, gamma, beta, y1, T * D, D, m1, r1, T, B, D, gelu, valid=valid)
    torch.cuda.synchronize()
    assert torch.equal(y1[live], y0[live]) and y1[~live].abs().max().item() == 0
    assert torch.equal(m1.view(B, T)[live], m0.view(B, T)[live]) and torch.equal(r1.view(B, T)[live], r0.view(B, T)[live])
    # backward
    dy = bf(torch.randn(B, T, D, device=dev)) * live.unsqueeze(-1)
    dres = bf(torch.randn(B, T, D, device=dev)) * live.unsqueeze(-1)
    outs = []
    for v in (None, valid):
        dx = torch.full_like(x, float("nan"))
        dg, db, cs = torch.zeros(D, device=dev), torch.zeros(D, device=dev), torch.zeros(D, device=dev)
        # dense run: statistics of the padded rows come from the dense forward; their dy is zero, so they add nothing
        ops.layer_norm_bwd(dy, T * D, D, x, T * D, D, m0, r0, gamma, beta, dres, T * D, D, dx, T * D, D, dg, db, cs, T, B, D,
                           gelu, valid=v)
        outs.append((dx, dg, db, cs))
    torch.cuda.synchronize()
    (dx0, dg0, db0, cs0), (dx1, dg1, db1, cs1) = outs
    assert torch.equal(dx1[live], dx0[live]) and dx1[~live].abs().max().item() == 0
    for a_, b_ in ((dg0, dg1), (db0, db1), (cs0, cs1)):
        assert (a_ - b_).abs().max().item() <= 1e-3 * max(1.0, a_.abs().max().item())
    c0, c1 = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
    ops.colsum(dy, T * D, D, T, B, D, c0)
    ops.colsum(bf(torch.randn(B, T, D, device=dev)).masked_scatter_(live.unsqueeze(-1).expand(B, T, D), dy[live]), T * D, D, T, B, D,
               c1, valid=valid)   # garbage on the padded rows must not be counted
    torch.cuda.synchronize()
    assert (c0 - c1).abs().max().item() <= 1e-3 * max(1.0, c0.abs().max().item())


@pytest.mark.parametrize("H", [12, 16])
def test_ragged_gate_kernels(cuda_device, H):
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(50 + H)
    B, T, D = 3, 53, H * 64
    valid = torch.tensor([53, 9, 0], dtype=torch.int32, device=dev)
    live = (torch.arange(T, device=dev)[None, :] < valid[:, None])
    x = bf(torch.randn(B, T, D, device=dev))
    gamma, beta = torch.rand(D, device=dev) + 0.5, torch.randn(D, device=dev) * 0.1
    gw, gb, ga = torch.randn(8, 64, device=dev) * 0.2, torch.randn(8, device=dev) * 0.1, torch.rand(1, H, 1, 1, device=dev) + 0.5
    res = []
    for v in (None, valid):
        y = torch.full_like(x, float("nan"))
        mean, rstd = torch.empty(B * T, device=dev), torch.empty(B * T, device=dev)
        gate = torch.full((B, H, T), float("nan"), device=dev)
        ops.layer_norm_gate_fwd(x, T * D, D, gamma, beta, y, T * D, D, mean, rstd, T, B, D, gw, gb, ga, H, gate, valid=v)
        res.append((y, gate))
    torch.cuda.synchronize()
    (y0, g0), (y1, g1) = res
    lg = live[:, None, :].expand(B, H, T)
    assert torch.equal(y1[live], y0[live]) and y1[~live].abs().max().item() == 0
    assert torch.equal(g1[lg], g0[lg]) and bool((g1[~lg] == 1.0).all())
    dgate = torch.randn(B, H, T, device=dev) * lg
    outs = []
    for v in (None, valid):
        dxg = torch.full_like(x, float("nan"))
        dgw, dgb, dga = torch.zeros_like(gw), torch.zeros_like(gb), torch.zeros(H, device=dev)
        ops.gate_bwd(x, T * D, D, T, B, H, gw, gb, ga, dgate, dxg, T * D, D, dgw, dgb, dga, valid=v)
        outs.append((dxg, dgw, dgb, dga))
    torch.cuda.synchronize()
    (d0, w0, b0, a0), (d1, w1, b1, a1) = outs
    assert torch.equal(d1[live], d0[live]) and d1[~live].abs().max().item() == 0
    for p_, q_ in ((w0, w1), (b0, b1), (a0, a1)):
        assert (p_ - q_).abs().max().item() <= 1e-3 * max(1.0, p_.abs().max().item())
