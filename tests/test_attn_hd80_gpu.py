"""Attention at head width 80 (XLS-R 1B / MMS-1B / HuBERT X-Large: D = 1280, 16 heads), without the relative-position bias:
forward outputs and log-sum-exp against an fp64 reference, dQ / dK / dV through b200s_attn_bwd and b200s_attn_bwd_fused against
fp64 autograd, and attention dropout (keep bits equal to the hash, forward / backward equal to the reference run with those
bits).  The shapes cover a partial last query tile in which every row of the second consumer warpgroup lies beyond T (T = 300),
T = 1, a ragged batch with an utterance shorter than one tile, and a long utterance."""
import numpy as np
import pytest
import torch

from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu

LN2 = float(np.log(2.0))


def bf(t):
    return t.to(torch.bfloat16)


def ref_attn(qkv, pad, B, T, H, hd, keep=None, p=0.0):
    """fp64 attention of the fused [B, T, 3D] projection at head width hd; returns (out [B, T, D], natural-log lse [B, H, T])."""
    D = H * hd
    q, k, v = (t.reshape(B, T, H, hd).transpose(1, 2) for t in qkv.double().split(D, dim=-1))
    s = torch.matmul(q, k.transpose(-1, -2)) * hd ** -0.5
    if pad is not None:
        s = s.masked_fill(pad.bool()[:, None, None, :], float("-inf"))
    lse = torch.logsumexp(s, dim=-1)
    pr = torch.softmax(s, dim=-1)
    if keep is not None:
        pr = pr * keep.to(pr.dtype) / (1.0 - p)
    return torch.matmul(pr, v).transpose(1, 2).reshape(B, T, D), lse


def make_inputs(dev, B, T, H, hd, valid, seed):
    torch.manual_seed(seed)
    D = H * hd
    qkv = bf(torch.randn(B, T, 3 * D, device=dev))
    pad = None
    if valid is not None:
        pad = torch.zeros(B, T, device=dev, dtype=torch.uint8)
        for b, n in enumerate(valid):
            pad[b, n:] = 1
    dout = bf(torch.randn(B, T, D, device=dev))
    if pad is not None:
        dout[pad.bool()] = 0  # padded query frames carry no gradient in the model
    return qkv, pad, dout


def check_fwd(out, lse, qkv, pad, B, T, H, hd, keep=None, p=0.0):
    ref, ref_lse = ref_attn(qkv, pad, B, T, H, hd, keep, p)
    assert torch.isfinite(out.float()).all()
    rows = (pad == 0) if pad is not None else torch.ones(B, T, dtype=torch.bool, device=out.device)
    err = (out.double() - ref).abs()[rows].max().item()
    assert err < 0.04, err
    if keep is None:
        got = lse.double() * LN2   # the kernel keeps lse in the log2 domain
        e = (got - ref_lse).abs().permute(0, 2, 1)[rows].max().item()
        assert e < 1e-3 * max(1.0, ref_lse.abs().max().item()), e


def check_bwd(dqkv, qkv, pad, dout, B, T, H, hd, keep=None, p=0.0):
    D = H * hd
    qr = qkv.double().requires_grad_(True)
    ref_attn(qr, pad, B, T, H, hd, keep, p)[0].backward(dout.double())
    assert torch.isfinite(dqkv.float()).all()
    scale_ref = qr.grad.abs().max().item()
    err = (dqkv.double() - qr.grad).abs().max().item()
    assert err < 0.03 * max(1.0, scale_ref), (err, scale_ref)
    for name, lo in (("dq", 0), ("dk", D), ("dv", 2 * D)):
        g_, r_ = dqkv.double()[..., lo:lo + D], qr.grad[..., lo:lo + D]
        if r_.norm().item() < 1e-6:   # dQ is zero at T = 1 (one key): the max-abs check above covers it
            continue
        cos = (g_ * r_).sum() / (g_.norm() * r_.norm() + 1e-30)
        assert cos.item() > 0.999, (name, cos.item())


CASES = [  # B, T, H, valid frames per utterance (None: no padding)
    (2, 999, 16, None),
    (2, 999, 16, (999, 640)),
    (2, 300, 4, None),          # last query tile: rows 256..299, the second consumer warpgroup's rows are all beyond T
    (1, 1, 2, None),
    (3, 300, 2, (300, 57, 200)),  # ragged, one utterance shorter than one tile
]


@pytest.mark.parametrize("B,T,H,valid", CASES)
def test_attn_hd80_fwd_bwd(cuda_device, B, T, H, valid):
    from unispeech_b200 import ops
    dev, hd = cuda_device, 80
    D = H * hd
    qkv, pad, dout = make_inputs(dev, B, T, H, hd, valid, seed=T + B)
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    ops.attn_fwd(qkv, None, None, pad, out, lse, B, T, H, hd ** -0.5, head_dim=hd)
    torch.cuda.synchronize()
    check_fwd(out, lse, qkv, pad, B, T, H, hd)
    delta = torch.empty(B, H, T, device=dev)
    for fused in (True, False):
        dqkv = torch.full((B, T, 3 * D), 3.0, device=dev, dtype=torch.bfloat16)
        if fused:
            dq_acc = torch.zeros(B, T, D, device=dev)
            ops.attn_bwd_fused(qkv, out, dout, None, None, pad, lse, delta, dq_acc, dqkv, None, None, B, T, H, hd ** -0.5,
                               head_dim=hd)
            torch.cuda.synchronize()
            assert dq_acc.abs().max().item() == 0.0
        else:
            ops.attn_bwd(qkv, out, dout, None, None, pad, lse, delta, dqkv, None, None, B, T, H, hd ** -0.5, head_dim=hd)
            torch.cuda.synchronize()
        check_bwd(dqkv, qkv, pad, dout, B, T, H, hd)


def test_attn_hd80_long(cuda_device):
    from unispeech_b200 import ops
    dev, hd, B, T, H = cuda_device, 80, 1, 4096, 2
    D = H * hd
    qkv, pad, dout = make_inputs(dev, B, T, H, hd, None, seed=4096)
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    ops.attn_fwd(qkv, None, None, pad, out, lse, B, T, H, hd ** -0.5, head_dim=hd)
    delta = torch.empty(B, H, T, device=dev)
    dqkv = torch.empty(B, T, 3 * D, device=dev, dtype=torch.bfloat16)
    dq_acc = torch.zeros(B, T, D, device=dev)
    ops.attn_bwd_fused(qkv, out, dout, None, None, pad, lse, delta, dq_acc, dqkv, None, None, B, T, H, hd ** -0.5, head_dim=hd)
    torch.cuda.synchronize()
    check_fwd(out, lse, qkv, pad, B, T, H, hd)
    check_bwd(dqkv, qkv, pad, dout, B, T, H, hd)


def unpack_mask(words, B, T, H):
    """uint32 words [B*H, 4n, 128n] (bit i & 31 of word (i >> 5, j)) -> bool [B, H, T, T]."""
    n = (T + 127) // 128
    w = words.view(B * H, 4 * n, 128 * n).cpu().numpy().astype(np.uint32)
    bits = (w[:, :, None, :] >> np.arange(32, dtype=np.uint32)[None, None, :, None]) & 1
    return torch.from_numpy(bits.reshape(B * H, 128 * n, 128 * n)[:, :T, :T].astype(bool)).view(B, H, T, T)


@pytest.mark.parametrize("B,T,H,valid", [(2, 300, 3, (300, 200)), (1, 520, 2, None)])
def test_attn_hd80_dropout(cuda_device, B, T, H, valid):
    from unispeech_b200 import ops
    dev, hd, p = cuda_device, 80, 0.1
    D = H * hd
    qkv, pad, dout = make_inputs(dev, B, T, H, hd, valid, seed=T + 7)
    d = O.HashDropout(777 + T)
    site = O.HashDropout.layer_site(1, 3)
    key = tuple(int(v) for v in d.key(site))
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    words = torch.full((ops.attn_dropout_mask_words(B, T, H),), -1, dtype=torch.int32, device=dev)
    ops.attn_fwd_dropout(qkv, None, None, pad, out, lse, B, T, H, hd ** -0.5, p, key, words, head_dim=hd)
    torch.cuda.synchronize()
    got_keep = unpack_mask(words, B, T, H)
    want_keep = torch.from_numpy(d.keep_attn(site, B, H, T, p))
    if pad is not None:  # bits are specified where both the key and the query frame are valid
        ok = (pad == 0).cpu()
        sel = (ok[:, None, None, :] & ok[:, None, :, None]).expand_as(want_keep)
        assert torch.equal(got_keep[sel], want_keep[sel])
    else:
        assert torch.equal(got_keep, want_keep)
    keep = want_keep.to(dev)
    check_fwd(out, lse, qkv, pad, B, T, H, hd, keep, p)
    delta = torch.empty(B, H, T, device=dev)
    dqkv = torch.zeros(B, T, 3 * D, device=dev, dtype=torch.bfloat16)
    dq_acc = torch.zeros(B, T, D, device=dev)
    ops.attn_bwd_fused_dropout(qkv, out, dout, None, None, pad, lse, delta, dq_acc, dqkv, None, None, B, T, H, hd ** -0.5, p,
                               words, head_dim=hd)
    torch.cuda.synchronize()
    check_bwd(dqkv, qkv, pad, dout, B, T, H, hd, keep, p)


@pytest.mark.parametrize("ragged", [False, True])
def test_layer_norm_1280(cuda_device, ragged):
    """Warp-per-row LayerNorm forward and backward at D = 1280, dense and ragged, against fp64."""
    from unispeech_b200 import ops
    dev, B, T, D = cuda_device, 2, 37, 1280
    torch.manual_seed(1280)
    x = bf(torch.randn(B, T, D, device=dev) * 2 + 0.5)
    w = torch.randn(D, device=dev) * 0.5 + 1
    bias = torch.randn(D, device=dev) * 0.1
    dy = bf(torch.randn(B, T, D, device=dev))
    rows = torch.ones(B, T, dtype=torch.bool, device=dev)
    valid = None
    if ragged:
        valid = torch.tensor([T, 20], dtype=torch.int32, device=dev)
        rows[1, 20:] = False
        dy[~rows] = 0
    xr = x.double().requires_grad_(True)
    wr, br = w.double().requires_grad_(True), bias.double().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(xr, (D,), wr, br, eps=1e-5)
    yr.backward(dy.double())
    y = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    mean = torch.empty(B * T, device=dev)
    rstd = torch.empty(B * T, device=dev)
    ops.layer_norm_fwd(x, T * D, D, w, bias, y, T * D, D, mean, rstd, T, B, D, valid=valid)
    dx = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    dw = torch.zeros(D, device=dev)
    db = torch.zeros(D, device=dev)
    ops.layer_norm_bwd(dy, T * D, D, x, T * D, D, mean, rstd, w, bias, None, 0, 0, dx, T * D, D, dw, db, None, T, B, D,
                       valid=valid)
    torch.cuda.synchronize()
    assert (y.double() - yr)[rows].abs().max().item() < 0.05
    assert (dx.double() - xr.grad)[rows].abs().max().item() < 0.03 * max(1.0, xr.grad.abs().max().item())
    assert (dw.double() - wr.grad).abs().max().item() < 1e-2 * max(1.0, wr.grad.abs().max().item())
    assert (db.double() - br.grad).abs().max().item() < 1e-2 * max(1.0, br.grad.abs().max().item())
