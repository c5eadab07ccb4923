"""Attention backward cases that test_attn_bwd cannot express: padding on every utterance (to a different length each),
sequences that end one row into a tile, and T = 4096 with the relative-position bias through b200s_attn_bwd -- the largest
shared-memory layout of the kernel (32 key tiles of table and d tab accumulators).  The forward takes the bias only up to
T = 3840, so at T = 4096 the output and lse come from the fp32 reference."""
import math

import pytest
import torch

from test_kernels_gpu import _attn_ref, bf


def _ref_out_lse(qkv, gate, tab, pad, B, T, H, scale):
    """Attention output (bf16) and the forward kernel's lse (log2 domain) from the fp32 reference."""
    D = H * 64
    q, k, _ = qkv.float().split(D, dim=-1)
    q = q.view(B, T, H, 64).transpose(1, 2)
    k = k.view(B, T, H, 64).transpose(1, 2)
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    if tab is not None:
        i = torch.arange(T, device=qkv.device)[:, None]
        j = torch.arange(T, device=qkv.device)[None, :]
        s = s + gate.unsqueeze(-1) * tab[:, (j - i) + T - 1].unsqueeze(0)
    if pad is not None:
        s = s.masked_fill(pad.bool()[:, None, None, :], float("-inf"))
    lse = torch.logsumexp(s, dim=-1) / math.log(2.0)
    return bf(_attn_ref(qkv, gate, tab, pad, B, T, H, scale)), lse.contiguous()


def _check_bwd(dev, B, T, H, bias, lengths, fused, ref_forward=False):
    from unispeech_b200 import ops
    torch.manual_seed(T + 7)
    D = H * 64
    qkv = bf(torch.randn(B, T, 3 * D, device=dev))
    gate = (torch.rand(B, H, T, device=dev) * 2 + 0.2) if bias else None
    tab = torch.randn(H, 2 * T - 1, device=dev) if bias else None
    pad = None
    if lengths is not None:
        pad = torch.zeros(B, T, device=dev, dtype=torch.uint8)
        for b, n in enumerate(lengths):
            pad[b, n:] = 1
    if ref_forward:
        out, lse = _ref_out_lse(qkv, gate, tab, pad, B, T, H, 0.125)
    else:
        out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
        lse = torch.empty(B, H, T, device=dev)
        ops.attn_fwd(qkv, gate, tab, pad, out, lse, B, T, H, 0.125)
    dout = bf(torch.randn(B, T, D, device=dev))
    if pad is not None:  # padded query frames carry no gradient in the model
        dout[pad.bool()] = 0
    delta = torch.empty(B, H, T, device=dev)
    dqkv = torch.zeros(B, T, 3 * D, device=dev, dtype=torch.bfloat16)
    dgate = torch.zeros(B, H, T, device=dev) if bias else None
    dtab = torch.zeros(H, 2 * T - 1, device=dev) if bias else None
    if fused:
        dq_acc = torch.zeros(B, T, D, device=dev)
        ops.attn_bwd_fused(qkv, out, dout, gate, tab, pad, lse, delta, dq_acc, dqkv, dgate, dtab, B, T, H, 0.125)
        torch.cuda.synchronize()
        assert dq_acc.abs().max().item() == 0.0
    else:
        ops.attn_bwd(qkv, out, dout, gate, tab, pad, lse, delta, dqkv, dgate, dtab, B, T, H, 0.125)
    torch.cuda.synchronize()
    qr = qkv.float().requires_grad_(True)
    gr = gate.clone().requires_grad_(True) if bias else None
    tr = tab.clone().requires_grad_(True) if bias else None
    _attn_ref(qr, gr, tr, pad, B, T, H, 0.125).backward(dout.float())
    assert torch.isfinite(dqkv.float()).all()
    valid = pad == 0 if pad is not None else torch.ones(B, T, dtype=torch.bool, device=dev)
    err = (dqkv.float() - qr.grad)[valid].abs().max().item()
    assert err < 0.03 * max(1.0, qr.grad.abs().max().item()), err
    if bias:
        vg = valid[:, None, :].expand(B, H, T)
        e1 = (dgate - gr.grad)[vg].abs().max().item()
        assert e1 < 0.03 * max(1.0, gr.grad.abs().max().item()), e1
        e2 = (dtab - tr.grad).abs().max().item()
        assert e2 < 0.03 * max(1.0, tr.grad.abs().max().item()), e2


@pytest.mark.gpu
@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("B,T,H,bias,lengths", [
    (3, 385, 2, True, (385, 129, 300)),   # every utterance but the first padded, one to a single row into its second tile
    (3, 129, 2, True, (129, 1, 100)),     # T one row into a tile; an utterance of one frame
    (2, 385, 2, False, (257, 385)),
    (2, 129, 2, True, None),
])
def test_attn_bwd_ragged_edges(cuda_device, B, T, H, bias, lengths, fused):
    _check_bwd(cuda_device, B, T, H, bias, lengths, fused)


@pytest.mark.gpu
def test_attn_bwd_t4096_bias(cuda_device):
    _check_bwd(cuda_device, 1, 4096, 1, True, (4000,), False, ref_forward=True)
