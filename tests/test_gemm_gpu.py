"""GPU parity tests of the wgmma GEMM family against a plain PyTorch fp32 reference of the same op."""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16)


def _gemm_rows(L, a, a_bs, a_rs, rows, batches, K, w, N, out, out_bs, out_ld, epi=None):
    L.call("b200s_gemm_rows", L.ptr(a), L.ll(a_bs), L.ll(a_rs), C.c_int(rows), C.c_int(batches), C.c_int(K),
           L.ptr(w), C.c_int(N), L.ptr(out), L.ll(out_bs), L.ll(out_ld),
           C.byref(epi) if epi is not None else None, L.stream_ptr())


@pytest.mark.parametrize("M,K,N", [(300, 192, 256), (128, 64, 64), (1000, 768, 384), (77, 128, 72), (513, 512, 2304)])
def test_gemm_rows_plain(cuda_device, M, K, N):
    from unispeech_b200 import _lib as L
    torch.manual_seed(0)
    a = _bf(torch.randn(M, K, device=cuda_device))
    w = _bf(torch.randn(N, K, device=cuda_device) / K ** 0.5)
    out = torch.empty(M, N, device=cuda_device, dtype=torch.bfloat16)
    _gemm_rows(L, a, 0, K, M, 1, K, w, N, out, 0, N)
    ref = a.float() @ w.float().t()
    torch.cuda.synchronize()
    err = (out.float() - ref).abs().max().item()
    assert err < 0.03, err


def test_gemm_rows_epilogues(cuda_device):
    from unispeech_b200 import _lib as L
    torch.manual_seed(1)
    M, K, N = 333, 256, 384
    a = _bf(torch.randn(M, K, device=cuda_device))
    w = _bf(torch.randn(N, K, device=cuda_device) / K ** 0.5)
    bias = torch.randn(N, device=cuda_device)
    r1 = _bf(torch.randn(M, N, device=cuda_device))
    r2 = _bf(torch.randn(M, N, device=cuda_device))
    aux = _bf(torch.randn(M, N, device=cuda_device))
    acc = a.float() @ w.float().t() + bias

    # bias + gelu with pre-activation store + residual
    out = torch.empty(M, N, device=cuda_device, dtype=torch.bfloat16)
    pre = torch.empty_like(out)
    epi = L.make_epilogue(bias=bias, gelu=True, out_pre=pre, pre_ld=N, res1=r1, res1_ld=N)
    _gemm_rows(L, a, 0, K, M, 1, K, w, N, out, 0, N, epi)
    torch.cuda.synchronize()
    assert (pre.float() - acc).abs().max().item() < 0.03
    ref = F.gelu(acc) + r1.float()
    assert (out.float() - ref).abs().max().item() < 0.04

    # bias + dgelu + two residuals + column sums
    out2 = torch.empty(M, N, device=cuda_device, dtype=torch.bfloat16)
    colsum = torch.zeros(N, device=cuda_device)
    epi = L.make_epilogue(bias=bias, dgelu=True, gelu_aux=aux, aux_ld=N, res1=r1, res1_ld=N, res2=r2, res2_ld=N,
                          colsum=colsum)
    _gemm_rows(L, a, 0, K, M, 1, K, w, N, out2, 0, N, epi)
    torch.cuda.synchronize()
    x = aux.float().requires_grad_(True)
    g = torch.autograd.grad(F.gelu(x).sum(), x)[0]
    ref2 = acc * g + r1.float() + r2.float()
    assert (out2.float() - ref2).abs().max().item() < 0.06
    assert (colsum - out2.float().sum(0)).abs().max().item() < 0.05


@pytest.mark.parametrize("C_,k,s,T,B", [(64, 3, 2, 101, 3), (64, 2, 2, 300, 2), (512, 3, 2, 1001, 2)])
def test_gemm_rows_conv_view(cuda_device, C_, k, s, T, B):
    """Strided Conv1d on channels-last activations as an overlapping-row GEMM view."""
    from unispeech_b200 import _lib as L
    torch.manual_seed(2)
    Tpad = T + (T % 2)  # keep the batch stride a multiple of the row stride
    x = torch.zeros(B, Tpad, C_, device=cuda_device, dtype=torch.bfloat16)
    x[:, :T] = _bf(torch.randn(B, T, C_, device=cuda_device))
    w = _bf(torch.randn(C_, C_, k, device=cuda_device) / (C_ * k) ** 0.5)  # [co, ci, k] reference layout
    wk = w.permute(0, 2, 1).contiguous().view(C_, k * C_)                  # [co, (j, ci)]
    T_out = (T - k) // s + 1
    out = torch.empty(B, T_out, C_, device=cuda_device, dtype=torch.bfloat16)
    _gemm_rows(L, x, Tpad * C_, s * C_, T_out, B, k * C_, wk, C_, out, T_out * C_, C_)
    torch.cuda.synchronize()
    ref = F.conv1d(x[:, :T].float().transpose(1, 2), w.float(), stride=s).transpose(1, 2)
    assert (out.float() - ref).abs().max().item() < 0.03


@pytest.mark.parametrize("rows,B,N,K", [(200, 1, 256, 128), (333, 3, 384, 192), (1000, 2, 64, 64), (70, 2, 72, 136)])
def test_gemm_wgrad(cuda_device, rows, B, N, K):
    from unispeech_b200 import _lib as L
    torch.manual_seed(3)
    y = _bf(torch.randn(B, rows, N, device=cuda_device))
    x = _bf(torch.randn(B, rows, K, device=cuda_device))
    dw = torch.zeros(N, K, device=cuda_device)
    L.call("b200s_gemm_wgrad", L.ptr(y), L.ll(rows * N), L.ll(N), L.ptr(x), L.ll(rows * K), L.ll(K),
           C.c_int(rows), C.c_int(B), C.c_int(N), C.c_int(K), L.ptr(dw), L.ll(K), L.stream_ptr())
    torch.cuda.synchronize()
    ref = torch.einsum("brn,brk->nk", y.float(), x.float())
    err = (dw - ref).abs().max().item()
    assert err < 1e-2 * max(1.0, ref.abs().max().item()), err


def test_gemm_wgrad_conv_view(cuda_device):
    from unispeech_b200 import _lib as L
    torch.manual_seed(4)
    C_, k, s, T, B = 64, 3, 2, 201, 2
    Tpad = T + (T % 2)
    x = torch.zeros(B, Tpad, C_, device=cuda_device, dtype=torch.bfloat16)
    x[:, :T] = _bf(torch.randn(B, T, C_, device=cuda_device))
    T_out = (T - k) // s + 1
    dy = _bf(torch.randn(B, T_out, C_, device=cuda_device))
    dw = torch.zeros(C_, k * C_, device=cuda_device)
    L.call("b200s_gemm_wgrad", L.ptr(dy), L.ll(T_out * C_), L.ll(C_), L.ptr(x), L.ll(Tpad * C_), L.ll(s * C_),
           C.c_int(T_out), C.c_int(B), C.c_int(C_), C.c_int(k * C_), L.ptr(dw), L.ll(k * C_), L.stream_ptr())
    torch.cuda.synchronize()
    xw = x[:, :T].float().transpose(1, 2).requires_grad_(False)
    w = torch.zeros(C_, C_, k, device=cuda_device, requires_grad=True)
    (F.conv1d(xw, w, stride=s) * dy.float().transpose(1, 2)).sum().backward()
    ref = w.grad.permute(0, 2, 1).reshape(C_, k * C_)
    assert (dw - ref).abs().max().item() < 1e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("D,G,T,B", [(128, 16, 70, 2), (768, 16, 200, 2), (1024, 16, 150, 1)])
def test_posconv(cuda_device, D, G, T, B):
    from unispeech_b200 import _lib as L
    torch.manual_seed(5)
    taps, Cg = 128, D // G
    x = _bf(torch.randn(B, T, D, device=cuda_device))
    w = _bf(torch.randn(D, Cg, taps, device=cuda_device) / (Cg * taps) ** 0.5)  # reference Conv1d layout
    bias = torch.randn(D, device=cuda_device)
    Tp = T + 128
    xpad = torch.zeros(B, Tp, D, device=cuda_device, dtype=torch.bfloat16)
    xpad[:, 64:64 + T] = x
    wp = torch.zeros(G, 64, taps, 64, device=cuda_device, dtype=torch.bfloat16)
    wp[:, :Cg, :, :Cg] = w.view(G, Cg, Cg, taps).permute(0, 1, 3, 2)
    out = torch.empty(B, T, D, device=cuda_device, dtype=torch.bfloat16)
    pre = torch.empty_like(out)
    x_res = xpad[:, 64:]
    epi = L.make_epilogue(bias=bias, gelu=True, out_pre=pre, pre_bs=T * D, pre_ld=D, res1=x_res, res1_bs=Tp * D,
                          res1_ld=D)
    L.call("b200s_posconv_gemm", L.ptr(xpad), L.ll(Tp * D), C.c_int(T), C.c_int(B), C.c_int(D), C.c_int(G),
           C.c_int(taps), L.ptr(wp), L.ptr(out), L.ll(T * D), L.ll(D), C.byref(epi), L.stream_ptr())
    torch.cuda.synchronize()
    conv = F.conv1d(x.float().transpose(1, 2), w.float(), bias, padding=64, groups=G)[:, :, :-1].transpose(1, 2)
    assert (pre.float() - conv).abs().max().item() < 0.05
    ref = F.gelu(conv) + x.float()
    assert (out.float() - ref).abs().max().item() < 0.05

    # weight gradient
    dy = _bf(torch.randn(B, T, D, device=cuda_device))
    dwp = torch.zeros(G, Cg, taps, 64, device=cuda_device)
    L.call("b200s_posconv_wgrad", L.ptr(dy), L.ll(T * D), L.ll(D), L.ptr(xpad), L.ll(Tp * D), C.c_int(T), C.c_int(B),
           C.c_int(D), C.c_int(G), C.c_int(taps), L.ptr(dwp), L.stream_ptr())
    torch.cuda.synchronize()
    wf = w.float().clone().requires_grad_(True)
    (F.conv1d(x.float().transpose(1, 2), wf, None, padding=64, groups=G)[:, :, :-1] * dy.float().transpose(1, 2)).sum().backward()
    ref_dw = wf.grad.view(G, Cg, Cg, taps).permute(0, 1, 3, 2)  # [g, co, j, ci]
    got = dwp[:, :, :, :Cg]
    assert (got - ref_dw).abs().max().item() < 1e-2 * max(1.0, ref_dw.abs().max().item())
