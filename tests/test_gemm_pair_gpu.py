"""GPU parity tests of the GEMM entry points at layer-sized shapes (many tiles, split-K weight gradients, ragged tails) against
PyTorch fp32 references."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def bf(t):
    return t.to(torch.bfloat16)


@pytest.mark.parametrize("M,K,N", [(3000, 768, 768), (2048, 512, 256), (11984, 768, 2304), (4100, 3072, 768), (2500, 256, 520)])
def test_pair_gemm_rows(cuda_device, M, K, N):
    from unispeech_b200 import _lib as L
    from unispeech_b200 import ops
    torch.manual_seed(M)
    dev = cuda_device
    a = bf(torch.randn(M, K, device=dev))
    w = bf(torch.randn(N, K, device=dev) / K ** 0.5)
    bias = torch.randn(N, device=dev)
    r1 = bf(torch.randn(M, N, device=dev))
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    pre = torch.empty_like(out)
    epi = L.make_epilogue(bias=bias, gelu=True, out_pre=pre, pre_ld=N, res1=r1, res1_ld=N)
    ops.gemm_rows(a, 0, K, M, 1, K, w, N, out, 0, N, epi)
    torch.cuda.synchronize()
    acc = a.float() @ w.float().t() + bias
    assert (pre.float() - acc).abs().max().item() < 0.05
    assert (out.float() - (F.gelu(acc) + r1.float())).abs().max().item() < 0.06
    # dgelu + two residuals + column sums
    aux = bf(torch.randn(M, N, device=dev))
    r2 = bf(torch.randn(M, N, device=dev))
    out2 = torch.empty_like(out)
    colsum = torch.zeros(N, device=dev)
    epi = L.make_epilogue(bias=bias, dgelu=True, gelu_aux=aux, aux_ld=N, res1=r1, res1_ld=N, res2=r2, res2_ld=N, colsum=colsum)
    ops.gemm_rows(a, 0, K, M, 1, K, w, N, out2, 0, N, epi)
    torch.cuda.synchronize()
    x = aux.float().requires_grad_(True)
    g = torch.autograd.grad(F.gelu(x).sum(), x)[0]
    ref2 = acc * g + r1.float() + r2.float()
    assert (out2.float() - ref2).abs().max().item() < 0.08
    assert (colsum - out2.float().sum(0)).abs().max().item() < 0.02 * max(1.0, out2.float().sum(0).abs().max().item())


@pytest.mark.parametrize("C_,k,s,T,B", [(512, 3, 2, 9001, 2), (512, 2, 2, 3000, 3)])
def test_pair_conv_view(cuda_device, C_, k, s, T, B):
    from unispeech_b200 import ops
    torch.manual_seed(T)
    dev = cuda_device
    Tpad = T + (T % 2)
    x = torch.zeros(B, Tpad, C_, device=dev, dtype=torch.bfloat16)
    x[:, :T] = bf(torch.randn(B, T, C_, device=dev))
    w = bf(torch.randn(C_, C_, k, device=dev) / (C_ * k) ** 0.5)
    wk = w.permute(0, 2, 1).contiguous().view(C_, k * C_)
    T_out = (T - k) // s + 1
    out = torch.empty(B, T_out, C_, device=dev, dtype=torch.bfloat16)
    ops.gemm_rows(x, Tpad * C_, s * C_, T_out, B, k * C_, wk, C_, out, T_out * C_, C_, None)
    torch.cuda.synchronize()
    ref = F.conv1d(x[:, :T].float().transpose(1, 2), w.float(), stride=s).transpose(1, 2)
    assert (out.float() - ref).abs().max().item() < 0.04


@pytest.mark.parametrize("rows,B,N,K", [(3000, 1, 768, 512), (2000, 2, 256, 1536), (11984, 1, 2304, 768), (1500, 3, 520, 264)])
def test_pair_wgrad(cuda_device, rows, B, N, K):
    from unispeech_b200 import ops
    torch.manual_seed(rows)
    dev = cuda_device
    y = bf(torch.randn(B, rows, N, device=dev))
    x = bf(torch.randn(B, rows, K, device=dev))
    dw = torch.zeros(N, K, device=dev)
    ops.gemm_wgrad(y, rows * N, N, x, rows * K, K, rows, B, N, K, dw, K)
    torch.cuda.synchronize()
    ref = torch.einsum("brn,brk->nk", y.float(), x.float())
    err = (dw - ref).abs().max().item()
    assert err < 1e-2 * max(1.0, ref.abs().max().item()), err


def test_pair_wgrad_conv_view(cuda_device):
    from unispeech_b200 import ops
    torch.manual_seed(4)
    dev = cuda_device
    C_, k, s, T, B = 512, 3, 2, 4001, 2
    Tpad = T + (T % 2)
    x = torch.zeros(B, Tpad, C_, device=dev, dtype=torch.bfloat16)
    x[:, :T] = bf(torch.randn(B, T, C_, device=dev))
    T_out = (T - k) // s + 1
    dy = bf(torch.randn(B, T_out, C_, device=dev))
    dw = torch.zeros(C_, k * C_, device=dev)
    ops.gemm_wgrad(dy, T_out * C_, C_, x, Tpad * C_, s * C_, T_out, B, C_, k * C_, dw, k * C_)
    torch.cuda.synchronize()
    w = torch.zeros(C_, C_, k, device=dev, requires_grad=True)
    (F.conv1d(x[:, :T].float().transpose(1, 2), w, stride=s) * dy.float().transpose(1, 2)).sum().backward()
    ref = w.grad.permute(0, 2, 1).reshape(C_, k * C_)
    assert (dw - ref).abs().max().item() < 1e-2 * max(1.0, ref.abs().max().item())


@pytest.mark.parametrize("M,K,N", [(3000, 768, 768), (300, 256, 192)])  # many tiles / one tile column
def test_gelu_derivative_modes(cuda_device, M, K, N):
    """gelu = 2: the forward epilogue stores gelu'(pre-activation); dgelu = 2: the backward epilogue multiplies by it."""
    from unispeech_b200 import _lib as L
    from unispeech_b200 import ops
    torch.manual_seed(M + 1)
    dev = cuda_device
    a = bf(torch.randn(M, K, device=dev))
    w = bf(torch.randn(N, K, device=dev) / K ** 0.5)
    bias = torch.randn(N, device=dev)
    out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    grad = torch.empty_like(out)
    ops.gemm_rows(a, 0, K, M, 1, K, w, N, out, 0, N, L.make_epilogue(bias=bias, gelu=2, out_pre=grad, pre_ld=N))
    torch.cuda.synchronize()
    acc = (a.float() @ w.float().t() + bias).requires_grad_(True)
    y = F.gelu(acc)
    g_ref = torch.autograd.grad(y.sum(), acc)[0]
    assert (out.float() - y.detach()).abs().max().item() < 0.05
    assert (grad.float() - g_ref).abs().max().item() < 0.02
    # backward-style GEMM: acc2 * stored derivative + residual, column sums
    r1 = bf(torch.randn(M, N, device=dev))
    out2 = torch.empty_like(out)
    colsum = torch.zeros(N, device=dev)
    ops.gemm_rows(a, 0, K, M, 1, K, w, N, out2, 0, N,
                  L.make_epilogue(dgelu=2, gelu_aux=grad, aux_ld=N, res1=r1, res1_ld=N, colsum=colsum))
    torch.cuda.synchronize()
    ref2 = (a.float() @ w.float().t()) * grad.float() + r1.float()
    assert (out2.float() - ref2).abs().max().item() < 0.08
    assert (colsum - out2.float().sum(0)).abs().max().item() < 0.02 * max(1.0, out2.float().sum(0).abs().max().item())
    # elementwise kernel with a stored derivative
    dy = bf(torch.randn(M, N, device=dev))
    o3 = torch.empty_like(out)
    ops.dgelu_mul(dy, 0, N, grad, 0, N, o3, 0, N, M, 1, N, None, pre_is_grad=True)
    torch.cuda.synchronize()
    assert (o3.float() - dy.float() * grad.float()).abs().max().item() < 0.02


@pytest.mark.parametrize("B,T,K,N,lengths", [(4, 1419, 1024, 1024, [1419, 205, 500, 999]), (3, 700, 768, 3072, [256, 700, 1]),
                                             (2, 1000, 4096, 1024, [999, 1000])])
def test_ragged_gemm_rows_and_wgrad(cuda_device, B, T, K, N, lengths):
    """Ragged batches (BASELINE.json configs[4]): `b200s_gemm_rows_ragged` computes exactly what the dense call computes on every
    M tile that holds a valid row and writes ZEROS on the tiles that start beyond an utterance's valid frames (output and saved
    GELU derivative); `b200s_gemm_wgrad_ragged` equals the weight gradient over the live 64-row blocks."""
    from unispeech_b200 import _lib as L
    from unispeech_b200 import ops
    torch.manual_seed(T + K)
    dev = cuda_device
    a = bf(torch.randn(B, T, K, device=dev))
    w = bf(torch.randn(N, K, device=dev) / K ** 0.5)
    bias = torch.randn(N, device=dev)
    r1 = bf(torch.randn(B, T, N, device=dev))
    valid = torch.tensor(lengths, dtype=torch.int32, device=dev)
    out = torch.full((B, T, N), float("nan"), device=dev, dtype=torch.bfloat16)
    pre = torch.full((B, T, N), float("nan"), device=dev, dtype=torch.bfloat16)
    epi = L.make_epilogue(bias=bias, gelu=2, out_pre=pre, pre_bs=T * N, pre_ld=N, res1=r1, res1_bs=T * N, res1_ld=N)
    ops.gemm_rows(a, T * K, K, T, B, K, w, N, out, T * N, N, epi, valid=valid)
    dense = torch.empty_like(out)
    pre_d = torch.empty_like(out)
    epi_d = L.make_epilogue(bias=bias, gelu=2, out_pre=pre_d, pre_ld=N, res1=r1, res1_ld=N)
    ops.gemm_rows(a, 0, K, B * T, 1, K, w, N, dense.view(B * T, N), 0, N, epi_d)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all() and torch.isfinite(pre.float()).all()   # padded rows stay finite
    for b, n in enumerate(lengths):
        live_rows = min(T, -(-n // 128) * 128)   # M tiles of 128 rows per utterance: every tile that starts below n is computed
        assert (out[b, :live_rows].float() - dense[b, :live_rows].float()).abs().max().item() < 0.03
        assert (pre[b, :live_rows].float() - pre_d[b, :live_rows].float()).abs().max().item() < 0.03
        if live_rows < T:
            assert float(out[b, live_rows:].float().abs().max()) == 0.0 and float(pre[b, live_rows:].float().abs().max()) == 0.0
    # weight gradient: dw[n, k] = sum over live rows of y[b, t, n] x[b, t, k]; rows of a live 64-block beyond `valid` still count
    y = bf(torch.randn(B, T, N, device=dev))
    dw = torch.zeros(N, K, device=dev)
    ops.gemm_wgrad(y, T * N, N, a, T * K, K, T, B, N, K, dw, K, valid=valid)
    torch.cuda.synchronize()
    want = torch.zeros(N, K, device=dev)
    for b, n in enumerate(lengths):
        live = min(T, -(-n // 64) * 64)
        want += y[b, :live].float().t() @ a[b, :live].float()
    scale = want.abs().max().item()
    assert (dw - want).abs().max().item() < 0.01 * scale + 0.05, ((dw - want).abs().max().item(), scale)


def test_reserved_sms_do_not_change_results(cuda_device):
    """`b200s_reserve_sms` is deprecated and has no effect: a caller that still sets it (parallel.configure_overlap) gets the same
    results -- rows GEMM bit-identical, split-K weight gradient equal up to fp32 summation order."""
    from unispeech_b200 import ops
    dev = cuda_device
    torch.manual_seed(12)
    M, K, N = 6000, 1024, 1024
    a = bf(torch.randn(M, K, device=dev))
    w = bf(torch.randn(N, K, device=dev) / K ** 0.5)
    y = bf(torch.randn(M, N, device=dev))
    res = []
    try:
        for keep in (0, 6):
            ops.reserve_sms(keep)
            out = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
            ops.gemm_rows(a, 0, K, M, 1, K, w, N, out, 0, N, None)
            dw = torch.zeros(N, K, device=dev)
            ops.gemm_wgrad(y, 0, N, a, 0, K, M, 1, N, K, dw, K)
            torch.cuda.synchronize()
            res.append((out, dw))
    finally:
        ops.reserve_sms(0)
    assert torch.equal(res[0][0], res[1][0])
    ref = y.float().t() @ a.float()
    for _, dw in res:
        assert (dw - ref).abs().max().item() <= 2e-3 * ref.abs().max().item()
