"""GPU parity tests of the persistent 128 x 256 stream-K weight gradient (b200s_gemm_wgrad with K >= 256) against a plain PyTorch
fp32 reference: partial M and N tiles, stream-K ranges that start and end inside tiles (several CTAs per tile and several tiles
per CTA), accumulation onto non-zero dW at a wider row stride, the strided-Conv1d overlapping-row view with per-batch K blocks,
and ragged batches whose valid rows include a zero-length utterance between live ones."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16)


def _check(dw, dw0, ref, K):
    """dw = dw0 + ref on the first K columns; the columns past K (row stride > K) untouched."""
    want = dw0[:, :K] + ref
    scale = max(1.0, ref.abs().max().item())
    err = (dw[:, :K] - want).abs().max().item()
    assert err < 2e-3 * scale, (err, scale)
    assert torch.equal(dw[:, K:], dw0[:, K:])


@pytest.mark.parametrize("rows,B,N,K", [
    (333, 3, 200, 264),      # partial M tile (200 rows of dW) and partial N tile (8 of 256 columns)
    (20000, 1, 128, 256),    # one tile over 313 K blocks: every range starts and ends inside it
    (3000, 2, 1000, 520),    # 8 x 3 tiles over 94 K blocks: ranges of ~17 blocks, a tile split 5-6 ways
    (64, 1, 4096, 2048),     # 256 tiles of one K block: about two tiles per CTA
    (100, 1, 3072, 1024),    # 96 tiles of two K blocks: pieces of one and two blocks
])
def test_wgrad_ws_accumulate(cuda_device, rows, B, N, K):
    from unispeech_b200 import ops
    torch.manual_seed(rows + N + K)
    y = _bf(torch.randn(B, rows, N, device=cuda_device))
    x = _bf(torch.randn(B, rows, K, device=cuda_device))
    ld = K + 8
    dw0 = torch.randn(N, ld, device=cuda_device)
    dw = dw0.clone()
    ops.gemm_wgrad(y, rows * N, N, x, rows * K, K, rows, B, N, K, dw, ld)
    torch.cuda.synchronize()
    _check(dw, dw0, torch.einsum("brn,brk->nk", y.float(), x.float()), K)


@pytest.mark.parametrize("k,s,T,B", [(3, 2, 1001, 3), (2, 2, 700, 2)])
def test_wgrad_ws_conv_view(cuda_device, k, s, T, B):
    """Conv1d(C, C, k, stride s) weight gradient: X read through the overlapping-row view (row stride s * C, k * C columns),
    K blocks iterating over (utterance, 64 output frames)."""
    from unispeech_b200 import ops
    torch.manual_seed(20 + k)
    C_ = 512
    Tpad = T + (T % 2)
    x = torch.zeros(B, Tpad, C_, device=cuda_device, dtype=torch.bfloat16)
    x[:, :T] = _bf(torch.randn(B, T, C_, device=cuda_device))
    T_out = (T - k) // s + 1
    dy = _bf(torch.randn(B, T_out, C_, device=cuda_device))
    dw0 = torch.randn(C_, k * C_, device=cuda_device)
    dw = dw0.clone()
    ops.gemm_wgrad(dy, T_out * C_, C_, x, Tpad * C_, s * C_, T_out, B, C_, k * C_, dw, k * C_)
    torch.cuda.synchronize()
    w = torch.zeros(C_, C_, k, device=cuda_device, requires_grad=True)
    (F.conv1d(x[:, :T].float().transpose(1, 2), w, stride=s) * dy.float().transpose(1, 2)).sum().backward()
    _check(dw, dw0, w.grad.permute(0, 2, 1).reshape(C_, k * C_), k * C_)


@pytest.mark.parametrize("T,N,K,lengths", [(1000, 1024, 1024, [1000, 0, 130, 777]), (700, 3072, 1024, [0, 64, 0, 1]),
                                           (500, 512, 1536, [0, 0, 0])])
def test_wgrad_ws_ragged(cuda_device, T, N, K, lengths):
    """Ragged batch: the 64-row blocks that start at or past an utterance's valid rows are skipped (a zero-length utterance
    contributes nothing); every other block counts in full, including its rows past `valid`."""
    from unispeech_b200 import ops
    torch.manual_seed(T + N)
    B = len(lengths)
    y = _bf(torch.randn(B, T, N, device=cuda_device))
    x = _bf(torch.randn(B, T, K, device=cuda_device))
    valid = torch.tensor(lengths, dtype=torch.int32, device=cuda_device)
    dw0 = torch.randn(N, K, device=cuda_device)
    dw = dw0.clone()
    ops.gemm_wgrad(y, T * N, N, x, T * K, K, T, B, N, K, dw, K, valid=valid)
    torch.cuda.synchronize()
    ref = torch.zeros(N, K, device=cuda_device)
    for b, n in enumerate(lengths):
        live = min(T, -(-n // 64) * 64)
        ref += y[b, :live].float().t() @ x[b, :live].float()
    _check(dw, dw0, ref, K)
