"""GPU parity tests of the persistent 128 x 256 row GEMM (b200s_gemm_rows with N >= 256) against a plain PyTorch fp32
reference: every fused epilogue the model engine passes, partial M and N tiles, more tiles than SMs, the strided-Conv1d
overlapping-row view with a strided output; and a ragged batch at the same widths, which the row GEMM hands to the tiled kernel."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _bf(t):
    return t.to(torch.bfloat16)


def _dgelu(x):
    x = x.float().requires_grad_(True)
    return torch.autograd.grad(F.gelu(x).sum(), x)[0]


def _operands(dev, M, K, N, seed):
    torch.manual_seed(seed)
    a = _bf(torch.randn(M, K, device=dev))
    w = _bf(torch.randn(N, K, device=dev) / K ** 0.5)
    return a, w, a.float() @ w.float().t()


# (name, epilogue) pairs of the layer GEMMs: forward qkv / out_proj / fc1 / fc2, input gradients fc2 / fc1 / out_proj / qkv
EPILOGUES = ["bias", "bias_res1", "bias_gelu_grad", "bias_gelu_pre", "dgelu_grad_colsum", "dgelu_colsum", "res1", "none",
             "res1_res2"]


@pytest.mark.parametrize("M,K,N", [(1000, 256, 640), (333, 192, 264), (128, 128, 1024)])
@pytest.mark.parametrize("kind", EPILOGUES)
def test_gemm_ws_epilogues(cuda_device, M, K, N, kind):
    from unispeech_b200 import _lib as L
    from unispeech_b200 import ops
    a, w, acc = _operands(cuda_device, M, K, N, 10)
    bias = torch.randn(N, device=cuda_device)
    r1 = _bf(torch.randn(M, N, device=cuda_device))
    r2 = _bf(torch.randn(M, N, device=cuda_device))
    aux = _bf(torch.randn(M, N, device=cuda_device))
    out = torch.full((M, N), float("nan"), device=cuda_device, dtype=torch.bfloat16)
    pre = torch.full_like(out, float("nan"))
    colsum = torch.zeros(N, device=cuda_device)
    kw, ref, ref_pre, tol = {}, acc, None, 0.03
    if kind.startswith("bias"):
        kw["bias"] = bias
        ref = acc + bias
    if kind == "bias_res1":
        kw.update(res1=r1, res1_ld=N)
        ref, tol = ref + r1.float(), 0.04
    elif kind == "bias_gelu_grad":
        kw.update(gelu=2, out_pre=pre, pre_ld=N)
        ref_pre, ref = _dgelu(ref), F.gelu(ref)
    elif kind == "bias_gelu_pre":
        kw.update(gelu=True, out_pre=pre, pre_ld=N)
        ref_pre, ref = ref, F.gelu(ref)
    elif kind == "dgelu_grad_colsum":
        g = _dgelu(aux)
        auxg = _bf(g)  # what a gelu=2 forward stored
        kw.update(dgelu=2, gelu_aux=auxg, aux_ld=N, colsum=colsum)
        ref = acc * auxg.float()
    elif kind == "dgelu_colsum":
        kw.update(dgelu=True, gelu_aux=aux, aux_ld=N, colsum=colsum)
        ref = acc * _dgelu(aux)
    elif kind == "res1":
        kw.update(res1=r1, res1_ld=N)
        ref, tol = acc + r1.float(), 0.04
    elif kind == "res1_res2":
        kw.update(res1=r1, res1_ld=N, res2=r2, res2_ld=N)
        ref, tol = acc + r1.float() + r2.float(), 0.06
    ops.gemm_rows(a, 0, K, M, 1, K, w, N, out, 0, N, L.make_epilogue(**kw) if kw else None)
    torch.cuda.synchronize()
    assert (out.float() - ref).abs().max().item() < tol
    if ref_pre is not None:
        assert (pre.float() - ref_pre).abs().max().item() < 0.03
    if "colsum" in kind:
        assert (colsum - out.float().sum(0)).abs().max().item() < 0.05


def test_gemm_ws_persistent_wrap(cuda_device):
    """8000 x 2048: 63 x 8 tiles, several per CTA, with the out_proj / fc2 epilogue."""
    from unispeech_b200 import _lib as L
    from unispeech_b200 import ops
    M, K, N = 8000, 512, 2048
    a, w, acc = _operands(cuda_device, M, K, N, 11)
    bias = torch.randn(N, device=cuda_device)
    r1 = _bf(torch.randn(M, N, device=cuda_device))
    out = torch.empty(M, N, device=cuda_device, dtype=torch.bfloat16)
    ops.gemm_rows(a, 0, K, M, 1, K, w, N, out, 0, N, L.make_epilogue(bias=bias, res1=r1, res1_ld=N))
    torch.cuda.synchronize()
    assert (out.float() - (acc + bias + r1.float())).abs().max().item() < 0.04


@pytest.mark.parametrize("k,s,T,B", [(3, 2, 1001, 2), (2, 2, 700, 3)])
def test_gemm_ws_conv_view_strided_out(cuda_device, k, s, T, B):
    """Conv1d(C, C, k, stride s) as the overlapping-row view, written into every s-th row of a wider buffer at a row offset
    (the layout of the conv input-gradient phase GEMMs)."""
    from unispeech_b200 import ops
    torch.manual_seed(12)
    C_ = 512
    Tpad = T + (T % 2)
    x = torch.zeros(B, Tpad, C_, device=cuda_device, dtype=torch.bfloat16)
    x[:, :T] = _bf(torch.randn(B, T, C_, device=cuda_device))
    wt = _bf(torch.randn(C_, C_, k, device=cuda_device) / (C_ * k) ** 0.5)
    wk = wt.permute(0, 2, 1).contiguous().view(C_, k * C_)
    T_out = (T - k) // s + 1
    R = s * T_out + 2
    dst = torch.full((B, R, C_), 7.0, device=cuda_device, dtype=torch.bfloat16)
    rho = 1
    ops.gemm_rows(x, Tpad * C_, s * C_, T_out, B, k * C_, wk, C_, dst.view(-1)[rho * C_:], R * C_, s * C_)
    torch.cuda.synchronize()
    ref = F.conv1d(x[:, :T].float().transpose(1, 2), wt.float(), stride=s).transpose(1, 2)
    got = dst[:, rho:rho + s * T_out:s]
    assert (got.float() - ref).abs().max().item() < 0.03
    untouched = torch.ones(R, dtype=torch.bool, device=cuda_device)
    untouched[rho:rho + s * T_out:s] = False
    assert bool((dst[:, untouched] == 7.0).all())


def test_gemm_ws_ragged(cuda_device):
    """A ragged row GEMM with N >= 256 (routed to the tiled kernel): dead M tiles (at or past an utterance's valid rows; here
    whole utterances between live ones) are written as zeros, in the output and in the pre-activation output; live tiles are
    computed in full."""
    from unispeech_b200 import _lib as L
    from unispeech_b200 import ops
    torch.manual_seed(13)
    T, B, K, N = 1000, 4, 256, 1024
    a = _bf(torch.randn(B, T, K, device=cuda_device))
    w = _bf(torch.randn(N, K, device=cuda_device) / K ** 0.5)
    bias = torch.randn(N, device=cuda_device)
    valid = torch.tensor([1000, 300, 0, 777], dtype=torch.int32, device=cuda_device)
    out = torch.full((B, T, N), float("nan"), device=cuda_device, dtype=torch.bfloat16)
    pre = torch.full_like(out, float("nan"))
    epi = L.make_epilogue(bias=bias, gelu=2, out_pre=pre, pre_bs=T * N, pre_ld=N)
    ops.gemm_rows(a, T * K, K, T, B, K, w, N, out, T * N, N, epi, valid=valid)
    torch.cuda.synchronize()
    acc = a.float() @ w.float().t() + bias
    for b, v in enumerate(valid.tolist()):
        live = min(((v + 127) // 128) * 128, T)  # rows of the tiles that start below v
        if live:
            assert (out[b, :live].float() - F.gelu(acc[b, :live])).abs().max().item() < 0.03
            assert (pre[b, :live].float() - _dgelu(acc[b, :live])).abs().max().item() < 0.03
        assert bool((out[b, live:] == 0).all()) and bool((pre[b, live:] == 0).all())
