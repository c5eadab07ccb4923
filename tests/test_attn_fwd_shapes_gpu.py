"""Attention forward at the WavLM-Large benchmark shape (B = 2, T = 999, 16 heads) and at a length whose last query tile has
rows only in its first 64 (T % 128 in [1, 64]): there the second consumer warpgroup of the forward kernel computes rows that all
lie beyond T.  Same checks as test_kernels_gpu.py::test_attn_fwd and test_dropout_gpu.py::test_attn_dropout_fwd_bwd (including
the keep bits against the hash, bit for bit), run at these shapes."""
import pytest

import test_dropout_gpu
import test_kernels_gpu

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("B,T,H,bias,padded", [(2, 999, 16, True, True), (2, 999, 16, True, False), (1, 300, 2, True, False)])
def test_attn_fwd_shapes(cuda_device, B, T, H, bias, padded):
    test_kernels_gpu.test_attn_fwd(cuda_device, B, T, H, bias, padded)


@pytest.mark.parametrize("B,T,H,bias,padded,p", [(2, 999, 16, True, True, 0.1), (2, 999, 16, True, False, 0.1),
                                                 (1, 300, 2, True, False, 0.1)])
def test_attn_dropout_fwd_bwd_shapes(cuda_device, B, T, H, bias, padded, p):
    test_dropout_gpu.test_attn_dropout_fwd_bwd(cuda_device, B, T, H, bias, padded, p)
