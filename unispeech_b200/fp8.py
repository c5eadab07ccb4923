"""Reference of the e4m3 quantisation rule of the fp8 inference path (csrc/fp8.cuh), in torch on any device.

One scale per row, amax = max |x| of the row in fp32:  q = e4m3(x * (448 / amax)) (round to nearest even),  s = amax / 448;
amax < 2^-119 (zero rows included) gives q = 0, s = 0.  |x * 448 / amax| never reaches 464, where torch's cast would give NaN
instead of saturating, so this is bit-exact against the kernels (`extract_features(fp8=True)`, tests/test_fp8_*.py).
"""
from __future__ import annotations

import torch

E4M3_MAX = 448.0
# rows with a smaller amax count as zero: 448 / amax would overflow fp32 below about 1.3e-36
MIN_AMAX = 2.0 ** -119


def quantize_rows_reference(x: torch.Tensor):
    """x: [..., K] (bf16 values are quantised from their bf16 value).  Returns (q float8_e4m3fn [..., K], s fp32 [...])."""
    xf = x.float()
    amax = xf.abs().amax(-1)
    c = torch.full_like(amax, E4M3_MAX)
    live = amax >= MIN_AMAX
    # tensor / tensor: an IEEE division on every device (torch turns a division by or of a Python number into a multiplication
    # by a reciprocal, which can differ in the last bit)
    rinv = torch.where(live, c / torch.where(live, amax, c), torch.zeros_like(amax))
    q = (xf * rinv.unsqueeze(-1)).to(torch.float8_e4m3fn)
    return q, torch.where(live, amax / c, torch.zeros_like(amax))


def dequantize_rows(q: torch.Tensor, s: torch.Tensor, dtype=torch.float64) -> torch.Tensor:
    return q.to(dtype) * s.to(dtype).unsqueeze(-1)
