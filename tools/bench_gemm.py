"""Micro-benchmark of the wgmma GEMM family on the shapes of the WavLM-Base 16 x 15 s step (needs an H100).

    python tools/bench_gemm.py [--reps 20] [--only NAME]
Prints one line per shape: time, TFLOP/s, fraction of the measured bf16 peak.
"""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unispeech_b200 import _lib as L  # noqa: E402
from unispeech_b200 import ops  # noqa: E402

BF = torch.bfloat16


def timeit(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--only", default=None)
    ap.add_argument("--large", action="store_true", help="WavLM-Large 8 x 20 s shapes (7992 rows, D = 1024, F = 4096), layer GEMMs only")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    L.check_device()
    peak = 1386.5
    try:
        peak = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops"]
    except Exception:
        pass
    M = 16 * 749
    cases = []
    # (name, kind, rows, batches, K, N, a_rs, extra)
    for name, K, N in (("qkv", 768, 2304), ("out_proj", 768, 768), ("fc1", 768, 3072), ("fc2", 3072, 768), ("proj", 512, 768),
                       ("qkv_dgrad", 2304, 768)):
        cases.append((name, "rows", M, 1, K, N))
    for name, N, K in (("wgrad_qkv", 2304, 768), ("wgrad_o", 768, 768), ("wgrad_fc1", 3072, 768), ("wgrad_fc2", 768, 3072)):
        cases.append((name, "wgrad", M, 1, K, N))
    for name, T_out, k in (("conv1", 23999, 3), ("conv2", 11999, 3), ("conv3", 5999, 3), ("conv4", 2999, 3), ("conv5", 1499, 2),
                           ("conv6", 749, 2)):
        cases.append((name, "conv", T_out, 16, k * 512, 512))
        cases.append((name + "_wgrad", "convw", T_out, 16, k * 512, 512))
    if args.large:
        M = 8 * 999
        cases = []
        for name, K, N in (("qkv", 1024, 3072), ("out_proj", 1024, 1024), ("fc1", 1024, 4096), ("fc2", 4096, 1024),
                           ("qkv_dgrad", 3072, 1024)):
            cases.append((name, "rows", M, 1, K, N))
        for name, N, K in (("wgrad_qkv", 3072, 1024), ("wgrad_o", 1024, 1024), ("wgrad_fc1", 4096, 1024), ("wgrad_fc2", 1024, 4096)):
            cases.append((name, "wgrad", M, 1, K, N))
    print(f"{'case':14s} {'ms':>8s} {'TFLOP/s':>9s} {'frac':>6s}")
    for name, kind, rows, batches, K, N in cases:
        if args.only and name not in args.only.split(','):
            continue
        flops = 2.0 * rows * batches * K * N
        if kind == "rows":
            a = torch.randn(rows, K, device=dev).to(BF)
            w = torch.randn(N, K, device=dev).to(BF)
            out = torch.empty(rows, N, device=dev, dtype=BF)
            bias = torch.randn(N, device=dev)
            epi = L.make_epilogue(bias=bias)
            fn = lambda: ops.gemm_rows(a, 0, K, rows, 1, K, w, N, out, 0, N, epi)
        elif kind == "wgrad":
            y = torch.randn(rows, N, device=dev).to(BF)
            x = torch.randn(rows, K, device=dev).to(BF)
            dw = torch.zeros(N, K, device=dev)
            fn = lambda: ops.gemm_wgrad(y, 0, N, x, 0, K, rows, 1, N, K, dw, K)
        elif kind == "conv":
            C, k = 512, K // 512
            T_in = 2 * rows + k
            T_in += T_in % 2
            x = torch.randn(batches, T_in, C, device=dev).to(BF)
            w = torch.randn(N, K, device=dev).to(BF)
            out = torch.empty(batches, rows + rows % 2, N, device=dev, dtype=BF)
            pre = torch.empty_like(out)
            epi = L.make_epilogue(gelu=True, out_pre=pre, pre_bs=out.shape[1] * N, pre_ld=N)
            fn = lambda: ops.gemm_rows(x, T_in * C, 2 * C, rows, batches, K, w, N, out, out.shape[1] * N, N, epi)
        else:
            C, k = 512, K // 512
            T_in = 2 * rows + k
            T_in += T_in % 2
            x = torch.randn(batches, T_in, C, device=dev).to(BF)
            dy = torch.randn(batches, rows + 2, C, device=dev).to(BF)
            dw = torch.zeros(C, K, device=dev)
            fn = lambda: ops.gemm_wgrad(dy, (rows + 2) * C, C, x, T_in * C, 2 * C, rows, batches, C, K, dw, K)
        ms = timeit(fn, args.reps)
        tf = flops / (ms * 1e-3) / 1e12
        print(f"{name:14s} {ms:8.4f} {tf:9.1f} {tf / peak:6.3f}")


if __name__ == "__main__":
    main()
