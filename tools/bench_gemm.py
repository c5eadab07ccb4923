"""Micro-benchmark of the wgmma GEMM family (needs an H100).

    python tools/bench_gemm.py [--reps 20] [--only NAME] [--large]
Default: the shapes of the WavLM-Base 16 x 15 s step.  --large: every b200s_gemm_rows call of one WavLM-Large 8 x 20 s training
step (pre-LN encoder, conv stack in layer_norm mode), each with the epilogue the engine passes, then every b200s_gemm_wgrad call of
the same step with the views the engine passes.
Prints one line per shape: time, algorithmic TFLOP/s, fraction of the bf16 peak and, for --large, the shape's FLOP-weighted share
of its family in one step.  Each --large shape is checked once against an fp32 torch reference.
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

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


def load_peak():
    try:
        return json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["bf16_tflops_sustained"], \
            "MEASURED_PEAKS.json bf16_tflops_sustained"
    except (OSError, KeyError, ValueError):
        return 989.0, "H100 SXM data sheet (989, dense bf16)"


def _even(n):
    return n + (n & 1)


def large_rows_cases():
    """(name, calls per step, rows, batches, K, N, a_rs, a_bs, out_ld, out_bs, out_off, epilogue kinds) of every gemm_rows
    call of one WavLM-Large 8 x 20 s step.  Strides in elements; a_bs / out_bs = 0 for a single batch."""
    B, T, D, Fd, C, layers = 8, 999, 1024, 4096, 512, 24
    M = B * T
    cases = [
        ("qkv", layers, M, 1, D, 3 * D, D, 0, 3 * D, 0, 0, ("bias",)),
        ("out_proj", layers, M, 1, D, D, D, 0, D, 0, 0, ("bias", "res1")),
        ("fc1", layers, M, 1, D, Fd, D, 0, Fd, 0, 0, ("bias", "gelu2")),
        ("fc2", layers, M, 1, Fd, D, Fd, 0, D, 0, 0, ("bias", "res1")),
        ("fc2_dgrad", layers, M, 1, D, Fd, D, 0, Fd, 0, 0, ("dgelu2", "colsum")),
        ("fc1_dgrad", layers, M, 1, Fd, D, Fd, 0, D, 0, 0, ("res1",)),
        ("out_proj_dgrad", layers, M, 1, D, D, D, 0, D, 0, 0, ()),
        ("qkv_dgrad", layers, M, 1, 3 * D, D, 3 * D, 0, D, 0, 0, ("res1", "res2")),
        ("proj", 1, T, B, C, D, C, T * C, D, T * D, 0, ("bias",)),
        ("proj_dgrad", 1, T, B, D, C, D, T * D, C, T * C, 0, ()),
    ]
    convs = [(C, 10, 5)] + [(C, 3, 2)] * 4 + [(C, 2, 2)] * 2
    L_ = 20 * 16000
    Ts, t = [], L_
    for (_, k, s) in convs:
        t = (t - k) // s + 1
        Ts.append(t)
    Tp = [_even(t) for t in Ts]
    for i in range(1, len(convs)):
        _, k, s = convs[i]
        cases.append((f"conv{i}", 1, Ts[i], B, k * C, C, s * C, Tp[i - 1] * C, C, Tp[i] * C, 0, ()))
    for i in range(len(convs) - 1, 0, -1):
        _, k, s = convs[i]
        lead = (k + s - 1) // s - 1
        Tg = _even((Ts[i - 1] + s - 1) // s + lead + 1)
        for rho in range(min(s, k)):
            nm = (k - rho + s - 1) // s
            n_u = (Ts[i - 1] - rho + s - 1) // s
            cases.append((f"conv{i}_dgrad_p{rho}", 1, n_u, B, nm * C, C, C, Tg * C, s * C, Tp[i - 1] * C, rho * C, ()))
    return cases


def large_wgrad_cases():
    """(name, calls per step, rows, batches, N, K, y_rs, y_bs, y_off, x_rs, x_bs) of every b200s_gemm_wgrad call of one WavLM-Large
    8 x 20 s step, with the views the engine passes: the layer GEMMs over all B*T frames, conv1-6 per utterance with X read through
    the overlapping-row view (row stride s*C) and dY from the lead-row gradient buffer, post_extract_proj per utterance."""
    B, T, D, Fd, C, layers = 8, 999, 1024, 4096, 512, 24
    M = B * T
    cases = [
        ("qkv", layers, M, 1, 3 * D, D, 3 * D, 0, 0, D, 0),
        ("out_proj", layers, M, 1, D, D, D, 0, 0, D, 0),
        ("fc1", layers, M, 1, Fd, D, Fd, 0, 0, D, 0),
        ("fc2", layers, M, 1, D, Fd, D, 0, 0, Fd, 0),
        ("post_extract_proj", 1, T, B, D, C, D, T * D, 0, C, T * C),
    ]
    convs = [(C, 10, 5)] + [(C, 3, 2)] * 4 + [(C, 2, 2)] * 2
    Ts, t = [], 20 * 16000
    for (_, k, s) in convs:
        t = (t - k) // s + 1
        Ts.append(t)
    Tp = [_even(t) for t in Ts]
    for i in range(1, len(convs)):
        _, k, s = convs[i]
        lead = (k + s - 1) // s - 1
        Tg = _even((Ts[i - 1] + s - 1) // s + lead + 1)
        cases.append((f"conv{i}", 1, Ts[i], B, C, k * C, C, Tg * C, lead * C, s * C, Tp[i - 1] * C))
    return cases


def run_large_wgrad(args, dev, peak):
    cases = large_wgrad_cases()
    total = sum(n * 2.0 * rows * b * N * K for (_, n, rows, b, N, K, *_r) in cases)
    print(f"gemm_wgrad family, one WavLM-Large 8 x 20 s step: {total / 1e12:.2f} TFLOP")
    print(f"{'case':18s} {'calls':>5s} {'rows':>7s} {'N':>5s} {'K':>5s} {'ms':>8s} {'TFLOP/s':>8s} {'frac':>6s} {'share':>6s} "
          f"{'rel_err':>8s}")
    fam_ms = 0.0
    for name, n, rows, b, N, K, y_rs, y_bs, y_off, x_rs, x_bs in cases:
        if args.only and name not in args.only.split(','):
            continue
        torch.manual_seed(0)
        y_elems = y_off + ((b - 1) * y_bs if b > 1 else 0) + (rows - 1) * y_rs + N
        x_elems = ((b - 1) * x_bs if b > 1 else 0) + (rows - 1) * x_rs + K
        y = torch.randn(y_elems, device=dev).to(BF)
        x = torch.randn(x_elems, device=dev).to(BF)
        yv = y[y_off:]
        dw = torch.zeros(N, K, device=dev)
        fn = lambda: ops.gemm_wgrad(yv, y_bs, y_rs, x, x_bs, x_rs, rows, b, N, K, dw, K)  # noqa: E731
        # one checked call (onto zeros), then the timed ones (accumulating)
        fn()
        torch.cuda.synchronize()
        ref = torch.zeros(N, K, device=dev)
        for bb in range(b):
            ref += y.as_strided((rows, N), (y_rs, 1), y_off + bb * y_bs).float().t() @ \
                x.as_strided((rows, K), (x_rs, 1), bb * x_bs).float()
        err = ((dw - ref).abs().max() / ref.abs().max()).item()
        del ref
        ms = timeit(fn, args.reps)
        flops = 2.0 * rows * b * N * K
        tf = flops / (ms * 1e-3) / 1e12
        fam_ms += n * ms
        print(f"{name:18s} {n:5d} {rows * b:7d} {N:5d} {K:5d} {ms:8.4f} {tf:8.1f} {tf / peak:6.3f} {n * flops / total:6.3f} "
              f"{err:8.1e}", flush=True)
        del y, x, yv, dw
        torch.cuda.empty_cache()
    if not args.only:
        print(f"family: {fam_ms:.2f} ms per step, {total / (fam_ms * 1e-3) / 1e12:.1f} TFLOP/s "
              f"({total / (fam_ms * 1e-3) / 1e12 / peak:.3f} of peak)")


def run_large_rows(args, dev, peak):
    cases = large_rows_cases()
    total = sum(n * 2.0 * rows * b * K * N for (_, n, rows, b, K, N, *_r) in cases)
    print(f"gemm_rows family, one WavLM-Large 8 x 20 s step: {total / 1e12:.2f} TFLOP")
    print(f"{'case':18s} {'calls':>5s} {'rows':>7s} {'K':>5s} {'N':>5s} {'ms':>8s} {'TFLOP/s':>8s} {'frac':>6s} {'share':>6s} "
          f"{'max_err':>8s}  epilogue")
    fam_ms = 0.0
    for name, n, rows, b, K, N, a_rs, a_bs, out_ld, out_bs, out_off, kinds in cases:
        if args.only and name not in args.only.split(','):
            continue
        torch.manual_seed(0)
        a_elems = (b - 1) * a_bs + (rows - 1) * a_rs + K if b > 1 else (rows - 1) * a_rs + K
        x = (torch.randn(a_elems, device=dev) * 0.5).to(BF)
        w = (torch.randn(N, K, device=dev) / K ** 0.5).to(BF)
        o_elems = out_off + ((b - 1) * out_bs if b > 1 else 0) + (rows - 1) * out_ld + N
        out = torch.zeros(o_elems, device=dev, dtype=BF)
        ovw = out[out_off:]
        kw, t_bs = {}, rows * N  # epilogue tensors are dense [b, rows, N]
        ep = {}
        if "bias" in kinds:
            ep["bias"] = kw["bias"] = torch.randn(N, device=dev)
        for r in ("res1", "res2"):
            if r in kinds:
                ep[r] = kw[r] = torch.randn(b, rows, N, device=dev).to(BF)
                kw[r + "_ld"], kw[r + "_bs"] = N, t_bs
        if "gelu2" in kinds:
            ep["pre"] = kw["out_pre"] = torch.empty(b, rows, N, device=dev, dtype=BF)
            kw.update(gelu=2, pre_ld=N, pre_bs=t_bs)
        if "dgelu2" in kinds:
            ep["aux"] = kw["gelu_aux"] = torch.rand(b, rows, N, device=dev).to(BF)
            kw.update(dgelu=2, aux_ld=N, aux_bs=t_bs)
        if "colsum" in kinds:
            ep["colsum"] = kw["colsum"] = torch.zeros(N, device=dev)
        epi = L.make_epilogue(**kw) if kw else None
        fn = lambda: ops.gemm_rows(x, a_bs, a_rs, rows, b, K, w, N, ovw, out_bs, out_ld, epi)  # noqa: E731
        # one checked call, then the timed ones
        fn()
        torch.cuda.synchronize()
        err = 0.0
        for bb in sorted({0, b - 1}):
            av = x.as_strided((rows, K), (a_rs, 1), bb * a_bs).float()
            acc = av @ w.float().t()
            if "bias" in ep:
                acc = acc + ep["bias"]
            if "pre" in ep:
                xg = acc.clone().requires_grad_(True)
                g = torch.autograd.grad(F.gelu(xg).sum(), xg)[0]
                err = max(err, (ep["pre"][bb].float() - g).abs().max().item())
                acc = F.gelu(acc)
            if "aux" in ep:
                acc = acc * ep["aux"][bb].float()
            for r in ("res1", "res2"):
                if r in ep:
                    acc = acc + ep[r][bb].float()
            got = out.as_strided((rows, N), (out_ld, 1), out_off + bb * out_bs).float()
            err = max(err, ((got - acc).abs() / (1.0 + acc.abs())).max().item())
            del av, acc, got
        if "colsum" in ep:
            full = out[:rows * N].view(rows, N).float().sum(0)
            err = max(err, ((ep["colsum"] - full).abs() / (1.0 + full.abs())).max().item())
        ms = timeit(fn, args.reps)
        flops = 2.0 * rows * b * K * N
        tf = flops / (ms * 1e-3) / 1e12
        fam_ms += n * ms
        print(f"{name:18s} {n:5d} {rows * b:7d} {K:5d} {N:5d} {ms:8.4f} {tf:8.1f} {tf / peak:6.3f} {n * flops / total:6.3f} "
              f"{err:8.4f}  {'+'.join(kinds) or '-'}", flush=True)
        del x, w, out, ovw, kw, ep, epi
        torch.cuda.empty_cache()
    if not args.only:
        print(f"family: {fam_ms:.2f} ms per step, {total / (fam_ms * 1e-3) / 1e12:.1f} TFLOP/s "
              f"({total / (fam_ms * 1e-3) / 1e12 / peak:.3f} of peak)")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--only", default=None)
    ap.add_argument("--large", action="store_true", help="WavLM-Large 8 x 20 s step: every gemm_rows call, then the layer wgrads")
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    L.check_device()
    peak, src = load_peak()
    print(f"peak: {peak} TFLOP/s ({src}); GPU: {torch.cuda.get_device_name(0)}")
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
        run_large_rows(args, dev, peak)
        run_large_wgrad(args, dev, peak)
        return
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
