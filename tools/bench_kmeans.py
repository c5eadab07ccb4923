"""K-means on the GPU: the library's kernels against the reference recipe's formulas.

  assignment  b200s_kmeans_assign vs dump_km_label.py's ApplyKmeans in torch (|x|^2 - 2 x C^T + |C|^2, argmin), fp32 and bf16
              matmul, at N = 4 M / 16 M rows, D = 768 / 1024, K = 500 / 1000.  The torch arms run in 1 M-row chunks (the [N, K]
              distance matrix of 16 M rows does not fit in memory).  TFLOP/s from 2 N K D; share of the 989 TFLOP/s dense BF16
              figure of the H100 SXM data sheet.
  update      b200s_kmeans_update (counting sort + fixed-order sums) and the centre finalisation: ms and GB/s of one read of X.
  fit         KMeans(500).fit on 2 M x 768 rows, 20 Lloyd iterations (+ k-means++ on 30 000 rows), and scikit-learn's
              MiniBatchKMeans with the recipe's settings (learn_kmeans.py) on the host CPU for orientation.
CUDA events after a warm-up; the arms alternate.  GPU only.

    python tools/bench_kmeans.py [--quick] [--sklearn-rows N]
"""
import argparse
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from unispeech_b200 import ops  # noqa: E402
from unispeech_b200.kmeans import KMeans  # noqa: E402

PEAK_TFLOPS = 989.0   # H100 SXM, dense BF16, data sheet
CHUNK = 1 << 20


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return name, pl


def timed(fn, reps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def rand_rows(N, D, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.empty(N, D, dtype=torch.bfloat16, device="cuda")
    for i in range(0, N, CHUNK):
        x[i:i + CHUNK] = torch.randn(min(CHUNK, N - i), D, generator=g, device="cuda").to(torch.bfloat16)
    return x


def apply_kmeans(x, C, Cnorm, dtype, out):
    """dump_km_label.py ApplyKmeans.__call__ on chunks of rows."""
    Ct = C.t().to(dtype)
    for i in range(0, x.shape[0], CHUNK):
        xc = x[i:i + CHUNK].to(dtype)
        dist = xc.float().pow(2).sum(1, keepdim=True) - 2 * torch.matmul(xc, Ct).float() + Cnorm
        out[i:i + CHUNK] = dist.argmin(dim=1)


def bench_assign(quick):
    rows = (4 << 20,) if quick else (4 << 20, 16 << 20)
    print("\n## assignment (ms; TFLOP/s = 2 N K D / time; % of 989)")
    print("| N | D | K | kernel ms | TFLOP/s | % peak | torch fp32 ms | torch bf16 ms | labels = bf16 arm |")
    print("|---|---|---|---|---|---|---|---|---|")
    for D in (768, 1024):
        x = rand_rows(max(rows), D, D)
        for K in (500, 1000):
            C = torch.randn(K, D, device="cuda")
            km = KMeans.from_centers(C.cpu())
            cbf, cn = km._device_centers(x.device)
            Cb = cbf[:K].float()
            Cnorm = (Cb * Cb).sum(1)[None]
            for N in rows:
                xs = x[:N]
                lab = torch.empty(N, dtype=torch.int32, device="cuda")
                ref = torch.empty(N, dtype=torch.int64, device="cuda")
                kern = lambda: ops.kmeans_assign(xs, 0, D, N, 1, D, None, cbf, cn, K, lab)  # noqa: E731
                t32 = lambda: apply_kmeans(xs, Cb, Cnorm, torch.float32, ref)  # noqa: E731
                t16 = lambda: apply_kmeans(xs, Cb, Cnorm, torch.bfloat16, ref)  # noqa: E731
                for f in (kern, t32, t16):
                    f()
                reps = 10 if N <= (4 << 20) else 4
                ms_k, ms_32, ms_16 = [], [], []
                for _ in range(2):
                    ms_k.append(timed(kern, reps))
                    ms_32.append(timed(t32, max(1, reps // 4)))
                    ms_16.append(timed(t16, max(1, reps // 4)))
                mk, m32, m16 = min(ms_k), min(ms_32), min(ms_16)
                agree = float((lab.long() == ref).double().mean())
                tf = 2.0 * N * K * D / (mk * 1e-3) / 1e12
                print(f"| {N >> 20} M | {D} | {K} | {mk:.2f} | {tf:.0f} | {100 * tf / PEAK_TFLOPS:.0f} % | {m32:.1f} | {m16:.1f} "
                      f"| {100 * agree:.2f} % |", flush=True)
        del x
        torch.cuda.empty_cache()


def bench_update(quick):
    rows = (4 << 20,) if quick else (4 << 20, 16 << 20)
    print("\n## update (counting sort + fixed-order sums; GB/s = N D 2 bytes / time)")
    print("| N | D | K | update ms | GB/s | centres ms |")
    print("|---|---|---|---|---|---|")
    D, K = 768, 500
    x = rand_rows(max(rows), D, 7)
    C = torch.randn(K, D, device="cuda")
    km = KMeans.from_centers(C.cpu())
    cbf, cn = km._device_centers(x.device)
    for N in rows:
        xs = x[:N]
        lab = torch.empty(N, dtype=torch.int32, device="cuda")
        score = torch.empty(N, device="cuda")
        ops.kmeans_assign(xs, 0, D, N, 1, D, None, cbf, cn, K, lab, score)
        counts = torch.empty(K, dtype=torch.int32, device="cuda")
        sums = torch.empty(K, D, device="cuda")
        inertia = torch.empty(1, dtype=torch.float64, device="cuda")
        ws = torch.empty(ops.kmeans_update_workspace(N, K, D), dtype=torch.uint8, device="cuda")
        cent = C.clone()
        upd = lambda: ops.kmeans_update(xs, D, N, D, lab, score, K, ws, counts, sums, inertia)  # noqa: E731
        fin = lambda: ops.kmeans_centers(sums, counts, K, D, cent, cbf, cn)  # noqa: E731
        upd()
        fin()
        mu = min(timed(upd, 10) for _ in range(2))
        mf = min(timed(fin, 10) for _ in range(2))
        print(f"| {N >> 20} M | {D} | {K} | {mu:.2f} | {N * D * 2 / (mu * 1e-3) / 1e9:.0f} | {mf:.3f} |", flush=True)
    del x
    torch.cuda.empty_cache()


def bench_fit(sk_rows):
    N, D, K, iters = 2 << 20, 768, 500, 20
    print(f"\n## fit: {N >> 20} M x {D} rows, K = {K}")
    x = rand_rows(N, D, 11)
    KMeans(K, max_iter=2, init_size=30_000).fit(x)   # warm-up
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    km = KMeans(K, max_iter=iters, init_size=30_000, seed=0).fit(x)
    torch.cuda.synchronize()
    t_fit = time.perf_counter() - t0
    t0 = time.perf_counter()
    KMeans(K, max_iter=1, init_size=30_000, seed=0)._seed_centers(x)
    torch.cuda.synchronize()
    t_seed = time.perf_counter() - t0
    print(f"KMeans.fit ({km.n_iter_} Lloyd iterations + k-means++ on 30 000 rows): {t_fit * 1e3:.0f} ms "
          f"(k-means++ alone {t_seed * 1e3:.0f} ms), inertia/row {km.inertia_ / N:.2f}")
    if sk_rows > 0:
        import numpy as np
        from sklearn.cluster import MiniBatchKMeans
        xs = x[:sk_rows].float().cpu().numpy().astype(np.float64)
        mb = MiniBatchKMeans(n_clusters=K, init="k-means++", max_iter=100, batch_size=10000, tol=0.0, max_no_improvement=100,
                             init_size=None, n_init=20, reassignment_ratio=0.0, compute_labels=False, verbose=0)
        t0 = time.perf_counter()
        mb.fit(xs)
        t_sk = time.perf_counter() - t0
        lab = torch.empty(sk_rows, dtype=torch.int32, device="cuda")
        sc = torch.empty(sk_rows, device="cuda")
        sk = KMeans.from_centers(mb.cluster_centers_)
        cbf, cn = sk._device_centers(x.device)
        ops.kmeans_assign(x[:sk_rows], 0, D, sk_rows, 1, D, None, cbf, cn, K, lab, sc)
        sk_inertia = float((x[:sk_rows].float().pow(2).sum(1) + sc).double().sum()) / sk_rows
        gpu_lab = km.predict(x[:sk_rows])
        cc = km.cluster_centers_.to(torch.bfloat16).float()
        gpu_inertia = float((x[:sk_rows].float() - cc[gpu_lab.long()]).pow(2).sum().double()) / sk_rows
        print(f"scikit-learn MiniBatchKMeans (recipe settings) on {sk_rows} rows, host CPU, {os.cpu_count()} CPUs visible, "
              f"torch threads {torch.get_num_threads()}: {t_sk:.1f} s ({mb.n_steps_} steps); inertia/row on those rows: "
              f"sklearn {sk_inertia:.2f}, this fit {gpu_inertia:.2f}")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--quick", action="store_true", help="4 M rows only")
    ap.add_argument("--sklearn-rows", type=int, default=500_000, help="rows for the CPU MiniBatchKMeans arm (0: skip)")
    ap.add_argument("--skip", default="", help="comma list of assign,update,fit to skip")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kmeans needs a CUDA device")
    name, pl = card()
    print(f"# {name}, power limit {pl}")
    skip = set(a.skip.split(","))
    if "assign" not in skip:
        bench_assign(a.quick)
    if "update" not in skip:
        bench_update(a.quick)
    if "fit" not in skip:
        bench_fit(a.sklearn_rows)


if __name__ == "__main__":
    main()
