"""MFCC features of HuBERT's first iteration on the GPU (b200s_mfcc) and the iteration-1 label pass.

  mfcc      b200s_mfcc (features + the bf16 k-means rows) on 64 x 15 s and on a ragged batch of 64 utterances of 2-16 s:
            audio-s/s, GB/s from the bytes the op must move (4 B per sample read; 156 B of features + 128 B of bf16 row written
            per frame) and that rate's share of the 3.35 TB/s HBM3 figure of the H100 SXM data sheet.
  recipe    the same features through torchaudio (kaldi.mfcc + compute_deltas twice, fp32, one utterance at a time, as
            dump_mfcc_feature.py does) on the same GPU and on the host CPU: comparison arms only.
  labels    the iteration-1 label pass on the ragged batch: mfcc -> KMeans(100) fit on 100 000 valid rows (20 Lloyd iterations)
            -> predict over every frame.
CUDA events (host clock around a synchronised loop for the CPU arm) after a warm-up.  Prints one JSON line.  GPU only.

    python tools/bench_mfcc.py [--reps 50]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from unispeech_b200 import ops  # noqa: E402
from unispeech_b200.kmeans import KMeans  # noqa: E402
from unispeech_b200.mfcc import mfcc, num_frames  # noqa: E402

HBM_BYTES_PER_S = 3.35e12   # H100 SXM, HBM3, data sheet
SR = 16000


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:  # noqa: BLE001
        pl = "unknown"
    return name, pl


def timed(fn, reps):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / reps


def batch(lengths, seed):
    g = torch.Generator().manual_seed(seed)
    L = max(lengths)
    wav = (torch.rand(len(lengths), L, generator=g) * 2 - 1) * 0.3
    pad = torch.arange(L)[None, :] >= torch.tensor(lengths)[:, None]
    wav[pad] = 0.0
    return wav.cuda(), pad


def op_bytes(lengths):
    return sum(4.0 * n + num_frames(n) * (156.0 + 128.0) for n in lengths)


def mfcc_arm(lengths, reps, seed):
    """`kernel_ms`: b200s_mfcc alone (both kernels, lengths already on the device); `call_ms`: mfcc() with the collater's host
    padding mask (valid-sample count and frame mask on the host, output allocation)."""
    wav, pad = batch(lengths, seed)
    B, L = wav.shape
    Tm = num_frames(L)
    n = torch.tensor(lengths, dtype=torch.int32, device="cuda")
    feats = torch.empty(B, Tm, 39, device="cuda")
    rows = torch.empty(B, Tm, 64, dtype=torch.bfloat16, device="cuda")
    ms = timed(lambda: ops.mfcc(wav, L, L, n, B, Tm, feats, Tm * 39, rows, Tm * 64), reps)
    call_ms = timed(lambda: mfcc(wav, padding_mask=pad, kmeans_rows=True), reps)
    gbs = op_bytes(lengths) / (ms * 1e-3) / 1e9
    return dict(utterances=len(lengths), audio_s=round(sum(lengths) / SR, 1), kernel_ms=round(ms, 4),
                audio_s_per_s=round(sum(lengths) / SR / (ms * 1e-3)), GB_per_s=round(gbs, 1),
                share_of_hbm=round(gbs * 1e9 / HBM_BYTES_PER_S, 4), call_ms=round(call_ms, 3))


def recipe_arm(lengths, device, seed, reps=1):
    import torchaudio as ta
    wav, _ = batch(lengths, seed)
    utts = [wav[b, :n].to(device).view(1, -1) for b, n in enumerate(lengths)]

    def run():
        for u in utts:
            m = ta.compliance.kaldi.mfcc(waveform=u, sample_frequency=SR, use_energy=False).transpose(0, 1)
            d = ta.functional.compute_deltas(m)
            torch.cat([m, d, ta.functional.compute_deltas(d)], dim=0)
    run()
    if device == "cuda":
        ms = timed(run, reps)
    else:
        t0 = time.perf_counter()
        for _ in range(reps):
            run()
        ms = (time.perf_counter() - t0) * 1e3 / reps
    return dict(ms=round(ms, 2), audio_s_per_s=round(sum(lengths) / SR / (ms * 1e-3)))


def label_pass(lengths, seed):
    wav, pad = batch(lengths, seed)

    def run():
        _, pm, rows = mfcc(wav, padding_mask=pad, kmeans_rows=True)
        valid = rows[~pm]
        g = torch.Generator(device="cuda").manual_seed(0)
        sub = valid[torch.randperm(valid.shape[0], generator=g, device="cuda")[:100_000]]
        km = KMeans(100, max_iter=20, tol=0.0, seed=0).fit(sub)
        return km.predict(rows, pm), km
    run()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    labels, km = run()
    torch.cuda.synchronize()
    ms = (time.perf_counter() - t0) * 1e3
    return dict(ms=round(ms, 1), frames=int((labels >= 0).sum()), lloyd_iterations=int(km.n_iter_))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_mfcc.py measures the GPU kernels: no CUDA device is visible")
    name, pl = card()
    g = torch.Generator().manual_seed(1)
    dense = [15 * SR] * 64
    ragged = [int(v) for v in torch.randint(2 * SR, 16 * SR + 1, (64,), generator=g)]
    res = dict(card=name, power_limit=pl, cpu_threads=torch.get_num_threads())
    res["mfcc_64x15s"] = mfcc_arm(dense, args.reps, 2)
    res["mfcc_ragged_2_16s"] = mfcc_arm(ragged, args.reps, 3)
    res["torchaudio_gpu_ragged"] = recipe_arm(ragged, "cuda", 3, reps=3)
    res["torchaudio_cpu_ragged"] = recipe_arm(ragged[:16], "cpu", 3)
    res["torchaudio_cpu_ragged"]["utterances"] = 16
    res["label_pass_ragged"] = label_pass(ragged, 3)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
