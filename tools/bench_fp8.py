"""FP8 inference path against bf16 on one GPU (`extract_features(fp8=True)`).

  (a) every encoder projection GEMM of large / xlsr1b / xlsr2b at 8 x 20 s: ms and TFLOP/s, bf16 (b200s_gemm_rows) against fp8
      (b200s_gemm_rows_fp8); and, per layer, the two quantise passes and the fp8 LayerNorm;
  (b) extract_features in eval mode, audio-s/s, bf16 against fp8, for the same workloads and WavLM-Large on 1 x 300 s (attention
      is most of that forward, so little gain is expected there);
  (c) accuracy on the same batch: per-frame cosine similarity and relative error of fp8 against bf16, and the share of frames
      whose KMeans(500) label (centres fit on the bf16 layer-6 features) is unchanged under fp8.
bf16 and fp8 alternate round by round; times are CUDA events.  `--checkpoint PATH` runs (b) and (c) on a WavLM-format checkpoint
({'cfg': dict, 'model': state_dict}) instead of default-initialised models.  Prints the card name and power limit of the run and
writes the results as JSON to --out.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from unispeech_b200 import _lib as L  # noqa: E402
from unispeech_b200 import ops  # noqa: E402
from unispeech_b200 import workloads as W  # noqa: E402
from unispeech_b200.kmeans import KMeans  # noqa: E402
from unispeech_b200.wavlm import WavLM, WavLMConfig  # noqa: E402


def card():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0]
    except Exception as e:  # noqa: BLE001
        return f"{torch.cuda.get_device_name()} (nvidia-smi unavailable: {e})"


def timed(fns, rounds, inner):
    """fns: {name: callable}; alternates the callables round by round; returns {name: median ms per call}."""
    ts = {k: [] for k in fns}
    for k, f in fns.items():  # warm-up
        f()
    torch.cuda.synchronize()
    for _ in range(rounds):
        for k, f in fns.items():
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(inner):
                f()
            e1.record()
            e1.synchronize()
            ts[k].append(e0.elapsed_time(e1) / inner)
    return {k: sorted(v)[len(v) // 2] for k, v in ts.items()}


def gemms(name, rounds):
    cfg, B, secs = W.model_config(name)
    T = W.num_frames(secs * W.SR, cfg)
    D, F = cfg["encoder_embed_dim"], cfg["encoder_ffn_embed_dim"]
    dev = torch.device("cuda")
    M = B * T
    out, tot = [], {"bf16": 0.0, "fp8": 0.0}
    g = torch.Generator(device=dev).manual_seed(0)
    for proj, K, N, epi in (("qkv", D, 3 * D, "bias"), ("out_proj", D, D, "bias+res"), ("fc1", D, F, "bias+gelu"),
                            ("fc2", F, D, "bias+res")):
        a = torch.randn(M, K, device=dev, generator=g).to(torch.bfloat16)
        w = (torch.randn(N, K, device=dev, generator=g) * 0.02).to(torch.bfloat16)
        bias = torch.zeros(N, device=dev)
        res = torch.randn(M, N, device=dev, generator=g).to(torch.bfloat16)
        o = torch.empty(M, N, dtype=torch.bfloat16, device=dev)
        qa, sa = torch.empty(M, K, dtype=torch.uint8, device=dev), torch.empty(M, device=dev)
        ops.quantize_rows_fp8(a, 0, K, M, 1, K, qa, 0, K, sa)
        qw, sw = torch.empty(N, K, dtype=torch.uint8, device=dev), torch.empty(N, device=dev)
        ops.quantize_rows_fp8(w, 0, K, N, 1, K, qw, 0, K, sw)
        kw = dict(bias=bias)
        if epi == "bias+res":
            kw.update(res1=res, res1_ld=N)
        if epi == "bias+gelu":
            kw.update(gelu=2)
        e = L.make_epilogue(**kw)
        ms = timed({"bf16": lambda: ops.gemm_rows(a, 0, K, M, 1, K, w, N, o, 0, N, e),
                    "fp8": lambda: ops.gemm_rows_fp8(qa, sa, 0, K, M, 1, K, qw, sw, N, o, 0, N, e)}, rounds, 10)
        fl = 2.0 * M * K * N
        row = dict(model=name, proj=proj, M=M, K=K, N=N, epilogue=epi)
        for k in ("bf16", "fp8"):
            row[f"{k}_ms"] = round(ms[k], 4)
            row[f"{k}_tflops"] = round(fl / ms[k] / 1e9, 1)
            tot[k] += ms[k]
        out.append(row)
        print(json.dumps(row), flush=True)
    # per-layer row passes of the fp8 path: quantise the attention output (D) and the GELU output (F), and the fp8 LayerNorm
    x = torch.randn(M, D, device=dev, generator=g).to(torch.bfloat16)
    h = torch.randn(M, F, device=dev, generator=g).to(torch.bfloat16)
    q, s = torch.empty(M, F, dtype=torch.uint8, device=dev), torch.empty(M, device=dev)
    gamma, beta = torch.ones(D, device=dev), torch.zeros(D, device=dev)
    ms = timed({"quantize_D": lambda: ops.quantize_rows_fp8(x, 0, D, M, 1, D, q, 0, D, s),
                "quantize_F": lambda: ops.quantize_rows_fp8(h, 0, F, M, 1, F, q, 0, F, s),
                "layer_norm_fp8": lambda: ops.layer_norm_fwd_fp8(x, 0, D, gamma, beta, None, 0, 0, None, None, q, 0, D, s, M, 1,
                                                                 D)}, rounds, 10)
    extra = dict(model=name, **{f"{k}_ms": round(v, 4) for k, v in ms.items()},
                 projections_bf16_ms=round(tot["bf16"], 4), projections_fp8_ms=round(tot["fp8"], 4))
    print(json.dumps(extra), flush=True)
    return out, extra


def model_from(name=None, checkpoint=None):
    if checkpoint:
        ck = torch.load(checkpoint, map_location="cpu", weights_only=False)
        m = WavLM(WavLMConfig(ck["cfg"]))
        m.load_state_dict(ck["model"], strict=False)
    else:
        cfg, _, _ = W.model_config(name)
        torch.manual_seed(0)
        m = WavLM(WavLMConfig(cfg))
    for p in m.parameters():
        p.requires_grad_(False)
    return m.cuda().eval()


def forward(m, label, B, secs, rounds):
    wav = torch.randn(B, int(secs * W.SR), generator=torch.Generator().manual_seed(1)).cuda()
    with torch.no_grad():
        ms = timed({"bf16": lambda: m.extract_features(wav), "fp8": lambda: m.extract_features(wav, fp8=True)}, rounds, 1)
    row = dict(workload=label, batch=f"{B} x {secs} s", bf16_audio_s_per_s=round(B * secs / (ms["bf16"] / 1e3), 1),
               fp8_audio_s_per_s=round(B * secs / (ms["fp8"] / 1e3), 1), speedup=round(ms["bf16"] / ms["fp8"], 3))
    print(json.dumps(row), flush=True)
    return row, wav


def accuracy(m, label, wav):
    n_layers = len(m.encoder.layers)
    lay = min(6, n_layers)
    with torch.no_grad():
        xb, _ = m.extract_features(wav)
        x8, _ = m.extract_features(wav, fp8=True)
        lb, _ = m.extract_features(wav, output_layer=lay)
        l8, _ = m.extract_features(wav, output_layer=lay, fp8=True)
    a, b = xb.float().reshape(-1, xb.shape[-1]), x8.float().reshape(-1, x8.shape[-1])
    cos = torch.nn.functional.cosine_similarity(a, b, dim=-1)
    rel = ((a - b).norm() / a.norm()).item()
    fb, f8 = lb.reshape(-1, lb.shape[-1]).contiguous(), l8.reshape(-1, l8.shape[-1]).contiguous()
    km = KMeans(500, max_iter=20, seed=0).fit(fb)
    same = (km.predict(fb) == km.predict(f8)).float().mean().item()
    row = dict(workload=label, cos_min=round(cos.min().item(), 5), cos_mean=round(cos.mean().item(), 5), rel_err=round(rel, 5),
               kmeans_layer=lay, kmeans500_same_label=round(same, 4))
    print(json.dumps(row), flush=True)
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--models", default="large,xlsr1b,xlsr2b")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--skip-gemm", action="store_true")
    ap.add_argument("--skip-long", action="store_true", help="skip WavLM-Large on 1 x 300 s")
    ap.add_argument("--checkpoint", default=None, help="WavLM-format checkpoint: (b) and (c) on it at 8 x 20 s")
    ap.add_argument("--out", default=None, help="write the results as JSON here")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_fp8 measures on a CUDA device; none is visible")
    L.check_device()
    res = dict(card=card())
    print("card:", res["card"], flush=True)
    if args.checkpoint:
        m = model_from(checkpoint=args.checkpoint)
        row, wav = forward(m, os.path.basename(args.checkpoint), 8, 20, args.rounds)
        res["forward"], res["accuracy"] = [row], [accuracy(m, os.path.basename(args.checkpoint), wav)]
    else:
        names = [n for n in args.models.split(",") if n]
        if not args.skip_gemm:
            res["gemm"], res["row_passes"] = [], []
            for n in names:
                rows, extra = gemms(n, args.rounds)
                res["gemm"] += rows
                res["row_passes"].append(extra)
        res["forward"], res["accuracy"] = [], []
        for n in names:
            _, B, secs = W.model_config(n)
            m = model_from(n)
            row, wav = forward(m, n, B, secs, args.rounds)
            res["forward"].append(row)
            res["accuracy"].append(accuracy(m, n, wav))
            del m
            torch.cuda.empty_cache()
        if not args.skip_long and "large" in names:
            m = model_from("large")
            row, _ = forward(m, "large-300s", 1, 300, max(2, args.rounds // 2))
            res["forward"].append(row)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
