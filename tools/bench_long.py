"""Whole recordings through WavLM-Large (random init, the workloads.py configuration):
    python tools/bench_long.py [--reps 3] [--infer-s 300] [--train-s 120]
- extract_features under no_grad on one utterance of --infer-s seconds;
- forward + backward (a mean-square probe loss on the features) on one utterance of --train-s seconds.
Each line gives the time per call, audio seconds per second, and the attention kernels' share of it, from CUDA events recorded
around every attention call (forward and backward entry points) and around the whole call."""
import argparse, os, subprocess, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unispeech_b200 import ops, workloads
from unispeech_b200.wavlm import WavLM, WavLMConfig

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=3)
ap.add_argument("--infer-s", type=float, default=300.0)
ap.add_argument("--train-s", type=float, default=120.0)
args = ap.parse_args()
dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip()
except (OSError, subprocess.CalledProcessError):
    card = f"{torch.cuda.get_device_name(0)}, power limit unknown"
print(f"GPU: {card}", flush=True)

_attn_events = []


def _timed(fn):
    def run(*a, **k):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        r = fn(*a, **k)
        e1.record()
        _attn_events.append((e0, e1))
        return r
    return run


for name in ("attn_fwd", "attn_fwd_dropout", "attn_bwd", "attn_bwd_fused", "attn_bwd_fused_dropout"):
    setattr(ops, name, _timed(getattr(ops, name)))

cfg, _, _ = workloads.model_config("large")
torch.manual_seed(0)
m = WavLM(WavLMConfig(cfg)).to(dev)


def measure(tag, secs, step):
    L = int(secs * workloads.SR)
    wav = torch.randn(1, L, device=dev)
    step(wav)  # warm-up
    torch.cuda.synchronize()
    tot = attn = 0.0
    for _ in range(args.reps):
        _attn_events.clear()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(wav)
        e1.record()
        torch.cuda.synchronize()
        tot += e0.elapsed_time(e1)
        attn += sum(a.elapsed_time(b) for a, b in _attn_events)
    ms, T = tot / args.reps, workloads.num_frames(L, cfg)
    print(f"{tag:9s} 1 x {secs:5.0f} s (T = {T:5d}): {ms:9.1f} ms  {secs / (ms / 1e3):7.1f} audio-s/s  "
          f"attention {attn / tot:5.3f} of the time", flush=True)


def infer(wav):
    with torch.no_grad():
        m.extract_features(wav)


def train(wav):
    x, _ = m.extract_features(wav)
    x.float().pow(2).mean().backward()
    m.zero_grad(set_to_none=True)


m.eval()
measure("infer", args.infer_s, infer)
m.train()
measure("fwd+bwd", args.train_s, train)
