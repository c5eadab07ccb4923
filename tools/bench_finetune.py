"""Fine-tuning step cost of channel masking and conv biases: `Wav2VecEncoder` (apply_mask=True, training mode) around a WavLM-Large-width encoder
(the workloads.py configuration), a `proj` head of 32 outputs and a mean-square probe loss on it, forward + backward:
    python tools/bench_finetune.py [--batch 8] [--secs 20] [--steps 10] [--rounds 5]
Four configurations alternate round by round: conv biases off / on (two models, `conv_bias`) x span masking only
(mask_channel_prob 0) / span + channel masking (mask_channel_prob 0.5, mask_channel_length 64, the published ASR recipes).
Each step includes the host-side mask draws.  Prints the card name and power limit, then ms per step (median over rounds, with
the min-max range) for each configuration."""
import argparse
import os
import statistics
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unispeech_b200 import workloads  # noqa: E402
from unispeech_b200.fairseq_encoder import Wav2VecEncoder  # noqa: E402
from unispeech_b200.wavlm import WavLM, WavLMConfig  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--batch", type=int, default=8)
ap.add_argument("--secs", type=float, default=20.0)
ap.add_argument("--steps", type=int, default=10)
ap.add_argument("--rounds", type=int, default=5)
args = ap.parse_args()
dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip()
except (OSError, subprocess.CalledProcessError):
    card = f"{torch.cuda.get_device_name(0)}, power limit unknown"
print(f"GPU: {card}", flush=True)

cfg, _, _ = workloads.model_config("large")
cfg = dict(cfg, mask_channel_prob=0.5, mask_channel_length=64)
encs = {}
for bias in (False, True):
    torch.manual_seed(0)
    m = WavLM(WavLMConfig(dict(cfg, conv_bias=bias)))
    encs[bias] = Wav2VecEncoder(m, apply_mask=True, output_dim=32).to(dev).train()
L = int(args.secs * workloads.SR)
wav = torch.randn(args.batch, L, device=dev)
CONFIGS = {f"conv bias {'on ' if b else 'off'}, {name}": (b, p) for b in (False, True)
           for name, p in (("span mask only", 0.0), ("span + channel mask", 0.5))}


def step(enc):
    y = enc(wav, None)["encoder_out"]
    y.float().pow(2).mean().backward()
    enc.w2v_model.zero_grad_buffer()
    enc.proj.weight.grad = enc.proj.bias.grad = None


def timed(bias, p):
    enc = encs[bias]
    enc.w2v_model.mask_channel_prob = p
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.steps):
        step(enc)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.steps


for bias, p in CONFIGS.values():  # warm-up of every configuration
    encs[bias].w2v_model.mask_channel_prob = p
    for _ in range(3):
        step(encs[bias])
torch.cuda.synchronize()
res = {k: [] for k in CONFIGS}
for r in range(args.rounds):
    for k, bp in (CONFIGS.items() if r % 2 == 0 else reversed(list(CONFIGS.items()))):
        res[k].append(timed(*bp))
T = workloads.num_frames(L, cfg)
for k, v in res.items():
    print(f"{k:38s} {args.batch} x {args.secs:.0f} s (T = {T}): {statistics.median(v):8.2f} ms/step  "
          f"(rounds {min(v):.2f} .. {max(v):.2f})", flush=True)
