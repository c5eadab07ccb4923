"""The wide encoders on one GPU: `xlsr1b` (XLS-R 1B / MMS-1B shape, 48 x 1280, head width 80, the default) or `xlsr2b`
(XLS-R 2B, 48 x 1920, head width 120), chosen with --workload:

* one `Wav2VecCtc` fine-tuning step (forward, CTC loss, backward, `FusedAdam`) on 8 x 20 s: ms per step, median and range over
  rounds;
* `extract_features` in eval mode on the same batch: audio seconds per second;
* `torch.cuda.max_memory_allocated` over both;
* the card's name and power limit, read in the same run.

Weights are the modules' default initialisation (timing does not depend on them).  Prints one JSON line.

    python tools/bench_wide.py [--workload xlsr1b|xlsr2b] [--rounds 5] [--steps 5] [--warmup 2]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from unispeech_b200 import workloads as W  # noqa: E402
from unispeech_b200.ctc import CtcCriterion, Wav2VecCtc  # noqa: E402
from unispeech_b200.optim import FusedAdam  # noqa: E402
from unispeech_b200.wav2vec2 import Wav2Vec2Config, Wav2Vec2Model  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--workload", choices=("xlsr1b", "xlsr2b"), default="xlsr1b")
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--steps", type=int, default=5, help="timed steps per round")
ap.add_argument("--warmup", type=int, default=2)
ap.add_argument("--vocab", type=int, default=32)
args = ap.parse_args()

if not torch.cuda.is_available():
    sys.exit("bench_wide.py needs a CUDA device")
dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, timeout=30).stdout.strip()
except (OSError, subprocess.SubprocessError):
    card = ""
card = card or f"{torch.cuda.get_device_name(0)}, power limit unknown"

cfg, B, secs = W.model_config(args.workload)
cfg = dict(cfg, dropout=0.0, attention_dropout=0.0, mask_prob=0.65)
L = secs * W.SR
torch.manual_seed(0)
w2v = Wav2Vec2Model(Wav2Vec2Config(cfg))
model = Wav2VecCtc.build_model(w2v, args.vocab, apply_mask=True).to(dev).train()
g = torch.Generator().manual_seed(1)
wav = torch.randn(B, L, generator=g).to(dev)
pmask = torch.zeros(B, L, dtype=torch.bool)
S = 200  # target tokens per utterance (letters of ~20 s of speech)
target = torch.randint(3, args.vocab, (B, S + 1), generator=g)
target[:, S] = 2  # eos
sample = {"net_input": {"source": wav, "padding_mask": pmask}, "target": target, "id": torch.arange(B)}
crit = CtcCriterion()
np.random.seed(0)

torch.cuda.reset_peak_memory_stats()
opt = None


def step():
    global opt
    loss, _, _ = crit(model, sample)
    loss.backward()
    if opt is None:
        opt = FusedAdam(w2v, lr=1e-5)
    opt.step()
    w2v.zero_grad_buffer()
    model.w2v_encoder.proj.weight.grad = model.w2v_encoder.proj.bias.grad = None


for _ in range(args.warmup):
    step()
torch.cuda.synchronize()
step_ms = []
for _ in range(args.rounds):
    t0 = time.perf_counter()
    for _ in range(args.steps):
        step()
    torch.cuda.synchronize()
    step_ms.append((time.perf_counter() - t0) * 1e3 / args.steps)

model.eval()
with torch.no_grad():
    for _ in range(args.warmup):
        w2v.extract_features(wav, padding_mask=None)
    torch.cuda.synchronize()
    fwd_rate = []
    for _ in range(args.rounds):
        t0 = time.perf_counter()
        for _ in range(args.steps):
            w2v.extract_features(wav, padding_mask=None)
        torch.cuda.synchronize()
        fwd_rate.append(B * secs * args.steps / (time.perf_counter() - t0))

res = {
    "workload": f"{args.workload} ({cfg['encoder_layers']} x {cfg['encoder_embed_dim']} / {cfg['encoder_ffn_embed_dim']}, "
                f"{cfg['encoder_attention_heads']} heads of width {cfg['encoder_embed_dim'] // cfg['encoder_attention_heads']}, "
                f"pre-LN, no relative-position bias), batch {B} x {secs} s, Wav2VecCtc vocab {args.vocab}, mask_prob 0.65, dropout 0",
    "card": card,
    "finetune_ms_per_step": {"median": float(np.median(step_ms)), "min": min(step_ms), "max": max(step_ms),
                             "rounds": args.rounds, "steps_per_round": args.steps},
    "finetune_audio_s_per_s": B * secs / (float(np.median(step_ms)) / 1e3),
    "extract_features_audio_s_per_s": {"median": float(np.median(fwd_rate)), "min": min(fwd_rate), "max": max(fwd_rate)},
    "max_memory_allocated_gib": torch.cuda.max_memory_allocated() / 2 ** 30,
}
print(json.dumps(res))
