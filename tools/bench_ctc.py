"""CTC loss forward + backward on bf16 logits: the library's kernels against the ATen path they replace, and the whole fine-tuning
step with each loss:
    python tools/bench_ctc.py [--calls 50] [--rounds 5] [--no-step] [--step-steps 5]
(a) `F.log_softmax(logits.float())` + `F.ctc_loss(reduction="sum")`, forward + backward down to the bf16 logits' gradient;
(b) `unispeech_b200.ctc.ctc_loss`, the same.
Both read the T x B x V view of a [B*T, 64] buffer (the fine-tuning wrappers' layout) at V = 32, B = 8 / 32, T = 999 / 1499, with
seeded targets of about 15 characters per second (0.3 labels per frame).  (a) and (b) alternate round by round in one process and
are timed with CUDA events over `--calls` calls after a warm-up.  Prints the card name and power limit, then per call: ms (median
over rounds, min .. max), kernel launches (counted by torch.profiler in a run of its own), bytes moved computed from the shapes,
and ns per recursion step (ms / max input_len): the chain of input_len dependent steps is latency-bound, so that is the figure to
watch -- a share of the HBM or tensor-core peak means nothing for it.
Then the `Wav2VecEncoder` WavLM-Large fine-tuning step (8 x 20 s, span masking, `proj` of 32 outputs) with each loss."""
import argparse
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unispeech_b200 import workloads  # noqa: E402
from unispeech_b200.ctc import ctc_loss  # noqa: E402
from unispeech_b200.fairseq_encoder import Wav2VecEncoder  # noqa: E402
from unispeech_b200.wavlm import WavLM, WavLMConfig  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--calls", type=int, default=50)
ap.add_argument("--rounds", type=int, default=5)
ap.add_argument("--no-step", action="store_true")
ap.add_argument("--step-steps", type=int, default=5)
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_ctc.py measures on a GPU; none is visible")
dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip()
except (OSError, subprocess.CalledProcessError):
    card = f"{torch.cuda.get_device_name(0)}, power limit unknown"
print(f"GPU: {card}", flush=True)
V, VP = 32, 64


def make_case(B, T, seed=0):
    g = torch.Generator().manual_seed(seed)
    S = int(0.3 * T)
    buf = (torch.randn(B * T, VP, generator=g) * 2).to(torch.bfloat16).to(dev)
    x = buf[:, :V].reshape(B, T, V).transpose(0, 1).requires_grad_(True)
    tl = torch.randint(int(0.8 * S), S + 1, (B,), generator=g)
    tg = torch.randint(1, V, (B, S), generator=g)
    il = torch.full((B,), T, dtype=torch.long)
    return x, il.to(dev), tg.to(dev), tl.to(dev), S


def aten(x, il, tg, tl):
    x.grad = None
    F.ctc_loss(F.log_softmax(x.float(), -1), tg, il, tl, blank=0, reduction="sum").backward()


def ours(x, il, tg, tl):
    x.grad = None
    ctc_loss(x, il, tg, tl, reduction="sum").backward()


def timed(fn, case, calls):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(calls):
        fn(*case)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / calls


def launches(fn, case):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn(*case)
        torch.cuda.synchronize()
    return sum(e.count for e in prof.key_averages() if e.device_type == torch.autograd.DeviceType.CUDA)


def bytes_moved(B, T, S):
    """From the shapes.  Library: logits read by the statistics, alpha and beta kernels' gathers (counted twice: once whole for
    the statistics, once whole for the gradient rows), gradient written once, log_alpha written and read, lse written and read
    twice.  ATen: fp32 cast written + read, log-probs written + read by alpha, beta and the gradient kernel, log_alpha and
    log_beta written + read, the fp32 CTC gradient written + read, the fp32 log-softmax gradient written + read, the bf16 gradient
    written."""
    n, Lx = B * T, 2 * S + 1
    lib = 2 * n * VP * 2 + n * VP * 2 + 2 * n * Lx * 4 + 3 * n * 4
    at = n * V * 2 + 2 * n * V * 4 + 4 * n * V * 4 + 2 * 2 * n * Lx * 4 + 2 * n * V * 4 + 2 * n * V * 4 + n * V * 2
    return lib, at


print(f"{'case':>16s} {'path':>8s} {'ms/call':>9s} {'(min .. max)':>18s} {'launches':>9s} {'MB moved':>9s} {'ns/step':>8s}")
for B in (8, 32):
    for T in (999, 1499):
        case = make_case(B, T)
        S = case[4]
        fns = {"aten": aten, "library": ours}
        for fn in fns.values():
            for _ in range(5):
                fn(*case[:4])
        torch.cuda.synchronize()
        res = {k: [] for k in fns}
        for r in range(args.rounds):
            for k in (list(fns) if r % 2 == 0 else reversed(list(fns))):
                res[k].append(timed(fns[k], case[:4], args.calls))
        nl = {k: launches(fns[k], case[:4]) for k in fns}
        lib_b, at_b = bytes_moved(B, T, S)
        for k, nb in (("aten", at_b), ("library", lib_b)):
            med = statistics.median(res[k])
            print(f"{f'B={B} T={T} S<={S}':>16s} {k:>8s} {med:9.3f} {f'({min(res[k]):.3f} .. {max(res[k]):.3f})':>18s} {nl[k]:9d} "
                  f"{nb / 1e6:9.1f} {med * 1e6 / T:8.0f}", flush=True)

if not args.no_step:
    cfg, _, _ = workloads.model_config("large")
    torch.manual_seed(0)
    enc = Wav2VecEncoder(WavLM(WavLMConfig(dict(cfg))), apply_mask=True, output_dim=V).to(dev).train()
    Bs, L = 8, int(20.0 * workloads.SR)
    wav = torch.randn(Bs, L, device=dev)
    T = workloads.num_frames(L, cfg)
    _, il, tg, tl, S = make_case(Bs, T, seed=1)

    def step(loss_fn):
        y = enc(wav, None)["encoder_out"]
        if loss_fn is aten:
            F.ctc_loss(F.log_softmax(y.float(), -1), tg, il, tl, blank=0, reduction="sum").backward()
        else:
            ctc_loss(y, il, tg, tl, reduction="sum").backward()
        enc.w2v_model.zero_grad_buffer()
        enc.proj.weight.grad = enc.proj.bias.grad = None

    for fn in (aten, ours):
        for _ in range(2):
            step(fn)
    torch.cuda.synchronize()
    res = {"aten": [], "library": []}
    for r in range(args.rounds):
        for k, fn in ((("aten", aten), ("library", ours)) if r % 2 == 0 else (("library", ours), ("aten", aten))):
            res[k].append(timed(lambda: step(fn), (), args.step_steps))
    for k, v in res.items():
        print(f"fine-tuning step 8 x 20 s (T = {T}), loss = {k:8s}: {statistics.median(v):8.2f} ms/step  (rounds {min(v):.2f} .. {max(v):.2f})",
              flush=True)
