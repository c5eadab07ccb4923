"""CTC forced alignment: `unispeech_b200.ctc.forced_align` against `torchaudio.functional.forced_align` on the GPU and on the CPU.
    python tools/bench_align.py [--calls 10] [--cpu-calls 2] [--skip-cpu-long]
Shapes (V = 32 classes, bf16 logits in the fine-tuning wrappers' layout, the T x B x V view of a [B*T, 64] buffer, seeded
targets of about 0.3 labels per frame, i.e. 15 characters per second at 50 frames per second):
  finetune   B = 8, T = 999 (20 s), S = 300
  ragged     B = 8 utterances of 2 .. 30 s (T_b = 99 .. 1499), S_b = 0.3 T_b
  long30k    B = 1, T = 30 000 (10 min), S = 4 000
  long90k    B = 1, T = 90 000 (30 min), S = 6 000
Per shape: the library's whole call (statistics + Viterbi + backtrack) timed with CUDA events, median over `--calls`; the
Viterbi and backtrack kernels timed separately by torch.profiler in a run of its own, and us per recursion step (Viterbi kernel
time / max T_b: the recursion is a chain of T_b dependent steps); torchaudio's GPU forced_align one utterance at a time on the
fp32 log-probabilities it needs, with the time to build those (log_softmax of the whole batch) stated separately, and whether
its paths and frame scores equal the library's (given lp built from the library's lse); torchaudio on the host CPU one utterance
at a time, with torch's intra-op thread count.  Prints the card name and power limit first."""
import argparse
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from unispeech_b200 import ops  # noqa: E402
from unispeech_b200.ctc import forced_align  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--calls", type=int, default=10)
ap.add_argument("--cpu-calls", type=int, default=2)
ap.add_argument("--skip-cpu-long", action="store_true", help="leave torchaudio's CPU path out of the long-form shapes")
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_align.py measures on a GPU; none is visible")
import torchaudio.functional as TA  # noqa: E402

dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip()
except (OSError, subprocess.CalledProcessError):
    card = f"{torch.cuda.get_device_name(0)}, power limit unknown"
print(f"GPU: {card}", flush=True)
print(f"CPU: torch intra-op threads = {torch.get_num_threads()}", flush=True)
V, VP = 32, 64


def make_case(T_list, S_list, T, seed=0):
    B = len(T_list)
    g = torch.Generator().manual_seed(seed)
    buf = (torch.randn(B * T, VP, generator=g) * 3).to(torch.bfloat16).to(dev)
    x = buf[:, :V].reshape(B, T, V).transpose(0, 1)
    Smax = max(S_list)
    tg = torch.randint(1, V, (B, Smax), generator=g, dtype=torch.int32)
    return x, torch.tensor(T_list, dtype=torch.int32, device=dev), tg.to(dev), torch.tensor(S_list, dtype=torch.int32, device=dev)


def cuda_ms(fn, calls):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(calls):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        out.append(e0.elapsed_time(e1))
    return statistics.median(out)


def kernel_ms(fn):
    """Device time of each kernel of one call from the torch.profiler trace (CUDA activities).  The kernels are launched with
    programmatic dependent launch, so a kernel becomes resident while its predecessor still runs and waits for it: its span in
    the trace starts early.  Each kernel is therefore charged from the end of the previous one (or its own start) to its end."""
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    spans = {}
    for e in prof.events():
        if e.device_type == torch.autograd.DeviceType.CUDA:
            for key in ("ctc_stats", "ctc_align_viterbi", "ctc_align_backtrack"):
                if key in e.name:
                    spans[key] = (e.time_range.start, e.time_range.end)
    out, prev_end = {}, None
    for key in ("ctc_stats", "ctc_align_viterbi", "ctc_align_backtrack"):
        if key in spans:
            t0, t1 = spans[key]
            out[key] = (t1 - (t0 if prev_end is None else max(t0, prev_end))) / 1e3
            prev_end = t1
    return out


def host_ms(fn, calls):
    fn()
    out = []
    for _ in range(calls):
        t0 = time.perf_counter()
        fn()
        out.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(out)


def fmt(v):
    return "not measured" if v is None else f"{v:10.3f}"


shapes = {
    "finetune": ([999] * 8, [300] * 8, 999),
    "ragged": ([99 + 200 * i for i in range(8)], [int(0.3 * (99 + 200 * i)) for i in range(8)], 1499),
    "long30k": ([30000], [4000], 30000),
    "long90k": ([90000], [6000], 90000),
}
rows = []
for name, (T_list, S_list, T) in shapes.items():
    x, il, tg, tl = make_case(T_list, S_list, T)
    long = T >= 30000
    calls = 3 if long else args.calls
    ours = cuda_ms(lambda: forced_align(x, il, tg, tl), calls)
    ks = kernel_ms(lambda: forced_align(x, il, tg, tl))
    ours_out = [t.cpu() for t in forced_align(x, il, tg, tl)]

    def build_lp():
        return torch.log_softmax(x.float(), -1).transpose(0, 1).contiguous()   # [B, T, V] fp32, what torchaudio takes

    lp_ms = cuda_ms(build_lp, calls)
    # torchaudio is given lp = logit - lse with the library's lse (the same fp32 tensor up to the last bit): with it the paths
    # must agree exactly, ties included
    lse = torch.zeros(len(T_list), T, device=dev)
    ops.ctc_stats(x, x.stride(0), x.stride(1), il, len(T_list), T, V, lse, None)
    lp = (x.float().transpose(0, 1) - lse[..., None]).contiguous()
    tg_l, il_l, tl_l = tg.long(), il.tolist(), tl.tolist()

    def ta_gpu():
        return [TA.forced_align(lp[b:b + 1, :il_l[b]], tg_l[b:b + 1, :tl_l[b]], blank=0) for b in range(len(il_l))]

    try:
        ta_gpu_ms = cuda_ms(ta_gpu, calls)
        ta_res = ta_gpu()
        agree = all(torch.equal(p[0].cpu(), ours_out[0][b, :il_l[b]]) and torch.equal(sc[0].cpu(), ours_out[1][b, :il_l[b]])
                    for b, (p, sc) in enumerate(ta_res))
    except Exception as e:  # noqa: BLE001 -- reported, not hidden
        print(f"{name}: torchaudio GPU failed: {type(e).__name__}: {e}", flush=True)
        ta_gpu_ms, agree = None, None
    ta_cpu_ms = None
    if not (long and args.skip_cpu_long):
        lp_cpu, tg_cpu = lp.cpu(), tg_l.cpu()

        def ta_cpu():
            return [TA.forced_align(lp_cpu[b:b + 1, :il_l[b]], tg_cpu[b:b + 1, :tl_l[b]], blank=0) for b in range(len(il_l))]

        ta_cpu_ms = host_ms(ta_cpu, 1 if long else args.cpu_calls)
    vit = ks.get("ctc_align_viterbi")
    rows.append((name, len(T_list), max(T_list), max(S_list), ours, ks.get("ctc_stats"), vit, ks.get("ctc_align_backtrack"),
                 None if vit is None else vit * 1e3 / max(T_list), lp_ms, ta_gpu_ms, ta_cpu_ms, agree))
    print(f"{name}: done", flush=True)

print()
print(f"{'shape':>9s} {'B':>2s} {'T':>6s} {'S':>5s} | {'library ms':>10s} {'stats':>10s} {'viterbi':>10s} {'backtrack':>10s} "
      f"{'us/step':>8s} | {'lp build':>10s} {'TA gpu ms':>10s} {'TA cpu ms':>12s} {'same path':>9s}")
for r in rows:
    name, B, T, S, ours, st, vit, bt, us, lp_ms, tg_ms, tc_ms, agree = r
    print(f"{name:>9s} {B:2d} {T:6d} {S:5d} | {fmt(ours)} {fmt(st)} {fmt(vit)} {fmt(bt)} "
          f"{'not measured' if us is None else f'{us:8.3f}'} | {fmt(lp_ms)} {fmt(tg_ms)} {fmt(tc_ms):>12s} {str(agree):>9s}", flush=True)
