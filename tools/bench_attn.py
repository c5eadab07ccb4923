"""Micro-benchmark of the attention kernels at the WavLM-Base (16 x 749, 12 heads) and -Large (8 x 999, 16 heads) shapes.
    python tools/bench_attn.py [--reps 10] [--only base|large|long|wide] [--dropout 0.1]
`--only wide` times the forward, the forward with dropout (--dropout, else 0.1) and the fused backward without the bias at
8 x 999 with 16 heads at head widths 80 (the 1280-wide encoders) and 120 (XLS-R 2B) next to head width 64 at the same shape;
it runs only when asked.
`--only long` times one utterance with 16 heads at T = 8192 (164 s: the forward and both backward entry points) and
T = 16384 (the forward), and checks every call once against the fp32 reference one head at a time (one [T, T] fp32
matrix is 1 GB at T = 16384).
Each line gives the time, the algorithmic TFLOP/s and its fraction of the bf16 peak (MEASURED_PEAKS.json when present, else
the H100 SXM data sheet).  At the Large shape every backward is also checked once against autograd of the fp32 reference
(dq / dk / dv, d gate, d tab; the tolerances of tests/test_kernels_gpu.py::test_attn_bwd); with dropout the reference applies
the keep mask the forward kernel wrote."""
import argparse, os, subprocess, sys
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from unispeech_b200 import ops
from bench_gemm import load_peak

ap = argparse.ArgumentParser()
ap.add_argument("--reps", type=int, default=10)
ap.add_argument("--only", default=None)
ap.add_argument("--dropout", type=float, default=0.0, help="also time the kernels with dropout on the probabilities")
args = ap.parse_args()
dev = torch.device("cuda:0")
peak, peak_src = load_peak()
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip()
except (OSError, subprocess.CalledProcessError):
    card = f"{torch.cuda.get_device_name(0)}, power limit unknown"
print(f"GPU: {card}; peak: {peak} TFLOP/s ({peak_src})", flush=True)


def attn_ref(qkv, gate, tab, B, T, H, scale, keep=None, p=0.0):
    """fp32 attention with the gated relative-position bias; `keep` [B,H,T,T] (bool) drops probabilities, scaled by 1/(1-p)."""
    D = H * 64
    q, k, v = (x.view(B, T, H, 64).transpose(1, 2) for x in qkv.float().split(D, dim=-1))
    s = torch.matmul(q, k.transpose(-1, -2)) * scale
    if tab is not None:
        i = torch.arange(T, device=qkv.device)[:, None]
        j = torch.arange(T, device=qkv.device)[None, :]
        s = s + gate.unsqueeze(-1) * tab[:, (j - i) + T - 1].unsqueeze(0)
    pr = torch.softmax(s, dim=-1)
    if keep is not None:
        pr = pr * keep / (1.0 - p)
    return torch.matmul(pr, v).transpose(1, 2).reshape(B, T, D)


def keep_mask(words, B, T, H):
    """The forward's dropout keep bits as [B,H,T,T] bool: bit i & 31 of word [(b*H+h)*4N + i/32, j]."""
    N = (T + 127) // 128
    w = words.view(B * H, 4 * N, 128 * N)[:, :, :T]
    i = torch.arange(T, device=words.device)
    rows = w[:, i // 32, :]                                   # [BH, T, T]
    return ((rows >> (i % 32).view(1, T, 1).to(torch.int32)) & 1).bool().view(B, H, T, T)


def check_bwd(name, run, qkv, gate, tab, dout, dqkv, dgate, dtab, B, T, H, keep=None, p=0.0):
    """One more call of `run` against autograd of the fp32 reference; prints the worst error over each tolerance."""
    if dtab is not None:
        dtab.zero_()  # accumulated by every call
    run()
    torch.cuda.synchronize()
    qr = qkv.float().requires_grad_(True)
    gr = gate.clone().requires_grad_(True) if gate is not None else None
    tr = tab.clone().requires_grad_(True) if tab is not None else None
    attn_ref(qr, gr, tr, B, T, H, 0.125, keep, p).backward(dout.float())
    errs = [("dqkv", dqkv.float(), qr.grad)]
    if tab is not None:
        errs += [("dgate", dgate, gr.grad), ("dtab", dtab, tr.grad)]
    parts, ok = [], True
    for k, got, ref in errs:
        r = (got - ref).abs().max().item() / (0.03 * max(1.0, ref.abs().max().item()))
        ok &= r < 1.0
        parts.append(f"{k} {r:.3f}")
    print(f"       check {name}: error / tolerance: {', '.join(parts)} -> {'ok' if ok else 'FAIL'}", flush=True)
    del qr, gr, tr
    torch.cuda.empty_cache()
    return ok


def timed(fn):
    for _ in range(2):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(args.reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / args.reps


def head_cols(h, D):
    return torch.cat([torch.arange(h * 64, h * 64 + 64) + o for o in (0, D, 2 * D)]).to(dev)


def check_long(name, run, qkv, gate, tab, out, lse, dout, dqkv, dgate, dtab, B, T, H):
    """One more call of `run` against the fp32 reference, one head at a time: the forward's output and lse, or the backward's
    dq / dk / dv, d gate and d tab (tolerances of check_bwd)."""
    D = H * 64
    if dtab is not None:
        dtab.zero_()
    run()
    torch.cuda.synchronize()
    worst, fwd = 0.0, name.startswith("fwd")
    for h in range(H):
        c = head_cols(h, D)
        qr = qkv[..., c].float().requires_grad_(not fwd)
        gr = gate[:, h:h + 1].clone().requires_grad_(not fwd)
        tr = tab[h:h + 1].clone().requires_grad_(not fwd)
        if fwd:
            with torch.no_grad():
                ref = attn_ref(qr, gr, tr, B, T, 1, 0.125)
            pairs = [(out[..., h * 64:(h + 1) * 64].float(), ref)]
        else:
            attn_ref(qr, gr, tr, B, T, 1, 0.125).backward(dout[..., h * 64:(h + 1) * 64].float())
            pairs = [(dqkv[..., c].float(), qr.grad), (dgate[:, h], gr.grad[:, 0]), (dtab[h], tr.grad[0])]
        for got, want in pairs:
            worst = max(worst, (got - want).abs().max().item() / (0.03 * max(1.0, want.abs().max().item())))
        del qr, gr, tr, pairs
        torch.cuda.empty_cache()
    ok = worst < 1.0
    print(f"       check {name} T={T}: worst error / tolerance over the heads {worst:.3f} -> {'ok' if ok else 'FAIL'}", flush=True)
    return ok


all_ok = True
if args.only == "long":
    B, H = 1, 16
    D = H * 64
    for T, kinds in ((8192, ("fwd", "bwd_fused", "bwd_2kernel")), (16384, ("fwd",))):
        torch.manual_seed(0)
        qkv = torch.randn(B, T, 3 * D, device=dev).to(torch.bfloat16)
        gate = torch.rand(B, H, T, device=dev) * 2 + 0.2
        tab = torch.randn(H, 2 * T - 1, device=dev)
        out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
        lse = torch.empty(B, H, T, device=dev)
        dout = torch.randn(B, T, D, device=dev).to(torch.bfloat16)
        delta = torch.empty(B, H, T, device=dev)
        dqkv = torch.zeros(B, T, 3 * D, device=dev, dtype=torch.bfloat16)
        dgate = torch.zeros(B, H, T, device=dev)
        dtab = torch.zeros(H, 2 * T - 1, device=dev)
        dq_acc = torch.zeros(B, T, D, device=dev)
        fns = {
            "fwd": lambda: ops.attn_fwd(qkv, gate, tab, None, out, lse, B, T, H, 0.125),
            "bwd_fused": lambda: ops.attn_bwd_fused(qkv, out, dout, gate, tab, None, lse, delta, dq_acc, dqkv, dgate, dtab, B, T, H,
                                                    0.125),
            "bwd_2kernel": lambda: ops.attn_bwd(qkv, out, dout, gate, tab, None, lse, delta, dqkv, dgate, dtab, B, T, H, 0.125),
        }
        fl = 4.0 * B * H * T * T * 64
        for k in kinds:
            ms = timed(fns[k])
            tf = fl * (1.0 if k == "fwd" else 2.5) / ms / 1e9
            print(f"long   {k:18s} T={T:5d} {ms*1e3:10.1f} us   {tf:8.1f} TFLOP/s (algorithmic)  {tf / peak:6.3f} of peak", flush=True)
            all_ok &= check_long(k, fns[k], qkv, gate, tab, out, lse, dout, dqkv, dgate, dtab, B, T, H)
        del qkv, gate, tab, out, lse, dout, delta, dqkv, dgate, dtab, dq_acc, fns
        torch.cuda.empty_cache()
for name, B, T, H in (("base", 16, 749, 12), ("large", 8, 999, 16)):
    if args.only and args.only != name:
        continue
    D = H * 64
    torch.manual_seed(0)
    qkv = torch.randn(B, T, 3 * D, device=dev).to(torch.bfloat16)
    gate = torch.rand(B, H, T, device=dev) * 2 + 0.2
    tab = torch.randn(H, 2 * T - 1, device=dev)
    pad = torch.zeros(B, T, device=dev, dtype=torch.uint8)
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    dout = torch.randn(B, T, D, device=dev).to(torch.bfloat16)
    delta = torch.empty(B, H, T, device=dev)
    dqkv = torch.zeros(B, T, 3 * D, device=dev, dtype=torch.bfloat16)
    dgate = torch.zeros(B, H, T, device=dev)
    dtab = torch.zeros(H, 2 * T - 1, device=dev)
    dq_acc = torch.zeros(B, T, D, device=dev)
    fns = {
        "fwd": lambda: ops.attn_fwd(qkv, gate, tab, pad, out, lse, B, T, H, 0.125),
        "bwd_fused": lambda: ops.attn_bwd_fused(qkv, out, dout, gate, tab, pad, lse, delta, dq_acc, dqkv, dgate, dtab, B, T, H, 0.125),
        "bwd_2kernel": lambda: ops.attn_bwd(qkv, out, dout, gate, tab, pad, lse, delta, dqkv, dgate, dtab, B, T, H, 0.125),
    }
    # the same kernels without the gated relative-position bias (HuBERT / wav2vec2 encoders): what the bias path costs
    fns["fwd_nobias"] = lambda: ops.attn_fwd(qkv, None, None, pad, out, lse, B, T, H, 0.125)
    fns["bwd_fused_nobias"] = lambda: ops.attn_bwd_fused(qkv, out, dout, None, None, pad, lse, delta, dq_acc, dqkv, None, None, B, T, H, 0.125)
    if args.dropout > 0:
        words = torch.empty(ops.attn_dropout_mask_words(B, T, H), dtype=torch.int32, device=dev)
        fns["fwd_dropout"] = lambda: ops.attn_fwd_dropout(qkv, gate, tab, pad, out, lse, B, T, H, 0.125, args.dropout, (123, 456), words)
        fns["bwd_fused_dropout"] = lambda: ops.attn_bwd_fused_dropout(qkv, out, dout, gate, tab, pad, lse, delta, dq_acc, dqkv, dgate,
                                                                      dtab, B, T, H, 0.125, args.dropout, words)
    fl = 4.0 * B * H * T * T * 64
    for k, fn in fns.items():
        for _ in range(2):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / args.reps
        mult = 1.0 if k.startswith("fwd") else 2.5
        tf = fl * mult / ms / 1e9
        print(f"{name:6s} {k:18s} {ms*1e3:9.1f} us   {tf:8.1f} TFLOP/s (algorithmic)  {tf / peak:6.3f} of peak", flush=True)
        if name == "large" and k.startswith("bwd"):
            bias = k != "bwd_fused_nobias"
            keep = keep_mask(words, B, T, H) if k == "bwd_fused_dropout" else None
            all_ok &= check_bwd(k, fn, qkv, gate if bias else None, tab if bias else None, dout, dqkv, dgate, dtab if bias else None,
                                B, T, H, keep, args.dropout)
            del keep
# 1280-wide encoders (XLS-R 1B, MMS-1B, HuBERT X-Large) and XLS-R 2B: head widths 80 and 120, no relative-position bias, beside
# head width 64 at the same B, T, H.  Algorithmic FLOPs scale with the head width.
if args.only == "wide":
    B, T, H = 8, 999, 16
    p_w = args.dropout if args.dropout > 0 else 0.1
    for hd in (64, 80, 120):
        D = H * hd
        torch.manual_seed(0)
        qkv = torch.randn(B, T, 3 * D, device=dev).to(torch.bfloat16)
        out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
        lse = torch.empty(B, H, T, device=dev)
        dout = torch.randn(B, T, D, device=dev).to(torch.bfloat16)
        delta = torch.empty(B, H, T, device=dev)
        dqkv = torch.zeros(B, T, 3 * D, device=dev, dtype=torch.bfloat16)
        dq_acc = torch.zeros(B, T, D, device=dev)
        words = torch.empty(ops.attn_dropout_mask_words(B, T, H), dtype=torch.int32, device=dev)
        sc = hd ** -0.5
        fns = {
            "fwd": lambda: ops.attn_fwd(qkv, None, None, None, out, lse, B, T, H, sc, head_dim=hd),
            "fwd_dropout": lambda: ops.attn_fwd_dropout(qkv, None, None, None, out, lse, B, T, H, sc, p_w, (123, 456), words,
                                                        head_dim=hd),
            "bwd_fused": lambda: ops.attn_bwd_fused(qkv, out, dout, None, None, None, lse, delta, dq_acc, dqkv, None, None, B, T,
                                                    H, sc, head_dim=hd),
        }
        fl = 4.0 * B * H * T * T * hd
        for k, fn in fns.items():
            for _ in range(2):
                fn()
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            for _ in range(args.reps):
                fn()
            e1.record()
            torch.cuda.synchronize()
            ms = e0.elapsed_time(e1) / args.reps
            tf = fl * (1.0 if k.startswith("fwd") else 2.5) / ms / 1e9
            print(f"wide   hd={hd} {k:13s} {ms*1e3:9.1f} us   {tf:8.1f} TFLOP/s (algorithmic)  {tf / peak:6.3f} of peak", flush=True)
        del qkv, out, lse, dout, delta, dqkv, dq_acc, words, fns
        torch.cuda.empty_cache()
if not all_ok:
    sys.exit(1)
