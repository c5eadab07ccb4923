"""CTC beam-search decoding: `unispeech_b200.ctc.ctc_beam_search` against `greedy_collapse` and the encoder forward that
produces the logits.
    python tools/bench_decode.py [--calls 10] [--skip-long] [--skip-forward]
    python tools/bench_decode.py --lexicon [N] [--calls 10] [--skip-long]
Logits: bf16 in the fine-tuning wrappers' layout (the T x B x V view of a [B*T, 64] buffer), V = 32 (fairseq's letter
dictionary, "|" = 4), seeded, peaked like a trained model's (one class per frame raised by 4 nats on top of N(0, 1)).
LM: a seeded random 4-gram ARPA over 3 000 letter-spelled words (3 003 unigrams with <s>, </s>, <unk>,
and 60 000 n-grams of each order 2-4: 183 003 entries), written by this script to
a temporary directory; lm_weight 0.5, word_score 0.2.  Shapes:
  finetune   B = 8, T = 999 (20 s), beam 8 / 32 / 128, without and with the LM
  ragged     B = 8 utterances of 2 .. 30 s (T_b = 99 .. 1499), beam 32, without and with the LM
  long90k    B = 1, T = 90 000 (30 min), beam 32, without and with the LM
Library time = CUDA events around the whole call (statistics + search + backtrack), median over `--calls` (3 for long-form).
greedy_collapse = device argmax + host collapse.  extract_features = WavLM-Large (random weights, eval, no_grad) on the same
batch's audio length.
With --lexicon N (default 200 000) it measures the lexicon-constrained search instead: a seeded random lexicon of N distinct
words of 1-8 letters over the 27 letters (V = 32), and a seeded random 4-gram ARPA over those words (60 000 n-grams of each order
2-4); B = 8, T = 999 at beam 8 / 32 / 128 with smearing "none" and "max", the calls alternating with the lexicon-free search with
the same LM on the same logits (lm_weight 0.5, word_score 0.2, unk_score -1); and the 30-minute utterance at beam 32.
torchaudio's `cuda_ctc_decoder` is not compared here: on an H100 with torchaudio 2.11 its first call ends in an illegal-address
error inside torchaudio even with inputs that meet its binding's contract (DESIGN §5g records the evidence).  Prints the card
name and power limit first."""
import argparse
import os
import statistics
import subprocess
import sys
import tempfile
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import decode_oracle as DO  # noqa: E402
from unispeech_b200.ctc import ctc_beam_search, greedy_collapse  # noqa: E402
from unispeech_b200.ngram import NgramLM  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("--calls", type=int, default=10)
ap.add_argument("--skip-long", action="store_true", help="leave out the 30-minute utterance")
ap.add_argument("--skip-forward", action="store_true", help="leave out extract_features")
ap.add_argument("--lexicon", type=int, nargs="?", const=200000, default=None, metavar="N",
                help="measure the lexicon-constrained search with a random lexicon of N words")
args = ap.parse_args()
if not torch.cuda.is_available():
    sys.exit("bench_decode.py measures on a GPU; none is visible")

dev = torch.device("cuda:0")
try:
    card = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True, check=True).stdout.strip()
except (OSError, subprocess.CalledProcessError):
    card = f"{torch.cuda.get_device_name(0)}, power limit unknown"
print(f"GPU: {card}", flush=True)
LETTERS = "ETAONIHSRDLUMWCFGYPBVK'XJQZ"
SYMBOLS = ["<s>", "<pad>", "</s>", "<unk>", "|"] + list(LETTERS)
V, VP, BOUNDARY = 32, 64, 4

tmp = tempfile.mkdtemp(prefix="bench_decode_")


def bench_lexicon(n_words):
    from unispeech_b200.lexicon import Lexicon
    t0 = time.perf_counter()
    words = DO.random_words(LETTERS, n_words, seed=3, max_len=8)
    lex_path = os.path.join(tmp, "random.lex")
    with open(lex_path, "w") as f:
        f.write("\n".join(f"{w} {' '.join(w)} |" for w in words) + "\n")
    arpa4 = os.path.join(tmp, "lexicon4.arpa")
    DO.write_random_arpa(arpa4, words, order=4, seed=4, ngrams_per_order=60000)
    t1 = time.perf_counter()
    lm4 = NgramLM.from_arpa(arpa4, SYMBOLS, BOUNDARY)
    t2 = time.perf_counter()
    lex = {sm: Lexicon.from_file(lex_path, SYMBOLS, BOUNDARY, lm=lm4, smearing=sm) for sm in ("none", "max")}
    torch.cuda.synchronize()
    t3 = time.perf_counter()
    print(f"lexicon: {len(words)} words, {lex['max'].nodes} trie nodes, {lex['max'].nbytes / 2**20:.1f} MiB on the device; "
          f"4-gram LM: {len(lm4.words)} words; written in {t1 - t0:.1f} s, LM built in {t2 - t1:.1f} s, both tries in "
          f"{t3 - t2:.1f} s", flush=True)
    kw = dict(lm=lm4, lm_weight=0.5, word_score=0.2, unk_score=-1.0)
    shapes = [("finetune", [999] * 8, 999, (8, 32, 128))]
    if not args.skip_long:
        shapes.append(("long90k", [90000], 90000, (32,)))
    print(f"{'shape':>9s} {'B':>2s} {'T':>6s} {'beam':>4s} | {'free ms':>9s} {'lex none':>9s} {'lex max':>9s} | "
          f"{'us/frame':>9s}", flush=True)
    for name, T_list, T, beams in shapes:
        x, il = make_case(T_list, T)
        calls = 3 if T >= 30000 else args.calls
        for beam in beams:
            fns = {"free": lambda: ctc_beam_search(x, il, beam_size=beam, **kw),
                   "none": lambda: ctc_beam_search(x, il, beam_size=beam, lexicon=lex["none"], **kw),
                   "max": lambda: ctc_beam_search(x, il, beam_size=beam, lexicon=lex["max"], **kw)}
            ms = {k: [] for k in fns}
            for _ in range(calls):   # alternating, one call of each per round
                for k, fn in fns.items():
                    ms[k].append(cuda_ms(fn, 1))
            med = {k: statistics.median(v) for k, v in ms.items()}
            print(f"{name:>9s} {len(T_list):2d} {T:6d} {beam:4d} | {fmt(med['free'])} {fmt(med['none'])} {fmt(med['max'])} | "
                  f"{fmt(med['max'] * 1e3 / T)}", flush=True)
arpa = os.path.join(tmp, "random4.arpa")
t0 = time.perf_counter()
DO.write_random_arpa(arpa, DO.random_words(LETTERS[:20], 3000, seed=1, max_len=8), order=4, seed=2, ngrams_per_order=60000)
t1 = time.perf_counter()
lm = NgramLM.from_arpa(arpa, SYMBOLS, BOUNDARY)
torch.cuda.synchronize()
t2 = time.perf_counter()
print(f"LM: 4-gram, {len(lm.words)} words, {lm.ngram_keys.numel()} + {lm.spell_keys.numel()} table slots, {lm.dropped} dropped; "
      f"written in {t1 - t0:.1f} s, parsed + built in {t2 - t1:.1f} s", flush=True)
LM_KW = dict(lm=lm, lm_weight=0.5, word_score=0.2)


def make_case(T_list, T, seed=0):
    B = len(T_list)
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(B * T, VP, generator=g)
    lead = torch.randint(0, V, (B * T,), generator=g)
    lead[torch.rand(B * T, generator=g) < 0.5] = 0   # about half the frames lead with blank
    x[torch.arange(B * T), lead] += 4.0
    buf = x.to(torch.bfloat16).to(dev)
    return buf[:, :V].reshape(B, T, V).transpose(0, 1), torch.tensor(T_list, dtype=torch.int32, device=dev)


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


def host_ms(fn, calls):
    fn()
    torch.cuda.synchronize()
    out = []
    for _ in range(calls):
        t = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        out.append((time.perf_counter() - t) * 1e3)
    return statistics.median(out)


def fmt(v, w=9, p=3):
    return f"{'n/m':>{w}s}" if v is None else f"{v:{w}.{p}f}"


if args.lexicon is not None:
    bench_lexicon(args.lexicon)
    sys.exit(0)

shapes = [("finetune", [999] * 8, 999, (8, 32, 128)), ("ragged", [99 + 200 * i for i in range(8)], 1499, (32,))]
if not args.skip_long:
    shapes.append(("long90k", [90000], 90000, (32,)))
rows = []
for name, T_list, T, beams in shapes:
    x, il = make_case(T_list, T)
    calls = 3 if T >= 30000 else args.calls
    greedy = host_ms(lambda: greedy_collapse(x.argmax(-1).t().cpu(), T_list), calls)
    for beam in beams:
        plain = cuda_ms(lambda: ctc_beam_search(x, il, beam_size=beam), calls)
        with_lm = cuda_ms(lambda: ctc_beam_search(x, il, beam_size=beam, **LM_KW), calls)
        rows.append((name, len(T_list), max(T_list), beam, plain, with_lm, plain * 1e3 / max(T_list), greedy))
        print(f"{name} beam {beam}: done", flush=True)

fwd = {}
if not args.skip_forward:
    from unispeech_b200 import workloads as W
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    cfg, _, _ = W.model_config("large")
    torch.manual_seed(0)
    m = WavLM(WavLMConfig(cfg))
    for p in m.parameters():
        p.requires_grad_(False)
    m = m.to(dev).eval()
    for name, secs in (("finetune", 20.0),):
        wav = torch.randn(8, int(secs * W.SR), generator=torch.Generator().manual_seed(1)).to(dev)
        with torch.no_grad():
            fwd[name] = cuda_ms(lambda: m.extract_features(wav), 5)
    print(f"extract_features WavLM-Large 8 x 20 s: {fwd['finetune']:.2f} ms", flush=True)

print()
print(f"{'shape':>9s} {'B':>2s} {'T':>6s} {'beam':>4s} | {'no LM ms':>9s} {'4-gram ms':>9s} {'us/frame':>9s} | "
      f"{'greedy ms':>9s} | {'fwd ms':>9s}")
for name, B, T, beam, plain, with_lm, us, greedy in rows:
    print(f"{name:>9s} {B:2d} {T:6d} {beam:4d} | {fmt(plain)} {fmt(with_lm)} {fmt(us)} | {fmt(greedy)} | {fmt(fwd.get(name))}",
          flush=True)

