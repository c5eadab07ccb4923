"""Is the eager forward pass bit-reproducible?  Runs the tiny pre-LN model (and optionally 2 layers of WavLM-Large) several times on
the same batch and span mask, interleaved with a backward pass and with allocator churn, and reports per stage (conv features, every
layer's output) whether the results are bit-identical.  python tools/debug_determinism.py [--large]"""
import argparse, os, sys
import numpy as np
import torch
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import wavlm_oracle as O
from unispeech_b200.wavlm import WavLM, WavLMConfig

ap = argparse.ArgumentParser()
ap.add_argument("--large", action="store_true")
args = ap.parse_args()
dev = torch.device("cuda:0")
cfg = O.large_config(encoder_layers=2) if args.large else O.tiny_config(pre_ln=True, encoder_layers=3)
m = WavLM(WavLMConfig(vars(cfg)))
m.load_state_dict(O.deterministic_state_dict(cfg))
m = m.to(dev).train()
B, L = 2, 16000
wav, _ = O.deterministic_waveform(B, L, seed=3)
wav = wav.to(dev)
np.random.seed(5)
T = O.num_frames(L, cfg)
mask = m.apply_mask(B, T, None)

def run(backward, churn):
    if churn:  # leave garbage in the allocator's free blocks
        junk = [torch.full((n,), float("nan"), device=dev) for n in (1 << 20, 3 << 18, 1 << 16, 12345)]
        del junk
    if m._engine is not None and m._engine.flat is not None:
        m.zero_grad_buffer()
        m._engine.prepared_version = None
    (x, lr), _ = m.extract_features(wav, padding_mask=None, mask=True, mask_indices=mask, ret_layer_results=True,
                                    output_layer=cfg.encoder_layers)
    with torch.no_grad():
        feats = m.feature_extractor(wav).transpose(1, 2).clone()
    outs = [feats] + [h.detach().clone() for h, _ in lr]
    if backward:
        x.float().sum().backward()
    torch.cuda.synchronize()
    return outs

ref = run(False, False)
names = ["conv features"] + [f"layer {i}" for i in range(len(ref) - 1)]
for trial, (bw, ch) in enumerate([(False, False), (True, False), (False, True), (True, True), (False, True), (False, False)]):
    got = run(bw, ch)
    line = []
    for n, a, b in zip(names, ref, got):
        same = torch.equal(a, b)
        line.append(f"{n}: {'==' if same else 'DIFF max %.3g' % (a.float() - b.float()).abs().max().item()}")
    print(f"trial {trial} (backward={bw}, churn={ch}): " + "; ".join(line), flush=True)
