"""Whole-model parity at BASELINE scale: the FULL-DEPTH WavLM-Base / WavLM-Large encoders at the frame counts of
BASELINE.json's configs (T = 749 / 999 / 1499) against the fp32 CPU oracle run on the same box.

The oracle is pinned to the unmodified reference at these sizes by tests/test_oracle_golden.py::test_long_sequence_rows_match_reference
(T = 499 and T = 1499, log-bucket branch) -- here it is the checker of the CUDA path.

Stated tolerance (bf16 activations end to end vs an fp32 oracle; the reference's own bf16-vs-fp32 forward differs by 0.093
max-abs on WavLM-Base hidden states of magnitude <= 5, SURVEY.md S17).  Because the pre-LN residual stream of WavLM-Large grows
with depth (|h| up to ~25 at layer 24 with these weights) the bound is stated RELATIVE to each layer's own scale:
    max-abs diff  <=  MAX_REL  * max|h_layer|        (MAX_REL  = 0.03)
    mean-abs diff <=  MEAN_REL * mean|h_layer|       (MEAN_REL = 0.015; bf16 has 2^-8 = 0.4 % relative spacing per rounding)
and for the post-LN WavLM-Base (|h| <= ~6 everywhere) additionally the absolute max-abs < 0.12 of the small-model tests.
Every layer's numbers are printed as a table (pytest -s) and written to gpurun_out/parity_fullscale.json when that directory
is writable.
"""
import json
import os

import pytest
import torch

from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu

MAX_REL = 0.03
MEAN_REL = 0.015
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

_SD_CACHE = {}


def state_dict_for(name, cfg):
    key = (name, cfg.encoder_layers)
    if key not in _SD_CACHE:
        _SD_CACHE.clear()  # one architecture at a time (Large is 1.26 GB of fp32)
        _SD_CACHE[key] = O.deterministic_state_dict(cfg)
    return _SD_CACHE[key]


def build(cfg, sd, device, train=False):
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(sd, strict=True)
    m = m.to(device)
    return m.train() if train else m.eval()


def record(tag, rows):
    path = os.path.join(ROOT, "gpurun_out")
    try:
        os.makedirs(path, exist_ok=True)
        fn = os.path.join(path, "parity_fullscale.json")
        data = json.load(open(fn)) if os.path.exists(fn) else {}
        data[tag] = rows
        json.dump(data, open(fn, "w"), indent=1)
    except OSError:
        pass


def layer_table(tag, got_layers, want_layers, valid_tb=None, abs_tol=None):
    """got/want: lists of [T,B,D]; valid_tb: bool [T,B] of frames that count (None = all).  Returns the rows and asserts."""
    rows, bad = [], []
    print(f"\n{tag}: layer  max|h|  mean|h|  max-abs-diff  mean-abs-diff  rel-max  rel-mean")
    for i, (g, w) in enumerate(zip(got_layers, want_layers)):
        g = g.detach().float().cpu()
        w = w.detach().float()
        assert g.shape == w.shape, (tag, i, g.shape, w.shape)
        assert torch.isfinite(g).all(), (tag, i)
        if valid_tb is not None:
            g, w = g[valid_tb], w[valid_tb]
        d = (g - w).abs()
        hm, ha = w.abs().max().item(), w.abs().mean().item()
        dm, da = d.max().item(), d.mean().item()
        rows.append(dict(layer=i, max_h=hm, mean_h=ha, max_abs=dm, mean_abs=da, rel_max=dm / hm, rel_mean=da / ha))
        print(f"{tag}: {i:5d}  {hm:6.2f}  {ha:7.3f}  {dm:12.4f}  {da:13.5f}  {dm / hm:7.4f}  {da / ha:8.5f}")
        if dm > MAX_REL * hm or da > MEAN_REL * ha or (abs_tol is not None and dm > abs_tol):
            bad.append(rows[-1])
    record(tag, rows)
    assert not bad, (tag, bad)
    return rows


def run_forward_case(tag, cfg, sd, B, L, lengths, device, abs_tol=None):
    wav, pmask = O.deterministic_waveform(B, L, seed=3, lengths=lengths)
    pm = pmask if lengths is not None else None
    n = cfg.encoder_layers
    with torch.no_grad():
        want = O.extract_features(sd, wav, cfg, padding_mask=pm, output_layer=n)
        want_final = O.extract_features(sd, wav, cfg, padding_mask=pm)  # incl. the final encoder LayerNorm of pre-LN models
    m = build(cfg, sd, device)
    with torch.no_grad():
        (xl, got_lr), fpm = m.extract_features(wav.to(device), padding_mask=pm.to(device) if pm is not None else None,
                                               ret_layer_results=True, output_layer=n)
        xf, _ = m.extract_features(wav.to(device), padding_mask=pm.to(device) if pm is not None else None)
    torch.cuda.synchronize()
    valid_tb = None
    if pm is not None:
        assert torch.equal(fpm.cpu(), want["padding_mask"])
        valid_tb = (~want["padding_mask"]).t().contiguous()
    assert len(got_lr) == n + 1 == len(want["layer_results"])
    want_layers = [h[0] if isinstance(h, tuple) else h for h in want["layer_results"]]
    got_layers = [h for h, _ in got_lr]
    layer_table(tag, got_layers, want_layers, valid_tb, abs_tol)
    layer_table(tag + ":final", [xf.transpose(0, 1)], [want_final["x"].transpose(0, 1)], valid_tb, abs_tol)
    del m
    torch.cuda.empty_cache()


def test_base_full_depth_T749(cuda_device):
    """BASELINE configs[1] geometry: WavLM-Base, 12 layers, 15 s (T = 749), post-LN, GroupNorm extractor, rel-pos + gate."""
    cfg = O.base_config()
    run_forward_case("base12_T749", cfg, state_dict_for("base", cfg), 1, 240000, None, cuda_device, abs_tol=0.12)


def test_large_full_depth_T999(cuda_device):
    """BASELINE configs[2] geometry: WavLM-Large, 24 layers, 20 s (T = 999), pre-LN, LayerNorm extractor."""
    cfg = O.large_config()
    run_forward_case("large24_T999", cfg, state_dict_for("large", cfg), 1, 320000, None, cuda_device)


def test_large_full_depth_ragged_T1499(cuda_device):
    """BASELINE configs[4] geometry: WavLM-Large, ragged {30 s, 10.03 s} (T = 1499, 12 key tiles, padded tail of 998 frames),
    compared on the valid frames under the frame padding mask."""
    cfg = O.large_config()
    L = 480000
    run_forward_case("large24_T1499_ragged", cfg, state_dict_for("large", cfg), 2, L, [L, 160480], cuda_device)


GRAD_KINDS = [
    "feature_extractor.conv_layers.0.0.weight", "feature_extractor.conv_layers.3.0.weight",
    "feature_extractor.conv_layers.6.0.weight", "layer_norm.weight", "layer_norm.bias",
    "post_extract_proj.weight", "post_extract_proj.bias", "mask_emb",
    "encoder.pos_conv.0.weight_g", "encoder.pos_conv.0.weight_v", "encoder.pos_conv.0.bias",
    "encoder.layers.0.self_attn.relative_attention_bias.weight",
    "encoder.layers.0.self_attn.grep_linear.weight", "encoder.layers.0.self_attn.grep_linear.bias",
    "encoder.layers.0.self_attn.grep_a", "encoder.layers.2.self_attn.grep_a",
    "encoder.layers.1.self_attn.q_proj.weight", "encoder.layers.1.self_attn.k_proj.weight",
    "encoder.layers.1.self_attn.v_proj.weight", "encoder.layers.1.self_attn.out_proj.weight",
    "encoder.layers.1.self_attn.q_proj.bias", "encoder.layers.1.self_attn.v_proj.bias",
    "encoder.layers.1.self_attn.out_proj.bias",
    "encoder.layers.0.self_attn_layer_norm.weight", "encoder.layers.3.final_layer_norm.bias",
    "encoder.layers.0.fc1.weight", "encoder.layers.3.fc1.bias", "encoder.layers.3.fc2.weight", "encoder.layers.0.fc2.bias",
    "encoder.layer_norm.weight",
]

# bf16 activations / gradients vs fp32: cosine > 0.999 and norm within 2 % is what the yardstick allows for the GEMM-fed
# parameters.  Two kinds sit on noisier paths and get a stated looser bound: (a) the gate parameters and the bias table sum
# tiny per-element contributions of bf16-rounded dS over T^2 entries; (b) conv layer 0 sits under 7 bf16 layers of backward.
LOOSE = {"grep_linear.weight": (0.995, 0.04), "grep_linear.bias": (0.995, 0.04), "grep_a": (0.995, 0.04),
         "relative_attention_bias.weight": (0.997, 0.03), "conv_layers.0.0.weight": (0.995, 0.04),
         "weight_g": (0.997, 0.03)}


def grad_case(tag, cfg, sd, B, L, lengths, device, feature_grad_mult=1.0):
    cfg.feature_grad_mult = feature_grad_mult
    wav, pmask = O.deterministic_waveform(B, L, seed=5, lengths=lengths)
    T = O.num_frames(L, cfg)
    # deterministic masked frames (hash), as apply_mask would produce a bool [B,T]
    mi = O.hash_uniform("maskidx", (B, T), 0.0, 1.0) < 0.3
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = O.extract_features(sdr, wav, cfg, padding_mask=pmask, mask_indices=mi)
    ref_loss = O.probe_loss(ref["x"], ref["padding_mask"], seed=7)
    ref_loss.backward()
    if feature_grad_mult != 1.0:  # GradMultiply (WavLM/modules.py:60-69; WavLM.py:333-336): scales the extractor's gradients
        for k in sdr:
            if k.startswith("feature_extractor."):
                sdr[k].grad.mul_(feature_grad_mult)
    m = build(cfg, sd, device, train=True)
    m.dropout_seed = 0
    x, fpm = m.extract_features(wav.to(device), padding_mask=pmask.to(device), mask=True, mask_indices=mi)
    loss = O.probe_loss(x.float(), fpm, seed=7)
    loss.backward()
    torch.cuda.synchronize()
    rl = ref_loss.item()
    print(f"\n{tag}: loss {loss.item():.4f} vs oracle {rl:.4f}")
    scale = (ref["x"].detach().abs().mean().item() * (~ref["padding_mask"]).sum().item() * cfg.encoder_embed_dim) ** 0.5
    assert abs(loss.item() - rl) < 0.02 * scale + 0.01 * abs(rl), (loss.item(), rl, scale)
    params = dict(m.named_parameters())
    rows, bad = [], []
    print(f"{tag}: parameter  |g| oracle  |g| gpu  norm-ratio  cosine")
    for k in GRAD_KINDS:
        if k not in sdr or sdr[k].grad is None:
            continue
        want = sdr[k].grad.double()
        got = params[k].grad.detach().double().cpu()
        nw, ng = want.norm().item(), got.norm().item()
        cos = ((got * want).sum() / (got.norm() * want.norm() + 1e-300)).item()
        cmin, ntol = 0.999, 0.02
        for suffix, (c, n_) in LOOSE.items():
            if k.endswith(suffix):
                cmin, ntol = c, n_
        rows.append(dict(param=k, ref_norm=nw, gpu_norm=ng, ratio=ng / max(nw, 1e-300), cosine=cos, cos_min=cmin, norm_tol=ntol))
        print(f"{tag}: {k:62s} {nw:10.4e} {ng:10.4e} {ng / max(nw, 1e-300):8.4f} {cos:9.6f}")
        if not (cos > cmin and abs(ng - nw) <= ntol * nw):
            bad.append(rows[-1])
    record(tag, rows)
    assert not bad, bad
    del m
    torch.cuda.empty_cache()


def test_gradients_large_width_4l_T324(cuda_device):
    """Real WavLM-Large widths (D 1024, F 4096, 16 heads, pre-LN, LayerNorm extractor), 4 layers, ragged 2 x 6.5 s (T = 324,
    three key tiles), masked frames, one parameter of every kind incl. the bias table, gate, weight-norm g and conv 0."""
    cfg = O.large_config(encoder_layers=4)
    L = 104000
    grad_case("grad_large4_T324", cfg, state_dict_for("large4", cfg), 2, L, [L, 70000], cuda_device)


def test_gradients_base_width_4l_T324(cuda_device):
    """Real WavLM-Base widths (D 768, post-LN, GroupNorm extractor), 4 layers, same batch geometry."""
    cfg = O.base_config(encoder_layers=4)
    L = 104000
    grad_case("grad_base4_T324", cfg, state_dict_for("base4", cfg), 2, L, [L, 70000], cuda_device)


def test_feature_grad_mult_recipe_value(cuda_device):
    """`feature_grad_mult = 0.1` (the released recipes; WavLM/modules.py:60-69, WavLM.py:333-336): the extractor's gradients are
    the oracle's scaled by 0.1, everything above the extractor is unchanged."""
    cfg = O.base_config(encoder_layers=2)
    L = 48000
    grad_case("grad_base2_fgm0.1", cfg, state_dict_for("base2", cfg), 2, L, [L, 40000], cuda_device, feature_grad_mult=0.1)
