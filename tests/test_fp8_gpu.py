"""FP8 inference path on the GPU: the quantisation kernels bit-exact against the reference rule (unispeech_b200/fp8.py), the e4m3
row GEMM against the float64 product of its dequantised operands at every encoder projection shape, and `extract_features(fp8=True)`
against bf16 on real speech and at full depth.  The measured figures are printed (-s) and recorded in DESIGN.md section 5e."""
import os

import numpy as np
import pytest
import torch

from oracle import wavlm_oracle as O
from unispeech_b200 import _lib as L
from unispeech_b200 import ops
from unispeech_b200 import workloads as W
from unispeech_b200.fp8 import dequantize_rows, quantize_rows_reference
from unispeech_b200.wavlm import WavLM, WavLMConfig

pytestmark = pytest.mark.gpu
U8 = torch.uint8


def _ragged_valid(dev, rows, batches):
    v = [rows, max(1, rows * 4 // 7), 41][:batches]
    return torch.tensor(v, dtype=torch.int32, device=dev), v


def _quant(x, valid=None):
    B, T, D = x.shape
    q, s = torch.empty(B, T, D, dtype=U8, device=x.device), torch.empty(B * T, dtype=torch.float32, device=x.device)
    ops.quantize_rows_fp8(x, T * D, D, T, B, D, q, T * D, D, s, valid=valid)
    return q, s


def test_quantize_rows_bit_exact_ragged(cuda_device):
    g = torch.Generator(device=cuda_device).manual_seed(0)
    for D in (128, 768, 1920, 5120, 7680):
        B, T = 3, 133
        x = (torch.randn(B, T, D, device=cuda_device, generator=g) * torch.logspace(-6, 3, T, device=cuda_device)[None, :, None])
        x = x.to(torch.bfloat16)
        x[1, 5] = 0
        x[0, 3] = torch.tensor(2.0 ** -126, dtype=torch.bfloat16)  # amax below 2^-119 (448 / amax would overflow): q = 0, s = 0
        x[0, 3, ::3] = 0
        vd, v = _ragged_valid(cuda_device, T, B)
        q, s = _quant(x, vd)
        qr, sr = quantize_rows_reference(x)
        qr, sr = qr.view(U8).clone(), sr.view(B, T).clone()
        for b, n in enumerate(v):
            qr[b, n:] = 0
            sr[b, n:] = 0
        bad = (q != qr).reshape(B * T, -1).any(-1).nonzero().flatten().tolist()
        assert torch.equal(q, qr), (D, len(bad), bad[:8])
        assert torch.equal(s.view(B, T), sr), D
        assert torch.all(q[0, 3] == 0) and s.view(B, T)[0, 3].item() == 0


@pytest.mark.parametrize("D", [128, 256, 768, 1024, 1280, 1920])
def test_layer_norm_fp8(cuda_device, D):
    g = torch.Generator(device=cuda_device).manual_seed(D)
    B, T = 3, 77
    H = D // 64
    x = (torch.randn(B, T, D, device=cuda_device, generator=g) * 3 + 1).to(torch.bfloat16)
    gamma = torch.rand(D, device=cuda_device, generator=g) + 0.5
    beta = torch.randn(D, device=cuda_device, generator=g) * 0.1
    vd, v = _ragged_valid(cuda_device, T, B)
    f = lambda *s: torch.empty(*s, dtype=torch.float32, device=cuda_device)
    gate_ok = D == H * 64 and 256 <= D <= 1280
    gw, gb, ga = torch.randn(8, 64, device=cuda_device, generator=g) * 0.1, torch.randn(8, device=cuda_device, generator=g), \
        torch.randn(H, device=cuda_device, generator=g)
    y, m1, r1, q, s = torch.empty_like(x), f(B * T), f(B * T), torch.empty(B, T, D, dtype=U8, device=cuda_device), f(B * T)
    gate = f(B, H, T) if gate_ok else None
    ops.layer_norm_fwd_fp8(x, T * D, D, gamma, beta, y, T * D, D, m1, r1, q, T * D, D, s, T, B, D,
                           gw if gate_ok else None, gb if gate_ok else None, ga if gate_ok else None, H, gate, valid=vd)
    y0, m0, r0 = torch.empty_like(x), f(B * T), f(B * T)
    ops.layer_norm_fwd(x, T * D, D, gamma, beta, y0, T * D, D, m0, r0, T, B, D, valid=vd)
    def where(a, b):
        bad = (a != b).reshape(B * T, -1).any(-1).nonzero().flatten().tolist()
        return f"D={D}: {len(bad)} rows differ, first {bad[:8]}"
    assert torch.equal(y, y0), where(y, y0)
    assert torch.equal(m1, m0), where(m1, m0)
    assert torch.equal(r1, r0), where(r1, r0)
    qr, sr = quantize_rows_reference(y)
    assert torch.equal(q, qr.view(U8)), where(q, qr.view(U8))
    assert torch.equal(s, sr.view(-1)), where(s, sr.view(-1))
    for b, n in enumerate(v):
        assert torch.all(q[b, n:] == 0) and torch.all(s.view(B, T)[b, n:] == 0)
    # fp8 only (no y, no statistics): the same q and s
    q2, s2 = torch.empty_like(q), f(B * T)
    ops.layer_norm_fwd_fp8(x, T * D, D, gamma, beta, None, 0, 0, None, None, q2, T * D, D, s2, T, B, D, valid=vd)
    assert torch.equal(q2, q) and torch.equal(s2, s)
    if gate_ok:
        for b, n in enumerate(v):
            assert torch.all(gate[b, :, n:] == 1)                  # padded frames: gate 1
        # valid frames, at every width (b200s_gate_fwd sums in another order: not bit for bit)
        g0 = f(B, H, T)
        ops.gate_fwd(y, T * D, D, T, B, H, gw, gb, ga, g0)
        for b, n in enumerate(v):
            assert torch.allclose(gate[b, :, :n], g0[b, :, :n], atol=1e-5, rtol=0), (D, b)
    if gate_ok and D <= 1024:  # (b200s_layer_norm_gate_fwd takes D = 256 .. 1024)
        y1, g1 = torch.empty_like(x), f(B, H, T)
        ops.layer_norm_gate_fwd(x, T * D, D, gamma, beta, y1, T * D, D, f(B * T), f(B * T), T, B, D, gw, gb, ga, H, g1, valid=vd)
        # b200s_layer_norm_gate_fwd's own y may differ from b200s_layer_norm_fwd's in the last bit of a few rows (it forms the mean
        # differently, and at 512..1024 sums in another order): the gate is a function of the stored y, so rows whose y agrees
        # bit for bit have bit-identical gates, and the rest agree to the bf16 rounding of y
        same = (y1 == y).all(-1)
        assert same.float().mean().item() > 0.5
        assert torch.equal(g1.permute(0, 2, 1)[same], gate.permute(0, 2, 1)[same])
        assert torch.allclose(g1, gate, atol=2e-3, rtol=0)


def _shapes():
    out = []
    for name in ("tiny", "base", "large", "xlsr1b", "xlsr2b"):
        cfg, _, _ = W.model_config(name)
        D, F = cfg["encoder_embed_dim"], cfg["encoder_ffn_embed_dim"]
        for proj, K, N in (("qkv", D, 3 * D), ("out_proj", D, D), ("fc1", D, F), ("fc2", F, D)):
            out.append((name, proj, K, N))
    return out


def _prep_weight(w):
    N, K = w.shape
    import struct
    q, s = torch.empty(N, K, dtype=U8, device=w.device), torch.empty(N, dtype=torch.float32, device=w.device)
    d = torch.frombuffer(bytearray(struct.pack("<QQQii", w.data_ptr(), q.data_ptr(), s.data_ptr(), N, K)), dtype=U8).to(w.device)
    ops.prep_linear_fp8_batched(d, 1, N)
    return q, s


@pytest.mark.parametrize("name,proj,K,N", _shapes())
def test_gemm_fp8_against_float64(cuda_device, name, proj, K, N):
    g = torch.Generator(device=cuda_device).manual_seed(K * 7 + N)
    B, T = 3, 300
    vd, v = _ragged_valid(cuda_device, T, B)
    a = (torch.randn(B, T, K, device=cuda_device, generator=g) * (1 + torch.rand(B, T, 1, device=cuda_device, generator=g))).to(
        torch.bfloat16)
    w = torch.randn(N, K, device=cuda_device, generator=g) * 0.02
    bias = torch.randn(N, device=cuda_device, generator=g) * 0.1
    res = torch.randn(B, T, N, device=cuda_device, generator=g).to(torch.bfloat16)
    qa, sa = _quant(a, vd)
    qw, sw = _prep_weight(w)
    qwr, swr = quantize_rows_reference(w)
    assert torch.equal(qw, qwr.view(U8)) and torch.equal(sw, swr)       # weight preparation: the same rule, bit-exact
    A = dequantize_rows(qa.view(torch.float8_e4m3fn), sa.view(B, T))
    Wd = dequantize_rows(qw.view(torch.float8_e4m3fn), sw)
    prod = A @ Wd.T + bias.double()
    worst = []
    for epi in ("bias", "bias+gelu", "bias+res"):
        out = torch.full((B, T, N), float("nan"), dtype=torch.bfloat16, device=cuda_device)
        if epi == "bias":
            e, ref = L.make_epilogue(bias=bias), prod
        elif epi == "bias+gelu":
            e, ref = L.make_epilogue(bias=bias, gelu=2), torch.nn.functional.gelu(prod)
        else:
            e, ref = L.make_epilogue(bias=bias, res1=res, res1_bs=T * N, res1_ld=N), prod + res.double()
        ops.gemm_rows_fp8(qa, sa, T * K, K, T, B, K, qw, sw, N, out, T * N, N, e, valid=vd)
        for b, n in enumerate(v):
            dead = (n + 127) // 128 * 128
            assert torch.all(out[b, dead:] == 0), (epi, b)              # tiles past valid[b]: zeros
            d = (out[b, :n].double() - ref[b, :n]).abs().max().item()
            m = ref[b, :n].abs().max().item()
            worst.append(d / m)
            assert d <= 4e-3 * m, (name, proj, epi, b, d, m)
    print(f"fp8 GEMM {name} {proj} K={K} N={N}: max|out-ref|/max|ref| = {max(worst):.2e}")


def test_gemm_fp8_argument_errors(cuda_device):
    q = torch.zeros(128, 192, dtype=U8, device=cuda_device)
    s = torch.zeros(128, dtype=torch.float32, device=cuda_device)
    out = torch.empty(128, 128, dtype=torch.bfloat16, device=cuda_device)
    with pytest.raises(RuntimeError, match="multiple of 128"):
        ops.gemm_rows_fp8(q, s, 0, 192, 128, 1, 192, q, s, 128, out, 0, 128)
    with pytest.raises(RuntimeError, match="res1"):
        ops.gemm_rows_fp8(q, s, 0, 128, 128, 1, 128, q, s, 128, out, 0, 128, L.make_epilogue(res2=out, res2_ld=128))


# ------------------------------------------------------------------------------------------------ model level
GOLD = os.path.join(os.path.dirname(__file__), "golden", "vox_real_large2l.npz")


def _vox_batch(g):
    pcm, lengths = g["pcm"], [int(v) for v in g["lengths"]]
    B, Ln = pcm.shape
    wav = torch.zeros(B, Ln)
    pmask = torch.zeros(B, Ln, dtype=torch.bool)
    for b, n in enumerate(lengths):
        w = torch.from_numpy(pcm[b, :n].astype(np.float32)) / 32768.0
        wav[b, :n] = torch.nn.functional.layer_norm(w, (n,))
        pmask[b, n:] = True
    return wav, pmask


# fp8 error / bf16 error against the reference's numbers on real speech (measured on an H100: see DESIGN.md section 5e)
VOX_ERR_RATIO = 12.0


def test_real_speech_fp8_against_golden(cuda_device):
    g = np.load(GOLD)
    cfg = O.large_config(encoder_layers=2)
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(O.deterministic_state_dict(cfg))
    m = m.to(cuda_device).eval()
    wav, pmask = _vox_batch(g)
    with torch.no_grad():
        xb, _ = m.extract_features(wav.to(cuda_device), padding_mask=pmask)
        x8, fpm = m.extract_features(wav.to(cuda_device), padding_mask=pmask, fp8=True)
    rows = torch.from_numpy(g["rows"])
    keep = ~torch.from_numpy(g["frame_padding_mask"])[:, rows]
    want = torch.from_numpy(g["x_final"].astype(np.float32))
    err = {}
    for k, x in (("bf16", xb), ("fp8", x8)):
        d = (x[:, rows.to(x.device)].float().cpu() - want)[keep].abs()
        err[k] = (d.max().item(), d.mean().item())
    print(f"real speech, 2-layer Large vs golden (max, mean abs): bf16 {err['bf16']}, fp8 {err['fp8']}")
    assert err["fp8"][1] <= VOX_ERR_RATIO * err["bf16"][1], err
    assert err["fp8"][0] <= VOX_ERR_RATIO * err["bf16"][0], err


def _cos_frames(a, b):
    a, b = a.float().reshape(-1, a.shape[-1]), b.float().reshape(-1, b.shape[-1])
    return torch.nn.functional.cosine_similarity(a, b, dim=-1)


# per-frame cosine similarity of fp8 against bf16 (default init, seeded input; measured on an H100: DESIGN.md section 5e)
FULL_DEPTH_COS = {"large": 0.99, "xlsr2b": 0.985}


@pytest.mark.parametrize("name", ["large", "xlsr2b"])
def test_full_depth_cosine(cuda_device, name):
    cfg, _, _ = W.model_config(name)
    torch.manual_seed(0)
    m = WavLM(WavLMConfig(cfg)).to(cuda_device).eval()
    wav = torch.randn(2, 4 * W.SR, generator=torch.Generator().manual_seed(1)).to(cuda_device)
    worst = {}
    with torch.no_grad():
        for layer in (6, 12, None):
            xb, _ = m.extract_features(wav, output_layer=layer)
            x8, _ = m.extract_features(wav, output_layer=layer, fp8=True)
            c = _cos_frames(xb, x8)
            worst[layer] = (c.min().item(), c.mean().item())
    print(f"full depth {name}: per-frame cosine fp8 vs bf16 (min, mean) by output_layer: {worst}")
    for layer, (cmin, _) in worst.items():
        assert cmin >= FULL_DEPTH_COS[name], (name, layer, worst)


def _tiny(cuda_device, pre_ln):
    cfg = O.tiny_config(pre_ln=pre_ln)
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(O.deterministic_state_dict(cfg))
    return m.to(cuda_device).eval()


@pytest.mark.parametrize("pre_ln", [False, True])
def test_behaviour(cuda_device, pre_ln):
    m = _tiny(cuda_device, pre_ln)
    wav, pmask = O.deterministic_waveform(2, 8000, seed=1, lengths=[8000, 5000])
    wav, pmask = wav.to(cuda_device), pmask.to(cuda_device)
    with torch.no_grad():
        b0, fpm0 = m.extract_features(wav, padding_mask=pmask)
        f1, _ = m.extract_features(wav, padding_mask=pmask, fp8=True)
        f2, _ = m.extract_features(wav, padding_mask=pmask, fp8=True)
        b1, _ = m.extract_features(wav, padding_mask=pmask)
        assert torch.equal(f1, f2)                                   # deterministic
        assert torch.equal(b0, b1)                                   # the bf16 path is untouched by an fp8 call
        keep = ~fpm0.reshape(-1)                                     # valid frames (padded ones hold no defined value)
        assert _cos_frames(f1, b0)[keep].min().item() > 0.99
        # other arguments behave as in bf16
        (xl, lr8), fpm8 = m.extract_features(wav, padding_mask=pmask, ret_layer_results=True, output_layer=1, fp8=True)
        (_, lrb), fpmb = m.extract_features(wav, padding_mask=pmask, ret_layer_results=True, output_layer=1)
        assert torch.equal(fpm8, fpmb) and len(lr8) == len(lrb)
        c8, _ = m.extract_features(wav, padding_mask=pmask, ret_conv=True, fp8=True)
        cb, _ = m.extract_features(wav, padding_mask=pmask, ret_conv=True)
        assert torch.equal(c8, cb)                                   # the conv stack is bf16 either way
    # forward hooks fire on every layer
    seen = []
    hs = [lyr.register_forward_hook(lambda mod, inp, out, i=i: seen.append(i)) for i, lyr in enumerate(m.encoder.layers)]
    with torch.no_grad():
        m.extract_features(wav, padding_mask=pmask, fp8=True)
    for h in hs:
        h.remove()
    assert seen == list(range(len(m.encoder.layers)))
    # an in-place weight update changes the fp8 output exactly as for a fresh model with those weights
    with torch.no_grad():
        m.encoder.layers[0].fc1.weight.mul_(1.5)
        m.encoder.layers[-1].self_attn.q_proj.weight.add_(0.01)
        u1, _ = m.extract_features(wav, padding_mask=pmask, fp8=True)
    fresh = WavLM(m.cfg)
    fresh.load_state_dict(m.state_dict())
    fresh = fresh.to(cuda_device).eval()
    with torch.no_grad():
        u2, _ = fresh.extract_features(wav, padding_mask=pmask, fp8=True)
    assert not torch.equal(u1, f1) and torch.equal(u1, u2)


def test_errors_on_device(cuda_device):
    m = _tiny(cuda_device, False)
    wav = torch.zeros(1, 8000, device=cuda_device)
    with pytest.raises(RuntimeError, match="model.eval"):
        m.train().extract_features(wav, fp8=True)
    m.eval()
    with pytest.raises(RuntimeError, match="without a backward"):
        m.extract_features(wav, fp8=True)
    with torch.no_grad(), pytest.raises(RuntimeError, match="mask=True"):
        m.extract_features(wav, mask=True, fp8=True)


def test_post_ln_hand_off(cuda_device, monkeypatch):
    """Post-LN layers: layer i's final LayerNorm writes layer i+1's e4m3 input and its gate, and layer i+1 uses them (only
    layer 0 quantises its input and computes its gate).  A hook that edits a layer output in place makes the next layer redo
    both, and the result still equals the bf16-then-quantise path's."""
    cfg = O.tiny_config(pre_ln=False, encoder_layers=3, encoder_embed_dim=256, encoder_ffn_embed_dim=512,
                        encoder_attention_heads=4)
    torch.manual_seed(0)
    m = WavLM(WavLMConfig(vars(cfg))).to(cuda_device).eval()
    wav, pmask = O.deterministic_waveform(2, 8000, seed=1, lengths=[8000, 5000])
    wav, pmask = wav.to(cuda_device), pmask.to(cuda_device)
    calls = {"quantize": 0, "gate": 0}
    q0, g0 = ops.quantize_rows_fp8, ops.gate_fwd

    def q(*a, **k):
        calls["quantize"] += 1
        return q0(*a, **k)

    def g(*a, **k):
        calls["gate"] += 1
        return g0(*a, **k)

    monkeypatch.setattr(ops, "quantize_rows_fp8", q)
    monkeypatch.setattr(ops, "gate_fwd", g)
    L_ = cfg.encoder_layers
    with torch.no_grad():
        f1, _ = m.extract_features(wav, padding_mask=pmask, fp8=True)
    # layer 0's input (1) and every layer's attention and GELU outputs (2 L); one gate, layer 0's
    assert calls == {"quantize": 2 * L_ + 1, "gate": 1}, calls
    calls.update(quantize=0, gate=0)
    def edit_in_place(mod, inp, out):  # multiplies by one: the values stay, the version counter moves
        out[0].mul_(1.0)

    h = m.encoder.layers[0].register_forward_hook(edit_in_place)
    with torch.no_grad():
        f2, _ = m.extract_features(wav, padding_mask=pmask, fp8=True)
    h.remove()
    assert calls == {"quantize": 2 * L_ + 2, "gate": 2}, calls  # layer 1 redid both
    assert torch.equal(f1, f2)
