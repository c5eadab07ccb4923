"""Feature-extractor conv biases (`conv_bias=True`: wav2vec 2.0 Large / XLS-R-style `layer_norm` extractors) on the GPU.

* layer 0, op level, against a float64 restatement built from the kernel's own inputs: LayerNorm mode forward, d bias and the
  unchanged dw / dgamma / dbeta under all three backward variants (separate dconv workspace, workspace aliasing the incoming
  gradient, no workspace); GroupNorm mode, where the bias cancels exactly (output bit-identical to the bias-free call, d bias zero);
* layers 1-6 through the engine and the whole model against the fp32 oracle, both extractor modes, dense and ragged batches
  (including an utterance with a single valid frame);
* a few `Wav2VecEncoder` fine-tuning steps with channel masking and FusedAdam."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu


def _conv0_case(dev, C, B, L, kind, seed):
    g = torch.Generator(device=dev).manual_seed(seed)
    wav = torch.randn(B, L, device=dev, generator=g) * 0.3
    if kind == "dc":        # DC offset: the conv output carries a large per-channel constant the bias adds to
        wav += 0.5
    if kind == "ragged":    # zero-padded tails
        for b in range(1, B):
            wav[b, L * (b + 1) // (B + 1):] = 0
    k, s = 10, 5
    w = torch.randn(C, 1, k, device=dev, generator=g) * 0.3
    gamma = torch.rand(C, device=dev, generator=g) + 0.5
    beta = torch.randn(C, device=dev, generator=g) * 0.1
    bias = torch.randn(C, device=dev, generator=g) * 0.5
    T = (L - k) // s + 1
    return wav, w, gamma, beta, bias, k, s, T


def _ref_ln(wav, w, gamma, beta, bias, s, da):
    """float64: gelu(LayerNorm_C(conv1d(wav, w, bias))) and its gradients for the upstream gradient `da` [B,T,C]."""
    p = [t.double().clone().requires_grad_(True) for t in (w, gamma, beta, bias)]
    y = F.conv1d(wav.double().unsqueeze(1), p[0], p[3], stride=s).transpose(1, 2)
    y = F.gelu(F.layer_norm(y, (y.shape[-1],), p[1], p[2], 1e-5))
    (y * da.double()).sum().backward()
    return y.detach(), [q.grad for q in p]


def _close(name, got, want, rel):
    err = (got.double() - want).abs().max().item()
    scale = want.abs().max().item()
    assert err <= rel * scale + 1e-6, (name, err, scale)


@pytest.mark.parametrize("C,B,L,kind", [(512, 8, 320000, "noise"), (512, 16, 240000, "dc"), (512, 3, 16000, "ragged"),
                                        (64, 3, 16000, "ragged"), (64, 2, 8000, "dc")])
@pytest.mark.parametrize("ws", ["separate", "alias", "none"])
def test_conv0_layer_norm_bias(cuda_device, C, B, L, kind, ws):
    from unispeech_b200 import ops
    dev = cuda_device
    wav, w, gamma, beta, bias, k, s, T = _conv0_case(dev, C, B, L, kind, seed=C + B + len(kind))
    out = torch.empty(B, T, C, dtype=torch.bfloat16, device=dev)
    fmean, frstd = torch.empty(B, T, device=dev), torch.empty(B, T, device=dev)
    ops.conv0_fwd(wav, L, B, T, C, k, s, w, gamma, beta, 1, None, fmean, frstd, out, T * C, bias=bias)
    da = (torch.randn(B, T, C, device=dev) * 0.1).to(torch.bfloat16)
    want, (dw_r, dg_r, db_r, dbias_r) = _ref_ln(wav, w, gamma, beta, bias, s, da)
    # forward: bf16 output of an fp32 computation (half an ulp of bf16, 2^-9 relative, plus fp32 noise)
    err = (out.double() - want).abs()
    assert bool((err <= 2.0 ** -8 * want.abs() + 2e-3).all()), err.max().item()
    dw, dg, db, dbias = (torch.zeros_like(t) for t in (w, gamma, beta, bias))
    da_in = da.clone()
    wsbuf = {"separate": torch.empty(B, T, C, dtype=torch.bfloat16, device=dev), "alias": da_in, "none": None}[ws]
    ops.conv0_bwd(wav, L, B, T, C, k, s, w, gamma, beta, 1, None, None, fmean, frstd, da_in, T * C, dw, dg, db,
                  dconv_ws=wsbuf, ws_bs=T * C, bias=bias, dbias=dbias)
    torch.cuda.synchronize()
    # sums over B*T frames of fp32 (workspace variants: bf16-rounded dconv) terms: 1 % of the largest entry
    _close("dbias", dbias, dbias_r, 1e-2)
    _close("dw", dw, dw_r, 1e-2)
    _close("dgamma", dg, dg_r, 1e-2)
    _close("dbeta", db, db_r, 1e-2)


@pytest.mark.parametrize("C,B,L", [(512, 8, 320000), (64, 3, 16000)])
def test_conv0_group_norm_bias_cancels(cuda_device, C, B, L):
    """GroupNorm(C, C) normalises each (utterance, channel) over all frames: a per-channel constant shifts the mean by it and
    leaves the variance unchanged, so the bias has no effect and no gradient."""
    from unispeech_b200 import ops
    dev = cuda_device
    wav, w, gamma, beta, bias, k, s, T = _conv0_case(dev, C, B, L, "dc", seed=7)
    outs = []
    for b in (None, bias):
        out = torch.empty(B, T, C, dtype=torch.bfloat16, device=dev)
        stats = torch.empty(B * C * 2 + B * 128, dtype=torch.float64, device=dev)
        ops.conv0_fwd(wav, L, B, T, C, k, s, w, gamma, beta, 0, stats, None, None, out, T * C, bias=b)
        outs.append((out, stats))
    assert torch.equal(outs[0][0], outs[1][0])
    da = (torch.randn(B, T, C, device=dev) * 0.1).to(torch.bfloat16)
    dw, dg, db, dbias = (torch.zeros_like(t) for t in (w, gamma, beta, bias))
    bstats = torch.empty(B, C, 12, dtype=torch.float32, device=dev)
    ops.conv0_bwd(wav, L, B, T, C, k, s, w, gamma, beta, 0, outs[1][1], bstats, None, None, da, T * C, dw, dg, db,
                  bias=bias, dbias=dbias)
    torch.cuda.synchronize()
    assert dbias.abs().max().item() == 0
    if C == 64:   # the reference's own d bias is rounding noise next to the weight gradient
        p = [t.double().clone().requires_grad_(True) for t in (w, bias)]
        y = F.conv1d(wav.double().unsqueeze(1), p[0], p[1], stride=s)
        y = F.gelu(F.group_norm(y, C, gamma.double(), beta.double(), 1e-5)).transpose(1, 2)
        (y * da.double()).sum().backward()
        assert p[1].grad.abs().max().item() < 1e-9 * max(1.0, p[0].grad.abs().max().item())


# ------------------------------------------------------------------------------------------------------------------ model
def _cos_rel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double()
    cos = ((got * want).sum() / (got.norm() * want.norm() + 1e-30)).item()
    rel = abs(got.norm().item() - want.norm().item()) / (want.norm().item() + 1e-30)
    return cos, rel


MODELS = {
    # wav2vec 2.0 Large style: LayerNorm extractor with conv biases, pre-LN, no relative-position bias, D = 1024
    "w2v_large_style": lambda: O.large_config(encoder_layers=2, conv_bias=True, relative_position_embedding=False,
                                              gru_rel_pos=False),
    "default_mode_bias": lambda: O.base_config(encoder_layers=2, conv_bias=True),
}


@pytest.mark.parametrize("name", sorted(MODELS))
@pytest.mark.parametrize("lengths", [None, [16000, 9000, 320]])   # 320 samples: a single valid frame
def test_model_with_conv_bias_vs_oracle(cuda_device, name, lengths):
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    dev = cuda_device
    cfg = MODELS[name]()
    sd = O.deterministic_state_dict(cfg)
    assert all(f"feature_extractor.conv_layers.{i}.0.bias" in sd for i in range(7))
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(sd, strict=True)
    m = m.to(dev).train()
    B, L = (3, 16000) if lengths is not None else (2, 16000)
    wav, pmask = O.deterministic_waveform(B, L, seed=5, lengths=lengths)
    pm = pmask if lengths is not None else None
    x, fpm = m.extract_features(wav.to(dev), padding_mask=pm.to(dev) if pm is not None else None)
    O.probe_loss(x.float(), fpm, seed=3).backward()
    torch.cuda.synchronize()
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = O.extract_features(sdr, wav, cfg, padding_mask=pm)
    O.probe_loss(ref["x"], ref["padding_mask"], seed=3).backward()
    if lengths is not None:
        assert int((~ref["padding_mask"][2]).sum()) == 1
    d = x.detach().float().cpu() - ref["x"].detach()
    if ref["padding_mask"] is not None:
        d = d[~ref["padding_mask"]]
    # DESIGN.md section 1: hidden states max-abs < 0.12, mean-abs < 0.02
    assert d.abs().max().item() < 0.12 and d.abs().mean().item() < 0.02, (d.abs().max().item(), d.abs().mean().item())
    params = dict(m.named_parameters())
    ln_mode = cfg.extractor_mode == "layer_norm"
    bad = []
    for k, p in params.items():
        if not k.startswith("feature_extractor") and k != "post_extract_proj.weight":
            continue
        if k == "feature_extractor.conv_layers.0.0.bias" and not ln_mode:
            # GroupNorm cancels it: exactly zero here, rounding noise in the reference
            assert p.grad.abs().max().item() == 0
            assert sdr[k].grad.abs().max().item() < 1e-4 * sdr["feature_extractor.conv_layers.0.0.weight"].grad.abs().max().item()
            continue
        # DESIGN.md section 1: GEMM-fed weights cosine > 0.999 / norm within 2 %; conv 0, the norms and the bias vectors (column
        # sums of bf16 gradients) cosine > 0.995 / norm within 4 %
        gemm_fed = k.endswith(".0.weight") and not k.startswith("feature_extractor.conv_layers.0.") or k == "post_extract_proj.weight"
        cmin, rmax = (0.999, 0.02) if gemm_fed else (0.995, 0.04)
        cos, rel = _cos_rel(p.grad, sdr[k].grad)
        if not (cos > cmin and rel < rmax):
            bad.append((k, cos, rel))
    assert not bad, bad


def test_conv_bias_gradients_live_in_the_flat_buffer_and_train(cuda_device):
    """End to end: Wav2VecEncoder around the wav2vec 2.0 Large-style model with channel masking and a `proj` head, a few steps
    with FusedAdam: finite loss, conv-bias gradients are views of the flat buffer's conv range, the optimizer's table covers them
    and every parameter moves."""
    from unispeech_b200.engine import build_flat_grads
    from unispeech_b200.fairseq_encoder import Wav2VecEncoder
    from unispeech_b200.optim import FusedAdam
    from unispeech_b200.wav2vec2 import Wav2Vec2Config, Wav2Vec2Model
    dev = cuda_device
    cfg = O.large_config(encoder_layers=2, conv_bias=True, relative_position_embedding=False, gru_rel_pos=False,
                         mask_channel_prob=0.5, mask_channel_length=64)
    m = Wav2Vec2Model(Wav2Vec2Config(vars(cfg)))
    sd = O.deterministic_state_dict(cfg)
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys
    assert all(k.startswith(("quantizer.", "project_q.", "final_proj.")) for k in res.missing_keys), res.missing_keys
    enc = Wav2VecEncoder(m, apply_mask=True, output_dim=32).to(dev).train()
    wav, pmask = O.deterministic_waveform(2, 16000, seed=8, lengths=[16000, 12000])
    np.random.seed(5)
    enc(wav.to(dev), pmask)["encoder_out"].float().pow(2).mean().backward()
    opt = FusedAdam(m, lr=1e-3)
    proj_opt = torch.optim.SGD(enc.proj.parameters(), lr=1e-2)
    biases = [blk[0].bias for blk in m.feature_extractor.conv_layers]
    lo, hi = m._engine.flat.flat.data_ptr(), m._engine.flat.flat.data_ptr() + 4 * m._engine.flat.flat.numel()
    _, ranges, _ = build_flat_grads(m, "cpu")
    c0, c1 = ranges["conv"]
    owned = {id(p) for p, _ in opt._ptrs}
    for b in biases:
        assert lo <= b.grad.data_ptr() < hi
        off = m._engine.flat.offsets[id(b)]
        assert c0 <= off and off + b.numel() <= c1
        assert id(b) in owned
    before = {k: p.detach().clone() for k, p in m.named_parameters()}
    opt.zero_grad()
    proj_opt.zero_grad()
    T = O.num_frames(16000, cfg)
    tgt = torch.randint(1, 32, (2, 6), generator=torch.Generator().manual_seed(1)).to(dev)
    for step in range(3):
        out = enc(wav.to(dev), pmask)
        lp = F.log_softmax(out["encoder_out"].float(), dim=-1)
        in_len = (~out["padding_mask"]).sum(1)
        loss = F.ctc_loss(lp, tgt, in_len, torch.full((2,), 6, device=dev), blank=0)
        assert torch.isfinite(loss), step
        loss.backward()
        opt.step(zero_grad=True)
        proj_opt.step()
        proj_opt.zero_grad()
    torch.cuda.synchronize()
    for k, p in m.named_parameters():
        if k.startswith(("quantizer.", "project_q.", "final_proj.")) or before[k].shape != p.shape:
            continue
        assert torch.isfinite(p).all(), k
    for b, k in zip(biases, [f"feature_extractor.conv_layers.{i}.0.bias" for i in range(7)]):
        assert (b.detach() - before[k]).abs().max().item() > 0, k
    assert T > 0
