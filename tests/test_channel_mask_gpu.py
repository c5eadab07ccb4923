"""Channel masking (`mask_channel_prob > 0`, the second half of apply_mask, WavLM/WavLM.py:288-307) on the GPU.

* op level: `frame_mask_fwd/bwd` with a channel mask against a torch restatement, bit for bit except `d mask_emb` (fp32 atomics:
  summation-order bound stated at the check);
* model level: WavLM with injected span AND channel masks against the fp32 oracle's stages run with the same masks (DESIGN.md section 1
  tolerances);
* the fine-tuning wrappers (HubertEncoder / Wav2VecEncoder) drawing the masks themselves from a seeded numpy state, the whole-step CUDA
  graph with a channel mask, and the device sampler drawing channel masks."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu

HID_TOL, HID_MEAN_TOL = 0.12, 0.02   # DESIGN.md section 1: hidden states of small models, bf16 path vs fp32 oracle


def bf(t):
    return t.to(torch.bfloat16)


# ------------------------------------------------------------------------------------------------------------------ kernel
def _ref_fwd(x, mask, pad, emb, chan):
    """x[mask] = mask_emb; x[chan] = 0 (broadcast over time); x[pad] = 0 -- WavLM/WavLM.py:285-306, 574-575."""
    B, T, D = x.shape
    y = x.clone()
    if mask is not None:
        y = torch.where(mask.bool().unsqueeze(-1), bf(emb).expand(B, T, D), y)
    if chan is not None:
        y = y.masked_fill(chan.bool().unsqueeze(1), 0)
    if pad is not None:
        y = y.masked_fill(pad.bool().unsqueeze(-1), 0)
    return y


def _ref_bwd(dy, mask, pad, chan):
    """(dx, d mask_emb in float64, sum of |terms| per column): dx is zero wherever the forward overwrote x."""
    B, T, D = dy.shape
    over = torch.zeros(B, T, D, dtype=torch.bool, device=dy.device)
    if mask is not None:
        over |= mask.bool().unsqueeze(-1)
    if pad is not None:
        over |= pad.bool().unsqueeze(-1)
    if chan is not None:
        over |= chan.bool().unsqueeze(1)
    dx = dy.masked_fill(over, 0)
    sel = torch.zeros(B, T, D, dtype=torch.bool, device=dy.device)
    if mask is not None:
        sel = mask.bool().unsqueeze(-1).expand(B, T, D).clone()
        if pad is not None:
            sel &= ~pad.bool().unsqueeze(-1)
        if chan is not None:
            sel &= ~chan.bool().unsqueeze(1)
    terms = dy.double() * sel
    return dx, terms.sum((0, 1)), terms.abs().sum((0, 1)), int(sel.sum((0, 1)).max())


def _run(B, T, D, mask, pad, emb, chan, strided, seed):
    """Forward on a [B,T,D] view (the padded pos_conv buffer `xpad[:, 64:]` with batch stride (T + 128) D when `strided`) and
    backward on a contiguous gradient; returns the kernel results and the restatement's."""
    from unispeech_b200 import ops
    dev = emb.device
    g = torch.Generator(device=dev).manual_seed(seed)
    x0 = bf(torch.randn(B, T, D, device=dev, generator=g))
    if strided:
        buf = torch.zeros(B, T + 128, D, dtype=torch.bfloat16, device=dev)
        buf[:, 64:64 + T] = x0
        xv, bs = buf[:, 64:], (T + 128) * D
    else:
        buf = x0.clone()
        xv, bs = buf, T * D
    ops.frame_mask_fwd(xv, bs, D, T, B, D, mask, pad, emb, chan)
    dy0 = bf(torch.randn(B, T, D, device=dev, generator=g))
    dy = dy0.clone()
    demb = torch.zeros(D, device=dev)
    ops.frame_mask_bwd(dy, T * D, D, T, B, D, mask, pad, demb, chan)
    torch.cuda.synchronize()
    y = buf[:, 64:64 + T] if strided else buf
    if strided:   # the halo of the padded buffer is never written
        assert buf[:, :64].abs().max().item() == 0 and buf[:, 64 + T:].abs().max().item() == 0
    return y, dy, demb, _ref_fwd(x0, mask, pad, emb, chan), _ref_bwd(dy0, mask, pad, chan)


def _masks(B, T, D, dev, seed, time_mask=True, ragged=True, all_chan_utt=None):
    g = torch.Generator().manual_seed(seed)
    mask = (torch.rand(B, T, generator=g) < 0.65).to(torch.uint8) if time_mask else None
    pad = None
    if ragged:
        lengths = torch.randint(1, T + 1, (B,), generator=g)
        lengths[0] = T
        pad = (torch.arange(T)[None, :] >= lengths[:, None]).to(torch.uint8)
    chan = (torch.rand(B, D, generator=g) < 0.5).to(torch.uint8)
    if all_chan_utt is not None:
        chan[all_chan_utt] = 1
    to = lambda t: t.to(dev).contiguous() if t is not None else None
    return to(mask), to(pad), to(chan)


@pytest.mark.parametrize("B,T,D", [(8, 999, 1024), (16, 749, 768), (3, 37, 64)])
@pytest.mark.parametrize("time_mask", [True, False])
@pytest.mark.parametrize("strided", [True, False])
def test_frame_mask_with_channel_mask_matches_restatement(cuda_device, B, T, D, time_mask, strided):
    dev = cuda_device
    emb = torch.rand(D, device=dev) + 0.5
    mask, pad, chan = _masks(B, T, D, dev, seed=B * T + D, time_mask=time_mask, ragged=True, all_chan_utt=1)
    y, dy, demb, y_ref, (dx_ref, demb_ref, demb_abs, n_terms) = _run(B, T, D, mask, pad, emb, chan, strided, seed=D)
    assert torch.equal(y, y_ref)
    assert torch.equal(dy, dx_ref)
    # d mask_emb: the same bf16 terms summed in fp32 in another order; |error| <= (n - 1) u sum|terms| (u = 2^-24, n terms
    # per column), plus one rounding of the fp32 result
    bound = (n_terms * 2.0 ** -24) * demb_abs + 2.0 ** -24 * demb_ref.abs() + 1e-30
    err = (demb.double() - demb_ref).abs()
    assert bool((err <= bound).all()), (err - bound).max().item()
    if time_mask:
        # the all-channels-masked utterance contributes nothing and keeps nothing
        assert y[1].abs().max().item() == 0 and dy[1].abs().max().item() == 0
        assert demb_ref.abs().max().item() > 0
    else:
        assert demb.abs().max().item() == 0


@pytest.mark.parametrize("B,T,D", [(8, 999, 1024), (3, 37, 64)])
def test_frame_mask_without_channel_mask_is_the_old_call(cuda_device, B, T, D):
    """`chan_mask=None` (the default) runs the time-mask-only kernel: same result as the positional call without the argument."""
    from unispeech_b200 import ops
    dev = cuda_device
    emb = torch.rand(D, device=dev)
    mask, pad, _ = _masks(B, T, D, dev, seed=5)
    x = bf(torch.randn(B, T, D, device=dev))
    a, b = x.clone(), x.clone()
    ops.frame_mask_fwd(a, T * D, D, T, B, D, mask, pad, emb)
    ops.frame_mask_fwd(b, T * D, D, T, B, D, mask, pad, emb, chan_mask=None)
    da, db = x.clone(), x.clone()
    ga, gb = torch.zeros(D, device=dev), torch.zeros(D, device=dev)
    ops.frame_mask_bwd(da, T * D, D, T, B, D, mask, pad, ga)
    ops.frame_mask_bwd(db, T * D, D, T, B, D, mask, pad, gb, chan_mask=None)
    torch.cuda.synchronize()
    ref = _ref_fwd(x, mask, pad, emb, None)
    assert torch.equal(a, ref) and torch.equal(b, ref)
    dx_ref, demb_ref, demb_abs, n = _ref_bwd(x, mask, pad, None)
    assert torch.equal(da, dx_ref) and torch.equal(db, dx_ref)
    bound = (n * 2.0 ** -24) * demb_abs + 2.0 ** -24 * demb_ref.abs() + 1e-30
    assert bool(((gb.double() - demb_ref).abs() <= bound).all())


# ------------------------------------------------------------------------------------------------------------------ model
def _oracle_masked(sd, wav, cfg, pmask, mi, ci):
    """oracle.extract_features (WavLM/WavLM.py:323-375) with the channel half of apply_mask: after `x[mask_indices] = mask_emb`
    (:285-286) comes `x[mask_channel_indices] = 0` (:304-306), the channel mask broadcast over time."""
    feats = O.conv_feature_extractor(sd, wav, cfg).transpose(1, 2)
    C = feats.shape[-1]
    feats = F.layer_norm(feats, (C,), sd["layer_norm.weight"], sd["layer_norm.bias"], 1e-5)
    pm = O.frame_padding_mask(pmask, feats.size(1)) if pmask is not None else None
    x = F.linear(feats, sd["post_extract_proj.weight"], sd["post_extract_proj.bias"])
    x = torch.where(mi.unsqueeze(-1), sd["mask_emb"].to(x.dtype), x)
    x = x.masked_fill(ci.unsqueeze(1), 0.0)
    x, _ = O.encoder(sd, x, pm, cfg)
    return x, pm


def _cos_rel(got, want):
    got, want = got.detach().double().cpu(), want.detach().double()
    cos = ((got * want).sum() / (got.norm() * want.norm() + 1e-30)).item()
    rel = abs(got.norm().item() - want.norm().item()) / (want.norm().item() + 1e-30)
    return cos, rel


MODEL_CASES = {
    # name: (config, B, L, lengths)
    "tiny_ragged": (lambda: O.tiny_config(pre_ln=False), 2, 8000, [8000, 5000]),
    "base2l_ragged": (lambda: O.base_config(encoder_layers=2), 2, 16000, [16000, 11000]),
    "large2l": (lambda: O.large_config(encoder_layers=2), 1, 16000, None),
}


@pytest.mark.parametrize("name", sorted(MODEL_CASES))
def test_model_with_channel_mask_vs_oracle(cuda_device, name):
    from unispeech_b200.masking import compute_mask_indices
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    dev = cuda_device
    mk, B, L, lengths = MODEL_CASES[name]
    cfg = mk()
    D = cfg.encoder_embed_dim
    sd = O.deterministic_state_dict(cfg)
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(sd, strict=True)
    m = m.to(dev).train()
    wav, pmask = O.deterministic_waveform(B, L, seed=4, lengths=lengths)
    T = O.num_frames(L, cfg)
    fpm = O.frame_padding_mask(pmask, T) if lengths is not None else None
    np.random.seed(21)
    mi = torch.from_numpy(compute_mask_indices((B, T), fpm, 0.65, 10, "static", 0, min_masks=2))
    ci = torch.from_numpy(compute_mask_indices((B, D), None, 0.5, min(64, D // 4), "static", 0))
    assert ci.any() and not ci.all()
    x, fpm_got = m.extract_features(wav.to(dev), padding_mask=pmask.to(dev) if lengths is not None else None, mask=True,
                                    mask_indices=mi, mask_channel_indices=ci)
    loss = O.probe_loss(x.float(), fpm_got, seed=2)
    loss.backward()
    torch.cuda.synchronize()
    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    want, pm = _oracle_masked(sdr, wav, cfg, pmask if lengths is not None else None, mi, ci)
    O.probe_loss(want, pm, seed=2).backward()
    d = (x.detach().float().cpu() - want.detach())
    if pm is not None:
        d = d[~pm]
    assert torch.isfinite(x.float()).all()
    assert d.abs().max().item() < HID_TOL and d.abs().mean().item() < HID_MEAN_TOL, (d.abs().max().item(), d.abs().mean().item())
    params = dict(m.named_parameters())
    # DESIGN.md section 1: GEMM-fed parameters cosine > 0.999, norm within 2 %; conv 0 and mask_emb (a column sum of bf16
    # gradients over the masked frames) cosine > 0.995, norm within 4 %
    keys = {"post_extract_proj.weight": (0.999, 0.02), "post_extract_proj.bias": (0.999, 0.02), "mask_emb": (0.995, 0.04),
            "feature_extractor.conv_layers.0.0.weight": (0.995, 0.04)}
    for i in range(1, len(O.conv_layers_of(cfg))):
        keys[f"feature_extractor.conv_layers.{i}.0.weight"] = (0.999, 0.02)
    bad = []
    for k, (cmin, rmax) in keys.items():
        cos, rel = _cos_rel(params[k].grad, sdr[k].grad)
        if not (cos > cmin and rel < rmax):
            bad.append((k, cos, rel))
    assert not bad, bad
    # channels masked in every utterance get no mask_emb gradient at all
    dead = ci.all(0)
    if bool(dead.any()):
        assert params["mask_emb"].grad[dead.to(dev)].abs().max().item() == 0


# ------------------------------------------------------------------------------------------------------------------ wrappers
@pytest.mark.parametrize("kind", ["hubert", "wav2vec"])
def test_finetuning_wrapper_samples_and_applies_channel_mask(cuda_device, kind):
    """Training mode with apply_mask=True, mask_channel_prob 0.5 / length 64 (the published ASR recipes): the masks drawn from a
    seeded numpy state are the reference's two compute_mask_indices calls in its order, the output equals extract_features with
    those masks injected, and a CTC loss on `proj` back-propagates finite gradients."""
    from unispeech_b200.fairseq_encoder import HubertEncoder, Wav2VecEncoder
    from unispeech_b200.masking import compute_mask_indices
    from unispeech_b200.wav2vec2 import Wav2Vec2Config, Wav2Vec2Model
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    dev = cuda_device
    w2v = kind == "wav2vec"   # wav2vec 2.0 Large style: pre-LN, LayerNorm extractor, no relative-position bias
    cfg = O.tiny_config(pre_ln=w2v, encoder_embed_dim=256, encoder_attention_heads=4, mask_channel_prob=0.5,
                        mask_channel_length=64, relative_position_embedding=not w2v, gru_rel_pos=not w2v)
    sd = O.deterministic_state_dict(cfg)
    if kind == "hubert":
        m, Enc = WavLM(WavLMConfig(vars(cfg))), HubertEncoder
    else:
        m, Enc = Wav2Vec2Model(Wav2Vec2Config(vars(cfg))), Wav2VecEncoder
    res = m.load_state_dict(sd, strict=False)
    # the oracle's state dict is the encoder's; only wav2vec 2.0's pre-training heads (dropped by the wrapper) are not in it
    assert not res.unexpected_keys, res.unexpected_keys
    assert all(k.startswith(("quantizer.", "project_q.", "final_proj.")) for k in res.missing_keys), res.missing_keys
    assert kind == "wav2vec" or not res.missing_keys
    V = 32
    enc = Enc(m, apply_mask=True, output_dim=V).to(dev).train()
    B, L = 2, 16000
    wav, pmask = O.deterministic_waveform(B, L, seed=6, lengths=[16000, 12000])
    T, D = O.num_frames(L, cfg), cfg.encoder_embed_dim
    drawn = []   # the masks the model sampled for the forward pass
    sample_masks = m.sample_masks
    m.sample_masks = lambda *a: drawn.append(sample_masks(*a)) or drawn[-1]
    np.random.seed(123)
    out = enc(wav.to(dev), pmask)
    np.random.seed(123)
    fpm = O.frame_padding_mask(pmask, T)
    mi = compute_mask_indices((B, T), fpm, cfg.mask_prob, cfg.mask_length, "static", 0, min_masks=2, no_overlap=False,
                              min_space=1)
    ci = compute_mask_indices((B, D), None, 0.5, 64, "static", 0, no_overlap=False, min_space=1)
    assert len(drawn) == 1
    assert torch.equal(drawn[0][0].cpu(), torch.from_numpy(mi))
    assert torch.equal(drawn[0][1].cpu(), torch.from_numpy(ci))
    y = out["encoder_out"]                                        # T x B x V
    with torch.no_grad():
        x_inj, _ = m.extract_features(wav.to(dev), padding_mask=pmask, mask=True, mask_indices=torch.from_numpy(mi),
                                      mask_channel_indices=torch.from_numpy(ci))
        y_inj = F.linear(x_inj.float(), enc.proj.weight, enc.proj.bias).transpose(0, 1)
    valid = (~fpm).t().to(dev)
    # same masks, same encoder kernels; `proj` here is an fp32 linear on the bf16 encoder output while the wrapper runs the bf16
    # GEMM (bf16 weights and output): ~1e-2 at |y| of a few units.  A different mask moves masked channels by O(1).
    d = (y.float() - y_inj)[valid].abs().max().item()
    assert d < 0.05, d
    lp = F.log_softmax(y.float(), dim=-1)
    tgt = torch.randint(1, V, (B, 8), generator=torch.Generator().manual_seed(0)).to(dev)
    in_len = (~fpm).sum(1).to(dev)
    loss = F.ctc_loss(lp, tgt, in_len, torch.full((B,), 8, device=dev), blank=0, zero_infinity=False)
    assert torch.isfinite(loss)
    loss.backward()
    torch.cuda.synchronize()
    for k in ("mask_emb", "post_extract_proj.weight", "encoder.layers.0.fc1.weight"):
        g = dict(m.named_parameters())[k].grad
        assert g is not None and torch.isfinite(g).all() and g.abs().max().item() > 0, k
    assert torch.isfinite(enc.proj.weight.grad).all()


# ------------------------------------------------------------------------------------------------------------------ graph
def test_graphed_step_with_channel_mask_matches_eager(cuda_device):
    from unispeech_b200.graphed import GraphedForwardBackward
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    dev = cuda_device
    cfg = O.tiny_config(pre_ln=True, encoder_layers=3, mask_channel_prob=0.5, mask_channel_length=16)
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(O.deterministic_state_dict(cfg))
    m = m.to(dev).train()
    B, L = 2, 16000
    wav, _ = O.deterministic_waveform(B, L, seed=3)
    wav_host = wav.float().pin_memory()
    R = None

    def loss_fn(x):
        nonlocal R
        if R is None:
            R = O.hash_uniform("probe:graph", tuple(x.shape)).to(dev)
        return (x.float() * R).sum()

    g = GraphedForwardBackward(m, loss_fn, B, L, dev).capture()
    assert g.chan_dev is not None
    np.random.seed(11)
    seen = []
    for step in range(3):
        loss = g.step(wav_host)
        torch.cuda.synchronize()
        mask, chan = g.mask_host.clone(), g.chan_host.clone()
        assert torch.equal(g.chan_dev.cpu(), chan)
        seen.append(chan)
        got_loss, got = float(loss), m.grad_buffer().detach().clone()
        m.zero_grad_buffer()
        m._engine.prepared_version = None
        x, _ = m.extract_features(wav.to(dev), padding_mask=None, mask=True, mask_indices=mask, mask_channel_indices=chan)
        ref = loss_fn(x)
        ref.backward()
        torch.cuda.synchronize()
        want = m.grad_buffer().detach().clone()
        # the tolerances of test_graph_gpu.py: the same kernels, fp32 atomics in another order
        assert abs(got_loss - float(ref)) <= 2e-3 * max(1.0, abs(float(ref))), (step, got_loss, float(ref))
        scale = want.abs().max().item()
        assert (got - want).abs().max().item() <= 2e-2 * scale, (step, (got - want).abs().max().item(), scale)
    assert not torch.equal(seen[0], seen[1])   # a new channel mask every replay


# ------------------------------------------------------------------------------------------------------------------ sampler
def test_device_sampler_draws_channel_masks(cuda_device):
    """span_mask_device over the channel axis with the channel arguments (no padding mask, min_masks 0) against the host port of the
    reference sampler: exact rules (same masked count in every row, whole spans) and the masked fraction statistically."""
    from unispeech_b200.datapath import span_mask_device
    from unispeech_b200.masking import compute_mask_indices
    dev = cuda_device
    fr_dev, fr_host = [], []
    for B, D, p, L in [(8, 1024, 0.5, 64), (16, 768, 0.1, 64), (32, 1024, 0.25, 10)]:
        for seed in range(8):
            c = span_mask_device(B, D, dev, p, L, min_masks=0, padding_mask=None, seed=seed).cpu()
            assert c.shape == (B, D) and c.dtype == torch.bool
            per_row = c.sum(1)
            assert int(per_row.min()) == int(per_row.max())
            fr_dev.append((p, L, per_row[0].item() / D))
        np.random.seed(B)
        for _ in range(8):
            r = compute_mask_indices((B, D), None, p, L, "static", 0)
            fr_host.append((p, L, r[0].sum() / D))
    for p, L in {(p, L) for p, L, _ in fr_dev}:
        a = np.mean([f for q, l, f in fr_dev if (q, l) == (p, L)])
        b = np.mean([f for q, l, f in fr_host if (q, l) == (p, L)])
        # 8 draws each; the spread of one draw's masked fraction is about one span (L / D) -- allow 1.5 spans of difference
        assert abs(a - b) < 1.5 * L / D + 0.01, (p, L, a, b)
