"""Whole-model parity on the GPU: unispeech_b200.WavLM (bf16 kernels) vs the CPU oracle (fp32) and the committed golden
fixtures generated from the unmodified reference.  Tolerances are stated per check; the bf16 yardstick is the reference's
own bf16-vs-fp32 forward difference (max-abs 0.093 on WavLM-Base hidden states, SURVEY.md S17)."""
import os

import numpy as np
import pytest
import torch

from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(__file__), "golden")

HID_TOL = 0.12      # max-abs on hidden states (|h| up to ~5), bf16 activations end to end
HID_MEAN_TOL = 0.02  # mean-abs


def build(cfg, device):
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    m = WavLM(WavLMConfig(vars(cfg)))
    missing = m.load_state_dict(O.deterministic_state_dict(cfg), strict=True)
    return m.to(device).eval()


def cmp(name, got, want, tol=HID_TOL, mean_tol=HID_MEAN_TOL, mask=None):
    got = got.detach().float().cpu()
    want = torch.as_tensor(want).float()
    assert got.shape == want.shape, (name, got.shape, want.shape)
    d = (got - want).abs()
    if mask is not None:
        d = d[~mask]
    assert torch.isfinite(got).all(), name
    assert d.max().item() < tol, (name, d.max().item())
    assert d.mean().item() < mean_tol, (name, d.mean().item())


CASES = {
    "tiny_postln_ragged": (lambda: O.tiny_config(pre_ln=False), 2, 8000, [8000, 5000]),
    "tiny_preln_ragged": (lambda: O.tiny_config(pre_ln=True), 2, 6400, [6400, 4321]),
    "tiny_postln_nomask": (lambda: O.tiny_config(pre_ln=False), 1, 7777, None),
    "tiny_preln_norelpos": (lambda: O.tiny_config(pre_ln=True, relative_position_embedding=False, gru_rel_pos=False),
                            2, 4000, [4000, 3000]),
    "base2l_halfsec": (lambda: O.base_config(encoder_layers=2), 1, 8000, None),
    "large2l_halfsec": (lambda: O.large_config(encoder_layers=2), 1, 8000, None),
}


@pytest.mark.parametrize("name", sorted(CASES))
def test_forward_vs_golden(cuda_device, name):
    mk, B, L, lengths = CASES[name]
    cfg = mk()
    g = np.load(os.path.join(GOLD, name + ".npz"))
    m = build(cfg, cuda_device)
    wav, pmask = O.deterministic_waveform(B, L, seed=1, lengths=lengths)
    pm = pmask.to(cuda_device) if lengths is not None else None
    with torch.no_grad():
        conv = m.feature_extractor(wav.to(cuda_device))
        x, fpm = m.extract_features(wav.to(cuda_device), padding_mask=pm)
        (xl, layer_results), _ = m.extract_features(wav.to(cuda_device), padding_mask=pm, ret_layer_results=True,
                                                    output_layer=cfg.encoder_layers)
        feats, _ = m.extract_features(wav.to(cuda_device), padding_mask=pm, ret_conv=True)
    cmp("conv_out", conv, g["conv_out"], tol=0.1, mean_tol=0.01)
    cmp("features", feats, g["features"])
    pad = torch.from_numpy(g["frame_padding_mask"]) if "frame_padding_mask" in g else None
    if pad is not None:
        assert torch.equal(fpm.cpu(), pad)
    cmp("x_final", x, g["x_final"], mask=pad)
    assert len(layer_results) == g["layer_results"].shape[0]
    for i, (h, z) in enumerate(layer_results):
        assert z is None and h.shape == (g["layer_results"].shape[1], B, cfg.encoder_embed_dim)
        cmp(f"layer_{i}", h, g["layer_results"][i], mask=pad.t() if pad is not None else None)


@pytest.mark.parametrize("name", [n for n in sorted(CASES) if n.startswith("tiny")])
def test_gradients_vs_golden(cuda_device, name):
    mk, B, L, lengths = CASES[name]
    cfg = mk()
    g = np.load(os.path.join(GOLD, name + ".npz"))
    m = build(cfg, cuda_device)
    wav, pmask = O.deterministic_waveform(B, L, seed=1, lengths=lengths)
    pm = pmask.to(cuda_device) if lengths is not None else None
    mi = torch.from_numpy(g["mask_indices"]) if "mask_indices" in g else None
    x, fpm = m.extract_features(wav.to(cuda_device), padding_mask=pm, mask=mi is not None, mask_indices=mi)
    cmp("masked_x", x, g["masked_x"], mask=fpm.cpu() if fpm is not None else None)
    loss = O.probe_loss(x.float(), fpm, seed=2)
    loss.backward()
    torch.cuda.synchronize()
    assert abs(loss.item() - float(g["loss"])) < 0.05 * max(1.0, abs(float(g["loss"]))) + 1.0, (loss.item(), float(g["loss"]))
    norms = dict(zip(g["grad_norm_keys"].tolist(), g["grad_norms"].tolist()))
    params = dict(m.named_parameters())
    bad = []
    for k, n in norms.items():
        assert params[k].grad is not None, k
        got = params[k].grad.double().norm().item()
        # k_proj.bias has a mathematically zero gradient (softmax is invariant to a per-query constant); the bf16 path
        # leaves rounding noise there, so it only gets an absolute bound
        atol = 0.1 if k.endswith("k_proj.bias") else 2e-3
        if abs(got - n) > 0.06 * n + atol:
            bad.append((k, got, n))
    assert not bad, bad
    for key in g.files:
        if key.startswith("grad:"):
            k = key[5:]
            ref = torch.from_numpy(g[key]).double()
            got = params[k].grad.detach().double().cpu()
            cos = (got * ref).sum() / (got.norm() * ref.norm() + 1e-30)
            assert cos.item() > 0.995, (k, cos.item())


def test_random_inputs_vs_oracle(cuda_device):
    """Seeded random (not fixture) batch, 3-layer tiny model, ragged lengths crossing several attention tiles."""
    cfg = O.tiny_config(pre_ln=False, encoder_layers=3)
    m = build(cfg, cuda_device)
    sd = O.deterministic_state_dict(cfg)
    torch.manual_seed(1234)
    B, L = 3, 16000 * 3  # T = 149
    wav = torch.randn(B, L) * 0.5
    lengths = [L, 40000, 31111]
    pmask = torch.zeros(B, L, dtype=torch.bool)
    for b, n in enumerate(lengths):
        wav[b, n:] = 0
        pmask[b, n:] = True
    with torch.no_grad():
        want = O.extract_features(sd, wav, cfg, padding_mask=pmask)
        got, fpm = m.extract_features(wav.to(cuda_device), padding_mask=pmask.to(cuda_device))
    assert torch.equal(fpm.cpu(), want["padding_mask"])
    cmp("x", got, want["x"], mask=want["padding_mask"])


def test_layer_hooks_and_module_tree(cuda_device):
    """The s3prl-style contract: forward hooks on encoder.layers[i] see a T x B x C input; encoder(...) output[0] is B x T x C."""
    cfg = O.tiny_config(pre_ln=True)
    m = build(cfg, cuda_device)
    seen = {}
    hooks = [m.encoder.layers[i].register_forward_hook(lambda mod, inp, out, i=i: seen.__setitem__(i, inp[0].transpose(0, 1)))
             for i in range(len(m.encoder.layers))]
    hooks.append(m.encoder.register_forward_hook(lambda mod, inp, out: seen.__setitem__("enc", out[0])))
    wav, _ = O.deterministic_waveform(1, 6400, seed=1)
    with torch.no_grad():
        x, _ = m.extract_features(wav.to(cuda_device))
    for h in hooks:
        h.remove()
    T = O.num_frames(6400, cfg)
    assert seen[0].shape == (1, T, cfg.encoder_embed_dim) and seen["enc"].shape == (1, T, cfg.encoder_embed_dim)
    assert hasattr(m.encoder.layers[1], "self_attn") and len(m.encoder.layers) == cfg.encoder_layers
    assert torch.equal(seen["enc"], x)


def test_layer_called_alone_after_an_interrupted_call_computes_every_row(cuda_device):
    """The ragged lengths of a batch belong to that call: after a forward hook raises inside the layer loop, a layer called on
    its own with a same-size batch of longer utterances must compute what a model that never saw the first batch computes."""
    cfg = O.tiny_config(pre_ln=True)
    m, fresh = build(cfg, cuda_device), build(cfg, cuda_device)
    B, L = 2, 16000
    T, D = O.num_frames(L, cfg), cfg.encoder_embed_dim
    wav, pmask = O.deterministic_waveform(B, L, seed=2, lengths=[L, 6000])

    class _Stop(Exception):
        pass

    def fail(mod, inp, out):
        raise _Stop

    hook = m.encoder.layers[1].register_forward_hook(fail)
    with torch.no_grad(), pytest.raises(_Stop):
        m.extract_features(wav.to(cuda_device), padding_mask=pmask.to(cuda_device))
    hook.remove()
    x = torch.randn(T, B, D, generator=torch.Generator().manual_seed(5)).to(cuda_device)
    pad = torch.zeros(B, T, dtype=torch.bool, device=cuda_device)
    pad[1, T - 3:] = True
    with torch.no_grad():
        fresh.extract_features(wav.to(cuda_device))   # prepares the layer operands
        want, _, _ = fresh.encoder.layers[0](x, self_attn_padding_mask=pad)
        got, _, _ = m.encoder.layers[0](x, self_attn_padding_mask=pad)
    assert torch.equal(got, want), (got.float() - want.float()).abs().amax((0, 2))


def test_extract_features_keeps_no_reference_to_its_outputs(cuda_device):
    """Once the caller drops what extract_features returned, nothing in the model keeps it alive."""
    import gc
    import weakref
    cfg = O.tiny_config(pre_ln=True)
    m = build(cfg, cuda_device)
    wav, pmask = O.deterministic_waveform(2, 16000, seed=3, lengths=[16000, 9000])
    with torch.no_grad():
        (x, layer_results), fpm = m.extract_features(wav.to(cuda_device), padding_mask=pmask.to(cuda_device),
                                                     output_layer=cfg.encoder_layers, ret_layer_results=True)
    refs = [weakref.ref(x), weakref.ref(layer_results[1][0])]
    del x, layer_results, fpm
    gc.collect()
    assert [r() is None for r in refs] == [True, True]


def test_state_dict_keys_match_reference_layout():
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    for cfg in (O.tiny_config(pre_ln=False), O.tiny_config(pre_ln=True)):
        m = WavLM(WavLMConfig(vars(cfg)))
        assert {k: tuple(v.shape) for k, v in m.state_dict().items()} == O.parameter_shapes(cfg)


def test_encoder_variants_fairseq_and_sat(cuda_device):
    """Encoder-loop variants of the fairseq tree (SURVEY.md section 8 a10): `tgt_layer` as a list of 1-based layer numbers
    (fairseq WavLM) and `extract_layer` + `layer_norm_for_extract` (UniSpeech-SAT encoder), against the oracle restatement."""
    cfg = O.tiny_config(pre_ln=True, layer_norm_for_extract=True)
    m = build(cfg, cuda_device)
    sd = O.deterministic_state_dict(cfg)
    assert "encoder.layer_norm_for_extract.weight" in m.state_dict()
    wav, pmask = O.deterministic_waveform(2, 6400, seed=4, lengths=[6400, 5000])
    ref = O.extract_features(sd, wav, cfg, padding_mask=pmask)
    fpm = ref["padding_mask"]
    # oracle encoder on the projected features (what encoder() receives inside extract_features)
    xin = ref["features"]
    n = cfg.encoder_layers
    want_x, want_lr, want_er = O.encoder(sd, xin, fpm, cfg, tgt_layer=None, extract_layer=n - 2)
    want_x2, want_lr2 = O.encoder(sd, xin, fpm, cfg, tgt_layer=[1, n])
    with torch.no_grad():
        xd = xin.to(cuda_device)
        got_x, got_lr, got_er = m.encoder(xd, padding_mask=fpm.to(cuda_device), extract_layer=n - 2)
        got_x2, got_lr2 = m.encoder.extract_features(xd, padding_mask=fpm.to(cuda_device), tgt_layer=[1, n])
    cmp("x", got_x, want_x, mask=fpm)
    cmp("extract_result", got_er, want_er, mask=fpm)
    assert got_lr == [] and want_lr == []
    assert len(got_lr2) == 2 == len(want_lr2)
    for (g, _), w in zip(got_lr2, want_lr2):
        cmp("layer_result", g.transpose(0, 1), w.transpose(0, 1), mask=fpm)
    cmp("x2", got_x2, want_x2, mask=fpm)


def test_deepcopy_gets_its_own_engine(cuda_device):
    """EMA / teacher copies: a deep copy must derive its bf16 operands from ITS OWN masters, not from the original's (the engine's
    descriptor tables hold raw device pointers)."""
    import copy
    cfg = O.tiny_config(pre_ln=True)
    m = build(cfg, cuda_device)
    wav, _ = O.deterministic_waveform(1, 6400, seed=1)
    with torch.no_grad():
        x0, _ = m.extract_features(wav.to(cuda_device))
        c = copy.deepcopy(m)
        assert c._engine is None and m._engine is not None
        assert c.encoder.layers[0]._owner[0] is c
        c.encoder.layers[0].fc1.weight.mul_(1.5)
        c.post_extract_proj.bias.add_(0.3)
        x1, _ = m.extract_features(wav.to(cuda_device))
        y1, _ = c.extract_features(wav.to(cuda_device))
    assert torch.equal(x0, x1)                              # the original is untouched by the copy's parameter edits
    assert (y1.float() - x0.float()).abs().max().item() > 1e-2   # and the copy really uses its own (edited) weights
