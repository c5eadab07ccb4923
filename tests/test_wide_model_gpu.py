"""The 1280-wide encoders (XLS-R 1B, MMS-1B, HuBERT X-Large: D = 1280, F = 5120, 16 heads of width 80, pos_conv groups of 80
channels, pre-LN, LayerNorm extractor with conv biases, no relative-position bias) through the whole product path:
the pos_conv stem against float64 (the checks of test_conv_stem_gpu at this width, post-LN and pre-LN), a 4-layer model against
the oracle (hidden states of every layer and parameter gradients, dense and ragged, with the DESIGN section 1 bounds), the
full 48-layer encoder on 10 s against the CPU oracle, and the fine-tuning wrappers and k-means labels on top of it."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_conv_stem_gpu as S
import test_fullscale_gpu as FS
from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu


def wide_config(**kw):
    d = dict(encoder_embed_dim=1280, encoder_ffn_embed_dim=5120, encoder_attention_heads=16, relative_position_embedding=False,
             gru_rel_pos=False, conv_bias=True)
    d.update(kw)
    return O.large_config(**d)


_STEM = {}


def stem_model(post_ln, dev):
    """The xlsr1b configuration with one encoder layer, non-trivial normalisation affine terms, pos_conv bias and weight_g (as
    test_conv_stem_gpu.model does for the shipped widths)."""
    if post_ln not in _STEM:
        from unispeech_b200 import workloads as W
        from unispeech_b200.wavlm import WavLM, WavLMConfig
        cfg, B, secs = W.model_config("xlsr1b")
        torch.manual_seed(14 + post_ln)
        m = WavLM(WavLMConfig(dict(cfg, encoder_layers=1, layer_norm_first=not post_ln)))
        with torch.no_grad():
            for mod in m.modules():
                if isinstance(mod, (torch.nn.LayerNorm, torch.nn.GroupNorm)):
                    mod.weight.normal_(1.0, 0.2)
                    mod.bias.normal_(0.0, 0.1)
            pc = m.encoder.pos_conv[0]
            pc.bias.normal_(0.0, 0.1)
            pc.weight_g.mul_(torch.rand_like(pc.weight_g) + 0.5)
        _STEM[post_ln] = (m.to(dev).eval(), B, secs)
    return _STEM[post_ln]


def test_posconv_prep_1280(cuda_device, monkeypatch):
    """posconv_prep at D = 1280, G = 16: 80 channels in a 128-wide group tile, zero weights past 80."""
    dev = cuda_device
    m, _, _ = stem_model(False, dev)
    eng = m._begin(dev)
    torch.cuda.synchronize()
    pc = m.encoder.pos_conv[0]
    G, taps, D = m.cfg.conv_pos_groups, m.cfg.conv_pos, m.cfg.encoder_embed_dim
    Cg = D // G
    assert tuple(eng.pc_fwd.shape) == (G, 128, taps, 128)
    w = S.weight_norm64(pc.weight_v.detach().double(), pc.weight_g.detach().double())
    ref_f = w.view(G, Cg, Cg, taps).permute(0, 1, 3, 2)
    S.assert_close(eng.pc_fwd[:, :Cg, :, :Cg], ref_f, S.bf16_bound(ref_f, 2.0 ** -20 * ref_f.abs()), "forward taps")
    assert (eng.pc_fwd[:, Cg:] == 0).all() and (eng.pc_fwd[:, :, :, Cg:] == 0).all()
    assert torch.equal(eng.pc_dg, eng.pc_fwd.flip(2).permute(0, 3, 2, 1))


@pytest.mark.parametrize("post_ln", [True, False], ids=["postln", "preln"])
@pytest.mark.parametrize("B,T", [(1, 999), (2, 129), (2, 1)])
def test_posconv_stem_1280(cuda_device, monkeypatch, post_ln, B, T):
    """Forward, input gradient, tap gradient and the weight-norm gradients (weight_v, weight_g) at D = 1280, G = 16, taps = 128,
    against float64 (test_conv_stem_gpu.test_posconv_stem's checks and bounds, on this model)."""
    monkeypatch.setattr(S, "model", lambda name, dev: stem_model(post_ln, dev))
    S.test_posconv_stem(cuda_device, monkeypatch, "xlsr1b", B, T)


def test_wide_4l_hidden_states(cuda_device):
    """4 layers at 1280 width, 1 x 10 s: every layer's hidden state within 3 % of its max|h| of the oracle's."""
    cfg = wide_config(encoder_layers=4)
    FS.run_forward_case("wide4_T499", cfg, FS.state_dict_for("wide4", cfg), 1, 160000, None, cuda_device)


def test_wide_4l_hidden_states_ragged(cuda_device):
    """Same, ragged 2 x {8 s, 3.1 s} (an utterance shorter than two key tiles), on the valid frames."""
    cfg = wide_config(encoder_layers=4)
    L = 128000
    FS.run_forward_case("wide4_T399_ragged", cfg, FS.state_dict_for("wide4", cfg), 2, L, [L, 50000], cuda_device)


def test_wide_4l_gradients_ragged(cuda_device):
    """Parameter gradients of every kind (conv biases, pos_conv weight norm, attention, FFN, LayerNorms) against the oracle,
    ragged 2 x 6.5 s with masked frames: cosine > 0.999 and norm within 2 % for the GEMM-fed parameters."""
    cfg = wide_config(encoder_layers=4)
    L = 104000
    FS.grad_case("grad_wide4_T324", cfg, FS.state_dict_for("wide4", cfg), 2, L, [L, 70000], cuda_device)


def test_wide_4l_gradients_dense(cuda_device):
    cfg = wide_config(encoder_layers=4)
    L = 104000
    FS.grad_case("grad_wide4_T324_dense", cfg, FS.state_dict_for("wide4", cfg), 2, L, [L, L], cuda_device)


# Depth bound: the per-layer table's 3 % max-abs / 1.5 % mean-abs bounds were set on the 24-layer WavLM-Large, and they hold
# here for layers 0..24.  The bf16 residual stream keeps drifting from the fp32 oracle with depth (on an H100: max-abs 2.65 % of
# max|h| at layer 24, 3.4 % at layer 40, 3.85 % at layer 48, growing smoothly layer by layer; mean-abs 1.12 % -> 1.46 %), so
# layers 25..48 and the final LayerNorm output are held to max-abs <= 4.5 % with the same 1.5 % mean-abs bound.
DEEP_MAX_REL = 0.045


def test_wide_full_depth_T499(cuda_device, monkeypatch):
    """The whole 48-layer XLS-R 1B encoder, 1 x 10 s (T = 499), against the fp32 CPU oracle with test_fullscale_gpu's per-layer
    table: its bounds for the first 24 layers, DEEP_MAX_REL beyond."""
    cfg = wide_config(encoder_layers=48)
    sd = FS.state_dict_for("wide48", cfg)
    wav, _ = O.deterministic_waveform(1, 160000, seed=3, lengths=None)
    n = cfg.encoder_layers
    with torch.no_grad():
        want = O.extract_features(sd, wav, cfg, output_layer=n)
        want_final = O.extract_features(sd, wav, cfg)
    m = FS.build(cfg, sd, cuda_device)
    with torch.no_grad():
        (_, got_lr), _ = m.extract_features(wav.to(cuda_device), ret_layer_results=True, output_layer=n)
        xf, _ = m.extract_features(wav.to(cuda_device))
    torch.cuda.synchronize()
    want_layers = [h[0] if isinstance(h, tuple) else h for h in want["layer_results"]]
    got_layers = [h for h, _ in got_lr]
    assert len(got_layers) == n + 1 == len(want_layers)
    FS.layer_table("wide48_T499", got_layers[:25], want_layers[:25])
    monkeypatch.setattr(FS, "MAX_REL", DEEP_MAX_REL)
    FS.layer_table("wide48_T499:25-48", got_layers[25:], want_layers[25:])
    FS.layer_table("wide48_T499:final", [xf.transpose(0, 1)], [want_final["x"].transpose(0, 1)])


def _wide_model(kind, dev, layers=2, V=32):
    from unispeech_b200.ctc import HubertCtc, Wav2VecCtc
    from unispeech_b200.wav2vec2 import Wav2Vec2Config, Wav2Vec2Model
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    cfg = wide_config(encoder_layers=layers)
    sd = O.deterministic_state_dict(cfg)
    if kind == "wav2vec":
        m, Model = Wav2Vec2Model(Wav2Vec2Config(vars(cfg))), Wav2VecCtc
    else:
        m, Model = WavLM(WavLMConfig(vars(cfg))), HubertCtc
    res = m.load_state_dict(sd, strict=False)
    assert not res.unexpected_keys
    torch.manual_seed(0)
    return Model.build_model(m, V, apply_mask=True).to(dev), cfg


def _sample(B, L, lengths, V, dev, seed=0):
    wav, pmask = O.deterministic_waveform(B, L, seed=6, lengths=lengths)
    pad, eos, S_ = 1, 2, 9
    g = torch.Generator().manual_seed(seed)
    target = torch.full((B, S_ + 2), pad, dtype=torch.long)
    for b in range(B):
        n = S_ - 3 * b
        target[b, :n] = torch.randint(3, V, (n,), generator=g)
        target[b, n] = eos
    return {"net_input": {"source": wav.to(dev), "padding_mask": pmask}, "target": target, "id": torch.arange(B)}


def test_wav2vec_ctc_step_1280(cuda_device):
    """One Wav2VecCtc fine-tuning step at 1280 width (2 layers) with FusedAdam.  Before the update, the loss and the `proj` /
    encoder gradients match the same model driven by F.log_softmax + F.ctc_loss on its own logits (cosine > 0.999, norm within
    2 %); the update then changes the parameters and leaves them finite."""
    from unispeech_b200.ctc import CtcCriterion, prepare_targets
    from unispeech_b200.optim import FusedAdam
    dev = cuda_device
    V, B, L = 32, 2, 32000
    model, cfg = _wide_model("wav2vec", dev, V=V)
    model.train()
    enc, m = model.w2v_encoder, model.w2v_encoder.w2v_model
    sample = _sample(B, L, [32000, 21000], V, dev)
    crit = CtcCriterion()
    names = ["mask_emb", "post_extract_proj.weight", "encoder.pos_conv.0.weight_v", "encoder.layers.0.self_attn.q_proj.weight",
             "encoder.layers.1.fc1.weight", "encoder.layers.0.self_attn.out_proj.weight"]
    params = dict(m.named_parameters())

    np.random.seed(123)
    loss, _, _ = crit(model, sample)
    loss.backward()
    torch.cuda.synchronize()
    got = {k: params[k].grad.detach().clone() for k in names}
    got["proj.weight"] = enc.proj.weight.grad.detach().clone()
    m.zero_grad_buffer()
    enc.proj.weight.grad = enc.proj.bias.grad = None

    np.random.seed(123)
    out = model(**sample["net_input"])
    tg, tl = prepare_targets(sample["target"], 1, 2)
    in_len = (~out["padding_mask"]).sum(1)
    ref = F.ctc_loss(F.log_softmax(out["encoder_out"].float(), -1), tg.long().to(dev), in_len, tl.long().to(dev), blank=0,
                     reduction="sum")
    ref.backward()
    torch.cuda.synchronize()
    assert abs(float(loss) - float(ref)) <= 1e-4 * abs(float(ref)), (float(loss), float(ref))
    want = {k: params[k].grad for k in names}
    want["proj.weight"] = enc.proj.weight.grad
    for k in got:
        a, b = got[k].double().flatten(), want[k].double().flatten()
        cos = float((a * b).sum() / (a.norm() * b.norm()))
        rel = abs(float(a.norm() / b.norm()) - 1.0)
        assert cos > 0.999 and rel < 0.02, (k, cos, rel)

    before = {k: params[k].detach().clone() for k in names}
    opt = FusedAdam(m, lr=1e-4)
    opt.step()
    torch.cuda.synchronize()
    for k in names:
        assert torch.isfinite(params[k]).all() and not torch.equal(params[k], before[k]), k


def test_hubert_encoder_eval_and_kmeans_1280(cuda_device):
    """HubertEncoder forward in eval mode at 1280 width (finite, best-path shape), and KMeans.predict on a 1280-wide
    extract_features(output_layer=...) against the float64 nearest centre of the same bf16 features."""
    from unispeech_b200.kmeans import KMeans
    dev = cuda_device
    V, B, L = 32, 2, 32000
    model, cfg = _wide_model("hubert", dev, V=V)
    model.eval()
    sample = _sample(B, L, [32000, 21000], V, dev)
    with torch.no_grad():
        out = model(**sample["net_input"])
    y = out["encoder_out"]
    T = O.num_frames(L, cfg)
    assert tuple(y.shape) == (T, B, V) and torch.isfinite(y.float()).all()

    m = model.w2v_encoder.w2v_model
    wav, pmask = O.deterministic_waveform(B, L, seed=9, lengths=[32000, 21000])
    with torch.no_grad():
        x, fpm = m.extract_features(wav.to(dev), padding_mask=pmask.to(dev), output_layer=1)
    assert x.shape[-1] == 1280
    feats = x.to(torch.bfloat16)
    valid = feats[~fpm]
    km = KMeans(8, max_iter=5, seed=0).fit(valid.contiguous())
    labels = km.predict(feats, padding_mask=fpm)
    torch.cuda.synchronize()
    assert (labels[fpm] == -1).all()
    c = km.cluster_centers_.to(torch.bfloat16).double()
    d = torch.cdist(valid.double(), c)
    got = labels[~fpm].long()
    best = d.min(1).values
    # the kernel's fp32 scores may break near-ties differently; its pick is within fp32 rounding of the nearest centre
    picked = d.gather(1, got[:, None])[:, 0]
    assert (picked - best <= 1e-3 * best.clamp_min(1.0)).all()
    assert (got == d.argmin(1)).float().mean().item() > 0.99
