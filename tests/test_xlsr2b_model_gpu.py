"""The 1920-wide encoder (XLS-R 2B: D = 1920, F = 7680, 16 heads of width 120, pos_conv groups of 120 channels, pre-LN,
LayerNorm extractor with conv biases, no relative-position bias) through the product path, with the bounds of
test_wide_model_gpu: the pos_conv stem against float64 (post-LN and pre-LN), a 4-layer model against the oracle (hidden states
of every layer and parameter gradients, dense and ragged), one Wav2VecCtc step with FusedAdam, and HubertEncoder in eval mode
followed by KMeans.predict."""
import pytest
import torch

import test_conv_stem_gpu as S
import test_fullscale_gpu as FS
import test_wide_model_gpu as W
from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu

D2B = 1920
_wide_config = W.wide_config   # (the wrapper tests below swap W.wide_config for config_2b)


def config_2b(**kw):
    return _wide_config(encoder_embed_dim=D2B, encoder_ffn_embed_dim=4 * D2B, **kw)


_STEM = {}


def stem_model(post_ln, dev):
    """The xlsr2b configuration with one encoder layer and the non-trivial affine terms of test_wide_model_gpu.stem_model."""
    if post_ln not in _STEM:
        from unispeech_b200 import workloads as WL
        from unispeech_b200.wavlm import WavLM, WavLMConfig
        cfg, B, secs = WL.model_config("xlsr2b")
        torch.manual_seed(20 + post_ln)
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


def test_posconv_prep_1920(cuda_device):
    """posconv_prep at D = 1920, G = 16: 120 channels in a 128-wide group tile, zero weights past 120."""
    m, _, _ = stem_model(False, cuda_device)
    eng = m._begin(cuda_device)
    torch.cuda.synchronize()
    pc = m.encoder.pos_conv[0]
    G, taps, D = m.cfg.conv_pos_groups, m.cfg.conv_pos, m.cfg.encoder_embed_dim
    Cg = D // G
    assert Cg == 120 and tuple(eng.pc_fwd.shape) == (G, 128, taps, 128)
    w = S.weight_norm64(pc.weight_v.detach().double(), pc.weight_g.detach().double())
    ref_f = w.view(G, Cg, Cg, taps).permute(0, 1, 3, 2)
    S.assert_close(eng.pc_fwd[:, :Cg, :, :Cg], ref_f, S.bf16_bound(ref_f, 2.0 ** -20 * ref_f.abs()), "forward taps")
    assert (eng.pc_fwd[:, Cg:] == 0).all() and (eng.pc_fwd[:, :, :, Cg:] == 0).all()
    assert torch.equal(eng.pc_dg, eng.pc_fwd.flip(2).permute(0, 3, 2, 1))


@pytest.mark.parametrize("post_ln", [True, False], ids=["postln", "preln"])
@pytest.mark.parametrize("B,T", [(1, 999), (2, 129), (2, 1)])
def test_posconv_stem_1920(cuda_device, monkeypatch, post_ln, B, T):
    """Forward, input gradient, tap gradient and the weight-norm gradients at D = 1920, G = 16, taps = 128, against float64
    (test_conv_stem_gpu.test_posconv_stem's checks and bounds, on this model)."""
    monkeypatch.setattr(S, "model", lambda name, dev: stem_model(post_ln, dev))
    S.test_posconv_stem(cuda_device, monkeypatch, "xlsr2b", B, T)


def test_xlsr2b_4l_hidden_states(cuda_device):
    """4 layers at 1920 width, 1 x 10 s: every layer's hidden state within the oracle bounds of test_fullscale_gpu."""
    cfg = config_2b(encoder_layers=4)
    FS.run_forward_case("xlsr2b4_T499", cfg, FS.state_dict_for("xlsr2b4", cfg), 1, 160000, None, cuda_device)


def test_xlsr2b_4l_hidden_states_ragged(cuda_device):
    cfg = config_2b(encoder_layers=4)
    L = 128000
    FS.run_forward_case("xlsr2b4_T399_ragged", cfg, FS.state_dict_for("xlsr2b4", cfg), 2, L, [L, 50000], cuda_device)


@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
def test_xlsr2b_4l_gradients(cuda_device, ragged):
    """Parameter gradients of every kind against the oracle, 2 x 6.5 s (ragged: the second utterance 4.4 s)."""
    cfg = config_2b(encoder_layers=4)
    L = 104000
    FS.grad_case("grad_xlsr2b4_T324" + ("" if ragged else "_dense"), cfg, FS.state_dict_for("xlsr2b4", cfg), 2, L,
                 [L, 70000 if ragged else L], cuda_device)


def test_wav2vec_ctc_step_1920(cuda_device, monkeypatch):
    """test_wide_model_gpu's Wav2VecCtc + FusedAdam step (gradients against F.ctc_loss on the model's own logits, then a
    finite update) at 1920 width."""
    monkeypatch.setattr(W, "wide_config", lambda **kw: config_2b(**kw))
    W.test_wav2vec_ctc_step_1280(cuda_device)


def test_hubert_encoder_eval_and_kmeans_1920(cuda_device, monkeypatch):
    """HubertEncoder forward in eval mode at 1920 width (finite, best-path shape), and KMeans.predict on a 1920-wide
    extract_features(output_layer=...) against the float64 nearest centre of the same bf16 features."""
    from unispeech_b200.kmeans import KMeans
    monkeypatch.setattr(W, "wide_config", lambda **kw: config_2b(**kw))
    dev = cuda_device
    V, B, L = 32, 2, 32000
    model, cfg = W._wide_model("hubert", dev, V=V)
    model.eval()
    sample = W._sample(B, L, [32000, 21000], V, dev)
    with torch.no_grad():
        out = model(**sample["net_input"])
    y = out["encoder_out"]
    assert tuple(y.shape) == (O.num_frames(L, cfg), B, V) and torch.isfinite(y.float()).all()

    m = model.w2v_encoder.w2v_model
    wav, pmask = O.deterministic_waveform(B, L, seed=9, lengths=[32000, 21000])
    with torch.no_grad():
        x, fpm = m.extract_features(wav.to(dev), padding_mask=pmask.to(dev), output_layer=1)
    assert x.shape[-1] == D2B
    feats = x.to(torch.bfloat16)
    valid = feats[~fpm]
    km = KMeans(8, max_iter=5, seed=0).fit(valid.contiguous())
    labels = km.predict(feats, padding_mask=fpm)
    torch.cuda.synchronize()
    assert (labels[fpm] == -1).all()
    d = torch.cdist(valid.double(), km.cluster_centers_.to(torch.bfloat16).double())
    got = labels[~fpm].long()
    best = d.min(1).values
    # the kernel's fp32 scores may break near-ties differently; its pick is within fp32 rounding of the nearest centre
    assert (d.gather(1, got[:, None])[:, 0] - best <= 1e-3 * best.clamp_min(1.0)).all()
    assert (got == d.argmin(1)).float().mean().item() > 0.99
