"""UniSpeech-SAT pre-training step on the GPU (BASELINE.json configs[3]; SURVEY.md section 8f row 1, second half): the
utterance-contrastive loss + Gumbel vector quantizer kernels (csrc/sat.cu) against the oracle's restatement of
src/fairseq/models/unispeech_sat/unispeech_sat.py:487-557,699-758 and src/fairseq/modules/gumbel_vector_quantizer.py:141-201, which is
pinned to the reference's own source by tests/golden/sat_heads.npz (tests/test_oracle_golden.py).  Same weights, the same host
`torch.randint` instance draws (same seed, same call order), and in training mode the same Gumbel noise (counter-based generator
restated in the oracle).  Tolerances: the loss within 1 % (bf16 projections, fp32 cosine / BCE), statistics exact up to a few
sign flips of near-zero logits, gradients cosine > 0.99 / norm within 6 % (they pass through bf16 GEMMs twice)."""
import pytest
import torch

from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu
SITE_GUMBEL = 0x7F000002


def _extra_state(D, Dp, classes, G, V, vq_dim, quant):
    sd = {"final_proj.weight": O.hash_uniform("fp.w", (Dp, D), -0.08, 0.08), "final_proj.bias": O.hash_uniform("fp.b", (Dp,), -0.1, 0.1),
          "label_embs_concat": O.hash_uniform("lab", (classes, Dp), 0.0, 1.0),
          "spk_proj.weight": O.hash_uniform("spk.w", (Dp, D), -0.1, 0.1), "spk_proj.bias": O.hash_uniform("spk.b", (Dp,), -0.1, 0.1)}
    if quant:
        sd.update({"quantizer.vars": O.hash_uniform("q.vars", (1, G * V, vq_dim // G), 0.0, 1.0),
                   "quantizer.weight_proj.weight": O.hash_uniform("q.w", (G * V, D), -0.5, 0.5),
                   "quantizer.weight_proj.bias": O.hash_uniform("q.b", (G * V,), -0.1, 0.1),
                   "project_q.weight": O.hash_uniform("pq.w", (Dp, vq_dim), -0.1, 0.1), "project_q.bias": O.hash_uniform("pq.b", (Dp,), -0.1, 0.1)})
    else:
        sd.update({"project_q.weight": O.hash_uniform("pq.w", (Dp, D), -0.1, 0.1), "project_q.bias": O.hash_uniform("pq.b", (Dp,), -0.1, 0.1)})
    return sd


def _equal_count_mask(B, T, lengths_frames, n_mask):
    """bool [B, T] with exactly n_mask masked frames per utterance, all inside the valid part (what compute_mask_indices with a
    padding mask produces: the same number of spans for every row)."""
    mi = torch.zeros(B, T, dtype=torch.bool)
    for b in range(B):
        score = O.hash_uniform(f"satmask{b}", (lengths_frames[b],), 0.0, 1.0)
        mi[b, torch.topk(score, n_mask).indices] = True
    return mi


@pytest.mark.parametrize("quant,train", [(False, False), (True, False), (True, True)])
def test_sat_step_vs_oracle(cuda_device, quant, train):
    from unispeech_b200.unispeech_sat import UniSpeechSATConfig, UniSpeechSATForPretraining
    dev = cuda_device
    cfg = O.tiny_config(pre_ln=True, layer_norm_for_extract=True, relative_position_embedding=False, gru_rel_pos=False)
    D, Dp, C, G, V, vq_dim = cfg.encoder_embed_dim, 64, 30, 2, 32, 128
    n_inst, n_cross, layer = 3, 5, 1
    scfg = UniSpeechSATConfig(dict(vars(cfg), final_dim=Dp, logit_temp=0.1, utterance_contrastive_layer=layer, num_instances=n_inst,
                                   cross_sample_instances=n_cross, quantize_targets=quant, latent_vars=V, latent_groups=G,
                                   latent_dim=vq_dim, latent_temp=(2.0, 0.5, 0.999995)))
    m = UniSpeechSATForPretraining(scfg, [C])
    sd = O.deterministic_state_dict(cfg)
    ex = _extra_state(D, Dp, C, G, V, vq_dim, quant)
    m.load_state_dict({**sd, **ex}, strict=True)
    m = m.to(dev)
    m = m.train() if train else m.eval()
    m.noise_seed = 4242
    B, L = 3, 9600
    lengths = [9600, 8000, 7000]
    wav, pmask = O.deterministic_waveform(B, L, seed=1, lengths=lengths)
    T = O.num_frames(L, cfg)
    fpm = O.frame_padding_mask(pmask, T)
    valid = [int((~fpm[b]).sum()) for b in range(B)]
    mi = _equal_count_mask(B, T, valid, 9)
    tl = [(O.hash_uniform("tgt", (B, T), 0.0, 1.0) * C).long().clamp(max=C - 1)]
    lw = [10.0, 5.0, 0.0, 2.0] if quant else [10.0, 5.0, 0.0]

    torch.manual_seed(99)
    out = m(wav.to(dev), target_list=tl, padding_mask=pmask, mask=True, mask_indices=mi)
    loss, ss, log = m.criterion(out, pred_masked_weight=1.0, pred_nomask_weight=0.0, loss_weights=lw)
    loss.backward()
    torch.cuda.synchronize()

    # ---- oracle
    sdr = {k: v.clone().requires_grad_(True) for k, v in {**sd, **ex}.items()}
    conv = O.conv_feature_extractor(sdr, wav, cfg)
    feats = O.extract_features(sdr, wav, cfg, padding_mask=pmask, mask_indices=mi)
    xin = torch.where(mi.unsqueeze(-1), sdr["mask_emb"], feats["features"])
    x, _, spk_x = O.encoder(sdr, xin, fpm, cfg, tgt_layer=None, extract_layer=layer - 1)
    args = (sdr["final_proj.weight"], sdr["final_proj.bias"], sdr["label_embs_concat"], [C], False, 0.1)
    lm = O.masked_prediction_logits(x, torch.logical_and(~fpm, mi), tl, *args)
    main, want_ss, _ = O.wavlm_criterion(lm, [], 1.0, 0.0, None, None)
    qd = None
    if quant:
        noise = None
        if train:
            S = B * 9
            noise = O.gumbel_noise(4242, SITE_GUMBEL, S * G * V).view(S * G, V)
        qd = dict(weight_proj_w=sdr["quantizer.weight_proj.weight"], weight_proj_b=sdr["quantizer.weight_proj.bias"],
                  vars_=sdr["quantizer.vars"], groups=G, num_vars=V, noise=noise, tau=2.0)
    torch.manual_seed(99)
    l_spk, mean_t, acc, q = O.sat_utterance_contrastive_loss(
        spk_x, fpm, mi, sdr["spk_proj.weight"], sdr["spk_proj.bias"], n_inst, n_cross, 0.1, quantizer=qd,
        project_q=(sdr["project_q.weight"], sdr["project_q.bias"]) if quant else None)
    pen = conv.float().pow(2).mean()
    want = main + lw[0] * pen * want_ss + lw[1] * l_spk * want_ss
    if quant:
        nv = G * V
        want = want + lw[3] * ((nv - q["prob_perplexity"]) / nv) * want_ss
    want.backward()

    assert ss == want_ss
    got_spk = out["loss_spk_m"].item()
    assert abs(got_spk - l_spk.item()) < 0.01 * abs(l_spk.item()) + 2e-3, (got_spk, l_spk.item())
    assert abs(out["mean_targets"].item() - mean_t.item()) < 1e-6
    assert abs(out["contrastive_acc"].item() - acc.item()) < 0.02
    if quant:
        assert abs(out["prob_perplexity"].item() - q["prob_perplexity"].item()) < 0.02 * q["prob_perplexity"].item()
        assert abs(out["code_perplexity"].item() - q["code_perplexity"].item()) < 0.05 * q["code_perplexity"].item() + 0.05
        assert out["num_vars"] == G * V and abs(out["temp"] - 2.0) < 1e-9
    assert abs(loss.item() - want.item()) < 0.02 * abs(want.item()) + 0.5, (loss.item(), want.item())
    params = dict(m.named_parameters())
    keys = ["spk_proj.weight", "spk_proj.bias", "encoder.layers.0.fc1.weight", "encoder.layers.0.self_attn.v_proj.weight",
            "post_extract_proj.weight", "encoder.layer_norm_for_extract.weight", "final_proj.weight"]
    if quant:
        keys += ["project_q.weight", "project_q.bias", "quantizer.vars", "quantizer.weight_proj.weight", "quantizer.weight_proj.bias"]
    bad = []
    for k in keys:
        w_ = sdr[k].grad
        assert w_ is not None, k
        w_, g_ = w_.double(), params[k].grad.detach().double().cpu()
        cos = ((g_ * w_).sum() / (g_.norm() * w_.norm() + 1e-30)).item()
        rel = abs(g_.norm().item() - w_.norm().item()) / (w_.norm().item() + 1e-30)
        if cos < 0.99 or rel > 0.06:
            bad.append((k, round(cos, 4), round(rel, 4)))
    assert not bad, bad


def test_sat_kernel_matches_reference_fixture(cuda_device):
    """The committed fixture of the REFERENCE's own code (tools/make_sat_golden.py executes the source text of
    unispeech_sat.py's sample_instances / compute_nce / compute_pred_spk): same hash-generated inputs, same `torch.randint`
    draws -> the CUDA loss kernel reproduces the reference's loss / mean_targets / accuracy (non-quantized cases; the
    projections are rounded to bf16 for the kernel, so 1 % on the loss)."""
    import os
    import numpy as np
    import torch.nn.functional as F
    from unispeech_b200 import ops
    from unispeech_b200.heads import sample_instances
    dev = cuda_device
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "sat_heads.npz"))
    B, T, C, Dp, temp = 3, 14, 16, 8, 0.1
    n_checked = 0
    for i, (use_q, n_inst, cross, seed) in enumerate(g["cases"].tolist()):
        if use_q:
            continue
        tag = f"sat{int(use_q)}{n_inst}{cross}"
        spk_x = O.hash_uniform(tag + ".x", (B, T, C), -1.0, 1.0)
        mask = torch.from_numpy(g[f"mask_{i}"])
        sw, sb = O.hash_uniform(tag + ".sw", (Dp, C), -0.5, 0.5), O.hash_uniform(tag + ".sb", (Dp,), -0.1, 0.1)
        x_m = spk_x[mask].view(B, -1, C)
        M = x_m.shape[1]
        S, N = B * M, int(n_inst) + int(cross)
        proj = F.linear(x_m, sw, sb).reshape(S, Dp)
        torch.manual_seed(int(seed))
        inst = sample_instances(B, M, int(n_inst), int(cross))
        inst_ns = inst.view(B, N, M).permute(1, 0, 2).reshape(N, S)
        same = (inst_ns // M) == (torch.arange(S) // M).unsqueeze(0)
        pb = proj.to(torch.bfloat16).to(dev).contiguous()
        gbuf = torch.empty(S, N + 1, device=dev)
        loss = torch.zeros(1, dtype=torch.float64, device=dev)
        stats = torch.zeros(2, dtype=torch.int32, device=dev)
        ops.sat_nce_fwd(pb, Dp, pb, Dp, inst_ns.to(torch.int32).contiguous().to(dev), same.to(torch.uint8).contiguous().to(dev), S, N,
                        Dp, temp, gbuf, loss, stats)
        torch.cuda.synchronize()
        want = g[f"out_{i}"]
        assert abs(loss.item() - want[0]) < 0.01 * abs(want[0]) + 1e-3, (i, loss.item(), want[0])
        tot = S * (N + 1)
        assert abs(stats[1].item() / tot - want[1]) < 1e-6, (i, stats[1].item() / tot, want[1])
        assert abs(stats[0].item() / tot - want[2]) < 0.03, (i, stats[0].item() / tot, want[2])
        n_checked += 1
    assert n_checked >= 2
