"""HuBERT's first iteration end to end on the library's kernels: MFCC of a ragged batch -> KMeans(100) fit on the valid frames ->
labels -> a HubertModel(label_rate=100) step, at lengths whose 100 Hz labels are one short of 2 T (the forward trims the
features to T' = int(len(labels) / 2) frames), and at 160 000 samples, where they cover every frame.  Loss and gradients are
compared with the oracle run on the first T' frames with labels t[:, 2 arange(T')], under the tolerances of
tests/test_pretrain_gpu.py (loss 2 % + 0.5, gradient cosine >= 0.98, norm within 10 %)."""
import os

import numpy as np
import pytest
import torch

from oracle import mfcc_oracle as MO
from oracle import trim_oracle as TO
from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(__file__), "golden", "vox_real_large2l.npz")
U = 2.0 ** -23


def _speech(L, lengths):
    """Real speech (the fixture's five utterances back to back, repeated) cut into a zero-padded batch."""
    g = np.load(GOLD)
    s = np.concatenate([g["pcm"][b, :int(n)] for b, n in enumerate(g["lengths"])]).astype(np.float32) / 32768.0
    s = np.tile(s, -(-2 * L // len(s)))
    wav = torch.zeros(len(lengths), L)
    pad = torch.ones(len(lengths), L, dtype=torch.bool)
    for b, n in enumerate(lengths):
        wav[b, :n] = torch.from_numpy(s[b * 7919:b * 7919 + n])
        pad[b, :n] = False
    return wav, pad


def _check_labels(x, cbf, K, labels):
    """tests/test_kmeans_gpu.py's rule: the chosen fp64 score is within 2 bound of the minimum, and the label is the fp64 arg-min
    wherever the best two are further apart than 2 bound."""
    xd, cd = x.double(), cbf[:K].double()
    s = (cd * cd).sum(1)[None, :] - 2.0 * xd @ cd.T
    bound = 2 * x.shape[1] * U * (xd.abs() @ cd.abs().T).amax(1) + x.shape[1] * U * (cd * cd).sum(1).max()
    lab = labels.long()
    assert bool(((lab >= 0) & (lab < K)).all())
    chosen = s.gather(1, lab[:, None])[:, 0]
    assert bool((chosen - s.min(1).values <= 2 * bound).all())
    top2 = s.topk(2, dim=1, largest=False).values
    clear = (top2[:, 1] - top2[:, 0]) > 2 * bound
    assert torch.equal(lab[clear], s.argmin(1)[clear])


def _model(dev, cfg, label_rate, C):
    from unispeech_b200.hubert import HubertConfig, HubertModel
    m = HubertModel(HubertConfig(dict(vars(cfg), final_dim=64, label_rate=label_rate, logit_temp=0.1)), [C])
    sd = O.deterministic_state_dict(cfg)
    head = {"final_proj.weight": O.hash_uniform("fp.w", (64, cfg.encoder_embed_dim), -0.08, 0.08),
            "final_proj.bias": O.hash_uniform("fp.b", (64,), -0.1, 0.1),
            "label_embs_concat": O.hash_uniform("lab", (C, 64), 0.0, 1.0)}
    m.load_state_dict({**sd, **head}, strict=True)
    return m.to(dev).train(), {**sd, **head}


def _step_against_oracle(dev, cfg, m, sd, wav, pad, labels, ratio, C):
    """One masked-prediction step of `m` and of the oracle on the kept frames; returns T'."""
    B, L = wav.shape
    T = O.num_frames(L, cfg)
    T2 = TO.trimmed_frames(T, labels.shape[1], ratio)
    mi = O.hash_uniform("premask", (B, T2)) > 0.35
    out = m(wav.to(dev), target_list=[labels], padding_mask=pad, mask=True, mask_indices=mi)
    assert out["x"].shape[1] == T2 and out["padding_mask"].shape == (B, T2)
    loss, sample_size, log = m.criterion(out, pred_masked_weight=1.0, pred_nomask_weight=0.5, loss_weights=[10.0])
    loss.backward()
    torch.cuda.synchronize()

    sdr = {k: v.clone().requires_grad_(True) for k, v in sd.items()}
    ref = TO.extract_features(sdr, wav, cfg, T2, padding_mask=pad, mask_indices=mi)
    fpm = ref["padding_mask"]
    assert torch.equal(out["padding_mask"].cpu(), fpm)
    tl = [labels.cpu()[:, (torch.arange(T2).float() * ratio).long()]]
    assert torch.equal(out["target_list"][0].cpu(), tl[0])
    args = (sdr["final_proj.weight"], sdr["final_proj.bias"], sdr["label_embs_concat"], [C], False, 0.1)
    lm = O.masked_prediction_logits(ref["x"], torch.logical_and(~fpm, mi), tl, *args)
    lu = O.masked_prediction_logits(ref["x"], torch.logical_and(~fpm, ~mi), tl, *args)
    pen = ref["conv"].float().pow(2).mean()
    assert abs(out["features_pen"].item() - pen.item()) <= 0.02 * pen.item()
    want, want_ss, _ = O.wavlm_criterion(lm, lu, 1.0, 0.5, pen, [10.0])
    want.backward()
    assert sample_size == want_ss
    assert abs(loss.item() - want.item()) < 0.02 * abs(want.item()) + 0.5, (loss.item(), want.item())
    params = dict(m.named_parameters())
    bad = []
    for k, v in sdr.items():
        if v.grad is None or k.endswith("k_proj.bias"):
            continue
        w_, g_ = v.grad.double(), params[k].grad.detach().double().cpu()
        if w_.norm().item() < 1e-7:
            continue
        cos = ((g_ * w_).sum() / (g_.norm() * w_.norm() + 1e-30)).item()
        rel = abs(g_.norm().item() - w_.norm().item()) / w_.norm().item()
        if cos < 0.98 or rel > (0.1 if w_.numel() > 16 else 0.25):
            bad.append((k, round(cos, 4), round(rel, 4)))
    assert not bad, bad
    return T2


@pytest.mark.parametrize("L,lengths,trimmed", [(160_160, [160_160, 97_001], True), (250_000, [250_000, 123_457], True),
                                               (160_000, [160_000, 101_000], False)])
def test_iteration1_mfcc_kmeans_labels_then_pretraining_step(cuda_device, L, lengths, trimmed):
    from unispeech_b200.kmeans import KMeans
    from unispeech_b200.mfcc import mfcc
    dev = cuda_device
    cfg = O.tiny_config(pre_ln=False, relative_position_embedding=False, gru_rel_pos=False)
    wav, pad = _speech(L, lengths)
    feats, pm, rows = mfcc(wav.to(dev), padding_mask=pad, kmeans_rows=True)
    Tm = MO.num_frames(L)
    assert rows.shape == (2, Tm, 64)
    valid = rows[~pm]
    assert valid.shape[0] == sum(MO.num_frames(n) for n in lengths)
    km = KMeans(100, max_iter=20, seed=0).fit(valid)
    labels = km.predict(rows, pm)
    assert bool((labels[pm] == -1).all())
    cbf, _ = km._device_centers(dev)
    _check_labels(valid, cbf, 100, labels[~pm])
    assert int(labels[~pm].unique().numel()) > 50
    m, sd = _model(dev, cfg, 100, 100)
    T = O.num_frames(L, cfg)
    T2 = _step_against_oracle(dev, cfg, m, sd, wav, pad, labels.long().clamp(min=0), 2.0, 100)
    assert T2 == (T - 1 if trimmed else T)


def test_label_rate_50_with_cropped_labels_trims_to_their_length(cuda_device):
    """50 Hz labels one short of the T conv frames (a cropped label file): the model runs on T - 1 frames."""
    dev = cuda_device
    cfg = O.tiny_config(pre_ln=False, relative_position_embedding=False, gru_rel_pos=False)
    L = 32_000
    wav, pad = _speech(L, [32_000, 20_011])
    T = O.num_frames(L, cfg)
    labels = (O.hash_uniform("tgt", (2, T - 1), 0.0, 1.0) * 37).long().clamp(max=36).to(dev)
    m, sd = _model(dev, cfg, 50, 37)
    assert _step_against_oracle(dev, cfg, m, sd, wav, pad, labels, 1.0, 37) == T - 1


def test_features_only_and_untrimmed_forward_are_unchanged(cuda_device):
    """Labels that cover every frame leave the forward exactly as without labels; features_only never trims."""
    dev = cuda_device
    cfg = O.tiny_config(pre_ln=False, relative_position_embedding=False, gru_rel_pos=False)
    m, _ = _model(dev, cfg, 100, 100)
    m.eval()
    L = 160_000
    wav, pad = _speech(L, [L, 90_000])
    T = O.num_frames(L, cfg)
    with torch.no_grad():
        a = m(wav.to(dev), padding_mask=pad, mask=False, features_only=True)["x"]
        b = m(wav.to(dev), target_list=[torch.zeros(2, 2 * T, dtype=torch.long)], padding_mask=pad, mask=False)["x"]
        c = m(wav.to(dev), target_list=[torch.zeros(2, T, dtype=torch.long)], padding_mask=pad, mask=False,
              features_only=True)["x"]
    assert a.shape[1] == T and torch.equal(a, b) and torch.equal(a, c)
