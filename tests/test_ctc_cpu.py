"""CTC fine-tuning surface without a GPU: the float64 oracle (oracle/ctc_oracle.py) against torch.nn.functional.ctc_loss in float64
(loss and autograd gradient), the criterion's target handling on host tensors, best-path collapse, and the state_dict keys of
HubertCtc / Wav2VecCtc."""
import pytest
import torch
import torch.nn.functional as F

from oracle import ctc_oracle as CO
from oracle import wavlm_oracle as O


def _case(name):
    """(T, B, V, input_len, targets [B, Smax], target_len, blank)"""
    g = torch.Generator().manual_seed(sum(map(ord, name)))
    if name == "ragged":
        T, B, V, blank = 40, 4, 9, 0
        tl = [12, 0, 1, 7]
        il = [40, 25, 3, 31]
    elif name == "all_equal":            # every repeat needs a blank between
        T, B, V, blank = 30, 2, 5, 0
        tl, il = [6, 9], [30, 30]
    elif name == "min_feasible":         # targets (3,3,4): 3 labels + 1 forced blank = 4 frames; 4 is feasible, 3 is not
        T, B, V, blank = 6, 2, 6, 0
        tl, il = [3, 3], [4, 3]
    elif name == "blank_last":
        T, B, V, blank = 25, 3, 7, 6
        tl, il = [5, 8, 2], [25, 20, 9]
    else:
        raise KeyError(name)
    S = max(max(tl), 1)
    lo, hi = (1, V) if blank == 0 else (0, V - 1)
    targets = torch.randint(lo, hi, (B, S), generator=g)
    if name == "all_equal":
        targets[:] = 2
    if name == "min_feasible":
        targets[:] = torch.tensor([3, 3, 4])
    logits = torch.randn(T, B, V, generator=g, dtype=torch.float64) * 2.0
    return logits, torch.tensor(il), targets, torch.tensor(tl), blank


@pytest.mark.parametrize("name", ["ragged", "all_equal", "min_feasible", "blank_last"])
def test_oracle_matches_aten_float64(name):
    logits, il, targets, tl, blank = _case(name)
    x = logits.clone().requires_grad_(True)
    nll = CO.ctc_nll(x, il, targets, tl, blank)
    y = logits.clone().requires_grad_(True)
    ref = F.ctc_loss(F.log_softmax(y, -1), targets, il, tl, blank=blank, reduction="none", zero_infinity=False)
    finite = torch.isfinite(ref)
    assert torch.equal(torch.isfinite(nll), finite)
    if name == "min_feasible":
        assert finite.tolist() == [True, False]
    assert torch.allclose(nll[finite], ref[finite], rtol=1e-12, atol=1e-12)
    nll[finite].sum().backward()
    F.ctc_loss(F.log_softmax(y, -1), targets, il, tl, blank=blank, reduction="sum", zero_infinity=True).backward()
    # float64 on both sides: only the summation order differs
    assert torch.allclose(x.grad, y.grad, rtol=1e-9, atol=1e-11)
    past = torch.arange(logits.shape[0])[:, None] >= il[None, :]   # frames past the input length: exactly zero
    assert x.grad[past].abs().sum().item() == 0


def test_prepare_targets_strips_pad_and_eos():
    from unispeech_b200.ctc import prepare_targets
    pad, eos = 1, 2
    target = torch.tensor([[5, 6, 7, eos, pad, pad],
                           [9, eos, pad, pad, pad, pad],
                           [eos, pad, pad, pad, pad, pad],
                           [4, 4, 8, 3, 5, eos]])
    t, n = prepare_targets(target, pad, eos)
    assert t.dtype == torch.int32 and n.dtype == torch.int32
    assert n.tolist() == [3, 1, 0, 5]
    packed = target.masked_select((target != pad) & (target != eos))   # what the reference feeds F.ctc_loss
    assert torch.equal(torch.cat([t[b, :n[b]] for b in range(4)]).long(), packed)
    # lengths given by the sample win over the mask count
    _, n2 = prepare_targets(target, pad, eos, torch.tensor([2, 1, 0, 5]))
    assert n2.tolist() == [2, 1, 0, 5]


def test_criterion_sample_size_and_logging_on_host(monkeypatch):
    """sentence_avg, ntokens and the lengths the criterion hands to the loss, with the loss itself stubbed (it has no CPU path)."""
    from unispeech_b200 import ctc as C
    seen = {}

    def fake_loss(logits, input_len, targets, target_len, **kw):
        seen.update(input_len=input_len, targets=targets, target_len=target_len, kw=kw)
        return logits.float().sum()

    monkeypatch.setattr(C, "ctc_loss", fake_loss)

    class M(torch.nn.Module):
        def forward(self, source, padding_mask):
            pm = torch.zeros(2, 7, dtype=torch.bool)
            pm[1, 4:] = True
            return {"encoder_out": source, "padding_mask": pm}

        def get_logits(self, net_output):
            return net_output["encoder_out"]

    sample = {"net_input": {"source": torch.ones(7, 2, 5), "padding_mask": None}, "target": torch.tensor([[3, 4, 2], [4, 2, 1]]),
              "id": torch.tensor([10, 11])}
    loss, size, log = C.CtcCriterion(sentence_avg=False)(M().train(), sample)
    assert seen["input_len"].tolist() == [7, 4] and seen["target_len"].tolist() == [2, 1]
    assert seen["targets"][0, :2].tolist() == [3, 4] and seen["targets"][1, :1].tolist() == [4]
    assert seen["kw"] == {"blank": 0, "reduction": "sum", "zero_infinity": False, "return_argmax": False}
    assert int(size) == 3 and int(log["ntokens"]) == 3 and log["nsentences"] == 2 and float(log["loss"]) == float(loss)
    _, size, _ = C.CtcCriterion(sentence_avg=True)(M().train(), sample)
    assert size == 2
    monkeypatch.undo()
    with pytest.raises(ValueError):   # the real loss refuses host tensors: there is no CPU path
        C.ctc_loss(torch.zeros(3, 1, 4), torch.tensor([3]), torch.tensor([[1]]), torch.tensor([1]))


def test_greedy_collapse():
    from unispeech_b200.ctc import greedy_collapse
    am = torch.tensor([[0, 3, 3, 0, 3, 4, 4, 0], [5, 5, 0, 0, 5, 1, 1, 1], [0, 0, 0, 0, 0, 0, 0, 0]])
    assert greedy_collapse(am, [8, 5, 8]) == [[3, 3, 4], [5, 5], []]
    assert greedy_collapse(am, [8, 8, 8], blank=5) == [[0, 3, 0, 3, 4, 0], [0, 1], [0]]


@pytest.mark.parametrize("kind", ["hubert", "wav2vec"])
def test_ctc_model_state_dict_keys(kind):
    from unispeech_b200.ctc import HubertCtc, Wav2VecCtc
    from unispeech_b200.wav2vec2 import Wav2Vec2Config, Wav2Vec2Model
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    w2v = kind == "wav2vec"
    cfg = O.tiny_config(pre_ln=w2v, relative_position_embedding=not w2v, gru_rel_pos=not w2v)
    if kind == "hubert":
        model = HubertCtc.build_model(WavLM(WavLMConfig(vars(cfg))), 32)
    else:
        model = Wav2VecCtc.build_model(Wav2Vec2Model(Wav2Vec2Config(vars(cfg))), 32, apply_mask=True)
    keys = set(model.state_dict())
    assert {"w2v_encoder.proj.weight", "w2v_encoder.proj.bias"} <= keys
    assert tuple(model.state_dict()["w2v_encoder.proj.weight"].shape) == (32, cfg.encoder_embed_dim)
    enc_keys = {k for k in keys if k.startswith("w2v_encoder.w2v_model.")}
    assert enc_keys == {"w2v_encoder.w2v_model." + k for k in model.w2v_encoder.w2v_model.state_dict()}
    assert keys == enc_keys | {"w2v_encoder.proj.weight", "w2v_encoder.proj.bias"}
    assert "w2v_encoder.w2v_model.encoder.layers.0.fc1.weight" in keys
    model.set_num_updates(7)
    assert model.w2v_encoder.num_updates == 7
    with pytest.raises(ValueError):
        HubertCtc(type(model.w2v_encoder)(WavLM(WavLMConfig(vars(cfg)))))   # no proj: nothing to put a CTC loss on
