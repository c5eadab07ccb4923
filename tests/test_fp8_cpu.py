"""FP8 inference path, host side: the e4m3 quantisation rule the kernels implement (unispeech_b200/fp8.py) and the argument
errors of `extract_features(fp8=True)`, which are raised before anything touches a device."""
import pytest
import torch

from oracle import wavlm_oracle as O
from unispeech_b200.fp8 import quantize_rows_reference
from unispeech_b200.wavlm import WavLM, WavLMConfig

def test_scale_maps_row_amax_to_448():
    x = torch.tensor([[1.0, -3.0, 0.5], [0.0, 0.0, 0.0], [-2.5, 1e-3, 2.5]])
    q, s = quantize_rows_reference(x)
    assert q.float()[0].tolist() == [144.0, -448.0, 72.0]       # 149.3 -> 144 (spacing 16), 74.7 -> 72 (spacing 8)
    assert q.float()[2].abs().max().item() == 448.0
    assert torch.equal(s, torch.tensor([3.0, 0.0, 2.5]) / 448.0)  # fp32 division
    assert torch.all(q.float()[1] == 0)                       # zero row: q = 0, s = 0, no NaN
    assert not torch.isnan(q.float()).any()


def test_rows_below_min_amax_count_as_zero():
    # 448 / amax overflows fp32 below about 1.3e-36: such rows (bf16 subnormals, say) quantise to zeros with s = 0, not NaN
    x = torch.tensor([[2.0 ** -126, 0.0, -(2.0 ** -130)], [2.0 ** -119, 0.0, 2.0 ** -120]])
    q, s = quantize_rows_reference(x)
    assert q.float()[0].tolist() == [0.0, 0.0, 0.0] and s[0].item() == 0.0
    assert q.float()[1].tolist() == [448.0, 0.0, 224.0] and torch.equal(s[1], torch.tensor(2.0 ** -119) / torch.tensor(448.0))


def test_round_to_nearest_even_ties():
    # values in [256, 448): spacing 32 in e4m3.  With amax = 448 the scale is 1, so x itself is rounded.
    x = torch.tensor([[448.0, 272.0, 304.0, 336.0, 368.0, 273.0]])
    q, _ = quantize_rows_reference(x)
    # 272 = 256 + 16: tie -> even mantissa (256); 304 = 288 + 16: tie -> 320; 336 -> 320; 368 -> 384; 273 -> 288
    assert q.float()[0].tolist() == [448.0, 256.0, 320.0, 320.0, 384.0, 288.0]


def test_subnormals_down_to_2_pow_minus_9():
    tiny = 2.0 ** -9
    x = torch.tensor([[448.0, tiny, 3 * tiny, tiny / 2, tiny * 0.5001, 2.0 ** -6, 7 * tiny]])
    q, _ = quantize_rows_reference(x)
    # the smallest subnormal survives; half of it is a tie to even (0); just above half rounds up to the subnormal
    assert q.float()[0].tolist() == [448.0, tiny, 3 * tiny, 0.0, tiny, 2.0 ** -6, 7 * tiny]


def test_quantised_values_stay_within_448_for_random_rows():
    g = torch.Generator().manual_seed(0)
    x = (torch.randn(64, 1024, generator=g) * torch.logspace(-4, 4, 64).unsqueeze(1)).to(torch.bfloat16)
    q, s = quantize_rows_reference(x)
    qf = q.float()
    assert not torch.isnan(qf).any() and qf.abs().max().item() == 448.0
    assert torch.all(qf.abs().amax(1) == 448.0)
    rel = ((qf * s.unsqueeze(1) - x.float()).abs() / x.float().abs().amax(1, keepdim=True)).max().item()
    assert rel <= 16.0 / 448.0 * 1.0001                         # half the e4m3 spacing (32) next to 448, relative to amax


def _tiny_model():
    cfg = O.tiny_config(pre_ln=False)
    m = WavLM(WavLMConfig(vars(cfg)))
    return m


def test_fp8_errors_before_the_device():
    m = _tiny_model()                                           # CPU model, CPU input: any launch would raise a different error
    wav = torch.zeros(1, 8000)
    with pytest.raises(RuntimeError, match="model.eval"):
        m.train().extract_features(wav, fp8=True)
    m.eval()
    with pytest.raises(RuntimeError, match="without a backward"):
        m.extract_features(wav, fp8=True)
    with torch.no_grad(), pytest.raises(RuntimeError, match="mask=True"):
        m.extract_features(wav, mask=True, fp8=True)
    for p in m.parameters():
        p.requires_grad_(False)
    with pytest.raises(RuntimeError, match="mask=True"):    # grad enabled, but nothing requires it: only the mask is refused
        m.extract_features(wav, mask=True, fp8=True)


def test_fp8_is_keyword_only():
    m = _tiny_model().eval()
    with pytest.raises(TypeError):
        m.extract_features(torch.zeros(1, 8000), None, False, False, None, False, None, None, True)
