"""Attention and whole-model runs past the lengths the attention kernels used to accept: 3840 frames (76.8 s) for the forward
with the relative-position bias, 19,968 without, 4096 for b200s_attn_bwd and 2048 for the fused backward and attention dropout.
Both kernels now stage a constant amount of shared memory per tile, so the cases below cross each old cap by a tile or more.

Host memory: the fp32 references materialise [B*H, T, T] tensors, several at a time.  The kernel-level cases keep B*H small
(at most 2 GB per tensor at T = 20000, H = 1).  The model-level oracle runs all heads at once: 1.6 GB per tensor for WavLM-Large
at T = 4999 (16 heads) and 1.9 GB for WavLM-Base at B = 2, T = 4499 (12 heads), so those cases want some 16 GB of host memory."""
import math

import pytest
import torch

import test_dropout_gpu
from oracle import wavlm_oracle as O
from test_attn_bwd_edges_gpu import _check_bwd, _ref_out_lse
from test_fullscale_gpu import grad_case, run_forward_case, state_dict_for
from test_kernels_gpu import bf

pytestmark = pytest.mark.gpu


def _check_fwd(dev, B, T, H, bias, lengths):
    from unispeech_b200 import ops
    torch.manual_seed(T + 11)
    D = H * 64
    qkv = bf(torch.randn(B, T, 3 * D, device=dev))
    gate = (torch.rand(B, H, T, device=dev) * 2 + 0.2) if bias else None
    tab = torch.randn(H, 2 * T - 1, device=dev) if bias else None
    pad = None
    if lengths is not None:
        pad = torch.zeros(B, T, device=dev, dtype=torch.uint8)
        for b, n in enumerate(lengths):
            pad[b, n:] = 1
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    ops.attn_fwd(qkv, gate, tab, pad, out, lse, B, T, H, 0.125)
    torch.cuda.synchronize()
    assert torch.isfinite(out.float()).all()
    valid = pad == 0 if pad is not None else torch.ones(B, T, dtype=torch.bool, device=dev)
    # one head at a time: the reference's [T, T] score matrix is the memory bound
    for h in range(H):
        cols = torch.cat([torch.arange(h * 64, h * 64 + 64) + o for o in (0, D, 2 * D)]).to(dev)
        ref_out, ref_lse = _ref_out_lse(qkv[..., cols].contiguous(), gate[:, h:h + 1].contiguous() if bias else None,
                                        tab[h:h + 1].contiguous() if bias else None, pad, B, T, 1, 0.125)
        err = (out[..., h * 64:(h + 1) * 64].float() - ref_out.float())[valid].abs().max().item()
        assert err < 0.03, (h, err)
        lerr = (lse[:, h] - ref_lse[:, 0])[valid].abs().max().item()
        assert lerr < 1e-3 * max(1.0, ref_lse[:, 0][valid].abs().max().item()), (h, lerr)
        del ref_out, ref_lse
        torch.cuda.empty_cache()


@pytest.mark.parametrize("B,T,H,lengths", [
    (1, 3968, 1, None),           # 31 key tiles: the first length past the old cap with the bias
    (2, 5000, 1, (5000, 2001)),   # one utterance padded to 2001 frames
    (1, 8192, 2, None),
])
def test_attn_fwd_long_bias(cuda_device, B, T, H, lengths):
    _check_fwd(cuda_device, B, T, H, True, lengths)


def test_attn_fwd_long_nobias_T20000(cuda_device):
    """157 key tiles, past the old no-bias cap of 19,968 frames."""
    _check_fwd(cuda_device, 1, 20000, 1, False, None)


@pytest.mark.parametrize("fused", [True, False])
@pytest.mark.parametrize("B,T,H,lengths", [
    (2, 4224, 1, (4200, 2500)),   # 33 tiles, a different padding length per utterance
    (1, 8192, 1, (8065,)),        # the last valid frame one row into a tile
])
def test_attn_bwd_long_bias(cuda_device, B, T, H, lengths, fused):
    # the fused path checks that dq_acc comes back zeroed
    _check_bwd(cuda_device, B, T, H, True, lengths, fused)


@pytest.mark.parametrize("B,T,H,padded", [(1, 2176, 2, False), (2, 4224, 1, True)])
def test_attn_dropout_long(cuda_device, B, T, H, padded):
    """Keep bits equal O.HashDropout.keep_attn; outputs and gradients within test_attn_dropout_fwd_bwd's bounds."""
    test_dropout_gpu.test_attn_dropout_fwd_bwd(cuda_device, B, T, H, True, padded, 0.1)


def test_large_2l_100s_vs_oracle(cuda_device):
    """WavLM-Large widths, 2 layers, 1 x 100 s (T = 4999)."""
    cfg = O.large_config(encoder_layers=2)
    run_forward_case("large2_T4999", cfg, state_dict_for("large2", cfg), 1, 1600000, None, cuda_device)


def test_base_2l_ragged_90s_40s_vs_oracle(cuda_device):
    """WavLM-Base widths, 2 layers, ragged {90 s, 40 s} (T = 4499)."""
    cfg = O.base_config(encoder_layers=2)
    L = 1440000
    run_forward_case("base2_T4499_ragged", cfg, state_dict_for("base2", cfg), 2, L, [L, 640000], cuda_device, abs_tol=0.12)


def test_gradients_base_2l_84s(cuda_device):
    """WavLM-Base widths, 2 layers, 1 x 84 s (T = 4199): past the old b200s_attn_bwd cap of 4096 frames."""
    cfg = O.base_config(encoder_layers=2)
    L = 1344000
    grad_case("grad_base2_T4199", cfg, state_dict_for("base2", cfg), 1, L, [L], cuda_device)


def test_large_24l_300s_extract_features_runs(cuda_device):
    """WavLM-Large, all 24 layers, extract_features under no_grad on 1 x 300 s (T = 14999): runs, and every output is finite."""
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    cfg = O.large_config()
    torch.manual_seed(0)
    m = WavLM(WavLMConfig(vars(cfg))).to(cuda_device).eval()
    L = 4800000
    wav = torch.randn(1, L, device=cuda_device)
    with torch.no_grad():
        x, _ = m.extract_features(wav)
    torch.cuda.synchronize()
    assert x.shape[:2] == (1, O.num_frames(L, cfg)) and x.shape[1] == 14999
    assert torch.isfinite(x.float()).all()
    assert not math.isnan(x.float().std().item())
