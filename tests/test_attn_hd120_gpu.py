"""Attention at head width 120 (XLS-R 2B: D = 1920, 16 heads), without the relative-position bias: forward output and
log-sum-exp against fp64, dQ / dK / dV through b200s_attn_bwd and b200s_attn_bwd_fused against fp64 autograd with a sentinel in
dqkv (unwritten columns show), attention dropout (keep bits equal to the hash, forward / backward equal to the reference run
with those bits), neighbour isolation at head widths 64, 80 and 120 (a head is read and written as exactly its own columns through
the head-shaped tensor maps; at 120 the zero-filled tail of its second 64-column block never holds the next head's columns), and
LayerNorm (+GELU) at D = 1920."""
import pytest
import torch

from oracle import wavlm_oracle as O
from test_attn_hd80_gpu import bf, check_bwd, check_fwd, make_inputs, unpack_mask

pytestmark = pytest.mark.gpu

HD = 120
SENTINEL = 3.0

CASES = [  # B, T, H, valid frames per utterance (None: no padding)
    (2, 999, 16, None),
    (2, 999, 16, (999, 640)),
    (2, 300, 4, None),          # last query tile: rows 256..299, the second consumer warpgroup's rows are all beyond T
    (1, 1, 2, None),
    (3, 300, 2, (300, 57, 200)),  # ragged, one utterance shorter than one tile
]


def run_fwd(qkv, pad, B, T, H, hd=HD):
    from unispeech_b200 import ops
    out = torch.full((B, T, H * hd), SENTINEL, device=qkv.device, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=qkv.device)
    ops.attn_fwd(qkv, None, None, pad, out, lse, B, T, H, hd ** -0.5, head_dim=hd)
    return out, lse


def run_bwd(qkv, out, dout, lse, pad, B, T, H, fused=True, hd=HD):
    from unispeech_b200 import ops
    D = H * hd
    delta = torch.empty(B, H, T, device=qkv.device)
    dqkv = torch.full((B, T, 3 * D), SENTINEL, device=qkv.device, dtype=torch.bfloat16)
    if fused:
        dq_acc = torch.zeros(B, T, D, device=qkv.device)
        ops.attn_bwd_fused(qkv, out, dout, None, None, pad, lse, delta, dq_acc, dqkv, None, None, B, T, H, hd ** -0.5,
                           head_dim=hd)
        torch.cuda.synchronize()
        assert dq_acc.abs().max().item() == 0.0
    else:
        ops.attn_bwd(qkv, out, dout, None, None, pad, lse, delta, dqkv, None, None, B, T, H, hd ** -0.5, head_dim=hd)
        torch.cuda.synchronize()
    return dqkv


def assert_written(t, pad):
    """No sentinel survives on a valid row (a column the kernel skipped would keep it exactly)."""
    rows = (pad == 0) if pad is not None else torch.ones(t.shape[:2], dtype=torch.bool, device=t.device)
    assert not (t[rows] == SENTINEL).all(dim=0).any()


@pytest.mark.parametrize("B,T,H,valid", CASES)
def test_attn_hd120_fwd_bwd(cuda_device, B, T, H, valid):
    qkv, pad, dout = make_inputs(cuda_device, B, T, H, HD, valid, seed=T + B + 120)
    out, lse = run_fwd(qkv, pad, B, T, H)
    torch.cuda.synchronize()
    assert_written(out, pad)
    check_fwd(out, lse, qkv, pad, B, T, H, HD)
    for fused in (True, False):
        dqkv = run_bwd(qkv, out, dout, lse, pad, B, T, H, fused)
        assert_written(dqkv, pad)
        check_bwd(dqkv, qkv, pad, dout, B, T, H, HD)


def test_attn_hd120_long(cuda_device):
    B, T, H = 1, 4096, 2
    qkv, pad, dout = make_inputs(cuda_device, B, T, H, HD, None, seed=4096 + 120)
    out, lse = run_fwd(qkv, pad, B, T, H)
    dqkv = run_bwd(qkv, out, dout, lse, pad, B, T, H)
    check_fwd(out, lse, qkv, pad, B, T, H, HD)
    check_bwd(dqkv, qkv, pad, dout, B, T, H, HD)


@pytest.mark.parametrize("head", [0, 2, 3])
@pytest.mark.parametrize("hd", [64, 80, 120])
def test_attn_hd120_neighbours_isolated(cuda_device, hd, head):
    """Every column outside head `head` of q, k and v (the other heads, and the same head of the other two sections) holds
    +-1e3.  The head's output and log-sum-exp must equal those of a run with zeros there bit for bit, its gradients up to the
    rounding of the dQ reductions, and both must match fp64.  head = 3 is the last head of each section (at width 120 its
    second block's tail is the next section's first head, or the end of the row)."""
    B, T, H = 2, 300, 4
    D = H * hd
    qkv, pad, dout = make_inputs(cuda_device, B, T, H, hd, (300, 170), seed=head + 31)
    cols = torch.zeros(3 * D, dtype=torch.bool, device=cuda_device)
    for sec in range(3):
        cols[sec * D + head * hd: sec * D + (head + 1) * hd] = True
    own = torch.zeros(D, dtype=torch.bool, device=cuda_device)
    own[head * hd:(head + 1) * hd] = True
    g = torch.Generator(device=cuda_device).manual_seed(head)
    loud = torch.where(torch.rand(B, T, 3 * D, device=cuda_device, generator=g) < 0.5, -1e3, 1e3).to(torch.bfloat16)
    quiet = qkv.clone()
    quiet[..., ~cols] = 0
    noisy = torch.where(cols, qkv, loud)
    dout_h = dout.clone()
    dout_h[..., ~own] = 0
    res = []
    for x in (quiet, noisy):
        out, lse = run_fwd(x, pad, B, T, H, hd=hd)
        dqkv = run_bwd(x, out, dout_h, lse, pad, B, T, H, hd=hd)
        res.append((out, lse, dqkv))
    (o0, l0, g0), (o1, l1, g1) = res
    rows = pad == 0
    assert torch.equal(o0[..., own][rows], o1[..., own][rows])
    assert torch.equal(l0[:, head], l1[:, head])
    # dQ is summed over key tiles by fp32 reductions in no fixed order, so the gradients may differ by rounding; a leaked +-1e3
    # would be orders of magnitude larger
    ga, gb = g0[..., cols][rows].double(), g1[..., cols][rows].double()
    assert (ga - gb).abs().max().item() <= 2.0 ** -7 * ga.abs().max().item()
    # and the head's results are right
    check_fwd(o1[..., own].contiguous(), l1[:, head:head + 1].contiguous(), quiet[..., cols].contiguous(), pad, B, T, 1, hd)
    check_bwd(g1[..., cols].contiguous(), quiet[..., cols].contiguous(), pad, dout[..., own].contiguous(), B, T, 1, hd)


@pytest.mark.parametrize("B,T,H,valid", [(2, 300, 3, (300, 200)), (1, 520, 2, None)])
def test_attn_hd120_dropout(cuda_device, B, T, H, valid):
    from unispeech_b200 import ops
    dev, p = cuda_device, 0.1
    D = H * HD
    qkv, pad, dout = make_inputs(dev, B, T, H, HD, valid, seed=T + 120)
    d = O.HashDropout(1207 + T)
    site = O.HashDropout.layer_site(2, 3)
    key = tuple(int(v) for v in d.key(site))
    out = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    lse = torch.empty(B, H, T, device=dev)
    words = torch.full((ops.attn_dropout_mask_words(B, T, H),), -1, dtype=torch.int32, device=dev)
    ops.attn_fwd_dropout(qkv, None, None, pad, out, lse, B, T, H, HD ** -0.5, p, key, words, head_dim=HD)
    torch.cuda.synchronize()
    got_keep = unpack_mask(words, B, T, H)
    want_keep = torch.from_numpy(d.keep_attn(site, B, H, T, p))
    if pad is not None:  # bits are specified where both the key and the query frame are valid
        ok = (pad == 0).cpu()
        sel = (ok[:, None, None, :] & ok[:, None, :, None]).expand_as(want_keep)
        assert torch.equal(got_keep[sel], want_keep[sel])
    else:
        assert torch.equal(got_keep, want_keep)
    keep = want_keep.to(dev)
    check_fwd(out, lse, qkv, pad, B, T, H, HD, keep, p)
    delta = torch.empty(B, H, T, device=dev)
    dqkv = torch.full((B, T, 3 * D), SENTINEL, device=dev, dtype=torch.bfloat16)
    dq_acc = torch.zeros(B, T, D, device=dev)
    ops.attn_bwd_fused_dropout(qkv, out, dout, None, None, pad, lse, delta, dq_acc, dqkv, None, None, B, T, H, HD ** -0.5, p,
                               words, head_dim=HD)
    torch.cuda.synchronize()
    assert_written(dqkv, pad)
    check_bwd(dqkv, qkv, pad, dout, B, T, H, HD, keep, p)


@pytest.mark.parametrize("gelu", [False, True], ids=["ln", "ln_gelu"])
@pytest.mark.parametrize("ragged", [False, True], ids=["dense", "ragged"])
def test_layer_norm_1920(cuda_device, ragged, gelu):
    """Warp-per-row LayerNorm (and LayerNorm + GELU) forward and backward at D = 1920 (4 columns x 15 chunks per lane), dense
    and ragged, against fp64."""
    from unispeech_b200 import ops
    dev, B, T, D = cuda_device, 2, 37, 1920
    torch.manual_seed(1920 + gelu)
    x = bf(torch.randn(B, T, D, device=dev) * 2 + 0.5)
    w = torch.randn(D, device=dev) * 0.5 + 1
    bias = torch.randn(D, device=dev) * 0.1
    dy = bf(torch.randn(B, T, D, device=dev))
    rows = torch.ones(B, T, dtype=torch.bool, device=dev)
    valid = None
    if ragged:
        valid = torch.tensor([T, 20], dtype=torch.int32, device=dev)
        rows[1, 20:] = False
        dy[~rows] = 0
    xr = x.double().requires_grad_(True)
    wr, br = w.double().requires_grad_(True), bias.double().requires_grad_(True)
    yr = torch.nn.functional.layer_norm(xr, (D,), wr, br, eps=1e-5)
    if gelu:
        yr = torch.nn.functional.gelu(yr)
    yr.backward(dy.double())
    y = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    mean = torch.empty(B * T, device=dev)
    rstd = torch.empty(B * T, device=dev)
    ops.layer_norm_fwd(x, T * D, D, w, bias, y, T * D, D, mean, rstd, T, B, D, gelu=gelu, valid=valid)
    dx = torch.empty(B, T, D, device=dev, dtype=torch.bfloat16)
    dw = torch.zeros(D, device=dev)
    db = torch.zeros(D, device=dev)
    ops.layer_norm_bwd(dy, T * D, D, x, T * D, D, mean, rstd, w, bias, None, 0, 0, dx, T * D, D, dw, db, None, T, B, D,
                       gelu=gelu, valid=valid)
    torch.cuda.synchronize()
    assert (y.double() - yr.detach())[rows].abs().max().item() < 0.05
    assert (dx.double() - xr.grad)[rows].abs().max().item() < 0.03 * max(1.0, xr.grad.abs().max().item())
    assert (dw.double() - wr.grad).abs().max().item() < 1e-2 * max(1.0, wr.grad.abs().max().item())
    assert (db.double() - br.grad).abs().max().item() < 1e-2 * max(1.0, br.grad.abs().max().item())
