"""Pieces shared by the pre-training loss heads (pretrain.py, ils_hubert.py, unispeech_sat.py, wav2vec2.py) and the output
projection of fairseq_encoder.py: the selected-rows `nn.Linear` (gather -> wgmma GEMM with the bias in its epilogue, and its
backward), the Gumbel vector quantizer of the contrastive targets, the host draw of the contrastive negatives and the weighting
of the models' extra losses.  Everything here runs on the project's kernels; this module imports nothing model-specific.
"""
from __future__ import annotations

import torch
import torch.nn as nn

from . import _lib as L
from . import ops
from .engine import BF

_EPS = 1e-7   # inside the log of the perplexities, as in gumbel_vector_quantizer.py:152-170


def _rows(n, C, dtype, dev):
    return torch.empty(n, C, dtype=dtype, device=dev)


def bf16(t: torch.Tensor) -> torch.Tensor:
    """`t` as a contiguous bf16 tensor (no copy when it already is one)."""
    return t if (t.dtype == BF and t.is_contiguous()) else t.to(BF).contiguous()


def gather(x2d, idx):
    """bf16 rows x2d[idx] (idx: int32 device vector)."""
    S, D = idx.numel(), x2d.shape[1]
    xs = _rows(S, D, BF, x2d.device)
    ops.gather_rows(x2d, D, idx, S, D, xs, D)
    return xs


def scatter(dxs, idx, rows):
    """Backward of `gather`: a zero bf16 [rows, D] gradient with dxs added at the rows idx."""
    S, D = dxs.shape
    dx = torch.zeros(rows, D, dtype=BF, device=dxs.device)
    ops.scatter_add_rows(dxs, D, idx, S, D, dx, D)
    return dx


# ------------------------------------------------------------------------------------------------- nn.Linear on selected rows
def linear_operands(w):
    """bf16 GEMM operands (W, W^T) of an fp32 `nn.Linear` weight [N, K]."""
    N, K = w.shape
    W, WT = _rows(N, K, BF, w.device), _rows(K, N, BF, w.device)
    ops.prep_linear(w, N, K, 1.0, W, K, WT, N)
    return W, WT


def linear_rows(x, W, bias):
    """y = x W^T + bias for bf16 rows x [S, K]; bias fp32 [N]."""
    S, K = x.shape
    N = W.shape[0]
    y = _rows(S, N, BF, x.device)
    ops.gemm_rows(x, 0, K, S, 1, K, W, N, y, 0, N, L.make_epilogue(bias=bias))
    return y


def linear_rows_backward(dy, x, WT, g_w, g_b, res=None):
    """Backward of `linear_rows`: g_b += colsum(dy), g_w += dy^T x (fp32 views), returns dx = dy W (+ res, bf16 [S, K], added in
    the GEMM's epilogue)."""
    S, N = dy.shape
    K = x.shape[1]
    ops.colsum(dy, 0, N, S, 1, N, g_b)
    ops.gemm_wgrad(dy, 0, N, x, 0, K, S, 1, N, K, g_w, K)
    dx = _rows(S, K, BF, dy.device)
    ops.gemm_rows(dy, 0, N, S, 1, N, WT, K, dx, 0, K, None if res is None else L.make_epilogue(res1=res, res1_ld=K))
    return dx


# ------------------------------------------------------------------------------------------------- Gumbel vector quantizer
def perplexity(p, keepdim=False):
    """exp(entropy) of each row of a [G, V] distribution (gumbel_vector_quantizer.py:152-170)."""
    return torch.exp(-torch.sum(p * torch.log(p + _EPS), dim=-1, keepdim=keepdim))


def perplexity_grad(p, dppl):
    """dppl * d(sum_g perplexity(p)_g) / dp, flattened to [G * V]."""
    return (dppl.float() * perplexity(p, keepdim=True) * (-torch.log(p + _EPS) - p / (p + _EPS))).reshape(-1).contiguous()


class GumbelVectorQuantizer(nn.Module):
    """Parameters, temperature schedule (src/fairseq/modules/gumbel_vector_quantizer.py:13-201; time_first, combine_groups=False,
    weight_proj_depth=1) and the forward / backward of hard codes on selected rows."""

    def __init__(self, dim, num_vars, temp, groups, vq_dim):
        super().__init__()
        assert vq_dim % groups == 0
        self.groups, self.num_vars, self.input_dim = groups, num_vars, dim
        self.vars = nn.Parameter(torch.FloatTensor(1, groups * num_vars, vq_dim // groups))
        nn.init.uniform_(self.vars)
        self.weight_proj = nn.Linear(dim, groups * num_vars)
        nn.init.normal_(self.weight_proj.weight, mean=0, std=1)
        nn.init.zeros_(self.weight_proj.bias)
        self.max_temp, self.min_temp, self.temp_decay = temp
        self.curr_temp = self.max_temp

    def set_num_updates(self, num_updates):
        self.curr_temp = max(self.max_temp * self.temp_decay ** num_updates, self.min_temp)

    def forward_rows(self, x, key, stats_out):
        """Quantize the bf16 rows x [S, dim] (gumbel_vector_quantizer.py:141-201): weight_proj GEMM, then per group the arg-max
        code (eval) or the Gumbel hard sample with the counter-based noise of `key` (training).  Returns q (bf16 [S, vq_dim], the
        chosen code vectors) and the state `backward_rows` needs (`codes`: int32 [S * groups], `avg_probs`: [groups, num_vars]
        mean softmax, the input of prob_perplexity); fills `code_perplexity`, `num_vars` and `temp` of stats_out."""
        S, dev = x.shape[0], x.device
        G, V, dv = self.groups, self.num_vars, self.vars.shape[-1]
        GV = G * V
        w, wT = linear_operands(self.weight_proj.weight)
        logits = linear_rows(x, w, self.weight_proj.bias)
        codes = torch.empty(S * G, dtype=torch.int32, device=dev)
        q = _rows(S, G * dv, BF, dev)
        counts = torch.zeros(GV, dtype=torch.float32, device=dev)
        probs = torch.zeros(GV, dtype=torch.float32, device=dev)
        ops.vq_hard(logits, GV, self.vars, S, G, V, dv, codes, q, G * dv, counts, probs, gumbel=self.training, key=key)
        # perplexities: tiny [G, V] reductions of the kernel's accumulators
        stats_out["code_perplexity"] = perplexity((counts / S).view(G, V)).sum()
        stats_out["num_vars"] = GV
        stats_out["temp"] = self.curr_temp
        return q, dict(x=x, wT=wT, logits=logits, codes=codes, avg_probs=(probs / S).view(G, V), training=self.training,
                       tau=float(self.curr_temp), key=key)

    def backward_rows(self, st, dq, dppl, g):
        """Backward of `forward_rows` for dq = d loss / d q and dppl = d loss / d prob_perplexity (None: not used): accumulates the
        `vars` and `weight_proj` gradients into their views g(param) and returns the gradient of the input rows, or None when
        nothing reaches the logits (eval mode without the diversity term)."""
        S, dev = dq.shape[0], dq.device
        G, V, dv = self.groups, self.num_vars, self.vars.shape[-1]
        GV, vq_dim = G * V, G * dv
        ops.vq_dvars(dq, vq_dim, st["codes"], S, G, V, dv, g(self.vars).view(GV, dv))
        # gradient of the logits: diversity term (through avg_probs) and, in training mode, the straight-through estimator of
        # F.gumbel_softmax(hard=True)
        c = None if dppl is None else perplexity_grad(st["avg_probs"], dppl)
        h = None
        if st["training"]:
            vb, _ = linear_operands(self.vars.view(GV, dv))
            h = _rows(S, GV, BF, dev)
            for grp in range(G):   # h[s, g, v] = dq[s, g, :] . vars[g, v, :]
                ops.gemm_rows(dq.view(-1)[grp * dv:], 0, vq_dim, S, 1, dv, vb[grp * V:(grp + 1) * V], V, h.view(-1)[grp * V:], 0,
                              GV, None)
        if c is None and h is None:
            return None
        dlogits = _rows(S, GV, BF, dev)
        ops.vq_logits_bwd(st["logits"], GV, S, G, V, c, h, GV, st["tau"], st["key"], dlogits, GV)
        return linear_rows_backward(dlogits, st["x"], st["wT"], g(self.weight_proj.weight), g(self.weight_proj.bias))


# ------------------------------------------------------------------------------------------------- host side
def sample_instances(bsz: int, num: int, n_instances: int, cross_sample_instances: int, generator=None) -> torch.Tensor:
    """Flat row indices [bsz, (n + c) * num] into y.view(-1, C) drawn exactly like unispeech_sat.py:487-533 and wav2vec2.py:488-523
    (host RNG: the same `torch.randint` calls in the same order; `idx[idx >= tszs] += 1` is written as `idx += (idx >= tszs)`,
    which is the same update without the boolean gather / scatter -- half of the reference formulation's host time)."""
    cross_high, high = num * bsz, num
    assert high > 1, (bsz, num)
    if n_instances > 0:
        tszs = torch.arange(num).unsqueeze(-1).expand(-1, n_instances).flatten()
        instance_idxs = torch.randint(low=0, high=high - 1, size=(bsz, n_instances * num), generator=generator)
        instance_idxs += (instance_idxs >= tszs)
    if cross_sample_instances > 0:
        tszs = torch.arange(num).unsqueeze(-1).expand(-1, cross_sample_instances).flatten()
        cross_instance_idxs = torch.randint(low=0, high=cross_high - 1, size=(bsz, cross_sample_instances * num), generator=generator)
        cross_instance_idxs += (cross_instance_idxs >= tszs)
    if n_instances > 0:
        instance_idxs += (torch.arange(bsz) * high).unsqueeze(1)
    else:
        instance_idxs = cross_instance_idxs
    if cross_sample_instances > 0 and n_instances > 0:
        instance_idxs = torch.cat([instance_idxs, cross_instance_idxs], dim=1)
    return instance_idxs


def weighted_extra_losses(extra_losses, loss_weights, sample_size):
    """(position, coef * loss * sample_size) of every extra loss with a non-zero weight and a value (wavlm_criterion.py:89-103,
    the same rule in wav2vec_criterion.py): a single weight applies to every extra loss, otherwise the weights are positional."""
    lw = list(loss_weights)
    if len(lw) == 1 and len(extra_losses) != 1:
        lw = [lw[0]] * len(extra_losses)
    assert len(extra_losses) == len(lw), f"{len(extra_losses)}, {len(lw)}"
    return [(i, coef * p.float() * sample_size) for i, (p, coef) in enumerate(zip(extra_losses, lw)) if coef != 0 and p is not None]
