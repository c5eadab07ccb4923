"""float64 restatement of log-softmax + CTC (Graves et al. 2006), the reference the CTC kernels are tested against.

A plain alpha recursion over the extended label sequence (blank, l_1, blank, ..., l_S, blank): a Python loop over frames,
vectorised over the batch and the positions, built from differentiable torch operations only.  Gradients of the reference come
from `torch.autograd` through this recursion, never from the alpha-beta closed form the kernels use.  tests/test_ctc_cpu.py
checks it against `torch.nn.functional.ctc_loss` in float64.
"""
import torch

NEG = -1e30   # stands for log 0: exp(NEG - m) is exactly 0 in float64 and, unlike -inf, keeps autograd free of inf - inf


def ctc_nll(logits_tbv: torch.Tensor, input_len, targets: torch.Tensor, target_len, blank: int = 0) -> torch.Tensor:
    """Per-utterance negative log-likelihood [B] (float64; +inf where no alignment exists).
    logits_tbv: T x B x V (any float dtype, promoted to float64; may require grad); targets: [B, Smax] padded; lengths: [B].
    Frames at t >= input_len[b] do not enter the result, but must be finite (their zero gradient is 0 * value)."""
    x = logits_tbv.double()
    lp = torch.log_softmax(x, dim=-1)
    T, B, V = lp.shape
    input_len = torch.as_tensor(input_len, dtype=torch.long)
    target_len = torch.as_tensor(target_len, dtype=torch.long)
    S = targets.shape[1]
    L = 2 * S + 1
    ext = torch.full((B, L), blank, dtype=torch.long)
    ext[:, 1::2] = targets.long().clamp(0, V - 1)
    skip = torch.zeros(B, L, dtype=torch.bool)
    skip[:, 2:] = (ext[:, 2:] != blank) & (ext[:, 2:] != ext[:, :-2])
    pos = torch.arange(L)[None, :]
    inside = pos < (2 * target_len + 1)[:, None]   # positions of each utterance's own extended sequence
    alpha = torch.full((B, L), NEG, dtype=torch.float64)
    alpha[:, 0] = 0.0   # before frame 0 all mass sits in front of position 0
    pad1 = torch.full((B, 1), NEG, dtype=torch.float64)
    pad2 = torch.full((B, 2), NEG, dtype=torch.float64)
    for t in range(T):
        a1 = torch.cat([pad1, alpha[:, :-1]], 1)
        a2 = torch.cat([pad2, alpha[:, :-2]], 1).masked_fill(~skip, NEG)
        new = torch.logsumexp(torch.stack([alpha, a1, a2]), 0) + lp[t].gather(1, ext)
        new = new.masked_fill(~inside, NEG).clamp(min=NEG)
        alpha = torch.where((t < input_len)[:, None], new, alpha)
    last = (2 * target_len)[:, None]
    end = alpha.gather(1, last)
    before = torch.where(last > 0, alpha.gather(1, (last - 1).clamp(min=0)), torch.full_like(end, NEG))
    ll = torch.logsumexp(torch.cat([end, before], 1), 1)
    return torch.where(ll < 0.5 * NEG, torch.full_like(ll, float("inf")), -ll)
