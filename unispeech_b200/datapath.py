"""On-device versions of the two host steps in front of every pre-training batch (SURVEY.md section 8f row 3): the span sampler of
`apply_mask` (WavLM/WavLM.py:35-159,271-287) and utterance mixing (src/fairseq/data/audio/utterance_mixing_dataset.py:373-438).

The reference runs both with numpy's RNG on the host (one `.item()` device sync per row in the sampler).  numpy's streams cannot be
reproduced on a GPU, so the device versions use the library's counter-based generator and are held to the reference statistically
(tests/test_datapath_gpu.py), keeping every deterministic rule.  The bit-exact host ports stay available (`masking.py`, `mixing.py`).
"""
from __future__ import annotations

import struct
from typing import Optional

import numpy as np
import torch

from . import dropout as DR
from . import ops

_SITE_MASK = 0x7F000003


def span_mask_device(B: int, T: int, device, mask_prob: float, mask_length: int, min_masks: int = 2,
                     padding_mask: Optional[torch.Tensor] = None, seed: Optional[int] = None) -> torch.Tensor:
    """bool [B, T] on `device`: the masked frames of one batch (static span length, overlapping spans -- the released recipes).
    `padding_mask`: bool [B, T] frame-level mask ON THE DEVICE (padded tail True) or None.  No host synchronisation.
    The same call draws the channel mask of apply_mask (WavLM/WavLM.py:288-307) when given the channel axis and the reference's
    channel arguments: `span_mask_device(B, encoder_embed_dim, device, mask_channel_prob, mask_channel_length, min_masks=0)`
    (no padding mask; T <= 4096 covers every released width)."""
    if seed is None:
        seed = int(torch.randint(0, 2 ** 62, (1,)).item())
    valid = None
    if padding_mask is not None:
        valid = (T - padding_mask.to(torch.int32).sum(1)).to(torch.int32).contiguous()
    mask = torch.empty(B, T, dtype=torch.uint8, device=device)
    counts = torch.empty(B, dtype=torch.int32, device=device)
    ops.span_mask(valid, B, T, float(mask_prob), int(mask_length), int(min_masks), DR.site_key(seed, _SITE_MASK), mask, counts)
    return mask.bool()


def draw_mix_plan(B: int, T: int, mixing_prob: float = 0.5, mixing_max_len: int = -1):
    """The random scalars of one batch's mixing, drawn on the host with numpy in the reference's order (mixing_num = 1):
    per utterance `random() < p`, source utterance, chunk length, source end, destination end, SNR (utterance_mixing_dataset.py:
    405-428).  Returns a list of (c, len, c_start, s_start, snr_db); c = -1 for utterances that are not mixed."""
    limit = T // 2 if mixing_max_len < 0 else T // mixing_max_len
    limit = min(limit, T)
    plan = []
    for _ in range(B):
        if not (np.random.random() < mixing_prob):
            plan.append((-1, 0, 0, 0, 0.0))
            continue
        c = int(np.random.choice(range(B), 1, replace=True)[0])
        c_len = int(np.random.randint(0, limit + 1))
        c_end = int(np.random.randint(c_len, T + 1))
        s_end = int(np.random.randint(c_len, T + 1))
        snr = float(np.random.uniform(-5, 5))
        plan.append((c, c_len, c_end - c_len, s_end - c_len, snr))
    return plan


def mix_utterances_device(source: torch.Tensor, plan, normalize: bool = False) -> torch.Tensor:
    """Apply a mixing plan on the device: source fp32 [B, T] (CUDA).  Returns the mixed batch (a new tensor).  Every chunk is taken
    from the ORIGINAL batch and scaled by the original powers (the reference mixes in place, so a source utterance that was itself
    mixed earlier in the loop carries its added chunk: a second-order difference, absent from the per-utterance statistics)."""
    assert source.is_cuda and source.dtype == torch.float32 and source.dim() == 2 and source.is_contiguous()
    B, T = source.shape
    dev = source.device
    rec = b"".join(struct.pack("<iiiif", *p) for p in plan)
    plan_d = torch.frombuffer(bytearray(rec), dtype=torch.uint8).to(dev, non_blocking=True)
    power = torch.zeros(B, dtype=torch.float64, device=dev)
    ops.row_power(source, T, B, T, power)
    out = source.clone()
    ops.mix_apply(source, T, B, T, plan_d, power, out)
    if normalize:
        stats = torch.zeros(B, 2, dtype=torch.float64, device=dev)
        ops.row_normalize(out, T, B, T, None, stats, plan_d)
    return out
