"""Label-driven feature trimming of the pre-training forward (fairseq HubertModel.forward_targets, restated by the fork's
wavlm.py:440-451): when the labels do not cover the T conv frames (feat2tar_ratio * T > targ_tsz), the model runs on the first
int(targ_tsz / feat2tar_ratio) frames.  The frame padding mask is then built on the kept frames, and so is everything after the
conv stack.  Written on top of the building blocks of wavlm_oracle (fp32 torch, autograd for the gradients)."""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
import torch.nn.functional as F
from torch import Tensor

from . import wavlm_oracle as O


def trimmed_frames(T: int, targ_tsz: int, feat2tar_ratio: float) -> int:
    """Frames the forward keeps: all T when the labels cover them, else int(targ_tsz / feat2tar_ratio)."""
    return int(targ_tsz / feat2tar_ratio) if feat2tar_ratio * T > targ_tsz else T


def frame_padding_mask(padding_mask: np.ndarray, T: int) -> np.ndarray:
    """WavLM.forward_padding_mask on T frames (numpy): drop the L % T trailing samples, chunk the rest into T groups, all()."""
    extra = padding_mask.shape[1] % T
    if extra > 0:
        padding_mask = padding_mask[:, :-extra]
    return padding_mask.reshape(padding_mask.shape[0], T, -1).all(-1)


def extract_features(sd, source: Tensor, cfg, frames: int, padding_mask: Optional[Tensor] = None,
                     mask_indices: Optional[Tensor] = None):
    """wavlm_oracle.extract_features on the first `frames` conv frames (no dropout, every layer).  Returns the encoder output,
    the frame padding mask on `frames` frames, and the kept conv features (the feature penalty's input)."""
    conv = O.conv_feature_extractor(sd, source, cfg)[..., :frames]
    feats = conv.transpose(1, 2)
    feats = F.layer_norm(feats, (feats.shape[-1],), sd["layer_norm.weight"], sd["layer_norm.bias"], 1e-5)
    fpm = O.frame_padding_mask(padding_mask, frames) if padding_mask is not None else None
    x = F.linear(feats, sd["post_extract_proj.weight"], sd["post_extract_proj.bias"])
    if mask_indices is not None:
        x = torch.where(mask_indices.unsqueeze(-1), sd["mask_emb"].to(x.dtype), x)
    x, _ = O.encoder(sd, x, fpm, cfg)
    return {"x": x, "padding_mask": fpm, "conv": conv}
