"""`FairseqEncoder`-style wrappers the reference's fine-tuning models put around the pre-trained encoder (SURVEY.md section 8b, B2):

  * `HubertEncoder.forward(source, padding_mask, tbc=True)`   src/fairseq/models/hubert/hubert_asr.py:314-340
        -> {"encoder_out": T x B x C, "encoder_padding_mask": B x T, "padding_mask": B x T}
  * `Wav2VecEncoder.forward(source, padding_mask, tbc=True)`  src/fairseq/models/wav2vec/wav2vec2_asr.py:390-421
        -> {"encoder_out": T x B x C, "encoder_padding_mask": T x B, "padding_mask": B x T, "layer_results": [...]}
    (it indexes the DICT form of extract_features: `res["x"]`, which is what `WavLM.forward(features_only=True)` returns)
  * `reorder_encoder_out`, `max_positions`, `set_num_updates`, `upgrade_state_dict_named`   fairseq_encoder.py:26-92

Both keep the reference's freeze logic (`freeze_finetune_updates`: the encoder runs under no_grad until that many updates) and
`apply_mask` (span masking, and channel masking when the model's `mask_channel_prob > 0`, in training only).  They are host glue around `unispeech_b200.wavlm.WavLM`: every tensor they return is a
view of the kernels' output.  `final_dropout` and the output projection `proj` (CTC vocabulary / decoder width,
hubert_asr.py:299-312,330-340) run on the same kernels as the encoder (`b200s_dropout_rows`, the wgmma GEMMs); `proj` keeps the
reference's parameter names (`proj.weight [V, D]`, `proj.bias`) and initialiser (xavier_uniform / zeros, `Linear()` of
hubert_asr.py:367-372).
"""
from __future__ import annotations

import contextlib
from typing import Optional

import torch
import torch.nn as nn

from . import dropout as DR
from . import heads as H
from . import ops
from .engine import BF
from .wavlm import WavLM, _on_forward_stream

_SITE_FINAL = 0x7F000001  # dropout site of `final_dropout` (distinct from every site of the encoder, dropout.py)


class _OutputProjFn(torch.autograd.Function):
    """y = proj(final_dropout(x)):  x bf16 [R, D] (R = T*B rows, any order), W fp32 [V, D], b fp32 [V].  Forward: counter-based
    dropout rows kernel + wgmma GEMM with the bias in its epilogue (the N dimension is padded to a multiple of 64 for the
    operand tiles, the padding columns are never returned).  Backward: column sum (bias), weight-gradient GEMM, input-gradient
    GEMM, the same dropout mask regenerated from its key."""

    @staticmethod
    def forward(ctx, x2d, w, b, p_drop, key):
        ctx.fwd_stream = torch.cuda.current_stream()
        dev = x2d.device
        R, D = x2d.shape
        V = w.shape[0]
        Vp = (V + 63) // 64 * 64
        wpad = torch.zeros(Vp, D, dtype=torch.float32, device=dev)
        wpad[:V] = w
        wp, wpT = H.linear_operands(wpad)
        bpad = torch.zeros(Vp, dtype=torch.float32, device=dev)
        bpad[:V] = b
        xd = x2d
        if p_drop > 0:
            xd = torch.empty_like(x2d)
            ops.dropout_rows(x2d, 0, D, None, 0, 0, xd, 0, D, R, 1, D, p_drop, key)
        y = H.linear_rows(xd, wp, bpad)
        ctx.xd, ctx.wpT, ctx.dims, ctx.drop = xd, wpT, (R, D, V, Vp), (p_drop, key)
        return y[:, :V]

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dy):
        R, D, V, Vp = ctx.dims
        dev = dy.device
        dyp = torch.zeros(R, Vp, dtype=BF, device=dev)
        dyp[:, :V] = dy
        db = torch.zeros(Vp, dtype=torch.float32, device=dev)
        dw = torch.zeros(Vp, D, dtype=torch.float32, device=dev)
        dx = H.linear_rows_backward(dyp, ctx.xd, ctx.wpT, dw, db)
        p_drop, key = ctx.drop
        if p_drop > 0:
            ops.dropout_rows(dx, 0, D, None, 0, 0, dx, 0, D, R, 1, D, p_drop, key)
        ctx.xd = None
        return dx, dw[:V], db[:V], None, None


class _DropOnlyFn(torch.autograd.Function):
    """final_dropout without an output projection."""

    @staticmethod
    def forward(ctx, x2d, p_drop, key):
        ctx.fwd_stream = torch.cuda.current_stream()
        R, D = x2d.shape
        y = torch.empty_like(x2d)
        ops.dropout_rows(x2d, 0, D, None, 0, 0, y, 0, D, R, 1, D, p_drop, key)
        ctx.drop = (p_drop, key)
        return y

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dy):
        R, D = dy.shape
        dx = torch.empty(R, D, dtype=BF, device=dy.device)
        p_drop, key = ctx.drop
        ops.dropout_rows(dy.contiguous(), 0, D, None, 0, 0, dx, 0, D, R, 1, D, p_drop, key)
        return dx, None, None


class _EncoderBase(nn.Module):
    def __init__(self, w2v_model: WavLM, apply_mask: bool = False, freeze_finetune_updates: int = 0, final_dropout: float = 0.0,
                 output_dim: Optional[int] = None):
        super().__init__()
        d = w2v_model.cfg.encoder_embed_dim
        if not 0.0 <= final_dropout < 1.0:
            raise ValueError(f"final_dropout={final_dropout} must be in [0, 1)")
        if hasattr(w2v_model, "remove_pretraining_modules"):
            w2v_model.remove_pretraining_modules()  # hubert_asr.py:290 / wav2vec2_asr.py:355
        self.w2v_model = w2v_model
        self.apply_mask = apply_mask
        self.freeze_finetune_updates = freeze_finetune_updates
        self.num_updates = 0
        self.final_dropout = nn.Dropout(final_dropout)  # parameter-free: kept for the attribute name, applied by the kernel
        self.dropout_seed: Optional[int] = None         # an int pins the final_dropout mask (tests)
        if output_dim is not None:
            # `tgt_dict is not None` -> Linear(d, len(tgt_dict)); `decoder_embed_dim != d` -> Linear(d, decoder_embed_dim)
            self.proj = nn.Linear(d, output_dim)
            nn.init.xavier_uniform_(self.proj.weight)
            nn.init.constant_(self.proj.bias, 0.0)
        else:
            self.proj = None

    def _tail(self, x_btc: torch.Tensor, tbc: bool):
        """final_dropout -> proj on the encoder output (hubert_asr.py:336-340 / wav2vec2_asr.py:411-414); returns T x B x C' if tbc."""
        p = float(self.final_dropout.p) if self.training else 0.0
        if self.proj is None and p == 0.0:
            return x_btc.transpose(0, 1) if tbc else x_btc
        B, T, D = x_btc.shape
        x2d = H.bf16(x_btc.reshape(B * T, D))
        seed = self.dropout_seed if self.dropout_seed is not None else int(torch.randint(0, 2 ** 62, (1,)).item())
        key = DR.site_key(seed, _SITE_FINAL)
        if self.proj is None:
            y = _DropOnlyFn.apply(x2d, p, key)
        else:
            y = _OutputProjFn.apply(x2d, self.proj.weight, self.proj.bias, p, key)
        y = y.reshape(B, T, -1)
        return y.transpose(0, 1) if tbc else y

    def set_num_updates(self, num_updates: int):
        self.num_updates = num_updates

    def _context(self):
        ft = self.freeze_finetune_updates <= self.num_updates
        return contextlib.ExitStack() if ft else torch.no_grad()

    def reorder_encoder_out(self, encoder_out, new_order):
        if encoder_out["encoder_out"] is not None:
            encoder_out["encoder_out"] = encoder_out["encoder_out"].index_select(1, new_order)
        if encoder_out["encoder_padding_mask"] is not None:
            encoder_out["encoder_padding_mask"] = encoder_out["encoder_padding_mask"].index_select(0, new_order)
        return encoder_out

    def max_positions(self):
        return None

    def upgrade_state_dict_named(self, state_dict, name):
        return state_dict


class HubertEncoder(_EncoderBase):
    """hubert_asr.py:314-340: tuple form of `extract_features`; `encoder_padding_mask` is B x T."""

    def forward(self, source, padding_mask, tbc: bool = True, **kwargs):
        with self._context():
            x, padding_mask = self.w2v_model.extract_features(source=source, padding_mask=padding_mask,
                                                              mask=self.apply_mask and self.training)
        x = self._tail(x, tbc)  # final_dropout, proj; B x T x C -> T x B x C
        return {"encoder_out": x, "encoder_padding_mask": padding_mask, "padding_mask": padding_mask}


class Wav2VecEncoder(_EncoderBase):
    """wav2vec2_asr.py:390-421: dict form (`res["x"]`), `encoder_padding_mask` is T x B, `layer_results` passed through."""

    def forward(self, source, padding_mask, tbc: bool = True, **kwargs):
        with self._context():
            res = self.w2v_model(source=source, padding_mask=padding_mask, mask=self.apply_mask and self.training,
                                 features_only=True)
            x, padding_mask = res["x"], res["padding_mask"]
        x = self._tail(x, tbc)
        return {"encoder_out": x,
                "encoder_padding_mask": padding_mask.transpose(0, 1) if padding_mask is not None else None,
                "padding_mask": padding_mask, "layer_results": res["layer_results"]}
