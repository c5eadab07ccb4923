"""H100 (sm_90a) WavLM / UniSpeech-SAT encoder with the reference's public surface.

Mirrors (names, arguments, return values, module tree and state_dict keys):
  * `WavLMConfig`, `WavLM.extract_features(source, padding_mask, mask, ret_conv, output_layer, ret_layer_results)`
    -- /root/reference/WavLM/WavLM.py:162-217, 220-375
  * `model.encoder.layers[i]` called with a T x B x C tensor, each exposing `.self_attn`; `model.encoder(x, padding_mask, layer)`
    returning `(x[B,T,C], layer_results)` -- the contract downstream heads hook (SURVEY.md section 8b, B3)
  * `WavLM.forward(source, padding_mask, mask, features_only, output_layer)` returning the fairseq-style dict
    (`x`, `padding_mask`, `features`, `layer_results`) -- src/fairseq/models/wavlm/wavlm.py:465-597 (encoder part).
The numerical work is done by hand-written sm_90a kernels through the C ABI (`engine.py`, `ops.py`); these modules only hold
the fp32 master parameters (so released checkpoints load with `load_state_dict`) and sequence the launches.
There is no CPU / PyTorch fallback: calling the model on a non-CUDA tensor raises.
"""
from __future__ import annotations

import math
from typing import List, Optional, Tuple

import numpy as np
import torch
import torch.nn as nn

from .dropout import DropState
from .engine import BF, Engine
from .masking import compute_mask_indices


class WavLMConfig:
    """Attribute bag with the reference defaults (WavLM/WavLM.py:162-217)."""

    def __init__(self, cfg=None):
        self.extractor_mode = "default"
        self.encoder_layers = 12
        self.encoder_embed_dim = 768
        self.encoder_ffn_embed_dim = 3072
        self.encoder_attention_heads = 12
        self.activation_fn = "gelu"
        self.layer_norm_first = False
        self.conv_feature_layers = "[(512,10,5)] + [(512,3,2)] * 4 + [(512,2,2)] * 2"
        self.conv_bias = False
        self.feature_grad_mult = 1.0
        self.normalize = False
        self.dropout = 0.1
        self.attention_dropout = 0.1
        self.activation_dropout = 0.0
        self.encoder_layerdrop = 0.0
        self.dropout_input = 0.0
        self.dropout_features = 0.0
        self.mask_length = 10
        self.mask_prob = 0.65
        self.mask_selection = "static"
        self.mask_other = 0
        self.no_mask_overlap = False
        self.mask_min_space = 1
        self.mask_channel_length = 10
        self.mask_channel_prob = 0.0
        self.mask_channel_selection = "static"
        self.mask_channel_other = 0
        self.no_mask_channel_overlap = False
        self.mask_channel_min_space = 1
        self.conv_pos = 128
        self.conv_pos_groups = 16
        self.relative_position_embedding = False
        self.num_buckets = 320
        self.max_distance = 1280
        self.gru_rel_pos = False
        if cfg is not None:
            self.update(cfg)

    def update(self, cfg):
        self.__dict__.update(cfg if isinstance(cfg, dict) else vars(cfg))


def _check_supported(cfg):
    bad = []
    if cfg.activation_fn != "gelu":
        bad.append("activation_fn != gelu")
    if eval(cfg.conv_feature_layers)[-1][0] == cfg.encoder_embed_dim:
        bad.append("conv feature width == encoder_embed_dim (the reference then has no post_extract_proj; the projection kernels assume one)")
    D, H = cfg.encoder_embed_dim, cfg.encoder_attention_heads
    head_dim = D // H if D % H == 0 else None
    if head_dim not in (64, 80, 120):
        bad.append(f"attention head width {D}/{H} (the attention kernels take head widths 64, 80 and 120)")
    elif cfg.relative_position_embedding and head_dim != 64:
        bad.append(f"relative_position_embedding at head width {head_dim} (the gated relative-position bias needs head width 64)")
    if D % cfg.conv_pos_groups != 0 or D // cfg.conv_pos_groups > 128:
        bad.append(f"pos_conv groups of {D}/{cfg.conv_pos_groups} channels (the pos_conv kernels take at most 128 channels per group)")
    return bad


# ----------------------------------------------------------------------------------------------------------------
# autograd glue: each Function runs the kernels of one stage and stashes what its backward needs
# ----------------------------------------------------------------------------------------------------------------
def _check_fp8_call(model, params=None):
    """The fp8 path is inference only (no backward): raised before anything touches the device."""
    if model.training:
        raise RuntimeError("fp8=True is an inference path: call model.eval() first")
    if torch.is_grad_enabled() and any(p.requires_grad for p in (params if params is not None else model.parameters())):
        raise RuntimeError("fp8=True is an inference path without a backward: run it under torch.no_grad() / "
                           "torch.inference_mode(), or with parameters that do not require grad")


def _fp8_tag(t):
    """What identifies a layer output for the fp8 hand-off: its memory (views share it) and its version counter."""
    return (t.data_ptr(), tuple(t.shape), t.stride(), t._version)


def _on_forward_stream(bwd):
    """Run a Function's backward on the stream its forward ran on (explicitly: the kernels are launched through ctypes on
    `torch.cuda.current_stream()`, and the autograd worker thread must not fall back to the legacy default stream -- this is
    what makes side-stream execution and CUDA-graph capture of the whole step legal)."""
    def wrapped(ctx, *grads):
        with torch.cuda.stream(ctx.fwd_stream):
            return bwd(ctx, *grads)
    return wrapped


class _ConvFn(torch.autograd.Function):
    """Conv stack + GradMultiply (WavLM/WavLM.py:333-336, WavLM/modules.py:60-69) + the feature penalty of the pre-training
    models (`features.float().pow(2).mean()` taken AFTER GradMultiply, src/fairseq/models/wavlm/wavlm.py:477-484): the penalty is
    an output of this Function, so its gradient and the gradient arriving from the projection reach the extractor together and
    BOTH are scaled by `feature_grad_mult` in one pass (`b200s_grad_multiply`).  `frames` (< the conv frame count, or None):
    only the first `frames` frames feed the model (label-driven trimming, pretrain.py), so the penalty is their mean and the
    gradient of every later frame is zero.  `valid_last`: see Engine.conv_forward."""

    @staticmethod
    def forward(ctx, anchor, eng: Engine, wav, want_pen, frames=None, valid_last=None):
        from . import ops
        ctx.fwd_stream = torch.cuda.current_stream()
        save = bool(ctx.needs_input_grad[0])
        st = eng.conv_forward(wav, save, valid_last)
        feats = st["a"][-1]
        B, Tp, C = feats.shape
        ctx.T_conv = st["geo"].T[-1]
        T = ctx.T_conv if frames is None else frames
        pen = None
        if want_pen:
            acc = torch.zeros(1, dtype=torch.float64, device=feats.device)
            ops.sumsq_rows(feats, Tp * C, C, T, B, C, acc)
            pen = (acc / float(B * T * C)).float().reshape(())
        ctx.eng, ctx.st, ctx.feats, ctx.T = eng, (st if save else None), (feats if save else None), T
        return feats, st, pen

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dfeat, _unused=None, dpen=None):
        from . import ops
        feats = ctx.feats
        B, Tp, C = feats.shape
        T = ctx.T
        if dfeat is None:  # only the penalty was used
            dfeat = torch.zeros_like(feats)
        g = dfeat if (dfeat.dtype == BF and dfeat.is_contiguous()) else dfeat.to(BF).contiguous()
        if T < ctx.T_conv:
            g[:, T:ctx.T_conv].zero_()  # trimmed frames: nothing downstream read them
        mult = float(ctx.eng.cfg.feature_grad_mult)
        if mult != 1.0 or dpen is not None:
            pg = dpen.float().contiguous() if dpen is not None else None
            ops.grad_multiply(g, Tp * C, C, feats, Tp * C, C, T, B, C, mult, pg, 2.0 / float(B * T * C))
        ctx.eng.conv_backward(ctx.st, g)
        ctx.st = ctx.feats = None
        ctx.eng.backward_stage_done("conv")
        return None, None, None, None, None, None


class _ProjFn(torch.autograd.Function):
    """LayerNorm(features) -> post_extract_proj -> dropout_input -> mask_emb / zero padded frames.  Outputs: the view of the padded
    pos_conv input buffer, `features` (projected, WavLM's ret_conv value) and -- `want_fn`, wav2vec 2.0 -- the LayerNorm output
    `unmasked_features` (src/fairseq/models/wav2vec/wav2vec2.py:578-580) whose gradient (quantizer branch) is added to the
    projection's in the backward pass -- and the stage state, whose `xpad` is the buffer the first output is a view of (the
    pos_conv stem reads the zero padding around it)."""

    @staticmethod
    def forward(ctx, feats, anchor, eng: Engine, T, mask_u8, pad_u8, want_features, want_fn=False, chan_u8=None):
        ctx.fwd_stream = torch.cuda.current_stream()
        save = bool(ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        st = eng.project_forward(feats, T, mask_u8, pad_u8, save, want_features, chan_u8)
        ctx.eng, ctx.st, ctx.T, ctx.mask, ctx.pad, ctx.chan = eng, st, T, mask_u8, pad_u8, chan_u8
        half = eng.cfg.conv_pos // 2
        xv = st["xpad"][:, half:half + T]
        return xv, st["features"], (st["fn"] if want_fn else None), st

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dxv, _dfeatures, dfn_extra=None, _unused=None):
        if dfn_extra is not None:
            dfn_extra = dfn_extra if (dfn_extra.dtype == torch.bfloat16 and dfn_extra.is_contiguous()) else \
                dfn_extra.to(torch.bfloat16).contiguous()
        dfeat = ctx.eng.project_backward(ctx.st, dxv.contiguous(), ctx.T, ctx.mask, ctx.pad, dfn_extra, ctx.chan)
        ctx.st = None  # (GradMultiply is applied where the gradient enters the extractor: _ConvFn.backward)
        ctx.eng.backward_stage_done("stem")
        return dfeat, None, None, None, None, None, None, None, None


class _StemFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, xv, anchor, eng: Engine, xpad, T):
        ctx.fwd_stream = torch.cuda.current_stream()
        save = bool(ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        x0, st = eng.posconv_forward(xpad, T, save)
        ctx.eng, ctx.st, ctx.T = eng, st, T
        return x0

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dx0):
        dxm = ctx.eng.posconv_backward(ctx.st, dx0.contiguous(), ctx.T)
        ctx.st = None
        return dxm, None, None, None, None


class _LayerFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, anchor, eng: Engine, idx, pad_u8, bias_state, rag):
        ctx.fwd_stream = torch.cuda.current_stream()
        save = bool(ctx.needs_input_grad[0] or ctx.needs_input_grad[1])
        tab = bias_state["tab"] if bias_state is not None else None
        out, st = eng.layer_forward(idx, x, pad_u8, tab, save, rag)
        ctx.eng, ctx.idx, ctx.st, ctx.bias_state = eng, idx, st, bias_state
        if bias_state is not None and save:
            ctx.first = not bias_state["has_first"]
            bias_state["has_first"] = True
        else:
            ctx.first = False
        return out

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dout):
        eng, bs = ctx.eng, ctx.bias_state
        dtab = bs["dtab"] if bs is not None else None
        dx = eng.layer_backward(ctx.idx, ctx.st, dout.contiguous(), dtab)
        if ctx.first and bs is not None:
            # every later layer has already added its share: scatter d tab into d relative_attention_bias (SURVEY.md S10)
            from . import ops
            emb = eng.m.encoder.layers[0].self_attn.relative_attention_bias.weight
            H = eng.cfg.encoder_attention_heads
            ops.relpos_table_bwd(dtab, bs["lut"], dtab.shape[1], H, eng.g(emb))
        ctx.st = None
        eng.backward_stage_done(("layer", ctx.idx))
        return dx, None, None, None, None, None, None


class _LNFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, eng: Engine, ln):
        ctx.fwd_stream = torch.cuda.current_stream()
        from . import ops
        B, T, D = x.shape
        y = torch.empty_like(x)
        mean = torch.empty(B * T, dtype=torch.float32, device=x.device)
        rstd = torch.empty(B * T, dtype=torch.float32, device=x.device)
        ops.layer_norm_fwd(x, T * D, D, ln.weight, ln.bias, y, T * D, D, mean, rstd, T, B, D)
        ctx.eng, ctx.ln, ctx.x, ctx.mean, ctx.rstd = eng, ln, x, mean, rstd
        return y

    @staticmethod
    @_on_forward_stream
    def backward(ctx, dy):
        from . import ops
        x, ln, eng = ctx.x, ctx.ln, ctx.eng
        B, T, D = x.shape
        dx = torch.empty_like(x)
        ops.layer_norm_bwd(dy.contiguous(), T * D, D, x, T * D, D, ctx.mean, ctx.rstd, ln.weight, ln.bias, None, 0, 0, dx,
                           T * D, D, eng.g(ln.weight), eng.g(ln.bias), None, T, B, D)
        return dx, None, None


# ----------------------------------------------------------------------------------------------------------------
# module tree (parameter containers with the reference names)
# ----------------------------------------------------------------------------------------------------------------
class _Placeholder(nn.Module):
    """Keeps the reference's Sequential indices (Dropout / TransposeLast / GELU / SamePad slots hold no parameters)."""

    def forward(self, x):
        return x


class ConvFeatureExtractionModel(nn.Module):
    """Parameter layout of WavLM/WavLM.py:378-449: conv_layers.{i}.0.weight, .2.{weight,bias} (GroupNorm, layer 0 of the
    `default` mode) or .2.1.{weight,bias} (LayerNorm of the `layer_norm` mode)."""

    def __init__(self, conv_layers, mode="default", conv_bias=False):
        super().__init__()
        assert mode in {"default", "layer_norm"}
        self.mode = mode
        self.conv_layers = nn.ModuleList()
        in_d = 1
        for i, (dim, k, stride) in enumerate(conv_layers):
            conv = nn.Conv1d(in_d, dim, k, stride=stride, bias=conv_bias)
            nn.init.kaiming_normal_(conv.weight)
            if mode == "layer_norm":
                blk = nn.Sequential(conv, _Placeholder(), nn.Sequential(_Placeholder(), nn.LayerNorm(dim), _Placeholder()),
                                    _Placeholder())
            elif i == 0:
                blk = nn.Sequential(conv, _Placeholder(), nn.GroupNorm(dim, dim, affine=True), _Placeholder())
            else:
                blk = nn.Sequential(conv, _Placeholder(), _Placeholder())
            self.conv_layers.append(blk)
            in_d = dim
        self._owner = None

    def forward(self, x):
        """[B, L] waveform -> [B, C, T] (channels-first view of the channels-last kernel output), as the reference returns."""
        feats, T, _ = self._owner[0]._extractor(x)
        return feats[:, :T].transpose(1, 2)


class _WeightNormConvParams(nn.Module):
    """encoder.pos_conv.0.{bias, weight_g, weight_v} exactly as nn.utils.weight_norm(dim=2) names them (WavLM.py:514-527)."""

    def __init__(self, D, groups, k):
        super().__init__()
        std = math.sqrt(4.0 / (k * D))
        v = torch.empty(D, D // groups, k).normal_(0, std)
        self.bias = nn.Parameter(torch.zeros(D))
        self.weight_g = nn.Parameter(v.norm(2, dim=(0, 1), keepdim=True).clone())
        self.weight_v = nn.Parameter(v)


class MultiheadAttention(nn.Module):
    """Parameter container for WavLM/modules.py:303-415 (q/k/v/out projections, grep_linear, grep_a, relative_attention_bias)."""

    def __init__(self, embed_dim, num_heads, has_relative_attention_bias=False, num_buckets=32, max_distance=128,
                 gru_rel_pos=False):
        super().__init__()
        self.embed_dim, self.num_heads = embed_dim, num_heads
        self.head_dim = embed_dim // num_heads
        self.has_relative_attention_bias = has_relative_attention_bias
        self.num_buckets, self.max_distance, self.gru_rel_pos = num_buckets, max_distance, gru_rel_pos
        self.fp32_attention = False  # attribute downstream code pokes (downstreams/.../ecapa_tdnn.py:199-202)
        self.k_proj = nn.Linear(embed_dim, embed_dim)
        self.v_proj = nn.Linear(embed_dim, embed_dim)
        self.q_proj = nn.Linear(embed_dim, embed_dim)
        self.out_proj = nn.Linear(embed_dim, embed_dim)
        if has_relative_attention_bias:
            self.relative_attention_bias = nn.Embedding(num_buckets, num_heads)
        if gru_rel_pos:
            self.grep_linear = nn.Linear(self.head_dim, 8)
            self.grep_a = nn.Parameter(torch.ones(1, num_heads, 1, 1))
        for lin in (self.k_proj, self.v_proj, self.q_proj):
            nn.init.xavier_uniform_(lin.weight, gain=1 / math.sqrt(2))
        nn.init.xavier_uniform_(self.out_proj.weight)
        nn.init.constant_(self.out_proj.bias, 0.0)
        if has_relative_attention_bias:
            nn.init.xavier_normal_(self.relative_attention_bias.weight)


class TransformerSentenceEncoderLayer(nn.Module):
    """One encoder layer; `forward` keeps the reference signature and T x B x C convention (WavLM/WavLM.py:615-742)."""

    def __init__(self, cfg, index, has_relative_attention_bias):
        super().__init__()
        D = cfg.encoder_embed_dim
        self.index = index
        self.embedding_dim = D
        self.layer_norm_first = cfg.layer_norm_first
        self.self_attn = MultiheadAttention(D, cfg.encoder_attention_heads,
                                            has_relative_attention_bias=has_relative_attention_bias,
                                            num_buckets=cfg.num_buckets, max_distance=cfg.max_distance,
                                            gru_rel_pos=cfg.gru_rel_pos)
        self.self_attn_layer_norm = nn.LayerNorm(D)
        self.fc1 = nn.Linear(D, cfg.encoder_ffn_embed_dim)
        self.fc2 = nn.Linear(cfg.encoder_ffn_embed_dim, D)
        self.final_layer_norm = nn.LayerNorm(D)
        self._owner = None  # set by WavLM (list wrapper, so the owner is not registered as a sub-module)

    def forward(self, x, self_attn_mask=None, self_attn_padding_mask=None, need_weights=False, pos_bias=None,
                valid_frames=None, fp8=False):
        """x: T x B x C.  `pos_bias` carries the shared relative-position state between layers (the reference passes the
        materialised [B*H,T,T] bias tensor here; we pass the per-head Toeplitz table instead).  `valid_frames` (int32 [B] on
        the device, with a padding mask only): frames of every utterance up to its last valid one; the row GEMMs and LayerNorms
        then skip the padded tail and write zeros there.  `fp8` (inference only, see WavLM.extract_features): the projections
        run as e4m3 GEMMs, and `pos_bias` (then always a dict) also carries this layer's e4m3 output to the next layer.
        Returns (x, None, pos_bias)."""
        assert self_attn_mask is None, "streaming / attention masks are not supported"
        model = self._owner[0]
        eng = model._engine_for(x.device)
        xb = x.transpose(0, 1)
        if xb.dtype != BF or not xb.is_contiguous():
            xb = xb.to(BF).contiguous()
        B, T, _ = xb.shape
        pad_u8, rag = None, None
        if self_attn_padding_mask is not None:
            pad_u8 = self_attn_padding_mask if self_attn_padding_mask.dtype == torch.uint8 else self_attn_padding_mask.to(torch.uint8)
            pad_u8, rag = pad_u8.contiguous(), valid_frames
        if pos_bias is None and model.encoder.relative_position_embedding:
            pos_bias = model.encoder._make_bias_state(T, x.device)
        if fp8:
            return self._forward_fp8(eng, xb, pad_u8, pos_bias, rag)
        out = _LayerFn.apply(xb, self.fc1.weight, eng, self.index, pad_u8, pos_bias, rag)
        return out.transpose(0, 1), None, pos_bias

    def _forward_fp8(self, eng, xb, pad_u8, pos_bias, rag):
        """The fp8 layer call.  The previous layer's e4m3 copy of its output (and the gate it computed for this layer) travel in
        `pos_bias["fp8_next"]`, tagged with the output's storage (address, shape, strides) and version counter: they are used only
        if `xb` views that same memory, unmodified -- `xb` is a new view of it (the layers pass T x B x C transposes), so identity
        cannot be the test.  A forward hook that replaced the output or modified it in place (the version counter is shared by all
        views) makes this layer quantise its input itself."""
        if pos_bias is None:
            pos_bias = {"tab": None}
        if not pos_bias.get("fp8_ready"):  # a direct layer call: check it, and make sure the e4m3 weights match the masters
            _check_fp8_call(self._owner[0])
            eng.prepare_fp8()
        x8 = gate = None
        nxt = pos_bias.pop("fp8_next", None)
        if nxt is not None and nxt[0] == _fp8_tag(xb):
            x8, gate = nxt[1], nxt[2]
        with torch.no_grad():
            out, out8, next_gate = eng.layer_forward_fp8(self.index, xb, pad_u8, pos_bias.get("tab"), rag, x8, gate)
        if out8 is not None:
            pos_bias["fp8_next"] = (_fp8_tag(out), out8, next_gate, out)  # (out held: its memory cannot be reused meanwhile)
        return out.transpose(0, 1), None, pos_bias


class TransformerEncoder(nn.Module):
    """pos_conv + layer stack (WavLM/WavLM.py:507-612)."""

    def __init__(self, cfg):
        super().__init__()
        D = cfg.encoder_embed_dim
        self.dropout = cfg.dropout
        self.embedding_dim = D
        self.pos_conv = nn.Sequential(_WeightNormConvParams(D, cfg.conv_pos_groups, cfg.conv_pos), _Placeholder(), _Placeholder())
        self.relative_position_embedding = getattr(cfg, "relative_position_embedding", False)
        self.num_buckets = cfg.num_buckets if self.relative_position_embedding else 0
        self.max_distance = cfg.max_distance if self.relative_position_embedding else 0
        self.layers = nn.ModuleList([
            TransformerSentenceEncoderLayer(cfg, i, has_relative_attention_bias=(self.relative_position_embedding and i == 0))
            for i in range(cfg.encoder_layers)
        ])
        self.layer_norm_first = cfg.layer_norm_first
        self.layer_norm = nn.LayerNorm(D)
        if self.layer_norm_first and getattr(cfg, "layer_norm_for_extract", False):
            # UniSpeech-SAT encoder (src/fairseq/models/unispeech_sat/unispeech_sat.py:1196-1197): same state_dict key
            self.layer_norm_for_extract = nn.LayerNorm(D)
        self.layerdrop = cfg.encoder_layerdrop
        self._owner = None
        # `self.apply(init_bert_params)` of the reference (WavLM/WavLM.py:560-562, WavLM/modules.py:168-200): EVERY nn.Linear of the
        # encoder -- q/k/v/out_proj, grep_linear, fc1/fc2 -- is re-drawn from N(0, 0.02) with a zero bias, and the
        # relative_attention_bias Embedding from N(0, 0.02) (it runs after MultiheadAttention.reset_parameters, so the xavier
        # values of the constructor do not survive)
        for mod in self.modules():
            if isinstance(mod, nn.Linear):
                mod.weight.data.normal_(mean=0.0, std=0.02)
                if mod.bias is not None:
                    mod.bias.data.zero_()
            elif isinstance(mod, nn.Embedding):
                mod.weight.data.normal_(mean=0.0, std=0.02)

    def _make_bias_state(self, T, device):
        from . import ops
        model = self._owner[0]
        eng = model._engine_for(device)
        H = model.cfg.encoder_attention_heads
        lut = eng.lut(T)
        tab = torch.empty(H, 2 * T - 1, dtype=torch.float32, device=device)
        ops.relpos_table_fwd(self.layers[0].self_attn.relative_attention_bias.weight, lut, 2 * T - 1, H, tab)
        dtab = torch.zeros(H, 2 * T - 1, dtype=torch.float32, device=device) if torch.is_grad_enabled() else None
        return dict(tab=tab, dtab=dtab, lut=lut, has_first=False)

    def forward(self, x, padding_mask=None, streaming_mask=None, layer=None, extract_layer=None, *, _xpad=None, _valid=None,
                fp8=False):
        """Returns (x, layer_results) like the reference WavLM encoder; with `extract_layer` (UniSpeech-SAT encoder,
        unispeech_sat.py:1202-1210) a third value: that layer's output, normalised by `layer_norm_for_extract` for pre-LN models.
        `_xpad` and `_valid` come from WavLM._extract only (see `_encode`)."""
        res = self._encode(x, padding_mask, streaming_mask, layer, extract_layer, _xpad, _valid, fp8)
        x, layer_results = res[0], res[1]
        er = res[2] if extract_layer is not None else None
        if self.layer_norm_first and layer is None:
            model = self._owner[0]
            xb = x if x.dtype == BF and x.is_contiguous() else x.to(BF).contiguous()
            x = _LNFn.apply(xb, model._engine_for(x.device), self.layer_norm)
            if er is not None and hasattr(self, "layer_norm_for_extract"):
                eb = er if er.dtype == BF and er.is_contiguous() else er.to(BF).contiguous()
                er = _LNFn.apply(eb, model._engine_for(x.device), self.layer_norm_for_extract)
        if extract_layer is not None:
            return x, layer_results, er
        return x, layer_results

    def extract_features(self, x, padding_mask=None, streaming_mask=None, tgt_layer=None, extract_layer=None):
        """x: [B,T,D] (projected, masked features).  Out-of-place restatement of WavLM/WavLM.py:572-612.  `tgt_layer` may
        also be a list of 1-based layer numbers (fairseq WavLM, src/fairseq/models/wavlm/wavlm.py:730-737: those layers' outputs
        are collected without early exit); `extract_layer` (0-based) adds that layer's output as a third return value
        (UniSpeech-SAT encoder, unispeech_sat.py:1236-1255)."""
        return self._encode(x, padding_mask, streaming_mask, tgt_layer, extract_layer)

    def _encode(self, x, padding_mask, streaming_mask, tgt_layer, extract_layer, xpad=None, valid=None, fp8=False):
        """`extract_features` body.  From WavLM._extract, `x` is a view of `xpad`, the zero-padded pos_conv input buffer
        the projection wrote, and `valid` (int32 [B] or None) the ragged lengths the layers skip the padded tails with."""
        assert streaming_mask is None, "streaming masks are not supported"
        model = self._owner[0]
        eng = model._engine_for(x.device)
        cfg = model.cfg
        B, T, D = x.shape
        half = cfg.conv_pos // 2
        if xpad is None:
            # external caller: make sure the bf16 operands exist for the current parameters, then stage into the zero-padded
            # pos_conv buffer and zero padded frames
            from . import ops
            eng = model._begin(x.device)
            xpad = torch.zeros(B, T + cfg.conv_pos, D, dtype=BF, device=x.device)
            xpad[:, half:half + T] = x.to(BF)
            if padding_mask is not None:
                ops.frame_mask_fwd(xpad[:, half:], (T + cfg.conv_pos) * D, D, T, B, D, None,
                                   padding_mask.to(torch.uint8).contiguous(), None)
            x = xpad[:, half:half + T]
        x0 = _StemFn.apply(x, self.pos_conv[0].bias, eng, xpad, T)
        x = x0.transpose(0, 1)  # B x T x C -> T x B x C (view)
        layer_results = []
        tgt_list = tgt_layer if isinstance(tgt_layer, (list, tuple)) else None
        if tgt_layer is not None and tgt_list is None:
            layer_results.append((x, None))
        r = None
        er = None
        pos_bias = self._make_bias_state(T, x.device) if self.relative_position_embedding else None
        if fp8:
            _check_fp8_call(model, eng._params)
            eng.prepare_fp8()
            pos_bias = dict(pos_bias or {"tab": None}, fp8_ready=True)
        lkw = dict(fp8=True) if fp8 else {}
        pad_u8 = padding_mask.to(torch.uint8).contiguous() if padding_mask is not None else None
        for i, layer in enumerate(self.layers):
            dropout_probability = np.random.random()
            if not self.training or (dropout_probability > self.layerdrop):
                x, _z, pos_bias = layer(x, self_attn_padding_mask=pad_u8, need_weights=False, pos_bias=pos_bias, valid_frames=valid,
                                        **lkw)
            if tgt_list is not None:
                if i + 1 in tgt_list:
                    layer_results.append((x, None))
            elif tgt_layer is not None:
                layer_results.append((x, None))
            if extract_layer is not None and i == extract_layer:
                er = x.transpose(0, 1)
            if tgt_list is None and i == tgt_layer:
                r = x
                break
        if r is not None:
            x = r
        if extract_layer is not None:
            return x.transpose(0, 1), layer_results, er
        return x.transpose(0, 1), layer_results


class WavLM(nn.Module):
    """Drop-in for the reference `WavLM` (WavLM/WavLM.py:220-375); same constructor, attributes and `extract_features`."""

    def __init__(self, cfg: WavLMConfig):
        super().__init__()
        bad = _check_supported(cfg)
        if bad:
            raise NotImplementedError("unsupported configuration for the CUDA hot path: " + "; ".join(bad))
        self.cfg = cfg
        self.conv_cfg = eval(cfg.conv_feature_layers)
        self.embed = self.conv_cfg[-1][0]
        self.feature_extractor = ConvFeatureExtractionModel(self.conv_cfg, mode=cfg.extractor_mode, conv_bias=cfg.conv_bias)
        self.post_extract_proj = nn.Linear(self.embed, cfg.encoder_embed_dim) if self.embed != cfg.encoder_embed_dim else None
        self.mask_prob, self.mask_selection, self.mask_other = cfg.mask_prob, cfg.mask_selection, cfg.mask_other
        self.mask_length, self.no_mask_overlap, self.mask_min_space = cfg.mask_length, cfg.no_mask_overlap, cfg.mask_min_space
        self.mask_channel_prob, self.mask_channel_selection = cfg.mask_channel_prob, cfg.mask_channel_selection
        self.mask_channel_other, self.mask_channel_length = cfg.mask_channel_other, cfg.mask_channel_length
        self.no_mask_channel_overlap, self.mask_channel_min_space = cfg.no_mask_channel_overlap, cfg.mask_channel_min_space
        self.dropout_input = nn.Dropout(cfg.dropout_input)
        self.dropout_features = nn.Dropout(cfg.dropout_features)
        self.feature_grad_mult = cfg.feature_grad_mult
        self.mask_emb = nn.Parameter(torch.FloatTensor(cfg.encoder_embed_dim).uniform_())
        self.encoder = TransformerEncoder(cfg)
        self.layer_norm = nn.LayerNorm(self.embed)
        owner = [self]
        self.feature_extractor._owner = owner
        self.encoder._owner = owner
        for lyr in self.encoder.layers:
            lyr._owner = owner
        self._engine: Optional[Engine] = None
        self.dropout_seed: Optional[int] = None  # None: draw a fresh seed per forward; an int pins the dropout masks (tests)
        # what the model's own forward pass needs from extract_features (set by the subclasses, honoured by every caller)
        self._want_features_pen = False      # pre-training models: the feature penalty (keeps every conv row, see _extractor)
        self._want_unmasked_features = False  # wav2vec 2.0: the LayerNorm'ed conv features of the quantizer branch
        self._extract_layer = None           # UniSpeech-SAT: 0-based `utterance_contrastive_layer - 1` (unispeech_sat.py:640-645)
        self._predict_layers = None          # ILS-HuBERT: 1-based layers whose outputs feed intermediate heads (ils_hubert.py:167-171)

    def __deepcopy__(self, memo):
        """`copy.deepcopy(model)` (EMA / teacher copies, checkpoint averaging): the engine holds raw device pointers to THIS model's
        masters (operand-preparation and optimizer descriptor tables), so the copy must not inherit it -- it builds its own on its
        first forward pass."""
        import copy
        new = self.__class__.__new__(self.__class__)
        memo[id(self)] = new
        for k, v in self.__dict__.items():
            new.__dict__[k] = None if k == "_engine" else copy.deepcopy(v, memo)
        return new

    # ---- engine plumbing
    def _engine_for(self, device) -> Engine:
        if device.type != "cuda":
            raise RuntimeError("unispeech_b200 runs on an H100 (sm_90) only: there is no CPU fallback for the hot path")
        if self._engine is None:
            self._engine = Engine(self)
        self._engine._ensure_device(device)
        return self._engine

    def _begin(self, device) -> Engine:
        if device.type != "cuda":
            raise RuntimeError("the hot path runs on a CUDA device (there is no CPU fallback)")
        if device.index is not None and device.index != torch.cuda.current_device():
            # kernels are launched on the CURRENT device's current stream (_lib.stream_ptr)
            raise RuntimeError(f"make cuda:{device.index} the current device (torch.cuda.set_device) before calling the model")
        eng = self._engine_for(device)
        # training-mode dropout: one seed per forward pass (torch CPU generator, or `self.dropout_seed` when a caller pins it)
        eng.drop = DropState.for_model(self.cfg, self.training, self.dropout_seed)
        if eng._params is None:  # Module.parameters() walks the module tree (~2 ms for WavLM-Base): once per engine
            eng._params = list(self.parameters())
        for p in eng._params:
            if p.device != device or p.dtype != torch.float32:
                raise RuntimeError("model parameters must be fp32 masters on the input's CUDA device (call model.float().cuda())")
        eng.prepare()
        if torch.is_grad_enabled() and any(p.requires_grad for p in eng._params):
            eng.flat.attach()
        return eng

    def grad_buffer(self) -> torch.Tensor:
        """The flat fp32 gradient buffer all `param.grad` alias; the data-parallel allreduce runs on it (one NCCL call)."""
        if self._engine is None or self._engine.flat is None:
            raise RuntimeError("run a forward pass on the GPU first")
        return self._engine.flat.flat

    def zero_grad_buffer(self):
        """Reset every gradient (the flat buffer all `param.grad` alias) on the current stream: the backward kernels ACCUMULATE,
        so this is the step's `optimizer.zero_grad()` when no `FusedAdam.step(zero_grad=True)` does it."""
        from . import ops
        ops.memset_zero(self.grad_buffer())

    def _extractor(self, source, valid_last=None, frames=None):
        """`valid_last` (int32 [B], host or device): frames of the extractor output up to every utterance's last valid one.  The
        conv stack then skips the padding beyond them (engine.conv_valid_rows) -- not when the feature penalty is wanted (the
        reference takes `features.pow(2).mean()` over the padded frames too, so they must hold the reference's values), and
        not when the caller asks for the conv features themselves (`ret_conv`: extract_features passes no `valid_last` then).
        `frames`: see _ConvFn.  Returns (features [B, Tp, C], conv frame count, feature penalty or None)."""
        eng = self._begin(source.device)
        wav = source.float().contiguous()
        w0 = self.feature_extractor.conv_layers[0][0].weight
        want_pen = self._want_features_pen
        valid_last = None if want_pen else valid_last
        if self.feature_grad_mult > 0:
            feats, st, pen = _ConvFn.apply(w0, eng, wav, want_pen, frames, valid_last)
        else:
            with torch.no_grad():
                feats, st, pen = _ConvFn.apply(w0, eng, wav, want_pen, frames, valid_last)
        return feats, st["geo"].T[-1], pen

    # ---- reference API
    def apply_mask(self, B, T, padding_mask):
        """Host-side span sampling identical to the reference (numpy RNG; WavLM/WavLM.py:271-287); returns bool [B,T] or None."""
        if self.mask_prob > 0:
            idx = compute_mask_indices((B, T), padding_mask, self.mask_prob, self.mask_length, self.mask_selection,
                                       self.mask_other, min_masks=2, no_overlap=self.no_mask_overlap,
                                       min_space=self.mask_min_space)
            return torch.from_numpy(idx)
        return None

    def apply_channel_mask(self, B):
        """Host-side channel sampling identical to the reference (numpy RNG; WavLM/WavLM.py:288-307): spans over the
        `encoder_embed_dim` channels, no padding mask, min_masks 0.  Returns bool [B, D] or None."""
        if self.mask_channel_prob > 0:
            idx = compute_mask_indices((B, self.cfg.encoder_embed_dim), None, self.mask_channel_prob, self.mask_channel_length,
                                       self.mask_channel_selection, self.mask_channel_other, no_overlap=self.no_mask_channel_overlap,
                                       min_space=self.mask_channel_min_space)
            return torch.from_numpy(idx)
        return None

    def sample_masks(self, B, T, padding_mask):
        """(span mask bool [B,T] or None, channel mask bool [B,D] or None), drawn from the numpy global RNG in the reference's
        order: the span mask first, then the channel mask."""
        mask_indices = self.apply_mask(B, T, padding_mask)
        return mask_indices, self.apply_channel_mask(B)

    def forward_padding_mask(self, T: int, padding_mask: torch.Tensor) -> torch.Tensor:
        """Sample-level mask -> frame-level mask (WavLM/WavLM.py:311-321)."""
        extra = padding_mask.size(1) % T
        if extra > 0:
            padding_mask = padding_mask[:, :-extra]
        padding_mask = padding_mask.view(padding_mask.size(0), T, -1)
        return padding_mask.all(-1)

    def extract_features(self, source, padding_mask=None, mask=False, ret_conv=False, output_layer=None,
                         ret_layer_results=False, mask_indices=None, mask_channel_indices=None, *, fp8=False):
        """Same contract as the reference.  `mask_indices` (bool [B,T], optional) and `mask_channel_indices` (bool [B,D],
        optional) let a caller inject the masked frames and channels instead of sampling them (used by the parity tests and the
        CUDA graph; the reference's sampler is host numpy RNG).  With `mask=True` both are sampled when neither is given;
        once either is given, the other one given as None means no mask of that kind.
        `fp8=True` (inference: eval mode, no gradient): the encoder layers' QKV, out_proj, fc1 and fc2 projections run as e4m3
        GEMMs with per-row activation and per-channel weight scales (the conv stack, post_extract_proj, pos_conv, attention and the
        LayerNorms stay bf16 / fp32).  RuntimeError in training mode, with gradients enabled on a model that requires them, or
        with `mask=True`."""
        if fp8:
            _check_fp8_call(self)
            if mask:
                raise RuntimeError("extract_features(fp8=True) is an inference path: mask=True is not supported")
        res = self._extract(source, padding_mask, mask, ret_conv, output_layer, mask_indices, mask_channel_indices, fp8=fp8)
        feature = res["features"] if ret_conv else res["x"]
        if ret_layer_results:
            feature = (feature, res["layer_results"])
        return feature, res["padding_mask"]

    def _extract(self, source, padding_mask, mask, ret_conv, output_layer, mask_indices, mask_channel_indices, frames=None,
                 fp8=False):
        """The forward pass behind `extract_features` and the models' `forward`: returns everything one call produced as a dict
        (`x`, `padding_mask`, `features`, `layer_results`, `mask_indices`, `mask_channel_indices`, `padding_mask_host`, `spk_x`,
        `unmasked_features`, `features_pen`).  `frames` (pre-training with labels shorter than the conv frames,
        WavLMForPretraining.forward): the model runs on the first `frames` frames -- frame mask, span / channel masks, projection
        and encoder all see that many."""
        from .engine import ConvGeom
        T_conv = ConvGeom(self.conv_cfg, source.shape[1]).T[-1]
        T = T_conv if frames is None else frames
        B = source.shape[0]
        # `padding_mask` may live on the host (as it does in the reference's collater): the frame mask and the span sampler
        # then run on the host without a device sync, and only the small uint8 masks are uploaded.
        fpm_host = None
        fpm = self.forward_padding_mask(T, padding_mask) if padding_mask is not None else None
        if fpm is not None and fpm.device.type == "cpu":
            fpm_host = fpm
            fpm = fpm.to(source.device, non_blocking=True)
        if mask and mask_indices is None and mask_channel_indices is None:
            if fpm is not None and fpm_host is None:
                fpm_host = fpm.cpu()  # device-resident mask: one sync, exactly like the reference's `.item()` per row
            mask_indices, mask_channel_indices = self.sample_masks(B, T, fpm_host)
        if mask_channel_indices is not None and tuple(mask_channel_indices.shape) != (B, self.cfg.encoder_embed_dim):
            raise ValueError(f"mask_channel_indices must be [B, encoder_embed_dim] = [{B}, {self.cfg.encoder_embed_dim}]; "
                             f"got {list(mask_channel_indices.shape)}")
        # ragged batch: frames of every utterance up to its last valid one (host arithmetic when the mask lives on the host; with
        # a device-only mask two tiny device ops, no synchronisation): `valid_last` for the conv stack, `valid` on the device for
        # the encoder layers, which skip the padded tail of every utterance.
        valid = valid_last = None
        if fpm is not None:
            if fpm_host is not None:
                if bool(fpm_host.any()):
                    last = ((~fpm_host).to(torch.int32) * torch.arange(1, T + 1, dtype=torch.int32)).amax(1)
                    valid_last = last.to(torch.int32).contiguous()
                    valid = valid_last.to(source.device, non_blocking=True)
            else:
                valid = valid_last = ((~fpm).to(torch.int32) * torch.arange(1, T + 1, dtype=torch.int32, device=fpm.device)) \
                    .amax(1).to(torch.int32).contiguous()
            fpm._b200_valid = valid  # for KMeans.predict on the returned mask (nothing in the model reads it)
        feats, T2, pen = self._extractor(source, None if ret_conv else valid_last, None if T == T_conv else T)
        assert T2 == T_conv
        eng = self._engine
        mask_u8 = mask_indices.to(device=source.device, dtype=torch.uint8).contiguous() if mask_indices is not None else None
        chan_u8 = mask_channel_indices.to(device=source.device, dtype=torch.uint8).contiguous() \
            if mask_channel_indices is not None else None
        pad_u8 = fpm.to(torch.uint8).contiguous() if fpm is not None else None
        xv, features, unmasked, proj_st = _ProjFn.apply(feats, self.post_extract_proj.weight, eng, T, mask_u8, pad_u8, ret_conv,
                                                        self._want_unmasked_features, chan_u8)
        el, pl = self._extract_layer, self._predict_layers
        lay = (list(pl) if (pl is not None and output_layer is None) else None) if output_layer is None else output_layer - 1
        enc = self.encoder(xv, padding_mask=fpm, layer=lay, extract_layer=el, _xpad=proj_st["xpad"], _valid=valid, fp8=fp8)
        return {"x": enc[0], "padding_mask": fpm, "features": features, "layer_results": enc[1],
                "mask_indices": mask_indices, "mask_channel_indices": mask_channel_indices, "padding_mask_host": fpm_host,
                "spk_x": enc[2] if el is not None else None, "unmasked_features": unmasked, "features_pen": pen}

    def forward(self, source, target_list=None, padding_mask=None, mask=True, features_only=False, output_layer=None):
        """fairseq-style entry (src/fairseq/models/wavlm/wavlm.py:465-523, encoder part): returns the result dict.
        The masked-prediction heads (final_proj / label embeddings) are outside the hot path (SURVEY.md section 8f)."""
        res = self._extract(source, padding_mask, mask, False, output_layer, None, None)
        out = {"x": res["x"], "padding_mask": res["padding_mask"], "features": res["features"],
               "layer_results": res["layer_results"]}
        if not features_only:
            out["mask_indices"] = res["mask_indices"]
        return out
