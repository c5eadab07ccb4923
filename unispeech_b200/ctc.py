"""CTC fine-tuning on the library's own kernels (csrc/ctc.cu): the loss, the criterion and the model surface of the reference's
ASR fine-tuning (src/fairseq/criterions/ctc.py, src/fairseq/models/hubert/hubert_asr.py `HubertCtc`,
src/fairseq/models/wav2vec/wav2vec2_asr.py `Wav2VecCtc`).

  * `ctc_loss(logits_tbv, input_len, targets, target_len, blank, reduction, zero_infinity)`: log-softmax + CTC on bf16 logits, one
    autograd Function.  Forward = row statistics + alpha recursion (all an eval pass needs); backward = beta recursion with the
    gradient through CTC and the log-softmax fused in.  The logits are read through their strides: the T x B x V view that the
    fine-tuning wrappers return over their [B*T, Vp] buffer is consumed, and its gradient produced, without a copy.  The loss stays
    on the device; nothing synchronises, so a fixed-shape fine-tuning step captures in a CUDA graph.
  * `CtcCriterion`: `forward(model, sample) -> (loss, sample_size, logging_output)` with the reference's contract (below).
  * `forced_align(logits_tbv, input_len, targets, target_len, blank)`: the most probable CTC path of each utterance's known
    transcript (csrc/ctc_align.cu), bit for bit what `torchaudio.functional.forced_align` returns for each utterance on
    lp = logits - logsumexp(logits) in fp32, but batched, on the bf16 logits themselves and for transcripts of up to
    `MAX_ALIGN_TARGET` labels.  `token_spans` turns its paths into per-token frame spans (`torchaudio.functional.merge_tokens`).
  * `ctc_beam_search(logits_tbv, input_len, beam_size, nbest, blank, beam_size_token, lm, lm_weight, word_score, unk_score)`:
    batched CTC prefix beam search (csrc/ctc_decode.cu) with an optional word n-gram LM (`ngram.NgramLM.from_arpa`) scored at
    word boundaries, lexicon-free, or with `lexicon` (`lexicon.Lexicon.from_file`) held to a word lexicon with LM look-ahead
    (csrc/ctc_decode_lex.cu); `hypotheses_to_words` spells the result.
  * `HubertCtc` / `Wav2VecCtc`: `w2v_encoder` = `HubertEncoder` / `Wav2VecEncoder`, `forward(**net_input)`, `get_logits`,
    `get_normalized_probs`, `set_num_updates`; `state_dict` keys `w2v_encoder.w2v_model.*`, `w2v_encoder.proj.*`.

Limits (the kernels fail beyond them, nothing is truncated): V <= 1024 classes, targets of at most `MAX_TARGET` labels.
An infeasible utterance (input too short for its target with one blank per repeated label; a label outside [0, V)) has
nll = +inf and an all-zero gradient, with and without `zero_infinity` (`torch.nn.functional.ctc_loss` leaves that gradient
unspecified without it); `zero_infinity` additionally replaces its +inf by 0 in the returned loss.
"""
from __future__ import annotations

from typing import List, NamedTuple, Optional

import torch
import torch.nn as nn
import torch.nn.functional as F

from . import ops
from .engine import BF
from .fairseq_encoder import HubertEncoder, Wav2VecEncoder
from .wavlm import _on_forward_stream

MAX_TARGET = 511   # B200S_CTC_MAX_TARGET: one thread per position of the extended label sequence, 2 * 511 + 1 <= 1024
MAX_CLASSES = 1024
MAX_ALIGN_TARGET = 8191   # B200S_CTC_ALIGN_MAX_TARGET: up to 32 positions of the extended label sequence per thread, 512 threads


class _CtcFn(torch.autograd.Function):
    """(nll [B] fp32, sum_b nll fp32 scalar, argmax [B, T] int32 or None) of bf16 logits T x B x V (unit class stride)."""

    @staticmethod
    def forward(ctx, logits, input_len, targets, target_len, blank, zero_infinity, want_argmax):
        ctx.fwd_stream = torch.cuda.current_stream()
        dev = logits.device
        T, B, V = logits.shape
        fs, bs = logits.stride(0), logits.stride(1)
        Smax = targets.shape[1]
        lse = torch.empty(B, T, dtype=torch.float32, device=dev)
        # frames past input_len are not visited: they decode to blank
        argmax = torch.full((B, T), blank, dtype=torch.int32, device=dev) if want_argmax else None
        log_alpha = torch.empty(B, T, 2 * Smax + 1, dtype=torch.float32, device=dev)
        nll = torch.empty(B, dtype=torch.float32, device=dev)
        total = torch.zeros(1, dtype=torch.float64, device=dev)
        ops.ctc_stats(logits, fs, bs, input_len, B, T, V, lse, argmax)
        ops.ctc_alpha(logits, fs, bs, lse, input_len, targets, Smax, target_len, B, T, V, blank, zero_infinity, log_alpha, nll, total)
        ctx.save_for_backward(logits, input_len, targets, target_len, lse, log_alpha, nll)
        ctx.blank = blank
        out = nll.masked_fill(nll == float("inf"), 0.0) if zero_infinity else nll.clone()
        if argmax is not None:
            ctx.mark_non_differentiable(argmax)
        return out, total.float().reshape(()), argmax

    @staticmethod
    @_on_forward_stream
    def backward(ctx, d_nll, d_total, _d_argmax=None):
        logits, input_len, targets, target_len, lse, log_alpha, nll = ctx.saved_tensors
        dev = logits.device
        T, B, V = logits.shape
        fs, bs = logits.stride(0), logits.stride(1)
        up = torch.zeros(B, dtype=torch.float32, device=dev)   # d loss / d nll[b]
        if d_nll is not None:
            up += d_nll.float()
        if d_total is not None:
            up += d_total.float()
        if bs == T * fs and fs >= V:
            # rows view of a [B*T, Vp] buffer: the gradient gets the same layout, its padding columns written as zeros
            buf = torch.empty(B * T, fs, dtype=BF, device=dev)
            grad, vpad = buf[:, :V].reshape(B, T, V).transpose(0, 1), fs
        else:
            grad, vpad = torch.empty_strided(logits.shape, logits.stride(), dtype=BF, device=dev), V
        ops.ctc_beta_grad(logits, fs, bs, lse, input_len, targets, targets.shape[1], target_len, B, T, V, ctx.blank, log_alpha, nll,
                          up, grad, fs, bs, vpad)
        return grad, None, None, None, None, None, None


def _i32(t: torch.Tensor, dev) -> torch.Tensor:
    return t.to(device=dev, dtype=torch.int32).contiguous()


def ctc_loss(logits_tbv: torch.Tensor, input_len: torch.Tensor, targets: torch.Tensor, target_len: torch.Tensor, blank: int = 0,
             reduction: str = "sum", zero_infinity: bool = False, return_argmax: bool = False):
    """CTC loss of bf16 logits T x B x V (log-softmax included).  `targets` [B, Smax] padded, `input_len` / `target_len` [B].
    reduction: "sum" (fp64 accumulation on the device), "mean" (F.ctc_loss's: nll / max(target_len, 1), averaged over the batch)
    or "none" ([B]).  With `return_argmax` also returns the per-frame first-argmax class [B, T] int32 (blank past input_len)."""
    if reduction not in ("sum", "mean", "none"):
        raise ValueError(f"ctc_loss: reduction={reduction!r}")
    if not logits_tbv.is_cuda or logits_tbv.dtype != BF or logits_tbv.dim() != 3:
        raise ValueError("ctc_loss: logits must be a CUDA bf16 tensor T x B x V (there is no CPU or fp32 path)")
    if logits_tbv.stride(2) != 1:
        raise ValueError("ctc_loss: the class dimension of the logits must have unit stride")
    if targets.dim() != 2 or targets.shape[0] != logits_tbv.shape[1]:
        raise ValueError(f"ctc_loss: targets must be [B, Smax] padded, got {tuple(targets.shape)}")
    dev = logits_tbv.device
    target_len = _i32(target_len, dev)
    nll, total, argmax = _CtcFn.apply(logits_tbv, _i32(input_len, dev), _i32(targets, dev), target_len, int(blank),
                                      bool(zero_infinity), bool(return_argmax))
    if reduction == "sum":
        loss = total
    elif reduction == "none":
        loss = nll
    else:
        loss = (nll / target_len.clamp(min=1).float()).mean()
    return (loss, argmax) if return_argmax else loss


def prepare_targets(target: torch.Tensor, pad_idx: int, eos_idx: int, target_lengths: Optional[torch.Tensor] = None):
    """`sample["target"]` [B, S] -> (int32 [B, S] with every pad / eos removed and the rest moved to the front in order, int32 [B]
    lengths).  The reference packs the kept labels with `masked_select` (a device synchronisation); this is the same selection
    kept per row, with device-side index arithmetic only."""
    keep = (target != pad_idx) & (target != eos_idx)
    B, S = target.shape
    pos = keep.long().cumsum(1) - 1
    out = torch.zeros(B, S + 1, dtype=target.dtype, device=target.device)
    out.scatter_(1, torch.where(keep, pos, torch.full_like(pos, S)), target)   # dropped entries land in the spare column
    lengths = keep.sum(-1) if target_lengths is None else target_lengths
    return out[:, :S].to(torch.int32).contiguous(), lengths.to(torch.int32)


def greedy_collapse(argmax: torch.Tensor, input_len, blank: int = 0) -> List[List[int]]:
    """Best-path decoding of per-frame argmax classes [B, T] (host side): per utterance, the first input_len[b] frames with
    consecutive duplicates merged and blanks removed."""
    rows, lens = argmax.tolist(), [int(n) for n in input_len]
    hyps = []
    for row, n in zip(rows, lens):
        out, prev = [], None
        for c in row[:n]:
            if c != prev and c != blank:
                out.append(int(c))
            prev = c
        hyps.append(out)
    return hyps


def forced_align(logits_tbv: torch.Tensor, input_len: torch.Tensor, targets: torch.Tensor, target_len: torch.Tensor,
                 blank: int = 0):
    """CTC forced alignment of bf16 logits T x B x V (log-softmax included) to padded `targets` [B, Smax] with lengths
    `target_len` [B] over `input_len` [B] valid frames -- the same inputs as `ctc_loss`.

    Returns (labels int32 [B, T], frame_scores fp32 [B, T], score fp32 [B]), all on the logits' device: the class of each frame
    on the most probable path through (blank, l_1, blank, ..., l_S, blank), lp = logit - logsumexp(logit) (fp32) at that class,
    and the path's log-probability.  Per utterance these are bit-identical to `torchaudio.functional.forced_align` (CPU) on the
    same fp32 lp, ties included.  Frames past input_len get (-1, 0).  An infeasible utterance (input too short for its target
    with one blank between equal neighbours, target_len outside [0, Smax], a label outside [0, V) or equal to blank) gets -1 on
    every frame and score -inf instead of an error, so nothing is read back: the call captures in a CUDA graph.  Limits:
    Smax <= MAX_ALIGN_TARGET, V <= MAX_CLASSES.  The backpointer workspace, B * T * ceil((2 Smax + 1) / 16) * 4 bytes, comes
    from the caching allocator."""
    if not logits_tbv.is_cuda or logits_tbv.dtype != BF or logits_tbv.dim() != 3:
        raise ValueError("forced_align: logits must be a CUDA bf16 tensor T x B x V (there is no CPU or fp32 path)")
    if logits_tbv.stride(2) != 1:
        raise ValueError("forced_align: the class dimension of the logits must have unit stride")
    if targets.dim() != 2 or targets.shape[0] != logits_tbv.shape[1]:
        raise ValueError(f"forced_align: targets must be [B, Smax] padded, got {tuple(targets.shape)}")
    dev = logits_tbv.device
    T, B, V = logits_tbv.shape
    fs, bs = logits_tbv.stride(0), logits_tbv.stride(1)
    Smax = targets.shape[1]
    input_len, targets, target_len = _i32(input_len, dev), _i32(targets, dev), _i32(target_len, dev)
    lse = torch.empty(B, T, dtype=torch.float32, device=dev)
    labels = torch.empty(B, T, dtype=torch.int32, device=dev)
    frame_scores = torch.empty(B, T, dtype=torch.float32, device=dev)
    score = torch.empty(B, dtype=torch.float32, device=dev)
    ws = ops.ctc_align_workspace_bytes(B, T, Smax)   # -1 past the limits: the call below then reports which one
    workspace = torch.empty(max(ws, 1), dtype=torch.uint8, device=dev)
    ops.ctc_stats(logits_tbv, fs, bs, input_len, B, T, V, lse, None)
    ops.ctc_align(logits_tbv, fs, bs, lse, input_len, targets, Smax, target_len, B, T, V, int(blank), workspace, labels,
                  frame_scores, score)
    return labels, frame_scores, score


class CtcHypotheses(NamedTuple):
    """`ctc_beam_search` result, best first per utterance: tokens int32 [B, nbest, T] (class ids, no blanks, repeats collapsed,
    -1 past `lengths`), lengths int32 [B, nbest], scores fp32 [B, nbest] (-inf, length 0 where fewer beams survived)."""
    tokens: torch.Tensor
    lengths: torch.Tensor
    scores: torch.Tensor


def ctc_beam_search(logits_tbv: torch.Tensor, input_len: torch.Tensor, beam_size: int = 32, nbest: int = 1, blank: int = 0,
                    beam_size_token: Optional[int] = None, lm=None, lm_weight: float = 0.0, word_score: float = 0.0,
                    unk_score: float = 0.0, lexicon=None) -> CtcHypotheses:
    """CTC prefix beam search over bf16 logits T x B x V (log-softmax included) with `input_len` [B] valid frames -- the inputs
    of `forced_align` -- in one CTA per utterance (csrc/ctc_decode.cu).  The semantics are written out in
    include/unispeech_b200.h (b200s_ctc_decode): lp = logit - logsumexp(logit) in fp32, prefixes carry
    (pb, pnb), ranking score = logaddexp(pb, pnb) + LM part, ties to the smaller 64-bit prefix hash, the best `beam_size` kept
    after every frame; `beam_size_token` (default all) non-blank classes of highest lp are tried per frame.
    `lm` (`ngram.NgramLM`): at each word boundary (its `word_boundary` class after a non-empty word) the score gains
    lm_weight * ln P(word | previous words) + word_score; a spelling the LM does not know scores as <unk> + unk_score; at the end
    the open word and </s> are scored.  Without `lm` the score is acoustic only.
    `lexicon` (`lexicon.Lexicon`, built for this `lm` or for none, csrc/ctc_decode_lex.cu): every word must be a lexicon word
    (flashlight's LexiconDecoder).  An extension must follow an edge of the lexicon's trie, a boundary may only end a lexicon
    word (scored as above, or by word_score alone without `lm`), a hypothesis that ends inside a word is dropped, and every
    allowed extension of every beam by the `beam_size_token` classes is tried.  With smearing="max" the ranking adds
    lm_weight * the best ln P(w | <s>) of the words the partial word can still become.
    Limits: 1 <= beam_size <= 128, nbest <= beam_size, 2 <= V <= MAX_CLASSES.  Nothing synchronises: the call captures in a CUDA
    graph.  The backpointer workspace, B * T * beam_size * 4 bytes, comes from the caching allocator."""
    if not logits_tbv.is_cuda or logits_tbv.dtype != BF or logits_tbv.dim() != 3:
        raise ValueError("ctc_beam_search: logits must be a CUDA bf16 tensor T x B x V (there is no CPU or fp32 path)")
    if logits_tbv.stride(2) != 1:
        raise ValueError("ctc_beam_search: the class dimension of the logits must have unit stride")
    dev = logits_tbv.device
    T, B, V = logits_tbv.shape
    fs, bs = logits_tbv.stride(0), logits_tbv.stride(1)
    input_len = _i32(input_len, dev)
    beam_token = V - 1 if beam_size_token is None else int(beam_size_token)
    lse = torch.empty(B, T, dtype=torch.float32, device=dev)
    tokens = torch.empty(B, max(int(nbest), 1), T, dtype=torch.int32, device=dev)
    lengths = torch.empty(B, max(int(nbest), 1), dtype=torch.int32, device=dev)
    scores = torch.empty(B, max(int(nbest), 1), dtype=torch.float32, device=dev)
    if lexicon is not None:
        lexicon.check(V, lm, dev, int(blank))
    ws = ops.ctc_decode_workspace_bytes(B, T, beam_size)   # -1 past the limits: the call below then reports which one
    workspace = torch.empty(max(ws, 1), dtype=torch.uint8, device=dev)
    ops.ctc_stats(logits_tbv, fs, bs, input_len, B, T, V, lse, None)
    if lexicon is not None:
        ops.ctc_decode_lexicon(logits_tbv, fs, bs, lse, input_len, B, T, V, int(blank), int(beam_size), int(nbest), beam_token,
                               lexicon.word_boundary, lm, lm_weight, word_score, unk_score, lexicon, workspace, tokens, lengths,
                               scores)
        return CtcHypotheses(tokens, lengths, scores)
    ops.ctc_decode(logits_tbv, fs, bs, lse, input_len, B, T, V, int(blank), int(beam_size), int(nbest), beam_token,
                   -1 if lm is None else lm.word_boundary, lm, lm_weight, word_score, unk_score, workspace, tokens, lengths, scores)
    return CtcHypotheses(tokens, lengths, scores)


def hypotheses_to_words(hyp: CtcHypotheses, symbols, word_boundary: int) -> List[List[List[str]]]:
    """Host side: per utterance and n-best entry, the words of the hypothesis (its symbols joined, split at `word_boundary`,
    empty words dropped)."""
    tokens, lengths = hyp.tokens.cpu().tolist(), hyp.lengths.cpu().tolist()
    out = []
    for tb, lb in zip(tokens, lengths):
        per = []
        for row, n in zip(tb, lb):
            words, cur = [], []
            for c in row[:n]:
                if c == word_boundary:
                    if cur:
                        words.append("".join(cur))
                    cur = []
                else:
                    cur.append(symbols[c])
            if cur:
                words.append("".join(cur))
            per.append(words)
        out.append(per)
    return out


class TokenSpan(NamedTuple):
    """One token of an aligned path: frames [start, end) (end exclusive), score = mean frame score over them."""
    token: int
    start: int
    end: int
    score: float


def token_spans(labels: torch.Tensor, frame_scores: torch.Tensor, input_len, blank: int = 0) -> List[List[TokenSpan]]:
    """Per-token spans of `forced_align` paths (host side), with `torchaudio.functional.merge_tokens` semantics on each
    utterance's first input_len[b] frames: runs of equal classes are merged, blank runs dropped, and each span's score is the
    mean of its frame scores.  An infeasible utterance (labels -1) has no spans.  Frames are the model's output frames: 320
    samples (20 ms) apart at 16 kHz, so frame f starts at f * 320 / 16000 seconds."""
    labels, frame_scores = labels.cpu(), frame_scores.cpu()
    out = []
    for b, n in enumerate(int(v) for v in input_len):
        n = min(max(n, 0), labels.shape[1])
        tok, sc = labels[b, :n], frame_scores[b, :n]
        if n == 0 or bool((tok < 0).any()):
            out.append([])
            continue
        edge = torch.tensor([-1], dtype=tok.dtype)
        cuts = torch.nonzero(torch.diff(tok, prepend=edge, append=edge) != 0).flatten().tolist()
        toks = tok.tolist()
        out.append([TokenSpan(toks[s], s, e, sc[s:e].mean().item()) for s, e in zip(cuts[:-1], cuts[1:]) if toks[s] != blank])
    return out


class CtcCriterion(nn.Module):
    """The reference's `ctc` criterion (src/fairseq/criterions/ctc.py) on `ctc_loss`.

    `forward(model, sample)` -> `(loss, sample_size, logging_output)`:
      * `net_output = model(**sample["net_input"])`, logits T x B x V from `model.get_logits(net_output)`;
      * input lengths = `sample["net_input"]["src_lengths"]` if present, else the number of False entries per row of
        `net_output["padding_mask"]` (all T when it is None);
      * every `pad_idx` / `eos_idx` entry of `sample["target"]` is dropped; target lengths = `sample["target_lengths"]` if
        present, else the number of kept labels;
      * loss = sum over the batch of the CTC negative log-likelihood (`reduction="sum"`, `blank_idx`, `zero_infinity`);
      * `sample_size` = number of sentences if `sentence_avg` else `ntokens` (`sample["ntokens"]`, else the sum of the target
        lengths); `logging_output` = {"loss", "ntokens", "nsentences", "sample_size"}.
    Where this differs: the reference packs the kept labels with `masked_select` and reads `ntokens` / the loss back with `.item()`;
    here targets stay padded [B, S] with lengths and `logging_output` carries device tensors, so a training step never waits for
    the device.  In eval mode `logging_output["hypotheses"]` holds the best path per utterance (per-frame argmax, consecutive
    duplicates merged, blanks removed) as lists of class ids; scoring them against text (WER / CER) is left to the caller."""

    def __init__(self, blank_idx: int = 0, pad_idx: int = 1, eos_idx: int = 2, zero_infinity: bool = False,
                 sentence_avg: bool = False):
        super().__init__()
        self.blank_idx, self.pad_idx, self.eos_idx = blank_idx, pad_idx, eos_idx
        self.zero_infinity, self.sentence_avg = zero_infinity, sentence_avg

    def forward(self, model, sample, reduce: bool = True):
        net_output = model(**sample["net_input"])
        logits = model.get_logits(net_output)
        T, B, _ = logits.shape
        if "src_lengths" in sample["net_input"]:
            input_lengths = sample["net_input"]["src_lengths"]
        elif net_output["padding_mask"] is not None:
            input_lengths = (~net_output["padding_mask"]).sum(-1)
        else:
            input_lengths = torch.full((B,), T, dtype=torch.int32, device=logits.device)
        targets, target_lengths = prepare_targets(sample["target"].to(logits.device), self.pad_idx, self.eos_idx,
                                                  sample.get("target_lengths"))
        eval_mode = not model.training
        res = ctc_loss(logits, input_lengths, targets, target_lengths, blank=self.blank_idx, reduction="sum",
                       zero_infinity=self.zero_infinity, return_argmax=eval_mode)
        loss, argmax = res if eval_mode else (res, None)
        ntokens = sample["ntokens"] if "ntokens" in sample else target_lengths.sum()
        sample_size = sample["target"].size(0) if self.sentence_avg else ntokens
        logging_output = {"loss": loss.detach(), "ntokens": ntokens,
                          "nsentences": sample["id"].numel() if "id" in sample else B, "sample_size": sample_size}
        if eval_mode:
            logging_output["hypotheses"] = greedy_collapse(argmax.cpu(), input_lengths.cpu(), self.blank_idx)
        return loss, sample_size, logging_output


class _CtcModel(nn.Module):
    """`BaseFairseqModel` surface of the reference's CTC fine-tuning models around one `w2v_encoder`."""

    def __init__(self, w2v_encoder):
        super().__init__()
        if w2v_encoder.proj is None:
            raise ValueError("a CTC model needs the encoder's output projection: build the encoder with output_dim = vocabulary size")
        self.w2v_encoder = w2v_encoder

    def forward(self, **kwargs):
        return self.w2v_encoder(**kwargs)

    def get_logits(self, net_output):
        """T x B x V bf16 logits.  The reference overwrites padded frames with (0, -inf, ...) here after a `padding_mask.any()`
        read-back; `ctc_loss` never reads frames past the input length, so they are returned as they are."""
        return net_output["encoder_out"]

    def get_normalized_probs(self, net_output, log_probs: bool, sample=None):
        """float (log-)softmax of `encoder_out` for callers that want probabilities; `CtcCriterion` does not go through it."""
        logits = net_output["encoder_out"].float()
        return F.log_softmax(logits, dim=-1) if log_probs else F.softmax(logits, dim=-1)

    def set_num_updates(self, num_updates: int):
        self.w2v_encoder.set_num_updates(num_updates)

    def max_positions(self):
        return self.w2v_encoder.max_positions()


class HubertCtc(_CtcModel):
    """hubert_asr.py `HubertCtc`: `w2v_encoder` is a `HubertEncoder` whose `proj` has the vocabulary's width."""

    @classmethod
    def build_model(cls, w2v_model, vocab_size: int, **encoder_kwargs):
        return cls(HubertEncoder(w2v_model, output_dim=vocab_size, **encoder_kwargs))


class Wav2VecCtc(_CtcModel):
    """wav2vec2_asr.py `Wav2VecCtc`: `w2v_encoder` is a `Wav2VecEncoder` whose `proj` has the vocabulary's width."""

    @classmethod
    def build_model(cls, w2v_model, vocab_size: int, **encoder_kwargs):
        return cls(Wav2VecEncoder(w2v_model, output_dim=vocab_size, **encoder_kwargs))
