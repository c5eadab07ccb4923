"""Data-parallel gradient exchange on the flat fp32 gradient buffer.

Mirrors `LegacyDistributedDataParallel.all_reduce_grads` (src/fairseq/legacy_distributed_data_parallel.py:76-165, called from
src/fairseq/trainer.py:781-785): gradients are averaged over the ranks.  The reference packs every gradient into a temporary
flat buffer, divides it by the world size, all-reduces and unpacks (two extra full-gradient copies + one scaling pass), strictly
after the backward pass.  Here the kernels already accumulate into ONE flat buffer laid out in backward-completion order
(`engine.grad_layout`), so
  * `all_reduce_grads(flat)` is a single in-place NCCL all-reduce with the AVG operator (no division pass), and
  * `OverlappedGradSync` issues that exchange in a few contiguous buckets WHILE the backward pass is still running: a bucket is
    sent as soon as the last layer it covers has produced its gradients (NCCL runs on its own stream over NVLink / NVSwitch and
    only the final bucket -- stem + conv stack -- is exposed at the end of the step).
One process per GPU, launched with torch.distributed.run; gloo (CPU tests) has no AVG operator and takes divide + SUM.
"""
from __future__ import annotations

from typing import List, Optional

import torch
import torch.distributed as dist


def _avg_all_reduce(t: torch.Tensor, group=None, async_op: bool = False):
    world = dist.get_world_size(group)
    if dist.get_backend(group) == "nccl":
        return dist.all_reduce(t, op=dist.ReduceOp.AVG, group=group, async_op=async_op)
    t.div_(world)
    return dist.all_reduce(t, op=dist.ReduceOp.SUM, group=group, async_op=async_op)


def all_reduce_grads(flat: torch.Tensor, group=None) -> torch.Tensor:
    """In-place average of the flat gradient buffer over the process group (no-op for a single process)."""
    if not dist.is_available() or not dist.is_initialized():
        return flat
    if dist.get_world_size(group) == 1:
        return flat
    _avg_all_reduce(flat, group)
    return flat


def configure_overlap(nccl_ctas: int = 0):
    """Optional knob for the overlapped exchange: bound NCCL to `nccl_ctas` CTAs (NCCL_MAX_CTAS, read when the communicator is created:
    call this BEFORE `init_process_group`; an explicit setting in the environment wins) and record that many SMs as reserved
    (`b200s_reserve_sms`; the GEMMs launch one CTA per tile, so no grid is sized around them).  The default (0) leaves NCCL alone."""
    import os
    from . import ops
    if int(nccl_ctas) <= 0:
        ops.reserve_sms(0)
        return 0
    ctas = int(os.environ.setdefault("NCCL_MAX_CTAS", str(int(nccl_ctas))))
    ops.reserve_sms(max(0, ctas))
    return ctas


class OverlappedGradSync:
    """Bucketed gradient averaging overlapped with the backward pass.

        sync = OverlappedGradSync(model, layers_per_bucket=6)      # after the first forward pass (the engine owns the layout)
        ...
        sync.begin(); loss.backward(); sync.finish()               # every step; gradients are averaged when finish() returns

    The engine calls `stage_done(stage)` from the backward of each stage ("head" is implied by the first layer that runs);
    stages the backward pass never reaches (layerdrop, frozen extractor) are swept up by `finish()`."""

    def __init__(self, model, layers_per_bucket: int = 6, group=None):
        eng = model._engine
        if eng is None or eng.flat is None:
            raise RuntimeError("run one forward pass on the GPU first: the engine owns the gradient layout")
        self.eng, self.group = eng, group
        self.flat = eng.flat.flat
        order = eng.stage_order                       # head, (layer, L-1), ..., (layer, 0), stem, conv
        layer_stages = [st for st in order if isinstance(st, tuple)]
        self.buckets: List[dict] = []
        lo = eng.stage_ranges[order[0]][0]
        k = max(1, int(layers_per_bucket))
        for j in range(0, len(layer_stages), k):
            chunk = layer_stages[j:j + k]
            hi = eng.stage_ranges[chunk[-1]][1]
            self.buckets.append({"lo": lo, "hi": hi, "trigger": chunk[-1]})   # complete when its LOWEST layer has run backward
            lo = hi
        tail_hi = eng.stage_ranges[order[-1]][1]
        if tail_hi > lo:
            self.buckets.append({"lo": lo, "hi": tail_hi, "trigger": order[-1]})
        self._rank = {st: i for i, st in enumerate(order)}
        self._works: List = []
        self._next = 0
        self.active = dist.is_available() and dist.is_initialized() and dist.get_world_size(group) > 1
        eng.grad_sync = self

    def begin(self):
        self._works, self._next = [], 0

    def _launch_through(self, upto: int):
        while self._next < upto:
            b = self.buckets[self._next]
            self._works.append(_avg_all_reduce(self.flat[b["lo"]:b["hi"]], self.group, async_op=True))
            self._next += 1

    def stage_done(self, stage):
        if not self.active:
            return
        r = self._rank.get(stage)
        if r is None:
            return
        n = self._next
        while n < len(self.buckets) and self._rank[self.buckets[n]["trigger"]] <= r:
            n += 1
        self._launch_through(n)

    def finish(self):
        if not self.active:
            return
        self._launch_through(len(self.buckets))
        for w in self._works:
            w.wait()   # NCCL: the current stream waits for the collective's stream (no host block)
        self._works = []

    def detach(self):
        if self.eng.grad_sync is self:
            self.eng.grad_sync = None


def shard_batch(n_items: int, rank: int, world: int):
    """Contiguous utterance shard of a global batch for this rank (utterances are independent: SURVEY.md section 8e)."""
    per = (n_items + world - 1) // world
    lo = min(rank * per, n_items)
    return lo, min(lo + per, n_items)
