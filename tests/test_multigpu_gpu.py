"""Data-parallel correctness on REAL GPUs (SURVEY.md section 4 item 4, section 8 a11): two ranks over NCCL, each with its shard of
a 4-utterance batch, gradients averaged on the flat fp32 buffer -- must equal the single-process gradients of the concatenated
batch (sum over utterances / world).  Mirrors `LegacyDistributedDataParallel.all_reduce_grads`
(src/fairseq/legacy_distributed_data_parallel.py:76-165): grads / world, all-reduce SUM.  Both exchange paths are checked: the
single all-reduce (`all_reduce_grads`) and the bucketed one overlapped with the backward pass (`OverlappedGradSync`).
Needs >= 2 GPUs on one machine; skipped where fewer are visible."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from oracle import wavlm_oracle as O

pytestmark = pytest.mark.gpu

LENGTHS = [16000, 12000, 14000, 9000]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _worker(rank, world, port, overlapped, out):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    from unispeech_b200.parallel import OverlappedGradSync, all_reduce_grads, shard_batch
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    cfg = O.tiny_config(pre_ln=True, encoder_layers=4)
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(O.deterministic_state_dict(cfg))
    m = m.to(dev).train()
    wav, pmask = O.deterministic_waveform(4, 16000, seed=1, lengths=LENGTHS)
    lo, hi = shard_batch(4, rank, world)
    # probe weights must be those of the utterance's position in the GLOBAL batch
    x, fpm = m.extract_features(wav[lo:hi].to(dev), padding_mask=pmask[lo:hi].to(dev), mask=False)
    R = O.hash_uniform("probe:2", (4,) + tuple(x.shape[1:]))[lo:hi].to(dev).masked_fill(fpm.unsqueeze(-1), 0.0)
    loss = (x.float() * R).sum()
    sync = None
    if overlapped:
        sync = OverlappedGradSync(m, layers_per_bucket=1)
        assert sync.active and len(sync.buckets) == cfg.encoder_layers + 1
        sync.begin()
    loss.backward()
    if overlapped:
        assert sync._next >= cfg.encoder_layers, sync._next   # the layer buckets were issued DURING the backward pass
        sync.finish()
    else:
        all_reduce_grads(m.grad_buffer())
    torch.cuda.synchronize()
    if rank == 0:
        out["flat"] = m.grad_buffer().detach().cpu()
        out["loss"] = loss.item()
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("overlapped", [False, True])
def test_two_rank_gradients_equal_single_process(cuda_device, overlapped):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    world = 2
    mgr = mp.Manager()
    out = mgr.dict()
    mp.spawn(_worker, args=(world, _free_port(), overlapped, out), nprocs=world, join=True)
    got = out["flat"]
    # single process, whole batch -- twice: the fp32 reductions that use atomics (dQ, split weight gradients, column sums) are
    # rounded to bf16 afterwards, so two runs of the SAME configuration differ by a few 1e-3 of the largest gradient; that run-to-run
    # spread is the yardstick for "equal"
    from unispeech_b200.wavlm import WavLM, WavLMConfig
    cfg = O.tiny_config(pre_ln=True, encoder_layers=4)
    m = WavLM(WavLMConfig(vars(cfg)))
    m.load_state_dict(O.deterministic_state_dict(cfg))
    m = m.to(cuda_device).train()
    wav, pmask = O.deterministic_waveform(4, 16000, seed=1, lengths=LENGTHS)
    runs = []
    for _ in range(2):
        if m._engine is not None and m._engine.flat is not None:
            m.zero_grad_buffer()
        x, fpm = m.extract_features(wav.to(cuda_device), padding_mask=pmask.to(cuda_device), mask=False)
        R = O.hash_uniform("probe:2", tuple(x.shape)).to(cuda_device).masked_fill(fpm.unsqueeze(-1), 0.0)
        (x.float() * R).sum().backward()
        torch.cuda.synchronize()
        runs.append(m.grad_buffer().detach().cpu() / world)   # sum over the 4 utterances / world = mean over ranks of the per-rank sums
    want = runs[0]
    assert got.shape == want.shape
    denom = want.abs().max().item()
    yard = (runs[0] - runs[1]).abs().max().item()
    err = (got - want).abs().max().item()
    cos = (got.double() * want.double()).sum() / (got.double().norm() * want.double().norm())
    assert err <= max(5e-3 * denom, 4.0 * yard) and err < 2e-2 * denom and cos.item() > 0.9999, (err, yard, denom, cos.item())
