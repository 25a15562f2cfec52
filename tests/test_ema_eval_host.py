"""Host logic of the data-parallel validation loss on the CPU: engine.allreduce_validation over a gloo world of two
processes gives every rank the mean of the ranks' values, which is the value of the global batch for a loss that is a
mean over equal shards."""
import os
import sys
import tempfile

import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rank(rank, world, init_file, out_dir):
    sys.path.insert(0, ROOT)
    from physicsinformeddiffusionmodels_b200.engine import allreduce_validation
    dist.init_process_group('gloo', init_method='file://' + init_file, rank=rank, world_size=world)
    try:
        g = torch.Generator().manual_seed(3)
        shards = torch.rand(world, 4, 5, generator=g)              # per-sample contributions of every rank's shard
        vals = shards[rank].mean(0)                                 # this rank's five values
        allreduce_validation(vals, world)
        torch.save(vals, os.path.join(out_dir, f'rank{rank}.pt'))
    finally:
        dist.destroy_process_group()


def test_validation_allreduce_gives_every_rank_the_global_batch_values():
    world = 2
    with tempfile.TemporaryDirectory() as d:
        mp.start_processes(_rank, args=(world, os.path.join(d, 'init'), d), nprocs=world, join=True, start_method='spawn')
        got = [torch.load(os.path.join(d, f'rank{r}.pt')) for r in range(world)]
    g = torch.Generator().manual_seed(3)
    whole = torch.rand(world, 4, 5, generator=g).reshape(world * 4, 5).mean(0)
    assert torch.equal(got[0], got[1])
    assert torch.allclose(got[0], whole, rtol=1e-6, atol=0)


def test_one_process_validation_values_are_left_alone():
    from physicsinformeddiffusionmodels_b200.engine import allreduce_validation
    v = torch.arange(5.)
    assert allreduce_validation(v, 1) is v and torch.equal(v, torch.arange(5.))
