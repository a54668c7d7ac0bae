"""shard.merge_best under gloo (world size 2 and 3, no GPU): every rank holds the best lists of all queries over its shard of the
reference axis, with local reference indices, and must end with the global best lists."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as td
import torch.multiprocessing as mp

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_shard_gloo import _free_port             # noqa: E402


def synthetic_grid(seed, q=31, r=53):
    rng = np.random.Generator(np.random.PCG64(seed))
    dist = rng.choice([0.0, 0.0625, 0.125, 0.25, 0.5], (q, r))     # ties inside and across shards
    ok = rng.random((q, r)) < 0.5
    ok[2] = False; ok[5] = True
    return dist, ok


def _worker(rank, world, port, n_best, tmp):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    td.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from mash_b200.shard import merge_best, shard_bounds
        from test_best_hits_model import shard_lists
        dist, ok = synthetic_grid(7 + n_best)
        b, e = shard_bounds(dist.shape[1], world)[rank]
        local = shard_lists(dist, ok, n_best, [(b, e)])[0]
        # as DistJob.run_best hands them out: numpy, unsigned, reference indices relative to the shard
        local = {k: v.numpy() for k, v in local.items()}
        local["ref"] = np.where(np.arange(n_best)[None, :] < local["n_hits"][:, None], local["ref"] - b, 0)
        for k in ("n_hits", "n_total", "ref", "numer", "denom"):
            local[k] = local[k].astype(np.uint32)
        got = merge_best(local, b, n_best)
        np.savez(os.path.join(tmp, f"best{rank}.npz"), **{k: v.numpy() for k, v in got.items()})
        td.barrier()
    finally:
        td.destroy_process_group()


@pytest.mark.parametrize("world,n_best", [(2, 1), (2, 8), (3, 8), (3, 64)])
def test_merge_best_equals_the_single_process_answer(tmp_path, world, n_best):
    from test_best_hits_model import global_lists
    mp.spawn(_worker, args=(world, _free_port(), n_best, str(tmp_path)), nprocs=world, join=True)
    dist, ok = synthetic_grid(7 + n_best)
    want = global_lists(dist, ok, n_best)
    for r in range(world):
        got = np.load(tmp_path / f"best{r}.npz")
        for k, v in want.items():
            assert np.array_equal(got[k], v.numpy()), (r, k)
