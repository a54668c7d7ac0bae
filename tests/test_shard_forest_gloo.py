"""shard.spanning_forest under gloo (world size 2 and 3, no GPU) and shard.merge_spanning_forests on its own: every rank holds the
minimum spanning forest of its share of the edges, and must end with the forest of the union, edge for edge and in forest order
(Kruskal's algorithm under (distance, col, row) in tests/forest_model.py is the reference)."""
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

from forest_model import kruskal                    # noqa: E402
from test_shard_gloo import _free_port             # noqa: E402


def random_edges(seed, n=300, e=400, levels=4):
    """distinct pairs {row > col} with quantized distances (0 among them) and made-up values"""
    rng = np.random.Generator(np.random.PCG64(seed))
    a, b = rng.integers(0, n, (2, e))
    keep = a != b
    pairs = np.unique(np.stack([np.maximum(a, b)[keep], np.minimum(a, b)[keep]], 1), axis=0)
    m = len(pairs)
    return n, {"row": pairs[:, 0], "col": pairs[:, 1], "numer": rng.integers(1, 1000, m), "denom": np.full(m, 1000),
               "distance": rng.integers(0, levels, m) / levels, "pvalue": rng.random(m)}


def take(edges, idx):
    return {k: v[idx] for k, v in edges.items()}


def local_forest(n, edges):
    return take(edges, kruskal(n, edges["row"], edges["col"], edges["distance"]))


def assert_forest(got, want):
    for k, v in want.items():
        g = got[k].cpu().numpy()
        assert g.shape == v.shape and np.array_equal(g, v.astype(g.dtype)), k


def _worker(rank, world, port, seed, tmp):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    td.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from mash_b200.shard import spanning_forest
        n, edges = random_edges(seed)
        owner = np.random.Generator(np.random.PCG64(seed + 1)).integers(0, world, len(edges["row"]))     # a random partition
        got = spanning_forest(local_forest(n, take(edges, owner == rank)))
        np.savez(os.path.join(tmp, f"f{rank}.npz"), **{k: v.numpy() for k, v in got.items()})
        td.barrier()
    finally:
        td.destroy_process_group()


@pytest.mark.parametrize("world,seed", [(2, 1), (2, 2), (3, 3), (3, 4)])
def test_spanning_forest_equals_the_forest_of_the_union(tmp_path, world, seed):
    mp.spawn(_worker, args=(world, _free_port(), seed, str(tmp_path)), nprocs=world, join=True)
    n, edges = random_edges(seed)
    want = local_forest(n, edges)
    assert 1 < len(want["row"]) < n - 1
    for r in range(world):
        got = np.load(tmp_path / f"f{r}.npz")
        assert_forest({k: torch.from_numpy(got[k]) for k in got.files}, want)


@pytest.mark.parametrize("shards", [2, 3, 5])
def test_a_path_split_in_alternating_order_with_equal_weights(shards):
    from mash_b200.shard import merge_spanning_forests
    n = 1000
    order = np.random.Generator(np.random.PCG64(shards)).permutation(n)     # the path visits the vertices in random order
    a, b = order[:-1], order[1:]
    m = n - 1
    path = {"row": np.maximum(a, b), "col": np.minimum(a, b), "numer": np.arange(m), "denom": np.full(m, 7),
            "distance": np.full(m, 0.25), "pvalue": np.zeros(m)}
    # every chord of a few vertices too, at the same weight: ties everywhere, and the answer is still unique
    extra = np.random.Generator(np.random.PCG64(9)).choice(n, 12, replace=False)
    i, j = np.tril_indices(12, -1)
    chords = {"row": np.maximum(extra[i], extra[j]), "col": np.minimum(extra[i], extra[j]), "numer": np.zeros(i.size, np.int64),
              "denom": np.full(i.size, 7), "distance": np.full(i.size, 0.25), "pvalue": np.ones(i.size)}
    both = {k: np.concatenate([path[k], chords[k]]) for k in path}
    _, first = np.unique(np.stack([both["row"], both["col"]], 1), axis=0, return_index=True)
    both = take(both, np.sort(first))
    parts = [local_forest(n, take(both, np.arange(s, len(both["row"]), shards))) for s in range(shards)]
    got = merge_spanning_forests([{k: torch.from_numpy(v) for k, v in p.items()} for p in parts], n)
    assert got["row"].dtype == torch.int64 and got["distance"].dtype == torch.float64
    assert_forest(got, local_forest(n, both))
    assert got["row"].numel() == n - 1


def test_merge_of_identical_empty_and_single_parts():
    from mash_b200.shard import merge_spanning_forests
    n, edges = random_edges(5, n=120, e=400)
    want = local_forest(n, edges)
    assert_forest(merge_spanning_forests([want], n), want)
    assert_forest(merge_spanning_forests([want, local_forest(n, take(edges, np.arange(0)))], n), want)
    empty = take(edges, np.arange(0))
    got = merge_spanning_forests([empty, empty], n)
    assert all(v.numel() == 0 for v in got.values())
    with pytest.raises(ValueError):
        merge_spanning_forests([], n)
