"""shard.merge_components under gloo (world size 2 and 3, no GPU) and shard.merge_component_labels on its own: every rank holds the
component labels of its share of the edges over all vertices, and must end with the components of the union of the edges,
labelled by their smallest vertex (scipy.sparse.csgraph.connected_components is the reference)."""
import os
import sys

import numpy as np
import pytest
import torch
import torch.distributed as td
import torch.multiprocessing as mp
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from test_shard_gloo import _free_port             # noqa: E402


def min_labels(n, edges):
    """label[i] = smallest vertex of i's component in the graph on n vertices with the edges (E, 2)"""
    edges = np.asarray(edges, np.int64).reshape(-1, 2)
    g = coo_matrix((np.ones(len(edges)), (edges[:, 0], edges[:, 1])), shape=(n, n))
    _, comp = connected_components(g, directed=False)
    first = np.full(comp.max() + 1 if n else 0, n, np.int64)
    np.minimum.at(first, comp, np.arange(n))
    return first[comp]


def random_graph(seed, n=400, e=300):
    rng = np.random.Generator(np.random.PCG64(seed))
    edges = rng.integers(0, n, (e, 2))
    chain = rng.permutation(n)[:120]                    # a long path through random vertices
    return n, np.concatenate([edges, np.stack([chain[:-1], chain[1:]], 1)])


def _worker(rank, world, port, seed, tmp):
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    td.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from mash_b200.shard import merge_components
        n, edges = random_graph(seed)
        owner = np.random.Generator(np.random.PCG64(seed + 1)).integers(0, world, len(edges))     # a random partition of the edges
        local = min_labels(n, edges[owner == rank]).astype(np.uint32)       # as DistJob.components hands them out
        got = merge_components(local)
        np.save(os.path.join(tmp, f"cc{rank}.npy"), got.numpy())
        td.barrier()
    finally:
        td.destroy_process_group()


@pytest.mark.parametrize("world,seed", [(2, 1), (2, 2), (3, 3), (3, 4)])
def test_merge_components_equals_the_components_of_the_union(tmp_path, world, seed):
    mp.spawn(_worker, args=(world, _free_port(), seed, str(tmp_path)), nprocs=world, join=True)
    n, edges = random_graph(seed)
    want = min_labels(n, edges)
    assert 1 < len(np.unique(want)) < n
    for r in range(world):
        assert np.array_equal(np.load(tmp_path / f"cc{r}.npy"), want), r


@pytest.mark.parametrize("shards", [2, 3, 5])
def test_a_path_split_in_alternating_order_needs_many_rounds(shards):
    from mash_b200.shard import merge_component_labels
    n = 1000
    order = np.random.Generator(np.random.PCG64(shards)).permutation(n)     # the path visits the vertices in random order
    path = np.stack([order[:-1], order[1:]], 1)
    parts = [torch.from_numpy(min_labels(n, path[s::shards])) for s in range(shards)]      # edge j goes to shard j mod shards
    got = merge_component_labels(parts)
    assert got.dtype == torch.int64 and torch.equal(got, torch.zeros(n, dtype=torch.int64))


def test_merge_of_disjoint_and_identical_parts():
    from mash_b200.shard import merge_component_labels
    n = 300
    rng = np.random.Generator(np.random.PCG64(9))
    edges = rng.integers(0, n, (200, 2))
    want = min_labels(n, edges)
    one = torch.from_numpy(want)
    assert torch.equal(merge_component_labels([one]), one)
    assert torch.equal(merge_component_labels([one, one.clone()]), one)
    ident = torch.arange(n)
    assert torch.equal(merge_component_labels([ident, ident]), ident)
    halves = [torch.from_numpy(min_labels(n, edges[:100])), torch.from_numpy(min_labels(n, edges[100:]))]
    assert np.array_equal(merge_component_labels(halves).numpy(), want)
    assert merge_component_labels([torch.zeros(0, dtype=torch.int64)] * 2).numel() == 0
