"""The greedy dereplication models (tests/representatives_model.py) on the CPU: the restatement of the device algorithm -- blocks,
covered flags, bit matrix rounds -- gives the sequential definition's representatives for every block size, on random graphs, ties and
zero distances, cliques and paths; the representatives are a maximal independent set in greedy order, every member goes to its nearest
adjacent representative under the spanning forest's key and lies in its component, and no block takes more rounds than rows."""
import numpy as np
import pytest
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from representatives_model import assign, device, sequential

BLOCKS = [1, 2, 7, 64, None]        # None: every row in one block


def random_graph(seed, n, p, levels):
    """edges {i, j}, j < i, each present with probability p, distances on `levels` values (0 among them)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    i, j = np.tril_indices(n, -1)
    keep = rng.random(i.size) < p
    d = rng.integers(0, levels, keep.sum()) / max(levels - 1, 1)
    return i[keep], j[keep], d


def duplicates(seed, n, groups):
    """sketches in `groups` groups of exact duplicates (distance 0 inside a group), groups joined at one tied distance"""
    rng = np.random.Generator(np.random.PCG64(seed))
    g = rng.integers(0, groups, n)
    i, j = np.tril_indices(n, -1)
    same = g[i] == g[j]
    near = np.abs(g[i] - g[j]) == 1
    keep = same | (near & (rng.random(i.size) < 0.3))
    return i[keep], j[keep], np.where(same[keep], 0.0, 0.05)


def cliques(seed, n, k):
    """k cliques over a shuffled order, all at one distance"""
    g = np.random.Generator(np.random.PCG64(seed)).integers(0, k, n)
    i, j = np.tril_indices(n, -1)
    keep = g[i] == g[j]
    return i[keep], j[keep], np.full(keep.sum(), 0.01)


def path(seed, n, shuffled):
    """a path whose chain position p is sketch perm[p]; in order the path is the worst case for rounds"""
    perm = np.random.Generator(np.random.PCG64(seed)).permutation(n) if shuffled else np.arange(n)
    a, b = perm[:-1], perm[1:]
    return np.maximum(a, b), np.minimum(a, b), np.full(n - 1, 0.02)


GRAPHS = {
    "random_sparse": lambda: (150, random_graph(1, 150, 0.03, 1000)),
    "random_dense": lambda: (120, random_graph(2, 120, 0.4, 5)),
    "random_tied": lambda: (200, random_graph(3, 200, 0.1, 2)),
    "duplicates": lambda: (160, duplicates(4, 160, 9)),
    "cliques": lambda: (140, cliques(5, 140, 6)),
    "one_clique": lambda: (60, cliques(6, 60, 1)),
    "path_in_order": lambda: (300, path(7, 300, False)),
    "path_shuffled": lambda: (300, path(8, 300, True)),
    "no_edges": lambda: (50, (np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0))),
}


def check_properties(n, i, j, d, is_rep, rep):
    i, j = np.asarray(i), np.asarray(j)
    assert not (is_rep[i] & is_rep[j]).any()                                   # independent
    start_rep = np.zeros(n, bool)
    e = is_rep[j] & ~is_rep[i]                                                 # member i with an earlier representative j
    start_rep[i[e]] = True
    assert (start_rep | is_rep).all()                                          # maximal in greedy order
    assert (rep[is_rep] == np.flatnonzero(is_rep)).all() and is_rep[rep].all()
    # nearest adjacent representative under (distance, min, max)
    for m in np.flatnonzero(~is_rep):
        sel = ((i == m) & is_rep[j]) | ((j == m) & is_rep[i])
        other = np.where(i[sel] == m, j[sel], i[sel])
        keys = sorted(zip(np.asarray(d)[sel], np.minimum(other, m), np.maximum(other, m), other))
        assert rep[m] == keys[0][3]
    if n:
        g = coo_matrix((np.ones(len(i)), (i, j)), shape=(n, n))
        _, comp = connected_components(g, directed=False)
        assert (comp[rep] == comp).all()


@pytest.mark.parametrize("block", BLOCKS)
@pytest.mark.parametrize("graph", list(GRAPHS))
def test_device_model_equals_the_definition(graph, block):
    n, (i, j, d) = GRAPHS[graph]()
    want = sequential(n, i, j)
    got, rounds = device(n, i, j, block)
    assert np.array_equal(got, want)
    rows = [min(block or n, n - q0) for q0 in range(1, n, block or max(n - 1, 1))]
    assert len(rounds) == len(rows) and all(r <= w for r, w in zip(rounds, rows))
    rep, edge = assign(n, got, i, j, d)
    check_properties(n, i, j, d, got, rep)
    assert ((edge >= 0) == ~got).all()


def test_path_in_order_is_the_worst_case_for_rounds():
    n = 300
    i, j, _ = path(7, n, False)
    _, rounds = device(n, i, j, None)
    assert rounds == [n - 2]                    # row 1 is covered by sketch 0; rows 2 .. n-1 decide one per round
    _, rounds = device(n, *path(8, n, True)[:2], None)
    assert rounds[0] < 20


def test_clique_has_one_representative_in_one_round():
    n = 60
    i, j, d = cliques(6, n, 1)
    is_rep, rounds = device(n, i, j, None)
    assert is_rep.sum() == 1 and is_rep[0] and rounds == [0]       # every row is covered by sketch 0
    rep, _ = assign(n, is_rep, i, j, d)
    assert (rep == 0).all()


@pytest.mark.parametrize("n", [0, 1, 2])
def test_tiny(n):
    i, j, d = (np.array([1]), np.array([0]), np.array([0.0])) if n == 2 else (np.zeros(0, np.int64),) * 2 + (np.zeros(0),)
    is_rep, rounds = device(n, i, j, None)
    assert np.array_equal(is_rep, sequential(n, i, j)) and sum(rounds) == 0
    rep, _ = assign(n, is_rep, i, j, d)
    assert rep.tolist() == ([0, 0] if n == 2 else list(range(n)))
