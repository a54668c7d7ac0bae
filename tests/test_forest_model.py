"""The spanning-forest models (tests/forest_model.py) on the CPU: the restatement of the device's Boruvka rounds equals Kruskal's
algorithm under the order (distance, col, row) on graphs with many ties and zero weights, the forest cut at every weight has the
components of the graph cut there, and its single-linkage dendrogram has scipy's cophenetic distances."""
import numpy as np
import pytest
from scipy.cluster.hierarchy import cophenet, linkage
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from forest_model import boruvka, edge_order, forest_labels, kruskal, to_linkage


def random_graph(seed, n, p, levels):
    """edges {i, j}, j < i, each present with probability p, weights on `levels` values (0 among them)"""
    rng = np.random.Generator(np.random.PCG64(seed))
    i, j = np.tril_indices(n, -1)
    keep = rng.random(i.size) < p
    w = rng.integers(0, levels, keep.sum()) / max(levels - 1, 1)
    return i[keep], j[keep], w


def components(n, row, col):
    g = coo_matrix((np.ones(len(row)), (row, col)), shape=(n, n))       # ones: a zero weight is still an edge
    _, comp = connected_components(g, directed=False)
    first = np.full(comp.max() + 1 if n else 0, n, np.int64)
    np.minimum.at(first, comp, np.arange(n))
    return first[comp]


def check(n, row, col, w):
    want = kruskal(n, row, col, w)
    got, rounds = boruvka(n, row, col, w)
    assert np.array_equal(got, want)
    assert np.array_equal(np.sort(want), np.unique(want))
    if n >= 2:
        assert 1 <= rounds <= int(np.ceil(np.log2(n))) + 1
    assert np.array_equal(forest_labels(n, row[want], col[want]), components(n, row, col))
    r = np.arange(want.size)
    assert np.array_equal(edge_order(row[want], col[want], w[want]), r)      # forest order
    return want


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("n,p,levels", [(60, 0.3, 3), (80, 0.05, 2), (50, 1.0, 4), (120, 0.02, 1), (40, 0.5, 1000)])
def test_rounds_equal_kruskal(seed, n, p, levels):
    row, col, w = random_graph(seed, n, p, levels)
    check(n, row, col, w)


def test_shapes():
    for n in (0, 1, 2):
        e = np.zeros(0, np.int64)
        assert check(n, e, e, np.zeros(0)).size == 0
    one = np.array([1]), np.array([0])
    assert check(2, *one, np.array([0.0])).tolist() == [0]
    n = 200
    star = np.arange(1, n), np.zeros(n - 1, np.int64)
    assert check(n, *star, np.zeros(n - 1)).size == n - 1
    perm = np.random.Generator(np.random.PCG64(1)).permutation(n)          # a path through shuffled vertices, equal weights
    a, b = perm[:-1], perm[1:]
    row, col = np.maximum(a, b), np.minimum(a, b)
    assert check(n, row, col, np.full(n - 1, 0.5)).size == n - 1
    # a path plus every chord at a larger weight: the forest is the path
    i, j = np.tril_indices(n, -1)
    on_path = set(zip(row.tolist(), col.tolist()))
    w = np.array([0.1 if (x, y) in on_path else 0.2 for x, y in zip(i.tolist(), j.tolist())])
    got = check(n, i, j, w)
    assert set(zip(i[got].tolist(), j[got].tolist())) == on_path
    # two disconnected cliques
    row, col, w = random_graph(3, 30, 1.0, 3)
    keep = (row < 15) == (col < 15)
    assert check(30, row[keep], col[keep], w[keep]).size == 28


@pytest.mark.parametrize("seed", range(4))
def test_cut_at_every_weight_has_the_components_of_the_graph(seed):
    n = 90
    row, col, w = random_graph(seed, n, 0.08, 5)
    f = kruskal(n, row, col, w)
    for t in np.unique(w):
        below = w <= t
        fb = f[w[f] <= t]
        assert np.array_equal(forest_labels(n, row[fb], col[fb]), components(n, row[below], col[below])), t


@pytest.mark.parametrize("seed", range(4))
@pytest.mark.parametrize("levels", [3, 50])
def test_cophenetic_distances_equal_single_linkage(seed, levels):
    # complete graphs only: the single-linkage cophenetic distances are unique under ties, the topology is not
    n = 40
    row, col, w = random_graph(seed, n, 1.0, levels)
    f = kruskal(n, row, col, w)
    z = to_linkage(n, row[f], col[f], w[f])
    dense = np.zeros((n, n))
    dense[row, col] = w
    dense = dense + dense.T
    condensed = dense[np.triu_indices(n, 1)]
    assert np.array_equal(cophenet(z), cophenet(linkage(condensed, method="single")))


def test_linkage_of_a_forest_joins_the_trees_at_one():
    row, col, w = np.array([1, 3]), np.array([0, 2]), np.array([0.1, 0.2])
    z = to_linkage(4, row, col, w)
    assert z.shape == (3, 4) and z[-1, 2] == 1.0 and z[-1, 3] == 4
    assert cophenet(z).max() == 1.0
