"""CPU checks of tests/linkage_model.py (DESIGN.md 3.11): the nearest-neighbour cache algorithm the device runs equals the naive
definition bit for bit, the definition agrees with scipy's average and complete linkage where the merge order is clear, and
ultrametric trees come back exactly."""
import numpy as np
import pytest
from scipy.cluster.hierarchy import cophenet, fcluster, linkage as scipy_linkage
from scipy.spatial.distance import squareform

from linkage_model import METHODS, as_z, clades, cut, linkage, linkage_cached, symmetric, tree, ultrametric


def same_bits(x, y):
    return all(np.array_equal(x[k], y[k]) for k in ("id_lo", "id_hi", "size")) and \
        np.array_equal(x["height"].view(np.uint64), y["height"].view(np.uint64))


def matrix(kind, n, rng):
    if kind == "random":
        return rng.random((n, n))
    if kind == "integer":                           # heavily tied
        return rng.integers(0, 4, (n, n)).astype(np.float64)
    if kind == "equal":
        return np.ones((n, n))
    base = symmetric(rng.random((8, 8)))            # duplicate rows: copies of 8 points, distance 0 between copies
    pick = rng.integers(0, 8, n)
    return base[np.ix_(pick, pick)]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("kind", ["random", "integer", "equal", "duplicate"])
def test_cached_algorithm_equals_the_definition(method, kind):
    rng = np.random.Generator(np.random.PCG64(7))
    for n in (2, 3, 4, 5, 9, 17, 40, 120):
        D = matrix(kind, n, rng)
        want = linkage(D, method)
        got, rows, read = linkage_cached(D, method)
        assert same_bits(got, want), (n, kind)
        assert n - 1 <= rows and read >= 0


def test_an_all_equal_matrix_rescans_only_the_merged_rows():
    for method in METHODS:
        _, rows, _ = linkage_cached(np.ones((200, 200)), method)
        assert rows == 199                          # one row per merge: case 1 of the update rule keeps every other cache


def test_the_upper_triangle_is_not_read():
    rng = np.random.Generator(np.random.PCG64(8))
    D = rng.random((30, 30))
    E = D.copy()
    E[np.triu_indices(30)] = np.nan
    for method in METHODS:
        assert same_bits(linkage(D, method), linkage(E, method))


def clear_matrix(n, rng):
    """random distances whose least pair is clear by more than 1e-9 at every step of both methods (so no tie can go another way
    in scipy's merge order)"""
    while True:
        D = symmetric(rng.random((n, n)))
        ok = True
        for method in METHODS:
            h = np.sort(np.unique(linkage(D, method)["height"]))
            ok &= bool(np.all(np.diff(h) > 1e-9))
        if ok:
            return D


def leaf_sets(Z, n):
    under = [frozenset([i]) for i in range(n)]
    for lo, hi, _, _ in Z:
        under.append(under[int(lo)] | under[int(hi)])
    return set(under[n:])


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("n", [3, 10, 60, 150])
def test_equals_scipy_on_random_matrices(method, n):
    rng = np.random.Generator(np.random.PCG64(100 + n))
    for _ in range(3):
        D = clear_matrix(n, rng)
        ours = as_z(linkage(D, method))
        ref = scipy_linkage(squareform(D, checks=False), method=method)
        assert leaf_sets(ours, n) == leaf_sets(ref, n)
        assert np.allclose(np.sort(ours[:, 2]), np.sort(ref[:, 2]), rtol=0, atol=1e-12)
        assert np.allclose(cophenet(ours), cophenet(ref), rtol=0, atol=1e-12)
        merges = linkage(D, method)
        for t in np.quantile(ref[:, 2], [0.1, 0.3, 0.5, 0.8]):
            want = fcluster(ref, t, "distance")
            got = cut(merges, n, t)
            assert len(set(zip(want, got))) == len(set(want)) == len(set(got))
            assert np.array_equal(fcluster(ours, t, "distance"), fcluster(ref, t, "distance"))


def test_cut_numbers_clusters_in_first_member_order():
    rng = np.random.Generator(np.random.PCG64(9))
    D = clear_matrix(40, rng)
    merges = linkage(D, "average")
    Z = as_z(merges)
    for t in (0.0, 0.2, 0.4, 1.0, 2.0):
        got = cut(merges, 40, t)
        f = fcluster(Z, t, "distance")
        first = {}
        want = [first.setdefault(x, len(first)) for x in f]
        assert got.tolist() == want
    assert cut(merges, 40, 2.0).tolist() == [0] * 40
    assert cut(merges, 40, -1.0).tolist() == list(range(40))


def test_cut_takes_the_largest_height_of_a_subtree():
    # a later merge lower than an earlier one (what rounding in the average can do by an ulp): the subtree is cut by its
    # largest height, as scipy's fcluster does
    merges = {"id_lo": np.array([0, 2], np.uint32), "id_hi": np.array([1, 3], np.uint32),
              "height": np.array([0.5, 0.4]), "size": np.array([2, 3], np.uint32)}
    assert cut(merges, 3, 0.45).tolist() == [0, 1, 2]
    assert cut(merges, 3, 0.5).tolist() == [0, 0, 0]


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("n", [2, 3, 20, 200])
def test_ultrametric_trees_come_back_exactly(method, n):
    D, want = ultrametric(n, np.random.Generator(np.random.PCG64(n)))
    merges = linkage(D, method)
    assert clades(merges, n) == want
    assert same_bits(linkage_cached(D, method)[0], merges)


def test_tree_heights_and_branches():
    merges = {"id_lo": np.array([0, 2], np.uint32), "id_hi": np.array([1, 3], np.uint32),
              "height": np.array([0.25, 1.0]), "size": np.array([2, 3], np.uint32)}
    parent, length = tree(merges, 3)
    assert parent.tolist() == [3, 3, 4, 4, 0xFFFFFFFF]
    assert length.tolist() == [0.125, 0.125, 0.5, 0.375, 0.0]
