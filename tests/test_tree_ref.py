"""CPU tests of tools/tree_ref.cpp, the C++ reference that the GPU tests hold neighbor joining and average / complete linkage to
at sizes the numpy models cannot reach (tests/test_gpu_trees_at_scale.py).  It is pinned here to tests/nj_model.py and
tests/linkage_model.py bit for bit, on the matrices where tie-breaks and operation order decide the result: continuous random
values, a handful of levels (massive ties), all-equal, duplicate rows, zero blocks, and junk past column n."""
import numpy as np
import pytest

import tree_ref
from linkage_model import METHODS, linkage
from nj_model import NONE, nj


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return tree_ref.build(tmp_path_factory.mktemp("tree_ref"))


def as_dict(tree):
    """nj_model.nj's (parent, length) in the layout of the reference and the engine"""
    return {"parent": tree[0], "length": tree[1]}


def matrices(n, seed):
    """(name, D) of the kinds of matrices the trees meet; the upper triangle and the diagonal hold NaN, which must not be read"""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = [("random", rng.random((n, n))),
           ("levels", rng.choice([0.0, 0.25, 0.5, 1.0], (n, n), p=[0.1, 0.2, 0.2, 0.5])),
           ("jaccard", 1.0 - rng.integers(0, 21, (n, n)) / 20.0),        # quantised like a sketch of 20 hashes
           ("equal", np.ones((n, n))),
           ("zero", np.zeros((n, n)))]
    base = rng.random((max(2, n // 4), max(2, n // 4)))
    base = np.tril(base, -1) + np.tril(base, -1).T
    pick = rng.integers(0, len(base), n)           # copies of a few rows: distance 0 between copies
    out.append(("duplicates", base[np.ix_(pick, pick)]))
    Z = rng.random((n, n))
    for _ in range(3):                              # blocks of zero distance, one of them off the diagonal
        i, j = sorted(rng.integers(0, n, 2))
        Z[i:j + 1, i:j + 1] = 0.0
    i, j = sorted(rng.integers(0, n, 2))
    Z[j:, :i + 1] = 0.0
    out.append(("zero_blocks", Z))
    for _, D in out:
        D[np.triu_indices(n)] = np.nan
    return out


SIZES = [3, 4, 5, 17, 64, 129, 257, 401]


@pytest.mark.parametrize("n", SIZES)
def test_nj_equals_the_model(exe, n):
    for name, D in matrices(n, 40 + n):
        got = tree_ref.run(exe, D, "nj")
        tree_ref.assert_nj_bits(got, as_dict(nj(D)))
        assert got["parent"][-1] == NONE, name


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("n", [2] + SIZES)
def test_linkage_equals_the_model(exe, method, n):
    for _, D in matrices(n, 70 + n):
        tree_ref.assert_linkage_bits(tree_ref.run(exe, D, method), linkage(D, method))


@pytest.mark.parametrize("n,ld", [(5, 6), (100, 101), (333, 384)])
def test_leading_dimension_with_junk(exe, n, ld):
    for _, D in matrices(n, 90 + n)[:3]:
        M = np.full((n, ld), np.nan)
        M[:, :n] = D
        tree_ref.assert_nj_bits(tree_ref.run(exe, M, "nj"), as_dict(nj(D)))
        for method in METHODS:
            tree_ref.assert_linkage_bits(tree_ref.run(exe, M, method), linkage(D, method))


def test_thread_count_does_not_change_the_result(exe):
    """the scan's per-thread minima are reduced by the same strict order (value, row, column), so ties resolve the same way"""
    for _, D in matrices(300, 11):
        tree_ref.assert_nj_bits(tree_ref.run(exe, D, "nj", threads=8), tree_ref.run(exe, D, "nj", threads=1))
        for method in METHODS:
            tree_ref.assert_linkage_bits(tree_ref.run(exe, D, method, threads=8), tree_ref.run(exe, D, method, threads=1))


def test_all_equal_matrix_gives_the_documented_shapes(exe):
    """every pair ties at every step: NJ joins positions 0 and 1 each time (nj_model's caterpillar), linkage merges slots 0 and 1"""
    n = 7
    got = tree_ref.run(exe, np.ones((n, n)), "nj")
    assert list(got["parent"]) == [7, 7, 8, 9, 10, 11, 11, 8, 9, 10, 11, NONE]
    got = tree_ref.run(exe, np.ones((n, n)), "average")
    assert list(got["id_lo"]) == [0, 2, 3, 4, 5, 6] and list(got["id_hi"]) == [1, 7, 8, 9, 10, 11]
    assert list(got["size"]) == [2, 3, 4, 5, 6, 7] and (got["height"] == 1.0).all()
