"""CPU checks of the linkage cut per component (tests/linkage_cut_model.py, DESIGN.md 3.13): the per-component route gives the whole
set's fcluster partition, and its merges up to t are the whole set's merges bit for bit, on matrices built to stress the argument --
planted clusters on an all-ones background, integer ties and duplicate rows, pairs at exactly t and one ulp either side, t = 0 and
t with T >= 1, for both methods."""
import numpy as np
import pytest

from linkage_cut_model import clades_at_most, components, linkage_cut, threshold, whole_cut
from linkage_model import METHODS, linkage_cached, symmetric


def check(D, method, t):
    n = len(D)
    labels, forest, n_comp = linkage_cut(D, method, t)
    assert np.array_equal(labels, whole_cut(D, method, t))
    assert len(forest["height"]) == n - n_comp
    whole = linkage_cached(D, method)[0]
    assert clades_at_most(forest, n, t) == clades_at_most(whole, n, t)
    return labels, n_comp


def planted(n, rng, spread=0.08, groups=12, near=0.0):
    """clusters of random sizes with distances in [0, spread) inside, 1 (no shared hash) between; with near > 0 some pairs of
    clusters sit at `near`, so components hold several flat clusters"""
    g = rng.integers(0, groups, n)
    D = np.where(g[:, None] == g[None, :], rng.random((n, n)) * spread, 1.0)
    if near:
        for a in range(0, groups - 1, 2):
            D[np.ix_(g == a, g == a + 1)] = near + rng.random() * 0.01
            D[np.ix_(g == a + 1, g == a)] = D[np.ix_(g == a, g == a + 1)].T
    return symmetric(D)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("t", [0.02, 0.05, 0.1, 0.3])
def test_planted_clusters(method, t):
    rng = np.random.Generator(np.random.PCG64(int(t * 1000)))
    for near in (0.0, 0.09, 0.2):
        labels, n_comp = check(planted(150, rng, near=near), method, t)
        assert n_comp >= 1


@pytest.mark.parametrize("method", METHODS)
def test_integer_ties_and_duplicate_rows(method):
    rng = np.random.Generator(np.random.PCG64(7))
    D = symmetric(rng.integers(0, 9, (120, 120)) / 8.0)            # distances k / 8, 1 for k = 8: heavy ties
    for t in (0.0, 0.125, 0.25, 0.5, 0.875):
        check(D, method, t)
    base = planted(30, rng, spread=0.2, groups=4)
    pick = rng.integers(0, 30, 140)                                 # copies of rows: distance 0 between them
    D = base[np.ix_(pick, pick)]
    D[np.arange(140), np.arange(140)] = 0
    for t in (0.0, 0.05, 0.15):
        check(D, method, t)


@pytest.mark.parametrize("method", METHODS)
def test_pairs_at_t_and_one_ulp_around_it(method):
    rng = np.random.Generator(np.random.PCG64(11))
    t = 0.1
    D = planted(100, rng, spread=0.05, groups=20)
    i, j = np.tril_indices(100, -1)
    pick = rng.choice(i.size, 60, replace=False)
    vals = np.array([t, np.nextafter(t, np.inf), np.nextafter(t, -np.inf)])[rng.integers(0, 3, 60)]
    D[i[pick], j[pick]] = vals
    D = symmetric(D)
    check(D, method, t)
    check(D, method, float(np.nextafter(t, np.inf)))
    check(D, method, float(np.nextafter(t, -np.inf)))


@pytest.mark.parametrize("method", METHODS)
def test_t_zero_and_one_component(method):
    rng = np.random.Generator(np.random.PCG64(13))
    D = planted(80, rng, spread=0.1, groups=8)
    D[5, 3] = D[3, 5] = D[40, 2] = D[2, 40] = 0.0
    labels, _ = check(D, method, 0.0)
    assert labels[5] == labels[3] == 3
    assert threshold(1.0, 80) > 1
    labels, n_comp = check(D, method, 1.0)          # T >= 1: the whole set is one component and one cluster
    assert n_comp == 1 and (labels == 0).all()
    assert (components(D, threshold(1.0, 80)) == 0).all()


@pytest.mark.parametrize("method", METHODS)
def test_pairs_at_distance_zero_join_across_the_background(method):
    """empty sketches: distance 0 to one another and 1 to everything else, scattered over the index range"""
    rng = np.random.Generator(np.random.PCG64(17))
    D = planted(90, rng, groups=9)
    empty = [4, 30, 31, 77]
    D[np.ix_(empty, empty)] = 0.0
    for t in (0.0, 0.05):
        labels, _ = check(symmetric(D), method, t)
        assert (labels[empty] == 4).all()


def test_threshold_is_above_t():
    for t in (0.0, 1e-300, 0.05, 0.1, 0.999):
        for n in (2, 1000, 10 ** 6):
            T = threshold(t, n)
            assert T > t and T >= t * (1 + 8 * n * 2.0 ** -53)
