"""CPU checks of the sparse screen finish's model (tests/screen_samples_model.py): it equals the dense definition at every sketch,
with and without -w, and the exact -w order equals the order of the double identity estimates."""
import functools
import math

import numpy as np
import pytest

import screen_samples_model as ssm


def check(ref, ref_n, cnt, k=21, lengths=None):
    index = ssm.build_index(ref, ref_n)
    for winner in (False, True):
        want = ssm.dense(ref, ref_n, cnt, k, winner=winner, lengths=lengths)
        rows, stats = ssm.sparse(index, cnt, ref_n, winner=winner, lengths=lengths)
        hit = np.flatnonzero(want["shared"] >= 1)
        assert np.array_equal(rows["ref"], hit)
        assert np.array_equal(rows["shared"], want["shared"][hit])
        assert np.array_equal(rows["median"], want["median"][hit])
        assert stats["hit_hashes"] == int((np.asarray(cnt) >= 1).sum())
        seg_n = np.diff(index["seg_start"])
        assert stats["hit_pairs"] == int(seg_n[np.asarray(cnt) >= 1].sum())
        if winner:
            assert int(rows["shared"].sum()) == stats["hit_hashes"]          # every hit goes to one sketch


def table(rng, n, s, universe, ragged=True):
    ref = np.full((n, s), np.uint64(2**64 - 1))
    ref_n = np.zeros(n, np.uint32)
    for r in range(n):
        m = int(rng.integers(0, s + 1)) if ragged else s
        h = np.sort(rng.choice(universe, size=m, replace=False).astype(np.uint64))
        ref[r, :m] = h
        ref_n[r] = m
    return ref, ref_n


def sample(rng, n_distinct, frac, depth=20):
    cnt = rng.integers(1, depth, n_distinct)
    cnt[rng.random(n_distinct) >= frac] = 0
    return cnt


@pytest.mark.parametrize("seed", range(6))
def test_random_tables(seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    ref, ref_n = table(rng, 40, 60, 900)
    lengths = rng.integers(0, 3, 40).astype(np.uint64)               # many length ties: the index decides
    nd = ssm.pairs(ref, ref_n)[0].size
    for frac in (0.05, 0.3, 0.9):
        check(ref, ref_n, sample(rng, nd, frac), k=int(rng.integers(9, 33)), lengths=lengths)


def test_duplicate_and_empty_sketches():
    rng = np.random.Generator(np.random.PCG64(7))
    ref, ref_n = table(rng, 12, 50, 400)
    ref = np.concatenate([ref, ref[:4], ref[:2]])
    ref_n = np.concatenate([ref_n, ref_n[:4], ref_n[:2]])
    ref_n[3] = 0                                                       # an empty sketch (and its duplicate is not)
    ref[3] = np.uint64(2**64 - 1)
    nd = ssm.pairs(ref, ref_n)[0].size
    check(ref, ref_n, sample(rng, nd, 0.5))
    check(ref, ref_n, sample(rng, nd, 0.5), lengths=np.arange(ref_n.size, dtype=np.uint64))


def test_hashes_held_by_thousands_of_sketches():
    rng = np.random.Generator(np.random.PCG64(8))
    base = np.sort(rng.choice(5000, 40, replace=False).astype(np.uint64))
    n = 3000
    ref = np.tile(base, (n, 1))
    ref_n = np.full(n, 40, np.uint32)
    ref_n[::7] = 25                                                    # a prefix: the same hashes, a different fraction
    nd = base.size
    check(ref, ref_n, sample(rng, nd, 0.6))
    check(ref, ref_n, sample(rng, nd, 0.6), lengths=(np.arange(n) % 5).astype(np.uint64))


def test_samples_hitting_nothing_or_everything():
    rng = np.random.Generator(np.random.PCG64(9))
    ref, ref_n = table(rng, 30, 40, 600)
    nd = ssm.pairs(ref, ref_n)[0].size
    check(ref, ref_n, np.zeros(nd, np.int64))
    check(ref, ref_n, np.ones(nd, np.int64))
    check(ref, ref_n, rng.integers(1, 1000, nd))


def right_farey_neighbour(a, b, n):
    """c / d: the successor of a / b (lowest terms) in the Farey sequence of order n (b c - a d = 1, d <= n maximal)."""
    d0 = (-pow(a, -1, b)) % b if b > 1 else 0
    d = d0 + ((n - d0) // b) * b
    c = (1 + a * d) // b
    assert b * c - a * d == 1 and d <= n
    return c, d


def estimate(shared, n, k):
    return 1.0 if shared == n else (0.0 if shared == 0 else math.pow(shared / n, 1.0 / k))


def test_exact_order_equals_double_order_on_farey_neighbours():
    n_max = 32768
    rng = np.random.Generator(np.random.PCG64(10))
    fracs = [(0, 1), (1, n_max), (n_max - 1, n_max), (1, 2), (16383, 32767)]
    while len(fracs) < 3000:
        b = int(rng.integers(2, n_max + 1))
        a = int(rng.integers(1, b))
        if math.gcd(a, b) == 1:
            fracs.append((a, b))
    for a, b in fracs:
        c, d = right_farey_neighbour(a, b, n_max) if b > 1 else (1, n_max)
        if a == 0:
            c, d = 1, n_max
        for k in range(1, 33):
            lo, hi = estimate(a, b, k), estimate(c, d, k)
            assert lo < hi, (a, b, c, d, k)
            # equal fractions in other terms give the same double
            m = n_max // max(b, d)
            if m >= 2:
                assert estimate(a * m, b * m, k) == lo and estimate(c * m, d * m, k) == hi


def test_exact_order_equals_double_order_on_random_fractions():
    rng = np.random.Generator(np.random.PCG64(11))
    n = rng.integers(1, 32769, 4000)
    s = np.array([int(rng.integers(0, m + 1)) for m in n])
    lengths = rng.integers(0, 4, n.size)
    for k in (1, 2, 7, 21, 32):
        want = sorted(range(n.size), key=lambda r: (-estimate(int(s[r]), int(n[r]), k), -int(lengths[r]), r))
        got = sorted(range(n.size), key=functools.cmp_to_key(lambda a, b: ssm.exact_before(a, b, s, n, lengths)))
        assert got == want
