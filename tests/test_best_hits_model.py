"""The best-hit protocol of dist on the CPU model (tests/best_hits_model.py): the tile-wise selection must equal a stable sort,
the block-halving driver must answer every query once and stop at the one-query floor, and the shard merge must be exact."""
import numpy as np
import pytest
import torch

from best_hits_model import select_streaming, run_blocks, TILE
from mash_b200.shard import merge_best_lists, BEST_LIST_KEYS


def tied_segment(rng, n, n_values):
    """n candidates with distinct references and distances drawn from n_values values (as equal numer/denom give; None: no ties)"""
    d = rng.random(n) if n_values is None else rng.choice(rng.random(n_values), n)
    ref = rng.permutation(4 * n + 7)[:n].astype(np.uint32)
    return d.view(np.uint64), ref


@pytest.mark.parametrize("n_best", [1, 10, 1024])
def test_streaming_selection_equals_stable_sort(n_best):
    rng = np.random.Generator(np.random.PCG64(n_best))
    lengths = {0, 1, 33, 257, TILE, TILE + 1, 3 * TILE + 5, n_best - 1, n_best, n_best + 1, 20 * n_best + 3, 40_000}
    for n in sorted(lengths):
        for n_values in (1, 3, None):
            d, ref = tied_segment(rng, n, n_values)
            got, flushes = select_streaming(d, ref, n_best)
            want = np.lexsort((ref, d))[:n_best]
            assert np.array_equal(got, want), (n, n_values)
            if n > 8 * TILE and n_values is None and n_best <= 10:
                assert flushes < n // TILE / 2          # the N-th-best test keeps most of a long segment out of the sorter


def test_non_negative_doubles_order_as_their_bits():
    rng = np.random.Generator(np.random.PCG64(5))
    d = np.concatenate([rng.random(1000), [0.0, 1.0, 5e-324, 1e-300]])
    assert np.array_equal(np.argsort(d, kind="stable"), np.argsort(d.view(np.uint64), kind="stable"))


@pytest.mark.parametrize("capacity", [0, 50, 51, 120, 1000, 10 ** 9])
def test_halving_driver_answers_every_query_once(capacity):
    rng = np.random.Generator(np.random.PCG64(capacity))
    q_count, n_ref = 137, 50
    hits = rng.integers(0, n_ref + 1, q_count)
    hits[40:60] = n_ref                                     # a stretch where every pair is a hit
    calls = []

    def capture(q0, qn):
        calls.append((q0, qn))
        return int(hits[q0:q0 + qn].sum())

    done, splits, runs = run_blocks(q_count, n_ref, capacity, 64, capture)
    assert [b for b, _ in done] == sorted(b for b, _ in done)                   # output order = query order
    covered = np.concatenate([np.arange(b, b + n) for b, n in done])
    assert np.array_equal(covered, np.arange(q_count))                          # every query exactly once
    cap = max(capacity, n_ref)
    assert all(hits[b:b + n].sum() <= cap for b, n in done)
    assert runs == len(done) + splits == len(calls)
    if capacity <= 51:
        assert any(n == 1 for _, n in done) and splits > 0                      # went down to the floor and stopped there
    if capacity >= 64 * n_ref:
        assert splits == 0                                                      # q * n_ref <= capacity cannot overflow
    # a block is never split while it fits: the work wasted is at most the sum over its split ancestors
    assert sum(n for _, n in calls) <= q_count * (2 + np.log2(64))


def shard_lists(dist, ref_ok, n_best, bounds):
    """per-shard best lists (global reference indices) of a dense (Q, R) distance grid with a hit mask"""
    parts = []
    q = dist.shape[0]
    for b, e in bounds:
        cols = {k: np.zeros((q, n_best), np.float64 if k in ("distance", "pvalue") else np.int64) for k in BEST_LIST_KEYS}
        hits = np.zeros(q, np.int64); total = np.zeros(q, np.int64)
        for i in range(q):
            r = np.flatnonzero(ref_ok[i, b:e]) + b
            r = r[np.argsort(dist[i, r], kind="stable")][:n_best]
            total[i] = ref_ok[i, b:e].sum(); hits[i] = r.size
            cols["ref"][i, :r.size] = r; cols["distance"][i, :r.size] = dist[i, r]
            cols["numer"][i, :r.size] = r + 1; cols["denom"][i, :r.size] = 2 * r + 1; cols["pvalue"][i, :r.size] = dist[i, r] / 2
        parts.append({**{k: torch.from_numpy(v) for k, v in cols.items()}, "n_hits": torch.from_numpy(hits), "n_total": torch.from_numpy(total)})
    return parts


def global_lists(dist, ref_ok, n_best):
    return shard_lists(dist, ref_ok, n_best, [(0, dist.shape[1])])[0]


@pytest.mark.parametrize("bounds", [[(0, 20), (20, 41)], [(0, 14), (14, 28), (28, 41)], [(0, 41), (41, 41)]])
@pytest.mark.parametrize("n_best", [1, 5, 64])
def test_shard_merge_is_exact_under_ties(bounds, n_best):
    rng = np.random.Generator(np.random.PCG64(n_best + len(bounds)))
    q, r = 23, 41
    dist = rng.choice([0.0, 0.125, 0.25, 0.5], (q, r))              # heavy ties, on both sides of every shard boundary
    ok = rng.random((q, r)) < 0.6
    ok[3] = False; ok[4] = True
    want = global_lists(dist, ok, n_best)
    got = merge_best_lists(shard_lists(dist, ok, n_best, bounds), n_best)
    for k in want:
        assert torch.equal(got[k], want[k]), k
