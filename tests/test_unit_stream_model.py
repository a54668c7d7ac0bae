"""CPU checks of the streaming unit job's model (no GPU): a running bottom-s with summed counts and the top's count at t*, merged stage
by stage, equals MinHashHeap with m = 1 (tests/reads_stream_model.py::ReferenceHeap, pinned to the reference's object code by
test_reads_stream_model.py) fed every hash in order -- for any stage boundaries."""
import numpy as np
import pytest

import reads_stream_model as R
import unit_stream_model as U


def _reference(flat, s):
    h = R.ReferenceHeap(s, m=1)
    for x in flat.tolist():
        h.try_insert(x)
    return h.result()


def _cut_sets(n, seed):
    rng = np.random.default_rng(seed)
    return [(), (n // 2,), tuple(rng.integers(0, n, 7).tolist()), tuple(rng.integers(0, n, 40).tolist()), tuple(range(1, n, 13))]


def _check(flat, s, cut_sets):
    want = _reference(flat, s)
    for cuts in cut_sets:
        h, c, _ = U.sketch_unit_stages(flat, s, cuts)
        assert np.array_equal(h, want[0]) and np.array_equal(c, want[1]), cuts


@pytest.mark.parametrize("seed", range(6))
@pytest.mark.parametrize("s,space", [(50, 1 << 40), (50, 400), (200, 1000), (16, 60)])
def test_random_streams_any_cuts(seed, s, space):
    rng = np.random.default_rng(seed * 31 + s)
    flat = rng.integers(0, space, 3000, dtype=np.uint64)
    _check(flat, s, _cut_sets(flat.size, seed))


def test_one_stage_per_kmer():
    rng = np.random.default_rng(3)
    flat = rng.integers(0, 300, 1500, dtype=np.uint64)
    _check(flat, 40, [tuple(range(1, flat.size))])


def test_s_equals_one():
    rng = np.random.default_rng(4)
    flat = rng.integers(0, 50, 800, dtype=np.uint64)
    _check(flat, 1, _cut_sets(flat.size, 4) + [tuple(range(1, flat.size))])


def test_heap_never_fills():
    rng = np.random.default_rng(5)
    flat = rng.integers(0, 30, 2000, dtype=np.uint64)         # 30 distinct hashes, s = 100
    want = _reference(flat, 100)
    assert want[0].size < 100
    _check(flat, 100, _cut_sets(flat.size, 5))


def test_top_arrives_last():
    # the final top is the last hash to enter: its count at t* is 1 whatever follows
    s = 10
    flat = np.array(list(range(100, 100 + s - 1)) * 3 + [500] + [500, 101, 500, 500], np.uint64)
    want = _reference(flat, s)
    assert want[0][-1] == 500 and want[1][-1] == 1
    _check(flat, s, _cut_sets(flat.size, 6) + [tuple(range(1, flat.size))])


@pytest.mark.parametrize("cut", [None, 5, 9, 12, 14])
def test_top_straddles_tstar(cut):
    # the top (900) occurs before and after t* (the first occurrence of 3, the last hash to enter): within one stage, or with
    # t* and the top's occurrences on either side of a stage boundary
    flat = np.array([900, 1, 2, 900, 900, 10, 900, 3, 900, 900, 2, 900, 1, 900, 900], np.uint64)
    s = 5
    want = _reference(flat, s)
    assert want[0][-1] == 900 and 0 < want[1][-1] < np.count_nonzero(flat == 900)
    cuts = () if cut is None else (cut,)
    h, c, recounts = U.sketch_unit_stages(flat, s, cuts)
    assert np.array_equal(h, want[0]) and np.array_equal(c, want[1])
    if cut is None:
        assert recounts == 1                 # first < t* < last inside one stage: counted over [stage start, t*]


def test_tiny_hash_space_heavy_duplication():
    rng = np.random.default_rng(8)
    for s in (1, 2, 3, 5):
        flat = rng.integers(0, 6, 5000, dtype=np.uint64)
        _check(flat, s, _cut_sets(flat.size, s) + [tuple(range(1, flat.size, 2))])


def test_repetitive_tail_after_tstar_across_stages():
    # the set is settled in the first stage; later stages only repeat the top and the others, which count in full except the top
    base = np.arange(1000, 1000 + 64, dtype=np.uint64)
    flat = np.concatenate([base, np.tile(base, 20)])
    want = _reference(flat, 64)
    assert want[1][-1] == 1 and want[1][0] == 21
    _check(flat, 64, [(64,), (32, 64, 500), tuple(range(64, flat.size, 64))])
