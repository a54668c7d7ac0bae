"""CPU model of the pair list between dist_probe_kernel and dist_pair_kernel (mash_b200/csrc/dist.cu).  A probe warp reserves
popc(want) slots (1-31) with one atomicAdd on pair_count and writes its (query, reference) pairs there if the whole reservation
fits the capacity; otherwise it writes nothing and sends the combination to the whole-tile merge.  The counter has moved either
way, so a reservation that straddles the capacity leaves the slots [at, capacity) unwritten.  The consumer must merge only
slots written by this run: below the start of the first reservation that did not fit (DistArgs::pair_full).  Bounding it by
min(pair_count, capacity) alone reads the unwritten slots -- whatever an earlier run of the job left in the reused buffer."""
import numpy as np
import pytest

STALE = (-1, -1)        # an earlier run's entry (in the kernel: a pair of another query range, or one merged twice)


def probe_run(rng, cap, n_warps, buf):
    """Warps in random atomic order.  Returns (pair_count, pair_full start or None, listed pairs, pairs sent to the dense path)."""
    count, full = 0, None
    listed, dense = [], []
    for w in rng.permutation(n_warps):
        n = int(rng.integers(1, 32))
        pairs = [(int(w), lane) for lane in range(n)]
        at = count
        count += n                                       # atomicAdd(pair_count, popc(want))
        if at + n <= cap:
            buf[at:at + n] = pairs
            listed += pairs
        else:
            full = at if full is None else min(full, at)     # atomicMax(pair_full, ~at)
            dense += pairs
    return count, full, listed, dense


def consumed_parent(count, full, cap):
    return min(count, cap)


def consumed_fixed(count, full, cap):
    return count if full is None else min(count, full)


def simulate(seed, cap, n_warps, consumed):
    rng = np.random.Generator(np.random.PCG64(seed))
    buf = [STALE] * cap                                  # DevBuf memory is not cleared, and the list is reused across runs
    count, full, listed, dense = probe_run(rng, cap, n_warps, buf)
    return buf[:consumed(count, full, cap)], listed, dense, count


CASES = [(seed, cap, n_warps) for seed in range(40) for cap, n_warps in ((64, 10), (100, 9), (1000, 80), (1 << 12, 400), (31, 3))]


def test_parent_rule_consumes_unwritten_slots():
    """The parent's bound min(pair_count, capacity): once the list overflows, the straddling reservation's slots are merged
    although no warp of this run wrote them."""
    hit = 0
    for seed, cap, n_warps in CASES:
        got, listed, dense, count = simulate(seed, cap, n_warps, consumed_parent)
        if count > cap:
            assert dense
            if STALE in got:
                hit += 1
                assert len(got) == cap and len(listed) < cap
    assert hit >= len(CASES) // 2          # a reservation that ends exactly on the capacity is the only way around it


@pytest.mark.parametrize("seed,cap,n_warps", CASES)
def test_fixed_rule_merges_exactly_the_listed_pairs(seed, cap, n_warps):
    got, listed, dense, count = simulate(seed, cap, n_warps, consumed_fixed)
    assert STALE not in got
    assert sorted(got) == sorted(listed)                 # every written entry once, nothing else
    assert not set(got) & set(dense)                     # a pair is merged by exactly one path ...
    assert len(got) + len(dense) == count                # ... and every pair by one
    if count > cap:
        assert cap - 31 < len(got) <= cap               # the list fills up to the first reservation that did not fit
    else:
        assert not dense and len(got) == count


def test_fixed_rule_on_a_reused_list():
    """Two runs on one buffer (one job, two query blocks): the second run never sees the first run's entries."""
    for seed in range(50):
        rng = np.random.Generator(np.random.PCG64(1000 + seed))
        cap = 500
        buf = [STALE] * cap
        probe_run(rng, cap, 60, buf)                     # run 1 overflows and fills the buffer
        buf = [(-2, e[1]) if e != STALE else STALE for e in buf]     # mark run 1's entries as stale for run 2
        count, full, listed, dense = probe_run(rng, cap, 45, buf)
        got = buf[:consumed_fixed(count, full, cap)]
        assert all(e[0] >= 0 for e in got) and sorted(got) == sorted(listed)
        assert len(got) + len(dense) == count
