"""CPU checks of the binomial-tail truth (tests/binom_truth.py) and of the oracle's long-double tail at large n.

The oracle is the comparison point of every dist / screen p-value parity test, so its own accuracy is pinned here against
the 60-digit sum on the grid that the device is held to (tests/test_gpu_pvalue_precision.py)."""
import mpmath as mp
import pytest

from binom_truth import GRID_N, GRID_R, grid_x, upper_tail


def test_truth_matches_the_golden_mpmath_values(golden):
    cases = golden.pvalue_cases
    assert len(cases) > 700
    with mp.workdps(60):
        for c in cases:
            want = mp.mpf(c["p"])
            got = upper_tail(c["x"], float(c["r"]), c["n"])
            if want == 0:
                assert got == 0, c
            else:
                assert abs(got - want) <= mp.mpf("1e-20") * want, (c, got)


def test_truth_edges_and_complement():
    assert upper_tail(0, 0.3, 10) == 1 and upper_tail(11, 0.3, 10) == 0
    assert upper_tail(5, 0.0, 10) == 0 and upper_tail(5, 1.0, 10) == 1
    # P[X >= n] = r^n and P[X >= 1] = 1 - (1-r)^n, for the exact binary r
    with mp.workdps(80):
        r = 0.63
        assert abs(upper_tail(100000, r, 100000) / mp.mpf(r) ** 100000 - 1) < mp.mpf("1e-50")
        assert abs(upper_tail(1, 1e-9, 4096) - (1 - (1 - mp.mpf(1e-9)) ** 4096)) < mp.mpf("1e-55")
    # the two branches agree across the mean: P[X >= x-200] - P[X >= x] = sum of the pmf over [x-200, x)
    n, r = 10000, 0.25
    with mp.workdps(60):
        for x in range(2480, 2521, 8):
            mid = mp.fsum(mp.binomial(n, k) * mp.mpf(r) ** k * (1 - mp.mpf(r)) ** (n - k) for k in range(x - 200, x))
            assert abs(upper_tail(x - 200, r, n) - upper_tail(x, r, n) - mid) < mp.mpf("1e-40")


@pytest.mark.parametrize("n", GRID_N)
def test_oracle_tail_matches_truth_at_large_n(oracle, n):
    worst = 0.0
    for r in GRID_R:
        for x in grid_x(n, r):
            truth = upper_tail(x, r, n)
            got = oracle.binomial_upper_tail(x, r, n)
            if truth > 1e-305:
                err = float(abs(mp.mpf(got) - truth) / truth)
                worst = max(worst, err)
                assert err <= 1e-13, (n, r, x, got, float(truth))
            else:
                assert got <= 1.0000001e-305, (n, r, x, got)
    assert worst > 0.0           # the comparison really ran
