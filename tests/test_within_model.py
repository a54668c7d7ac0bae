"""The closed form of containSketches that the `within` kernels implement (tests/within_model.py), checked pair by pair against
the reference's own object code (oracle/_ref/libmash_ref_contain.so).  CPU only."""
import numpy as np
import pytest

import within_model as wm

pytestmark = pytest.mark.skipif(not wm.RefContain.available(), reason="oracle/_ref/libmash_ref_contain.so not built (reference sources absent)")


@pytest.fixture(scope="module")
def ref():
    return wm.RefContain()


def _check_all_pairs(ref, rows, use64):
    H, n = wm.pack_rows(rows)
    score, error = ref.grid(H, n, H, n, use64=use64)
    k = 0
    for q in range(len(rows)):
        for r in range(len(rows)):
            common, j = wm.contain_closed_form(rows[r], rows[q])
            ws, we = wm.score_error(common, j)
            assert error[k].tobytes() == we.tobytes(), (q, r, error[k], we)
            assert score[k].tobytes() == ws.tobytes(), (q, r, score[k], ws)
            k += 1


@pytest.mark.parametrize("use64", [True, False])
def test_edge_rows(ref, use64):
    rng = np.random.Generator(np.random.PCG64(7))
    _check_all_pairs(ref, wm.edge_rows(rng, hi=2**64 if use64 else 2**32), use64)


@pytest.mark.parametrize("seed", range(6))
def test_fuzzed_rows(ref, seed):
    """Related rows of ragged lengths drawn from a narrow value range, so that every stop of the loop is common."""
    rng = np.random.Generator(np.random.PCG64(100 + seed))
    use64 = seed % 2 == 0
    top = 2**64 - 1 if use64 else 2**32 - 1
    span = (200, 5000, top)[int(rng.integers(0, 3))]
    base = np.unique(rng.integers(0, span, 60, dtype=np.uint64, endpoint=True))
    rows = []
    for _ in range(24):
        m = int(rng.integers(0, 80))
        fresh = np.unique(rng.integers(0, span, m, dtype=np.uint64, endpoint=True))
        keep = base[rng.random(base.size) < rng.random()]
        rows.append(np.union1d(keep, fresh)[: int(rng.integers(0, 90))])
    _check_all_pairs(ref, rows, use64)


def test_nan_bits_for_nothing_examined(ref):
    """j = 0 (empty R, or R entirely below Q): score is the x86 NaN with the sign bit set, error +inf."""
    for R, Q in (([], [1, 2, 3]), ([1, 2], [5, 6]), ([1, 2], [])):
        s, e = ref.pair(np.array(R, np.uint64), np.array(Q, np.uint64))
        assert s.tobytes() == wm.NEG_NAN.tobytes() and np.isinf(e) and e > 0


def test_examined_from_error_round_trips():
    j = np.arange(0, 200_000)
    _, e = wm.score_error(np.zeros_like(j), j)
    assert np.array_equal(wm.examined_from_error(e), j)
