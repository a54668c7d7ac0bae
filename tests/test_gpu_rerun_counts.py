"""GPU test of the exact re-run's top-of-heap count at `-m` 1-3: a unit that the planned threshold leaves with fewer than s hashes
is re-run alone, and its final top keeps occurring after t*, so its count comes from a recount over [unit start, t*]."""
import numpy as np
import pytest

from fixtures import synth_genome

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("m", [1, 2, 3])
def test_rerun_counts_top_up_to_tstar(gpu, oracle, m):
    s = 1000
    unit = bytes(synth_genome(41, 30_000)) * 20          # ~30k distinct k-mers, each ~20 times: few survive the planned threshold
    p, po = gpu.params(k=21, s=s, min_copies=m), oracle.params(k=21)
    oh, oc, _ = oracle.sketch_unit_m([unit], po, s=s, min_copies=m, counts=True)
    assert oh.size == s
    # the case the recount handles: the top was promoted (its m-th occurrence) before t* and occurs again after it
    pos = oracle.all_hashes(unit, po)
    promoted = [np.flatnonzero(pos == h)[m - 1] for h in oh]
    tstar, top = max(promoted), np.flatnonzero(pos == oh[-1])
    assert top[m - 1] < tstar < top[-1] and oc[-1] < top.size
    before = gpu.stats()["exact_reruns"]
    h, n, _, c = gpu.sketch([unit], p, counts=True)
    assert gpu.stats()["exact_reruns"] > before
    assert n[0] == s and np.array_equal(h[0, :s], oh) and np.array_equal(c[0, :s], oc)
