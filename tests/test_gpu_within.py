"""`mash within` through the C ABI (mashgpu_within_*) against the reference's own containSketches (tests/within_model.py): common,
examined, error and pass bit-identical, score bit-identical for j > 0 and the x86 NaN for j = 0, on every kernel path."""
import numpy as np
import pytest

import fixtures
import within_model as wm

pytestmark = pytest.mark.gpu

F32_005 = float(np.float32(0.05))


@pytest.fixture(scope="module")
def ref():
    if not wm.RefContain.available():
        pytest.skip("oracle/_ref/libmash_ref_contain.so not built")
    return wm.RefContain()


def _expect(ref, R, Rn, Q, Qn, max_error, use64=True):
    score, error = ref.grid(R, Rn, Q, Qn, use64=use64, threads=8)
    shp = (len(Qn), len(Rn))
    score, error = score.reshape(shp), error.reshape(shp)
    common, examined = wm.grid_closed_form(R, Rn, Q, Qn)
    assert np.array_equal(wm.examined_from_error(error), examined)        # the model agrees with the reference on these rows
    return dict(common=common, examined=examined, score=score, error=error, passed=error <= max_error)


def _check(got, want):
    assert np.array_equal(got["common"], want["common"])
    assert np.array_equal(got["examined"], want["examined"])
    assert got["error"].tobytes() == want["error"].tobytes()
    assert got["score"].tobytes() == want["score"].tobytes()        # NEG_NAN where examined == 0, as the reference
    assert np.array_equal(got["pass"], want["passed"])


def _run_all(gpu, R, Rn, Q=None, Qn=None, max_error=F32_005):
    job = gpu.within_open(R, Rn, Q, Qn, max_error=max_error)
    try:
        return job.run(0, job.n_qry)
    finally:
        job.close()


def test_golden_genomes(gpu, ref, golden):
    p = gpu.params(k=21, s=1000)
    recs, unit = [], []
    for u, (_, rs) in enumerate(golden.genomes):
        recs += [r[2] for r in rs]
        unit += [u] * len(rs)
    h, n, _ = gpu.sketch(recs, p, unit_of_record=np.array(unit, np.uint32), n_units=3)
    _check(_run_all(gpu, h, n), _expect(ref, h, n, h, n, F32_005))                      # all against all
    _check(_run_all(gpu, h[:1], n[:1], h[1:], n[1:]), _expect(ref, h[:1], n[:1], h[1:], n[1:], F32_005))   # `mash within g1 g2 g3`


# every kernel the job can select: rows of up to 1034 hashes tiled, 1035 and above one warp per pair
@pytest.mark.parametrize("s", [1, 2, 31, 32, 33, 1000, 1034, 1035, 10000, 28500])
def test_synth_families_all_paths(gpu, ref, s):
    n = 48 if s <= 1035 else 12
    R, Rn, _ = fixtures.synth_sketches(n, s, seed=s, ragged=True)
    Q, Qn, _ = fixtures.synth_sketches(n + 5, s, seed=s + 1, ragged=True)     # same families, other members: related and unrelated
    Q[:3] = R[:3]; Qn[:3] = Rn[:3]                                           # identical rows
    for max_error in (F32_005, 1.0):
        _check(_run_all(gpu, R, Rn, Q, Qn, max_error), _expect(ref, R, Rn, Q, Qn, max_error))
    _check(_run_all(gpu, R, Rn, None, None, F32_005), _expect(ref, R, Rn, R, Rn, F32_005))


@pytest.mark.parametrize("use64", [True, False])
def test_edge_rows(gpu, ref, use64):
    rng = np.random.Generator(np.random.PCG64(11))
    rows = wm.edge_rows(rng, hi=2**64 if use64 else 2**32)
    H, N = wm.pack_rows(rows, stride=64)
    for max_error in (F32_005, 1.0, float("inf")):
        _check(_run_all(gpu, H, N, None, None, max_error), _expect(ref, H, N, H, N, max_error, use64=use64))


def test_error_threshold_is_the_float(gpu):
    """j = 400 gives error 0.05 (double) <= float(0.05): passes; j = 399 fails.  -e inf passes j = 0 (error inf)."""
    base = np.arange(1, 1001, dtype=np.uint64) * np.uint64(1 << 40)
    rows = [base, base[:400], base[:399], np.zeros(0, np.uint64)]
    H, N = wm.pack_rows(rows)
    got = _run_all(gpu, H[:1], N[:1], H, N, F32_005)
    assert got["examined"][:, 0].tolist() == [1000, 400, 399, 0]
    assert got["pass"][:, 0].tolist() == [True, True, False, False]
    got = _run_all(gpu, H[:1], N[:1], H, N, float("inf"))
    assert got["pass"][:, 0].tolist() == [True] * 4
    assert np.isinf(got["error"][3, 0]) and got["score"][3, 0].tobytes() == wm.NEG_NAN.tobytes()


@pytest.mark.parametrize("s", [1000, 10000])
def test_subranges_repeats_self_and_device(gpu, s):
    import torch
    R, Rn, _ = fixtures.synth_sketches(70, s, seed=5, ragged=True)
    job = gpu.within_open(R, Rn, max_error=F32_005)
    twice = gpu.within_open(R, Rn, R, Rn, max_error=F32_005)
    try:
        full = job.run(0, 70)
        for a, b in ((0, 1), (3, 30), (33, 37), (69, 1), (0, 70)):
            part = job.run(a, b)
            for k in full:
                assert part[k].tobytes() == full[k][a:a + b].tobytes(), (k, a, b)
        other = twice.run(0, 70)
        for k in full:
            assert other[k].tobytes() == full[k].tobytes()
        dev = torch.device("cuda:0")
        d = dict(common=torch.zeros(70 * 70, dtype=torch.int32, device=dev), examined=torch.zeros(70 * 70, dtype=torch.int32, device=dev),
                 score=torch.zeros(70 * 70, dtype=torch.float64, device=dev), error=torch.zeros(70 * 70, dtype=torch.float64, device=dev),
                 passed=torch.zeros(70 * 70, dtype=torch.uint8, device=dev))
        job.run_dev(0, 70, d["common"].data_ptr(), d["examined"].data_ptr(), d["score"].data_ptr(), d["error"].data_ptr(),
                    d["passed"].data_ptr(), torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert np.array_equal(d["common"].cpu().numpy().view(np.uint32).reshape(70, 70), full["common"])
        assert np.array_equal(d["examined"].cpu().numpy().view(np.uint32).reshape(70, 70), full["examined"])
        assert d["score"].cpu().numpy().reshape(70, 70).tobytes() == full["score"].tobytes()
        assert d["error"].cpu().numpy().reshape(70, 70).tobytes() == full["error"].tobytes()
        assert np.array_equal(d["passed"].cpu().numpy().reshape(70, 70).astype(bool), full["pass"])
    finally:
        job.close()
        twice.close()


def test_run_crosses_output_chunk(gpu, ref):
    """mashgpu_within_run cuts its device outputs into chunks of 2^24 pairs: 4096 references x 4100 queries take two."""
    import torch
    rng = np.random.Generator(np.random.PCG64(3))
    rows = [np.unique(rng.integers(0, 4000, int(rng.integers(0, 12)), dtype=np.uint64)) for _ in range(4100)]
    H, N = wm.pack_rows(rows, stride=12)
    job = gpu.within_open(H[:4096], N[:4096], H, N, max_error=F32_005)
    try:
        got = job.run(0, 4100, outputs=("common", "examined"))
        dev = torch.device("cuda:0")
        dc = torch.zeros(4100 * 4096, dtype=torch.int32, device=dev)
        dx = torch.zeros(4100 * 4096, dtype=torch.int32, device=dev)
        job.run_dev(0, 4100, dc.data_ptr(), dx.data_ptr(), None, None, None, torch.cuda.current_stream().cuda_stream)
        torch.cuda.synchronize()
        assert np.array_equal(dc.cpu().numpy().view(np.uint32).reshape(4100, 4096), got["common"])
        assert np.array_equal(dx.cpu().numpy().view(np.uint32).reshape(4100, 4096), got["examined"])
    finally:
        job.close()
    # the reference on the queries around the chunk boundary (query 4096 starts the second chunk)
    score, error = ref.grid(H[:4096], N[:4096], H, N, pair_begin=4094 * 4096, pair_count=6 * 4096, threads=8)
    j = wm.examined_from_error(error).reshape(6, 4096)
    assert np.array_equal(got["examined"][4094:], j)
    with np.errstate(invalid="ignore"):
        common = np.where(j > 0, np.rint(score.reshape(6, 4096) * j), 0)
    assert np.array_equal(got["common"][4094:], common)


def test_row_longer_than_stride_is_refused(gpu):
    import mash_b200
    H = np.arange(8, dtype=np.uint64).reshape(2, 4)
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.within_open(H, np.array([4, 5], np.uint32))
    assert e.value.code == 1
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.within_open(H, np.array([4, 4], np.uint32), H, np.array([0, 9], np.uint32))
    assert e.value.code == 1
