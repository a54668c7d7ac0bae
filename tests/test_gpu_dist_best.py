"""GPU tests of the best hits of dist (mashgpu_dist_run_best): the n_best nearest references of every query, selected on the
device.  The result is defined as the first n_best rows of a stable sort of the query's row of the dense grid once the rows with
numer == 0 or pass == 0 are dropped, so it is compared with exactly that, computed from DistJob.run on the same job: indices
and counts equal, doubles bit-equal."""
import numpy as np
import pytest

from fixtures import synth_sketches
from test_gpu_dist_prefilter import mixed_sketches

pytestmark = pytest.mark.gpu

LISTS = ("ref", "numer", "denom", "distance", "pvalue")


def expected_best(grid, n_best, triangle_r0=None, q_begin=0):
    """best lists from a dense grid (dict of (Q, R) arrays as DistJob.run returns them)"""
    q_count, n_ref = grid["numer"].shape
    out = {"n_hits": np.zeros(q_count, np.uint32), "n_total": np.zeros(q_count, np.uint32),
           "ref": np.zeros((q_count, n_best), np.uint32), "numer": np.zeros((q_count, n_best), np.uint32),
           "denom": np.zeros((q_count, n_best), np.uint32), "distance": np.zeros((q_count, n_best)), "pvalue": np.zeros((q_count, n_best))}
    for i in range(q_count):
        hit = grid["pass"][i] & (grid["numer"][i] > 0)
        r = np.flatnonzero(hit)
        r = r[np.argsort(grid["distance"][i, r], kind="stable")][:n_best]
        out["n_total"][i] = hit.sum(); out["n_hits"][i] = r.size
        out["ref"][i, :r.size] = r
        for k in ("numer", "denom", "distance", "pvalue"):
            out[k][i, :r.size] = grid[k][i, r]
    return out


def assert_same(got, want):
    assert np.array_equal(got["n_total"], want["n_total"])
    assert np.array_equal(got["n_hits"], want["n_hits"])
    for k in ("ref", "numer", "denom"):
        assert np.array_equal(got[k], want[k]), k
    for k in ("distance", "pvalue"):
        assert np.array_equal(got[k].view(np.uint64), want[k].view(np.uint64)), k


def check_job(job, n_best, q_begin=0, q_count=None):
    q_count = job.n_qry - q_begin if q_count is None else q_count
    grid = job.run(q_begin, q_count)
    got = job.run_best(q_begin, q_count, n_best)
    assert_same(got, expected_best(grid, n_best))
    return got, grid


@pytest.mark.parametrize("s,k", [(1000, 21), (50, 11), (1, 21), (1034, 21), (1036, 21), (5000, 21)])
@pytest.mark.parametrize("prefilter", [0, 1])
def test_best_equals_sorted_grid_and_oracle(gpu, oracle, s, k, prefilter):
    H, N, L = synth_sketches(70, s, seed=3 + s, n_families=3, ragged=True)
    Hq, Nq, Lq = synth_sketches(45, s, seed=99 + s, n_families=3, ragged=True)
    Hq[:10] = H[:10]; Nq[:10] = N[:10]
    ks = 4.0 ** k
    job = gpu.dist_open(H, N, L, Hq, Nq, Lq, sketch_size=s, k=k, kmer_space=ks)
    try:
        job.set_prefilter(prefilter)
        for n_best in (1, 7, 1024):            # 1024 > n_ref
            got, _ = check_job(job, n_best)
    finally:
        job.close()
    want = oracle.compare_all(H, N, L, Hq, Nq, Lq, s, k, ks)
    hit = want["pass"].astype(bool) & (want["numer"] > 0)
    assert np.array_equal(got["n_total"], hit.sum(1))
    for i in range(45):
        r = got["ref"][i, :got["n_hits"][i]]
        assert np.array_equal(got["numer"][i, :r.size], want["numer"][i, r]) and np.array_equal(got["denom"][i, :r.size], want["denom"][i, r])
        d_o = np.sort(want["distance"][i, hit[i]])[:1024]
        assert np.all(np.abs(np.sort(got["distance"][i, :r.size]) - d_o) <= 1e-12)


@pytest.mark.parametrize("pair_max", ["4", "0"])
def test_best_through_the_pair_list(gpu, monkeypatch, pair_max):
    monkeypatch.setenv("MASHGPU_DIST_PAIR_MAX", pair_max)
    s, k, n = 1000, 21, 700
    rng = np.random.Generator(np.random.PCG64(2024))
    H, N, L = mixed_sketches(n, s, seed=91, n_related=0)
    Hf, Nf, _ = synth_sketches(44, s, 92, n_families=4, ragged=True)
    pos = rng.choice(n, 44, replace=False)
    H[pos], N[pos] = Hf, Nf
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        job.set_prefilter(1)
        got, _ = check_job(job, 7)
        if pair_max != "0":
            assert job.prefilter_stats()["pairs_from_lists"] >= 44 * 10
        assert got["n_hits"].max() == 7 and got["n_total"].max() >= 11
        # triangle: hits among the rows below the query only; then a sub-range, then a second range (no stale candidates)
        job.set_triangle(True)
        check_job(job, 7)
        check_job(job, 3, q_begin=100, q_count=333)
        check_job(job, 3, q_begin=0, q_count=50)
    finally:
        job.close()


@pytest.mark.parametrize("md,mp", [(1.0, 1.0), (0.1, 1.0), (1.0, 1e-10), (0.02, 1e-30), (-1.0, -1.0)])
def test_best_under_thresholds_and_query_ranges(gpu, md, mp):
    s, k = 500, 21
    H, N, L = mixed_sketches(200, s, seed=7)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=md, max_pvalue=mp)
    try:
        if md == 0.02:
            job.set_triangle(True)                       # without the query itself most queries have no reference this near
        got, _ = check_job(job, 5, q_begin=23, q_count=131)
        if md == 0.02:
            assert (got["n_hits"] == 0).any() and (got["n_hits"] > 0).any()         # some queries keep no hit at all
        check_job(job, 5, q_begin=150, q_count=50)
    finally:
        job.close()


def test_best_on_an_encoded_job_with_a_reference_offset(gpu):
    import torch
    from fixtures import dense_rank_rows
    s, k = 300, 21
    H, N, L = synth_sketches(90, s, seed=12, n_families=4, ragged=True)
    rows, n_eff = dense_rank_rows(H, N, s)
    d_rows = torch.from_numpy(rows.view(np.int32)).cuda(); d_neff = torch.from_numpy(n_eff.view(np.int32)).cuda()
    d_len = torch.from_numpy(L.view(np.int64)).cuda()
    job = gpu.dist_open_encoded(d_rows.data_ptr(), d_neff.data_ptr(), d_len.data_ptr(), 90, 30, 40, sketch_size=s, k=k, kmer_space=4.0 ** k,
                                keepalive=(d_rows, d_neff, d_len))
    try:
        got, grid = check_job(job, 6)                    # references are rows 30..69; ref is relative to row 30, like the grid's column
        assert grid["numer"].shape == (90, 40) and got["ref"].max() < 40
        job.set_triangle(True)
        check_job(job, 6)
    finally:
        job.close()


@pytest.mark.parametrize("capacity", [1, 300, 1000, 5000])
def test_overflowing_blocks_are_split_and_lose_nothing(gpu, capacity):
    # one family: every pair shares hashes, so a block of q queries has q * n_ref candidates
    s, k, n = 200, 21, 300
    H, N, L = synth_sketches(n, s, seed=2, n_families=1)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        want = job.run_best(0, n, 10)
        st0 = job.best_stats()
        assert st0["blocks_split"] == 0 and st0["blocks_run"] == 1 and st0["candidates"] == int(want["n_total"].sum())
        job.set_best_capacity(capacity)                 # 1 is raised to n_ref = 300: one query per block at the end
        got = job.run_best(0, n, 10)
        st = job.best_stats()
        assert st["blocks_split"] > 0
        assert st["candidates"] - st0["candidates"] == int(want["n_total"].sum())       # each hit kept exactly once
        assert_same(got, want)
        job.set_best_capacity(0)
        assert_same(job.run_best(0, n, 10), want)
        assert job.best_stats()["blocks_split"] == st["blocks_split"]
    finally:
        job.close()
    assert (want["n_total"] > 250).all()


def test_long_segments_and_ties_are_ordered_by_reference(gpu):
    # many identical sketches: equal distances, the list is in reference order; 3000 hits per query take the streaming path
    s, k = 64, 21
    H, N, L = synth_sketches(5, s, seed=8, n_families=1)
    idx = np.random.Generator(np.random.PCG64(1)).integers(0, 5, 3000)
    H, N, L = H[idx], N[idx], L[idx]
    job = gpu.dist_open(H, N, L, H[:40], N[:40], L[:40], sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        for n_best in (1, 10, 100, 1024):
            got, _ = check_job(job, n_best)
        same = np.flatnonzero(idx == idx[0])
        assert np.array_equal(got["ref"][0, :min(1024, same.size)], same[:1024]) and np.all(got["distance"][0, :same.size] == 0)
    finally:
        job.close()


def test_empty_and_tiny_sets_and_refused_arguments(gpu):
    import mash_b200
    s, k = 100, 21
    H, N, L = synth_sketches(9, s, seed=4, n_families=2)
    N[2] = 0; N[5] = 0                                   # empty sketches: numer == denom == 0, distance 0, not a hit
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        got, grid = check_job(job, 4)
        assert grid["distance"][2, 5] == 0 and grid["numer"][2, 5] == 0 and got["n_total"][2] == 0 and got["n_hits"][5] == 0
        assert job.run_best(3, 0, 4)["ref"].shape == (0, 4)
        check_job(job, 1, q_begin=8, q_count=1)
        for n_best, code in ((0, 1), (1025, 3)):         # MASHGPU_ERR_INVALID, MASHGPU_ERR_UNSUPPORTED
            with pytest.raises(mash_b200.MashGpuError) as e:
                job.run_best(0, 9, n_best)
            assert e.value.code == code
        with pytest.raises(mash_b200.MashGpuError):
            job.run_best(5, 5, 1)                        # range beyond the queries
    finally:
        job.close()
    job = gpu.dist_open(H[:0], N[:0], L[:0], H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)       # no references
    try:
        got = job.run_best(0, 9, 3)
        assert not got["n_hits"].any() and not got["n_total"].any()
    finally:
        job.close()
