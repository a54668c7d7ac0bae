"""GPU tests of average and complete linkage (DESIGN.md 3.11): mashgpu_linkage_matrix (Engine.linkage_matrix) and
mashgpu_dist_linkage (DistJob.linkage).  The want is tests/linkage_model.py, bit for bit: ids and sizes equal, heights equal as
uint64, and the rows rescanned equal to the cache model's count.  Ultrametric trees beyond the model's reach must come back exactly."""
import numpy as np
import pytest
import torch

import mash_b200
from fixtures import dense_rank_rows, on_device, random_matrix, synth_sketches
from linkage_model import METHODS, clades, linkage, linkage_cached, symmetric, ultrametric
from test_gpu_dist_nj import assert_unchanged, job_trees, threshold_trees

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED, ERR_NOMEM = 1, 3, 4


def assert_bits(got, want):
    for key, dtype in (("id_lo", np.uint32), ("id_hi", np.uint32), ("size", np.uint32), ("height", np.float64)):
        assert got[key].dtype == dtype
    assert np.array_equal(got["id_lo"], want["id_lo"])
    assert np.array_equal(got["id_hi"], want["id_hi"])
    assert np.array_equal(got["size"], want["size"])
    assert np.array_equal(got["height"].view(np.uint64), want["height"].view(np.uint64))


def assert_model(got, D, method):
    want, rows, _ = linkage_cached(D, method)
    assert_bits(got, want)
    assert got["rows_rescanned"] == rows


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("n", [2, 3, 17, 257, 1500])
def test_matrix_entry_equals_the_model(gpu, method, n):
    D = random_matrix(n, 100 + n)
    got = gpu.linkage_matrix(on_device(D), n, method=method)
    assert_model(got, D, method)
    if n <= 257:
        assert_bits(got, linkage(D, method))


@pytest.mark.parametrize("method", METHODS)
def test_tied_matrices(gpu, method):
    rng = np.random.Generator(np.random.PCG64(5))
    n = 300
    assert_model(gpu.linkage_matrix(on_device(np.ones((n, n))), n, method=method), np.ones((n, n)), method)
    base = symmetric(rng.random((60, 60)))
    pick = rng.integers(0, 60, 400)              # many leaves are copies of one another: distance 0 between them
    D = base[np.ix_(pick, pick)]
    assert_model(gpu.linkage_matrix(on_device(D), 400, method=method), D, method)
    D = rng.integers(0, 5, (500, 500)).astype(np.float64)
    assert_model(gpu.linkage_matrix(on_device(D), 500, method=method), D, method)


def test_all_equal_matrix_rescans_one_row_per_merge(gpu):
    n = 1000
    got = gpu.linkage_matrix(on_device(np.ones((n, n))), n)
    assert got["rows_rescanned"] == n - 1
    assert (got["height"] == 1.0).all()


@pytest.mark.parametrize("n,ld", [(100, 101), (333, 512), (1200, 1280)])
def test_leading_dimension(gpu, n, ld):
    D = random_matrix(n, 7 + n)
    for method in METHODS:
        M = on_device(D, ld)
        assert_model(gpu.linkage_matrix(M, n, method=method), D, method)
        assert torch.isnan(M[:, n:]).all()       # columns past n are neither read nor written
        flat = on_device(D, ld).reshape(-1)
        assert_model(gpu.linkage_matrix(flat, n, ld=ld, method=method), D, method)


def test_upper_triangle_is_not_read(gpu):
    D = random_matrix(80, 9)
    E = D.copy()
    E[np.triu_indices(80, 1)] = np.inf
    for method in METHODS:
        assert_bits(gpu.linkage_matrix(on_device(E), 80, method=method), linkage(D, method))


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("n", [2000, 20000])
def test_ultrametric_trees_are_recovered(gpu, method, n):
    D, want = ultrametric(n, np.random.Generator(np.random.PCG64(n)), depth=24)
    got = gpu.linkage_matrix(on_device(D), n, method=method)
    assert clades(got, n) == want


def test_z_is_scipys_layout(gpu):
    from scipy.cluster.hierarchy import is_valid_linkage
    D = random_matrix(50, 10)
    got = gpu.linkage_matrix(on_device(D), 50)
    Z = mash_b200.linkage_z(got)
    assert Z.shape == (49, 4) and Z.dtype == np.float64 and is_valid_linkage(Z)


def test_refusals(gpu):
    for bad in (np.nan, np.inf, -np.inf):
        D = random_matrix(50, 8)
        D[31, 7] = bad
        with pytest.raises(mash_b200.MashGpuError) as e:
            gpu.linkage_matrix(on_device(D), 50)
        assert e.value.code == ERR_INVALID
    for n in (0, 1):
        with pytest.raises(mash_b200.MashGpuError) as e:
            gpu.linkage_matrix(torch.zeros((3, 3), dtype=torch.float64, device="cuda"), n)
        assert e.value.code == ERR_INVALID
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.linkage_matrix(torch.zeros((4, 4), dtype=torch.float64, device="cuda").reshape(-1), 4, ld=3)
    assert e.value.code == ERR_INVALID
    for method in (2, -1):
        with pytest.raises(mash_b200.MashGpuError) as e:
            gpu.linkage_matrix(on_device(random_matrix(10, 1)), 10, method=method)
        assert e.value.code == ERR_INVALID
    with pytest.raises(ValueError):
        gpu.linkage_matrix(on_device(random_matrix(10, 1)), 10, method="ward")
    with pytest.raises(ValueError):
        gpu.linkage_matrix(torch.zeros((4, 4), dtype=torch.float32, device="cuda"), 4)


# ---- the job entry: the linkages of the job runs of test_gpu_dist_nj.py, one per input set
def job_linkage(gpu, golden, name, *params):
    grid, trees, after = job_trees(gpu, golden, name, *params)
    for method in METHODS:
        assert_model(trees[method], grid["distance"], method)
    assert_unchanged(grid, after)
    return trees, grid


def test_golden_genomes(gpu, golden):
    got, _ = job_linkage(gpu, golden, "golden")
    assert got["average"]["size"].tolist() == [2, 3]


@pytest.mark.parametrize("prefilter", [0, 1])
def test_families_of_mutated_genomes(gpu, prefilter):
    job_linkage(gpu, None, "families", prefilter)


@pytest.mark.parametrize("s,prefilter", [(1000, 0), (1000, 1), (300, -1), (10000, -1)])
def test_synthetic_sketches(gpu, s, prefilter):
    job_linkage(gpu, None, "synthetic", s, prefilter)


def test_mostly_unrelated_sketches(gpu):
    job_linkage(gpu, None, "mostly_unrelated")


def test_all_unrelated_sketches(gpu):
    got, grid = job_linkage(gpu, None, "all_unrelated")
    assert (grid["distance"][np.tril_indices(60, -1)] == 1.0).all()
    assert got["average"]["rows_rescanned"] == 59 and (got["complete"]["height"] == 1.0).all()


def test_thresholds_and_triangle_do_not_change_the_merges(gpu):
    base = job_linkage(gpu, None, "thresholds")[0]
    for before, trees, after in threshold_trees(gpu):
        for method in METHODS:
            assert_bits(trees[method], base[method])
            assert trees[method]["rows_rescanned"] == base[method]["rows_rescanned"]
        assert_unchanged(before, after)


def test_job_refusals(gpu):
    H, N, L = synth_sketches(40, 300, seed=2)
    rows, n_eff = dense_rank_rows(H, N, 300)
    d_rows = torch.from_numpy(rows.view(np.int32)).cuda()
    d_neff = torch.from_numpy(n_eff.view(np.int32)).cuda()
    d_len = torch.from_numpy(L.view(np.int64)).cuda()
    job = gpu.dist_open_encoded(d_rows.data_ptr(), d_neff.data_ptr(), d_len.data_ptr(), 40, 0, 40, sketch_size=300, k=21,
                                kmer_space=4.0 ** 21, keepalive=(d_rows, d_neff, d_len))
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.linkage()
        assert e.value.code == ERR_UNSUPPORTED
    finally:
        job.close()
    job = gpu.dist_open(H[:20], N[:20], L[:20], H[20:], N[20:], L[20:], sketch_size=300, k=21, kmer_space=4.0 ** 21)
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.linkage()
        assert e.value.code == ERR_INVALID
    finally:
        job.close()
    job = gpu.dist_open(H[:1], N[:1], L[:1], sketch_size=300, k=21, kmer_space=4.0 ** 21)
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.linkage()
        assert e.value.code == ERR_INVALID
    finally:
        job.close()
    job = gpu.dist_open(H[:5], N[:5], L[:5], sketch_size=300, k=21, kmer_space=4.0 ** 21)
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.linkage(7)
        assert e.value.code == ERR_INVALID
        assert_model(job.linkage("complete"), job.run(0, 5)["distance"], "complete")
    finally:
        job.close()


def test_matrix_larger_than_the_device_is_refused_before_allocating(gpu):
    total = torch.cuda.get_device_properties(0).total_memory
    n = int((total / 8) ** 0.5) + 1000              # 8 n^2 bytes beyond the whole device
    H = np.arange(n, dtype=np.uint64).reshape(n, 1) * np.uint64(7919)
    N = np.ones(n, np.uint32)
    L = np.full(n, 1000, np.uint64)
    job = gpu.dist_open(H, N, L, sketch_size=1, k=21, kmer_space=4.0 ** 21)
    try:
        torch.cuda.synchronize()
        before = torch.cuda.mem_get_info()[0]
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.linkage()
        assert e.value.code == ERR_NOMEM
        assert torch.cuda.mem_get_info()[0] >= before - (64 << 20)
    finally:
        job.close()
