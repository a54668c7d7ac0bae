"""GPU tests of neighbor joining (DESIGN.md 3.10): mashgpu_neighbor_joining_matrix (Engine.neighbor_joining_matrix) and
mashgpu_dist_neighbor_joining (DistJob.neighbor_joining).  The want is tests/nj_model.py's numpy restatement, bit for bit: parent
equal, length equal as uint64.  Larger additive trees, beyond the model's reach, must be recovered exactly."""
import functools

import numpy as np
import pytest
import torch

import mash_b200
from fixtures import dense_rank_rows, mutate, on_device, random_matrix, synth_genome, synth_sketches
from linkage_model import METHODS
from nj_model import NONE, TreeMatrix, nj, random_tree, splits
from test_gpu_dist_prefilter import mixed_sketches

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED, ERR_NOMEM = 1, 3, 4


def assert_bits(got, want):
    assert got["parent"].dtype == np.uint32 and got["length"].dtype == np.float64
    assert np.array_equal(got["parent"], want[0])
    assert np.array_equal(got["length"].view(np.uint64), want[1].view(np.uint64))


@pytest.mark.parametrize("n", [3, 4, 5, 17, 64, 257, 1000, 1500])
def test_matrix_entry_equals_the_model(gpu, n):
    D = random_matrix(n, 100 + n)
    want = nj(D)
    got = gpu.neighbor_joining_matrix(on_device(D), n)
    assert_bits(got, want)
    assert got["parent"][-1] == NONE and got["length"][-1] == 0.0


def test_all_equal_matrix(gpu):
    n = 300
    D = np.ones((n, n))
    assert_bits(gpu.neighbor_joining_matrix(on_device(D), n), nj(D))


def test_duplicate_rows_and_zero_distances(gpu):
    rng = np.random.Generator(np.random.PCG64(5))
    base = rng.random((80, 80))
    base = np.tril(base, -1) + np.tril(base, -1).T
    pick = rng.integers(0, 80, 200)              # many leaves are copies of one another: distance 0 between them
    D = base[np.ix_(pick, pick)]
    assert_bits(gpu.neighbor_joining_matrix(on_device(D), 200), nj(D))


def test_negative_lengths_are_kept(gpu):
    n = 120
    D = random_matrix(n, 6)
    D[5, :5] = 1e-3                               # a leaf close to everything: its neighbours' branches go negative
    D[40:, 5] = 1e-3
    want = nj(D)
    assert (want[1] < 0).any()
    assert_bits(gpu.neighbor_joining_matrix(on_device(D), n), want)


@pytest.mark.parametrize("n,ld", [(100, 101), (333, 512), (1200, 1280)])
def test_leading_dimension(gpu, n, ld):
    D = random_matrix(n, 7 + n, scale=3.0)
    M = on_device(D, ld)
    assert_bits(gpu.neighbor_joining_matrix(M, n), nj(D))
    assert torch.isnan(M[:, n:]).all()           # columns past n are neither read nor written
    flat = on_device(D, ld).reshape(-1)
    assert_bits(gpu.neighbor_joining_matrix(flat, n, ld=ld), nj(D))


@pytest.mark.parametrize("kind,n", [("random", 2000), ("caterpillar", 3000), ("balanced", 5000), ("random", 20000)])
def test_additive_trees_are_recovered(gpu, kind, n):
    parent, length = random_tree(n, kind, np.random.Generator(np.random.PCG64(n)))
    tm = TreeMatrix(parent, length, n)
    M = torch.empty((n, n), dtype=torch.float64, device="cuda")
    for i0 in range(0, n, 1024):
        rows = np.stack([tm.row(a) for a in range(i0, min(n, i0 + 1024))])
        M[i0:i0 + len(rows)] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    got = gpu.neighbor_joining_matrix(M, n)
    assert splits(got["parent"], got["length"], n) == splits(parent, length, n)


def test_refusals(gpu):
    for bad in (np.nan, np.inf, -np.inf):
        D = random_matrix(50, 8)
        D[31, 7] = bad
        with pytest.raises(mash_b200.MashGpuError) as e:
            gpu.neighbor_joining_matrix(on_device(D), 50)
        assert e.value.code == ERR_INVALID
    D = random_matrix(50, 8)
    D[7, 31] = np.inf                            # the upper triangle is not read
    assert_bits(gpu.neighbor_joining_matrix(on_device(D), 50), nj(D))
    for n in (0, 1, 2):
        with pytest.raises(mash_b200.MashGpuError) as e:
            gpu.neighbor_joining_matrix(torch.zeros((3, 3), dtype=torch.float64, device="cuda"), n)
        assert e.value.code == ERR_INVALID
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.neighbor_joining_matrix(torch.zeros((4, 4), dtype=torch.float64, device="cuda").reshape(-1), 4, ld=3)
    assert e.value.code == ERR_INVALID
    with pytest.raises(ValueError):
        gpu.neighbor_joining_matrix(torch.zeros((4, 4), dtype=torch.float32, device="cuda"), 4)


# ---- the job entry: one self job per input set gives its grid, the NJ tree and both linkages, which test_gpu_dist_linkage.py checks
def job_set(gpu, golden, name, *params):
    """(H, N, L, s, prefilter) of the job-entry input set `name`"""
    if name == "golden":
        sk = [golden.golden_sketch(i) for i in range(3)]
        H = np.stack([h for h, _, _, _ in sk])
        N = np.array([len(h) for h, _, _, _ in sk], np.uint32)
        L = np.array([l for _, l, _, _ in sk], np.uint64)
        return H, N, L, 1000, None
    if name == "families":
        seqs = []
        for f in range(4):
            g = synth_genome(70 + f, 40_000)
            for m in range(6):
                seqs.append(bytes(g))
                g = mutate(g, 0.003 * (m + 1), 10 * f + m)
        return (*gpu.sketch(seqs, gpu.params(k=21, s=1000)), 1000, params[0])
    if name == "synthetic":
        s, prefilter = params
        H, N, L = synth_sketches(150, s, seed=21 + s, n_families=6, ragged=True)
        N[[3, 8]] = 0                           # empty sketches
        H[20], N[20] = H[19], N[19]              # a duplicate
        return H, N, L, s, prefilter
    if name == "mostly_unrelated":
        return (*mixed_sketches(400, 1000, seed=4), 1000, 1)
    if name == "all_unrelated":
        rng = np.random.Generator(np.random.PCG64(3))
        H = np.sort(rng.integers(0, 2**62, (60, 200), dtype=np.uint64), axis=1)
        return H, np.full(60, 200, np.uint32), np.full(60, 5_000_000, np.uint64), 200, None
    assert name == "thresholds"
    return (*synth_sketches(120, 1000, seed=31, n_families=5, ragged=True), 1000, None)


def job_trees_of(job):
    return {"nj": job.neighbor_joining(), **{method: job.linkage(method) for method in METHODS}}


@functools.cache
def job_trees(gpu, golden, name, *params):
    """(grid, trees, grid after): the job's grid, then its NJ tree and both linkages, then its grid again"""
    H, N, L, s, prefilter = job_set(gpu, golden, name, *params)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=21, kmer_space=4.0 ** 21)
    try:
        if prefilter is not None:
            job.set_prefilter(prefilter)
        grid = job.run(0, job.n_qry)
        trees = job_trees_of(job)
        return grid, trees, job.run(0, job.n_qry)
    finally:
        job.close()


@functools.cache
def threshold_trees(gpu):
    """(grid before, trees, grid after) of the "thresholds" set under three thresholds, the trees taken with the triangle set"""
    H, N, L, s, _ = job_set(gpu, None, "thresholds")
    out = []
    for kw in ({"max_distance": 0.05}, {"max_pvalue": 1e-30}, {"max_distance": 0.0, "max_pvalue": 0.0}):
        job = gpu.dist_open(H, N, L, sketch_size=s, k=21, kmer_space=4.0 ** 21, **kw)
        try:
            before = job.run(0, job.n_qry)
            job.set_triangle(True)
            trees = job_trees_of(job)
            job.set_triangle(False)
            out.append((before, trees, job.run(0, job.n_qry)))
        finally:
            job.close()
    return out


def assert_unchanged(before, after):
    for key in before:
        assert np.array_equal(before[key], after[key]), key


def job_tree(gpu, golden, name, *params):
    grid, trees, after = job_trees(gpu, golden, name, *params)
    assert_bits(trees["nj"], nj(grid["distance"]))
    assert_unchanged(grid, after)
    return trees["nj"], grid


def test_golden_genomes(gpu, golden):
    got, _ = job_tree(gpu, golden, "golden")
    assert sorted(got["parent"][:3]) == [3, 3, 3]


@pytest.mark.parametrize("prefilter", [0, 1])
def test_families_of_mutated_genomes(gpu, prefilter):
    job_tree(gpu, None, "families", prefilter)


@pytest.mark.parametrize("s,prefilter", [(1000, 0), (1000, 1), (300, -1), (10000, -1)])
def test_synthetic_sketches(gpu, s, prefilter):
    job_tree(gpu, None, "synthetic", s, prefilter)


def test_mostly_unrelated_sketches(gpu):
    job_tree(gpu, None, "mostly_unrelated")


def test_all_unrelated_sketches(gpu):
    _, grid = job_tree(gpu, None, "all_unrelated")
    assert (grid["distance"][np.tril_indices(60, -1)] == 1.0).all()


def test_thresholds_and_triangle_do_not_change_the_tree(gpu):
    base = job_tree(gpu, None, "thresholds")[0]
    for before, trees, after in threshold_trees(gpu):
        assert_bits(trees["nj"], (base["parent"], base["length"]))
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
            job.neighbor_joining()
        assert e.value.code == ERR_UNSUPPORTED
    finally:
        job.close()
    job = gpu.dist_open(H[:20], N[:20], L[:20], H[20:], N[20:], L[20:], sketch_size=300, k=21, kmer_space=4.0 ** 21)
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.neighbor_joining()
        assert e.value.code == ERR_INVALID
    finally:
        job.close()
    for n in (1, 2):
        job = gpu.dist_open(H[:n], N[:n], L[:n], sketch_size=300, k=21, kmer_space=4.0 ** 21)
        try:
            with pytest.raises(mash_b200.MashGpuError) as e:
                job.neighbor_joining()
            assert e.value.code == ERR_INVALID
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
            job.neighbor_joining()
        assert e.value.code == ERR_NOMEM
        assert torch.cuda.mem_get_info()[0] >= before - (64 << 20)
    finally:
        job.close()
