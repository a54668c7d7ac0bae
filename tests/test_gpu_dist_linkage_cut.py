"""GPU tests of the linkage cut per component (DESIGN.md 3.13): mashgpu_dist_linkage_cut (DistJob.linkage_cut).  The labels must be
the dense route's cut (DistJob.linkage() then cut) and tests/linkage_cut_model.py's over run()'s grid; the merge forest must be the
model's per-component linkage bit for bit, and neither may depend on the tier a component goes through (the CTA kernel or the
matrix tier).  Beyond the dense route's memory the labels of each component must be those of a linkage_matrix run on its own grid."""
import numpy as np
import pytest
import torch

import mash_b200
from fixtures import dense_rank_rows, on_device
from linkage_cut_model import clades_at_most, components, linkage_cut, smallest_labels, threshold
from linkage_model import METHODS, cut

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED, ERR_NOMEM = 1, 3, 4


def families(sizes, s, seed, bits=64, ragged=False):
    """One family per entry of `sizes`, rows shuffled.  A family has a base of s hashes in the lower half of the hash range; each member
    keeps every base hash with its own probability (0.45 .. 0.99) and fills the rest from the upper half, so members of a family are
    at distances from ~0.001 to ~0.05 (k = 21) and members of different families share no hash.  Ragged: every 7th row is cut short and rows 3, 10
    and 50 are empty (at distance 0 from one another).
    Returns (hashes, n_hashes, lengths)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    n = int(sum(sizes))
    half = 1 << (bits - 1)
    H = np.full((n, s), np.uint64(0xFFFFFFFFFFFFFFFF), np.uint64)
    N = np.full(n, s, np.uint32)
    row = 0
    for m in sizes:
        base = np.unique(rng.integers(0, half, 2 * s, dtype=np.uint64))[:s]
        p = rng.uniform(0.45, 0.99, (m, 1))
        keep = rng.random((m, s)) < p
        fresh = rng.integers(half, (1 << bits) - 1, (m, s), dtype=np.uint64)
        H[row:row + m] = np.sort(np.where(keep, base[None, :].astype(np.uint64), fresh), axis=1)
        row += m
    perm = rng.permutation(n)
    H = H[perm]
    if ragged:
        for i in range(0, n, 7):
            c = int(rng.integers(1, s))
            N[i] = c
            H[i, c:] = np.uint64(0xFFFFFFFFFFFFFFFF)
        N[[3, 10, 50]] = 0
        H[[3, 10, 50]] = np.uint64(0xFFFFFFFFFFFFFFFF)
    return H, N, rng.integers(4_000_000, 6_000_000, n).astype(np.uint64)


SIZES = [1] * 40 + [2] * 20 + [3] * 10 + [5, 8, 13, 17, 31, 33, 40, 64, 65, 90, 128, 129, 160, 200, 238, 239, 300]


def open_job(gpu, H, N, L, s, k=21):
    return gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.3, max_pvalue=1e-5)


def grid(job):
    return job.run(0, job.n_qry, outputs=("distance",))["distance"]


def assert_forest(got, want):
    assert np.array_equal(got["id_lo"], want["id_lo"])
    assert np.array_equal(got["id_hi"], want["id_hi"])
    assert np.array_equal(got["size"], want["size"])
    assert np.array_equal(got["height"].view(np.uint64), want["height"].view(np.uint64))


def check_job(job, ts, methods=METHODS, dense=True, tiers=(0,)):
    D = grid(job)
    n = job.n_qry
    for method in methods:
        whole = job.linkage(method) if dense else None
        for t in ts:
            labels, forest, n_comp = linkage_cut(D, method, t)
            for tier in tiers:
                job.set_linkage_cut_cta_max(tier)
                got = job.linkage_cut(method, t, merges=True)
                assert np.array_equal(got["labels"], labels), (method, t, tier)
                assert got["n_components"] == n_comp
                assert got["n_clusters"] == len(np.unique(labels))
                assert got["largest_component"] == np.bincount(components(D, threshold(t, n))).max()
                assert_forest(got["merges"], forest)
                nolist = job.linkage_cut(method, t)
                assert np.array_equal(nolist["labels"], labels) and "merges" not in nolist
            if dense:
                assert np.array_equal(labels, smallest_labels(cut(whole, n, t)))
                assert clades_at_most(forest, n, t) == clades_at_most(whole, n, t)
    job.set_linkage_cut_cta_max(0)


def test_many_components_of_varied_sizes_every_tier(gpu):
    s = 200
    H, N, L = families(SIZES, s, seed=1)
    job = open_job(gpu, H, N, L, s)
    try:
        check_job(job, [0.0, 0.005, 0.02, 0.05], tiers=(0, 1, 32))
        job.linkage_cut("average", 0.02)
        ms = job.linkage_cut_stats()
        assert set(ms) == {"components", "grouping", "cta", "matrix"} and all(v >= 0 for v in ms.values())
    finally:
        job.close()


def test_one_family(gpu):
    s = 300
    H, N, L = families([700], s, seed=2)
    job = open_job(gpu, H, N, L, s)
    try:
        check_job(job, [0.01, 0.03, 0.06])
    finally:
        job.close()


def test_ragged_sketches(gpu):
    s = 400
    H, N, L = families(SIZES[40:], s, seed=3, ragged=True)
    job = open_job(gpu, H, N, L, s)
    try:
        check_job(job, [0.01, 0.04], tiers=(0, 1))
    finally:
        job.close()


def test_general_merge_path(gpu):
    """s > 1035: the tiled merge does not fit shared memory, so the matrix tier fills through the warp-per-pair merge"""
    s = 1100
    H, N, L = families([1, 1, 2, 5, 30, 120, 260], s, seed=4)
    job = open_job(gpu, H, N, L, s)
    try:
        check_job(job, [0.01, 0.03], tiers=(0, 1))
    finally:
        job.close()


def test_32_bit_hashes(gpu):
    s = 500
    H, N, L = families([1, 3, 9, 27, 81, 243], s, seed=5, bits=32)
    job = open_job(gpu, H, N, L, s, k=16)
    try:
        check_job(job, [0.01, 0.05], tiers=(0, 1))
    finally:
        job.close()


def test_cut_at_and_above_one(gpu):
    """T >= 1: the whole set is one component, linked in one CTA when it fits, else through the matrix tier"""
    s = 100
    H, N, L = families([3, 4, 5, 20], s, seed=6)
    job = open_job(gpu, H, N, L, s)
    try:
        for tier in (0, 1):
            job.set_linkage_cut_cta_max(tier)
            for method in METHODS:
                got = job.linkage_cut(method, 1.0, merges=True)
                assert got["n_components"] == 1 and got["largest_component"] == 32
                assert (got["labels"] == 0).all() and got["n_clusters"] == 1
                assert_forest(got["merges"], job.linkage(method))
    finally:
        job.close()


def test_past_the_dense_limit(gpu):
    """~110 000 sketches: the dense route needs 97 GB and refuses; the cut runs, and within each component (the components of a job
    opened at max_distance T) the labels are those of linkage_matrix on the component's own grid"""
    s, k, t = 12, 21, 0.05
    rng = np.random.Generator(np.random.PCG64(9))
    sizes = []
    while sum(sizes) < 110_000:
        sizes.append(int(rng.choice([1, 1, 2, 3, 4, 6, 10, 20, 50, 150, 400])))
    H, N, L = families(sizes, s, seed=10)
    n = len(N)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.linkage("average")
        assert e.value.code == ERR_NOMEM
        got = job.linkage_cut("average", t)
    finally:
        job.close()
    T = threshold(t, n)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=T, max_pvalue=1.0)
    try:
        comp_labels, _ = job.components()
    finally:
        job.close()
    comps = {}
    for i, r in enumerate(comp_labels.tolist()):
        comps.setdefault(r, []).append(i)
    assert got["n_components"] == len(comps) and got["largest_component"] == max(len(v) for v in comps.values())
    singles = [v[0] for v in comps.values() if len(v) == 1]
    assert (got["labels"][singles] == singles).all()
    multi = sorted((np.array(v) for v in comps.values() if len(v) > 1), key=len, reverse=True)
    pick = multi[:25] + [multi[i] for i in rng.choice(np.arange(25, len(multi)), min(25, max(len(multi) - 25, 0)), replace=False)]
    for mem in pick:
        sub = gpu.dist_open(H[mem], N[mem], L[mem], sketch_size=s, k=k, kmer_space=4.0 ** k)
        try:
            D = sub.run(0, len(mem), outputs=("distance",))["distance"]
        finally:
            sub.close()
        merges = gpu.linkage_matrix(on_device(D), len(mem), method="average")
        assert np.array_equal(mem[smallest_labels(cut(merges, len(mem), t))], got["labels"][mem])
    assert len(pick) >= 30


def test_refusals_and_tiny_sets(gpu):
    s = 100
    H, N, L = families([3, 4], s, seed=7)
    job = open_job(gpu, H, N, L, s)
    try:
        for bad in (np.nan, -0.01, -np.inf):
            with pytest.raises(mash_b200.MashGpuError) as e:
                job.linkage_cut("average", bad)
            assert e.value.code == ERR_INVALID
        for method in (2, -1):
            with pytest.raises(mash_b200.MashGpuError) as e:
                job.linkage_cut(method, 0.1)
            assert e.value.code == ERR_INVALID
        labels = np.zeros(7, np.uint32)
        lo = np.zeros(6, np.uint32)
        u64 = [mash_b200._capi.C.c_uint64(0) for _ in range(3)]
        rc = gpu.lib.mashgpu_dist_linkage_cut(job.h, 0, 0.1, labels.ctypes.data_as(mash_b200._capi.u32p), lo.ctypes.data_as(mash_b200._capi.u32p),
                                              None, None, None, *[mash_b200._capi.C.byref(x) for x in u64])
        assert rc == ERR_INVALID
        rc = gpu.lib.mashgpu_dist_linkage_cut(job.h, 0, 0.1, None, None, None, None, None, *[mash_b200._capi.C.byref(x) for x in u64])
        assert rc == ERR_INVALID
        before = job.run(0, 7, outputs=("pass",))["pass"]
        job.linkage_cut("complete", 0.05)
        assert np.array_equal(job.run(0, 7, outputs=("pass",))["pass"], before)     # thresholds of the job unchanged
    finally:
        job.close()
    job = gpu.dist_open(H[:3], N[:3], L[:3], H[3:], N[3:], L[3:], sketch_size=s, k=21, kmer_space=4.0 ** 21)
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.linkage_cut("average", 0.1)
        assert e.value.code == ERR_INVALID
    finally:
        job.close()
    rows, n_eff = dense_rank_rows(H, N, s)
    d_rows = torch.from_numpy(rows.view(np.int32)).cuda()
    d_neff = torch.from_numpy(n_eff.view(np.int32)).cuda()
    d_len = torch.from_numpy(L.view(np.int64)).cuda()
    job = gpu.dist_open_encoded(d_rows.data_ptr(), d_neff.data_ptr(), d_len.data_ptr(), 7, 0, 7, sketch_size=s, k=21,
                                kmer_space=4.0 ** 21, keepalive=(d_rows, d_neff, d_len))
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.linkage_cut("average", 0.1)
        assert e.value.code == ERR_UNSUPPORTED
    finally:
        job.close()
    for n in (0, 1):
        job = gpu.dist_open(H[:n], N[:n], L[:n], sketch_size=s, k=21, kmer_space=4.0 ** 21)
        try:
            got = job.linkage_cut("average", 0.1, merges=True)
            assert got["labels"].tolist() == list(range(n)) and got["n_clusters"] == got["n_components"] == got["largest_component"] == n
            assert len(got["merges"]["height"]) == 0
        finally:
            job.close()
