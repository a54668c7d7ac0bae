"""GPU tests of greedy dereplication (mashgpu_dist_representatives): representatives in index order on the graph of
mashgpu_dist_components, every member assigned to its nearest adjacent representative under (distance, min, max).  The want is the
numpy restatement of the device algorithm (tests/representatives_model.py) over the dense grid of DistJob.run on the same job, itself
checked against the sequential definition: rep, the rounds and the values must be equal bit for bit."""
import numpy as np
import pytest
import torch

from fixtures import mutate, synth_genome, synth_sketches
from representatives_model import edges_from_grid, from_grid, sequential
from test_gpu_dist_prefilter import mixed_sketches

pytestmark = pytest.mark.gpu

KEYS = ("rep", "numer", "denom", "distance", "pvalue")


def default_block(n):
    return min(2 ** 31 // max(n, 1), 32768)


def assert_same(got, want, exact=True, keys=KEYS):
    for k in keys:
        g, w = np.asarray(got[k]), np.asarray(want[k])
        assert g.shape == w.shape, k
        if g.dtype == np.float64 and exact:
            assert np.array_equal(g.view(np.uint64), w.astype(np.float64).view(np.uint64)), k
        elif g.dtype == np.float64:
            assert np.allclose(g, w, rtol=1e-12, atol=0), k
        else:
            assert np.array_equal(g, w.astype(g.dtype)), k


def check_job(job, block=None):
    """representatives() against the model over the job's own grid; block = the block size set on the job (None: the default)"""
    n = job.n_qry
    grid = job.run(0, n)
    got = job.representatives()
    want = from_grid(grid, min(block or default_block(n), 32768, max(n - 1, 1)))
    assert_same(got, want)
    assert got["n_reps"] == want["n_reps"] and got["rounds"] == want["rounds"]
    i, j, _ = edges_from_grid(grid)
    assert np.array_equal(got["rep"] == np.arange(n), sequential(n, i, j))
    return got


@pytest.mark.parametrize("s,k", [(1000, 21), (50, 11), (1, 21), (1034, 21), (1036, 21), (5000, 21)])
@pytest.mark.parametrize("prefilter", [0, 1])
def test_equals_the_model_over_the_grid(gpu, oracle, s, k, prefilter):
    H, N, L = synth_sketches(70, s, seed=3 + s, n_families=5, ragged=True)
    ks = 4.0 ** k
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=ks)
    try:
        job.set_prefilter(prefilter)
        got = check_job(job)
        job.set_triangle(True)                  # the job's own setting does not matter
        assert_same(check_job(job), got)
    finally:
        job.close()
    assert 1 < got["n_reps"] < 70
    want = oracle.compare_all(H, N, L, H, N, L, s, k, ks)
    want["pass"] = np.ones_like(want["numer"], dtype=np.uint8)
    assert_same(got, from_grid(want, default_block(70)), exact=False, keys=KEYS[:4])     # the p-values: test_gpu_pvalue_precision


@pytest.mark.parametrize("pair_max", ["4", "0"])
def test_through_the_pair_list(gpu, monkeypatch, pair_max):
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
        got = check_job(job)
        if pair_max != "0":
            assert job.prefilter_stats()["pairs_from_lists"] > 0
    finally:
        job.close()
    assert got["n_reps"] < n


@pytest.mark.parametrize("md,mp", [(1.0, 1.0), (0.1, 1.0), (1.0, 1e-10), (0.02, 1e-30)])
@pytest.mark.parametrize("ragged", [False, True])
def test_under_thresholds(gpu, md, mp, ragged):
    s, k = 500, 21
    H, N, L = synth_sketches(160, s, seed=7, n_families=6, ragged=ragged)
    if ragged:
        N[[3, 8, 40]] = 0                       # empty sketches: no shared hash, so each is its own representative
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=md, max_pvalue=mp)
    try:
        got = check_job(job)
    finally:
        job.close()
    if ragged:
        assert (got["rep"][[3, 8, 40]] == [3, 8, 40]).all()
        assert not np.isin([3, 8, 40], np.delete(got["rep"], [3, 8, 40])).any()


def test_duplicate_sketches(gpu):
    s, k = 300, 21
    H, N, L = synth_sketches(40, s, seed=8, n_families=3, ragged=True)
    idx = np.random.Generator(np.random.PCG64(4)).integers(0, 40, 120)
    H, N, L = H[idx], N[idx], L[idx]
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        got = check_job(job)
    finally:
        job.close()
    # copies of one sketch share a representative; the copies of a representative are its members at distance 0
    for v in np.unique(idx[N > 0]):
        copies = np.flatnonzero(idx == v)
        assert len(np.unique(got["rep"][copies])) == 1
        if got["rep"][copies[0]] == copies[0]:
            assert (got["distance"][copies[1:]] == 0).all() and not np.signbit(got["distance"][copies]).any()
    assert (got["distance"][got["rep"] != np.arange(120)] == 0).sum() >= 10


def test_block_sizes_give_one_result(gpu):
    s, k, n = 400, 21, 300
    H, N, L = synth_sketches(n, s, seed=21, n_families=9, ragged=True)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.2)
    try:
        results = []
        for block in (1, 7, 64, 0):
            job.set_representative_block(block)
            results.append(check_job(job, block or None))
        for r in results[1:]:
            assert_same(r, results[0])
        job.set_representative_block(7)
        out = {kk: torch.zeros(n, dtype=torch.int32 if kk in ("rep", "numer", "denom") else torch.float64, device="cuda") for kk in KEYS}
        reps, rounds = job.representatives_dev(*(out[kk].data_ptr() for kk in KEYS))
        dev = {kk: (v.cpu().numpy().view(np.uint32) if v.dtype == torch.int32 else v.cpu().numpy()) for kk, v in out.items()}
        assert_same(dev, results[1])
        assert reps == results[1]["n_reps"] and rounds == results[1]["rounds"]
    finally:
        job.close()


def one_family(n=20_000, s=64, k=21):
    """every member keeps the family's smallest s/2 hashes, so every pair shares a hash"""
    rng = np.random.Generator(np.random.PCG64(5))
    base = np.unique(rng.integers(0, 2 ** 60, 4 * s, dtype=np.uint64))
    H = np.empty((n, s), np.uint64)
    for i in range(n):
        H[i] = np.sort(np.concatenate([base[:s // 2], rng.choice(base[s // 2:], s // 2, replace=False)]))
    return H, np.full(n, s, np.uint32), np.full(n, 5_000_000, np.uint64)


def test_one_family_one_representative(gpu):
    n, s, k = 20_000, 64, 21
    H, N, L = one_family(n, s, k)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        got = job.representatives()
        assert got["n_reps"] == 1 and (got["rep"] == 0).all() and got["rounds"] == 0
        assert_same(job.representatives(), got)
        for m in np.random.Generator(np.random.PCG64(6)).choice(np.arange(1, n), 50, replace=False):
            row = job.run(int(m), 1)
            for kk in ("numer", "denom", "distance", "pvalue"):
                assert row[kk][0, 0].tobytes() == got[kk][m].tobytes(), kk
    finally:
        job.close()


def test_mutation_chain_in_order(gpu):
    # chain position i is sketch i: each sketch is near the ones just before it, a long dependency chain for the rounds
    n, s, k = 400, 1000, 21
    g = [synth_genome(11, 60_000)]
    for i in range(1, n):
        g.append(mutate(g[-1], 0.004, 100 + i))
    p = gpu.params(k=k, s=s)
    H, N, L = gpu.sketch([bytes(x) for x in g], p)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=p.kmer_space, max_distance=0.02)
    try:
        got = check_job(job)
        job.set_representative_block(64)
        check_job(job, 64)
    finally:
        job.close()
    assert got["rounds"] > 10 and 1 < got["n_reps"] < n


def shuffled_path(n=50_000, s=4, k=21):
    """sketch perm[p] is chain position p; adjacent positions share exactly one hash among the first s of their union, other pairs none"""
    rng = np.random.Generator(np.random.PCG64(77))
    breaks = np.zeros(n, bool)
    breaks[rng.choice(n - 1, 25, replace=False)] = True
    links = np.arange(1, 2 * n + 2, dtype=np.uint64)
    left = np.empty(n, np.uint64); right = np.empty(n, np.uint64)
    nxt = 0
    for j in range(n):
        if j == 0 or breaks[j - 1]:
            left[j] = links[nxt]; nxt += 1
        else:
            left[j] = right[j - 1]
        right[j] = links[nxt]; nxt += 1
    fill = np.unique(rng.integers(2 ** 40, 2 ** 62, 3 * n, dtype=np.uint64))[:2 * n]
    rng.shuffle(fill)
    perm = rng.permutation(n)
    H = np.empty((n, s), np.uint64)
    H[perm] = np.sort(np.stack([left, right, fill[:n], fill[n:]], 1), axis=1)
    return H, np.full(n, s, np.uint32), np.full(n, 5_000_000, np.uint64), perm, breaks


def test_shuffled_path_over_several_blocks(gpu):
    from representatives_model import assign, device
    n, s, k = 50_000, 4, 21
    H, N, L, perm, breaks = shuffled_path(n, s, k)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        assert default_block(n) < n - 1                     # more than one pass-1 block
        got = job.representatives()
        assert_same(job.representatives(), got)
        one = job.run(int(max(perm[0], perm[1])), 1)
    finally:
        job.close()
    p = np.flatnonzero(~breaks[:-1])
    a, b = perm[p], perm[p + 1]
    i, j = np.maximum(a, b), np.minimum(a, b)
    d = np.full(i.size, one["distance"][0, min(perm[0], perm[1])])
    is_rep, rounds = device(n, i, j, default_block(n))
    assert np.array_equal(is_rep, sequential(n, i, j))
    rep, _ = assign(n, is_rep, i, j, d)
    assert np.array_equal(got["rep"], rep) and got["rounds"] == sum(rounds) and got["n_reps"] == is_rep.sum()
    member = ~is_rep
    assert (got["numer"][member] == 1).all() and (got["denom"][member] == 4).all()
    assert (got["distance"][member] == d[0]).all() and (got["numer"][is_rep] == 0).all()


def test_refusals_and_tiny_sets(gpu):
    import ctypes as C
    import mash_b200
    from fixtures import dense_rank_rows
    s, k = 100, 21
    H, N, L = synth_sketches(9, s, seed=4, n_families=2)
    job = gpu.dist_open(H, N, L, H[:4], N[:4], L[:4], sketch_size=s, k=k, kmer_space=4.0 ** k)       # two sets
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.representatives()
        assert e.value.code == 1
    finally:
        job.close()
    rows, n_eff = dense_rank_rows(H, N, s)
    d_rows = torch.from_numpy(rows.view(np.int32)).cuda(); d_neff = torch.from_numpy(n_eff.view(np.int32)).cuda()
    d_len = torch.from_numpy(L.view(np.int64)).cuda()
    job = gpu.dist_open_encoded(d_rows.data_ptr(), d_neff.data_ptr(), d_len.data_ptr(), 9, 0, 9, sketch_size=s, k=k, kmer_space=4.0 ** k,
                                keepalive=(d_rows, d_neff, d_len))
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.representatives()
        assert e.value.code == 3
    finally:
        job.close()
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        n, r = C.c_uint64(0), C.c_uint64(0)
        u = np.zeros(9, np.uint32); d = np.zeros(9, np.float64)
        pu = u.ctypes.data_as(C.POINTER(C.c_uint32)); pd = d.ctypes.data_as(C.POINTER(C.c_double))
        assert gpu.lib.mashgpu_dist_representatives(job.h, None, pu, pu, pd, pd, C.byref(n), C.byref(r)) == 1
        assert gpu.lib.mashgpu_dist_representatives(job.h, pu, pu, pu, pd, pd, None, C.byref(r)) == 1
        assert gpu.lib.mashgpu_dist_representatives(job.h, pu, pu, pu, pd, pd, C.byref(n), None) == 1
        assert gpu.lib.mashgpu_dist_representatives_dev(job.h, None, None, None, None, None, C.byref(n), C.byref(r), None) == 1
        check_job(job)
    finally:
        job.close()
    for m in (0, 1, 2):
        job = gpu.dist_open(H[:m], N[:m], L[:m], sketch_size=s, k=k, kmer_space=4.0 ** k)
        try:
            got = job.representatives()
            if m < 2:
                assert got["rep"].tolist() == list(range(m)) and got["rounds"] == 0 and got["n_reps"] == m
            else:
                check_job(job)
        finally:
            job.close()
    H2 = np.stack([H[0], H[0]]); N2 = N[:2].copy(); N2[:] = N[0]
    job = gpu.dist_open(H2, N2, L[:2], sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        got = check_job(job)
        assert got["rep"].tolist() == [0, 0] and got["distance"].tolist() == [0.0, 0.0] and got["n_reps"] == 1 and got["rounds"] == 0
    finally:
        job.close()
