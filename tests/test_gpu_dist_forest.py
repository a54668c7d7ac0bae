"""GPU tests of the minimum spanning forest of dist (mashgpu_dist_spanning_forest): the graph of mashgpu_dist_components (pairs of
the lower triangle with pass == 1 and numer > 0), edges ordered by (distance, col, row).  The want is Kruskal's algorithm
(tests/forest_model.py) over the dense grid of DistJob.run on the same job, itself checked against the oracle: edges, order and
values must be equal bit for bit.  The two largest input sets are run once per session, with test_gpu_dist_components.py."""
import math
import os

import numpy as np
import pytest
import torch

from fixtures import dense_rank_rows, mutate, synth_genome, synth_sketches
from forest_model import forest_labels, kruskal
from test_gpu_dist_components import one_family_run, shuffled_path_run
from test_gpu_dist_prefilter import mixed_sketches

pytestmark = pytest.mark.gpu

KEYS = ("row", "col", "numer", "denom", "distance", "pvalue")


def max_rounds(n):
    return math.ceil(math.log2(n)) + 1 if n >= 2 else 0


def want_from_grid(grid, r0=0, hit=None):
    """the forest of a dense grid of a self job (r0 = 0) or of an encoded job whose references start at row r0"""
    n = grid["numer"].shape[0]
    if hit is None:
        hit = grid["pass"].astype(bool) & (grid["numer"] > 0)
    q, r = np.nonzero(hit)
    keep = r0 + r < q
    q, r = q[keep], r[keep]
    f = kruskal(n, q, r0 + r, grid["distance"][q, r])
    q, r = q[f], r[f]
    return {"row": q, "col": r0 + r, "numer": grid["numer"][q, r], "denom": grid["denom"][q, r], "distance": grid["distance"][q, r],
            "pvalue": grid["pvalue"][q, r]}


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


def check_job(job, r0=0):
    grid = job.run(0, job.n_qry)
    f = job.spanning_forest()
    assert_same(f, want_from_grid(grid, r0))
    assert f["row"].dtype == np.uint32 and f["distance"].dtype == np.float64
    assert f["rounds"] <= max_rounds(job.n_qry)
    return f


@pytest.mark.parametrize("s,k", [(1000, 21), (50, 11), (1, 21), (1034, 21), (1036, 21), (5000, 21)])
@pytest.mark.parametrize("prefilter", [0, 1])
def test_forest_equals_kruskal_over_the_grid(gpu, oracle, s, k, prefilter):
    H, N, L = synth_sketches(70, s, seed=3 + s, n_families=5, ragged=True)
    ks = 4.0 ** k
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=ks)
    try:
        job.set_prefilter(prefilter)
        f = check_job(job)
        job.set_triangle(True)                  # the job's own setting does not matter, and is left as it was
        assert_same(check_job(job), f)
        assert job.run(5, 1)["numer"][0, 5:].sum() == 0
    finally:
        job.close()
    assert len(f["row"]) > 0
    want = oracle.compare_all(H, N, L, H, N, L, s, k, ks)
    assert_same(f, want_from_grid(want, hit=want["numer"] > 0), exact=False, keys=KEYS[:5])      # the p-values: test_gpu_pvalue_precision


@pytest.mark.parametrize("pair_max", ["4", "0"])
def test_forest_through_the_pair_list(gpu, monkeypatch, pair_max):
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
        f = check_job(job)
        if pair_max != "0":
            assert job.prefilter_stats()["pairs_from_lists"] > 0
        assert len(f["row"]) > 0
    finally:
        job.close()


@pytest.mark.parametrize("md,mp", [(1.0, 1.0), (0.1, 1.0), (1.0, 1e-10), (0.02, 1e-30)])
@pytest.mark.parametrize("ragged", [False, True])
def test_forest_under_thresholds(gpu, md, mp, ragged):
    s, k = 500, 21
    H, N, L = synth_sketches(160, s, seed=7, n_families=6, ragged=ragged)
    if ragged:
        N[[3, 8, 40]] = 0                       # empty sketches: distance 0 to each other but no shared hash, never joined
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=md, max_pvalue=mp)
    try:
        f = check_job(job)
        if ragged:
            assert not np.isin([3, 8, 40], np.concatenate([f["row"], f["col"]])).any()
    finally:
        job.close()


def test_cut_at_t_has_the_components_at_t(gpu):
    s, k, n = 500, 21, 200
    H, N, L = synth_sketches(n, s, seed=17, n_families=8, ragged=True)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.3)
    try:
        f = check_job(job)
    finally:
        job.close()
    ts = [0.0, 0.01, 0.03, 0.08, 0.15, 0.3] + [float(x) for x in np.quantile(f["distance"], [0.25, 0.5, 0.75])]
    for t in ts:
        job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=t)
        try:
            labels, _ = job.components()
        finally:
            job.close()
        below = f["distance"] <= t
        assert np.array_equal(labels, forest_labels(n, f["row"][below], f["col"][below])), t


def test_duplicate_sketches_give_zero_weight_edges(gpu):
    s, k = 300, 21
    H, N, L = synth_sketches(40, s, seed=8, n_families=3, ragged=True)
    idx = np.random.Generator(np.random.PCG64(4)).integers(0, 40, 120)
    H, N, L = H[idx], N[idx], L[idx]
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        f = check_job(job)
        assert_same(job.spanning_forest(), f)
    finally:
        job.close()
    assert (f["distance"] == 0).sum() >= 40 and not np.signbit(f["distance"]).any()


def test_one_family_every_pair_an_edge(gpu):
    # every pair shares a hash: one tree, whose values are the grid's, and whose weights are those of every minimum spanning tree
    r = one_family_run(gpu)
    n, (first, second) = r["n"], r["forests"]
    for e, one, c in r["sample"]:
        assert one["numer"][0, c] == first["numer"][e] and one["denom"][0, c] == first["denom"][e]
        assert one["distance"][0, c].tobytes() == first["distance"][e].tobytes()
        assert one["pvalue"][0, c].tobytes() == first["pvalue"][e].tobytes()
    assert_same(first, second)
    assert len(first["row"]) == n - 1 and first["rounds"] <= max_rounds(n)
    assert (first["row"] > first["col"]).all()
    assert np.array_equal(forest_labels(n, first["row"], first["col"]), np.zeros(n))
    key = np.lexsort((first["row"], first["col"], first["distance"]))
    assert np.array_equal(key, np.arange(n - 1))
    assert np.allclose(r["grid_at_edges"], first["distance"], rtol=0, atol=0)
    assert np.array_equal(r["prim_weights"], first["distance"])


def test_mutation_chain(gpu):
    n, s, k = 400, 1000, 21
    g = [synth_genome(11, 60_000)]
    for i in range(1, n):
        g.append(mutate(g[-1], 0.004, 100 + i))
    perm = np.random.Generator(np.random.PCG64(12)).permutation(n)
    p = gpu.params(k=k, s=s)
    H, N, L = gpu.sketch([bytes(g[i]) for i in perm], p)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=p.kmer_space)
    try:
        f = check_job(job)
        assert_same(job.spanning_forest(), f)
    finally:
        job.close()
    # one tree, and mostly links between neighbours of the chain
    assert len(f["row"]) == n - 1
    assert (np.abs(perm[f["row"]] - perm[f["col"]]) == 1).mean() > 0.9         # sketch i is chain position perm[i]


def test_shuffled_path_over_several_query_blocks(gpu):
    # the forest is the chains' links, all at one distance, in (col, row) order; in shuffled order the trees of the union-find grow
    # deep over the rounds
    r = shuffled_path_run(gpu)
    n, perm, breaks = r["n"], r["perm"], r["breaks"]
    j = np.flatnonzero(~breaks[:-1])
    a, b = perm[j], perm[j + 1]
    row, col = np.maximum(a, b), np.minimum(a, b)
    o = np.lexsort((row, col))
    f = r["forests"][0]
    assert_same(r["forests"][1], f)
    assert np.array_equal(f["row"], row[o]) and np.array_equal(f["col"], col[o])
    assert (f["numer"] == 1).all() and (f["denom"] == 4).all() and len(np.unique(f["distance"])) == 1
    assert f["rounds"] <= max_rounds(n)


@pytest.mark.parametrize("shards", [2, 3])
def test_encoded_shards_merge_to_the_self_job(gpu, shards):
    from mash_b200.shard import merge_spanning_forests, shard_bounds
    s, k, n = 300, 21, 150
    H, N, L = synth_sketches(n, s, seed=12 + shards, n_families=7, ragged=True)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.3)
    try:
        want = check_job(job)
    finally:
        job.close()
    rows, n_eff = dense_rank_rows(H, N, s)
    d_rows = torch.from_numpy(rows.view(np.int32)).cuda(); d_neff = torch.from_numpy(n_eff.view(np.int32)).cuda()
    d_len = torch.from_numpy(L.view(np.int64)).cuda()
    parts = []
    for b, e in shard_bounds(n, shards):
        assert b > 0 or e < n
        job = gpu.dist_open_encoded(d_rows.data_ptr(), d_neff.data_ptr(), d_len.data_ptr(), n, b, e - b, sketch_size=s, k=k,
                                    kmer_space=4.0 ** k, max_distance=0.3, keepalive=(d_rows, d_neff, d_len))
        try:
            f = check_job(job, r0=b)
            out = {"row": torch.empty(n - 1, dtype=torch.int32, device="cuda"), "col": torch.empty(n - 1, dtype=torch.int32, device="cuda"),
                   "numer": torch.empty(n - 1, dtype=torch.int32, device="cuda"), "denom": torch.empty(n - 1, dtype=torch.int32, device="cuda"),
                   "distance": torch.empty(n - 1, dtype=torch.float64, device="cuda"), "pvalue": torch.empty(n - 1, dtype=torch.float64, device="cuda")}
            m, rounds = job.spanning_forest_dev(*(out[k].data_ptr() for k in KEYS))
            assert m == len(f["row"]) and rounds == f["rounds"]
            dev = {k: v[:m].cpu().numpy() for k, v in out.items()}
            assert_same({k: (v.view(np.uint32) if v.dtype == np.int32 else v) for k, v in dev.items()}, f)
        finally:
            job.close()
        assert (f["col"] >= b).all() and (f["col"] < e).all()
        parts.append({k: torch.from_numpy(v.astype(np.int64) if v.dtype == np.uint32 else v).cuda() for k, v in f.items() if k in KEYS})
    got = merge_spanning_forests(parts, n)
    assert got["row"].is_cuda
    assert_same({k: v.cpu().numpy() for k, v in got.items()}, want)


def test_refusals_and_tiny_sets(gpu):
    import ctypes as C
    import mash_b200
    s, k = 100, 21
    H, N, L = synth_sketches(9, s, seed=4, n_families=2)
    job = gpu.dist_open(H, N, L, H[:4], N[:4], L[:4], sketch_size=s, k=k, kmer_space=4.0 ** k)       # two sets
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.spanning_forest()
        assert e.value.code == 1
    finally:
        job.close()
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        n, r = C.c_uint64(0), C.c_uint64(0)
        u = np.zeros(8, np.uint32); d = np.zeros(8, np.float64)
        pu = u.ctypes.data_as(C.POINTER(C.c_uint32)); pd = d.ctypes.data_as(C.POINTER(C.c_double))
        assert gpu.lib.mashgpu_dist_spanning_forest(job.h, None, pu, pu, pu, pd, pd, C.byref(n), C.byref(r)) == 1
        assert gpu.lib.mashgpu_dist_spanning_forest(job.h, pu, pu, pu, pu, pd, pd, None, C.byref(r)) == 1
        assert gpu.lib.mashgpu_dist_spanning_forest(job.h, pu, pu, pu, pu, pd, pd, C.byref(n), None) == 1
        assert gpu.lib.mashgpu_dist_spanning_forest_dev(job.h, None, None, None, None, None, None, C.byref(n), C.byref(r), None) == 1
        check_job(job)
    finally:
        job.close()
    for m in (0, 1, 2):
        job = gpu.dist_open(H[:m], N[:m], L[:m], sketch_size=s, k=k, kmer_space=4.0 ** k)
        try:
            f = job.spanning_forest()
            if m < 2:
                assert len(f["row"]) == 0 and f["rounds"] == 0
            else:
                check_job(job)
        finally:
            job.close()
    H2 = np.stack([H[0], H[0]]); N2 = N[:2].copy(); N2[:] = N[0]
    job = gpu.dist_open(H2, N2, L[:2], sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        f = check_job(job)
        assert f["row"].tolist() == [1] and f["col"].tolist() == [0] and f["distance"].tolist() == [0.0] and f["rounds"] == 1
    finally:
        job.close()


def test_small_sets_against_the_oracle(gpu, oracle):
    s, k = 200, 15
    for seed, md in ((1, 1.0), (2, 0.05), (3, 0.2)):
        H, N, L = synth_sketches(25, s, seed=seed, n_families=4, ragged=True)
        job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=md)
        try:
            f = job.spanning_forest()
        finally:
            job.close()
        want = oracle.compare_all(H, N, L, H, N, L, s, k, 4.0 ** k)
        assert_same(f, want_from_grid(want, hit=(want["distance"] <= md) & (want["numer"] > 0)), exact=False, keys=KEYS[:5])


def _nccl_worker(rank, world, port, tmp):
    import torch.distributed as td
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    td.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import mash_b200
        from mash_b200.shard import shard_bounds, spanning_forest
        s, k, n = 300, 21, 200
        H, N, L = synth_sketches(n, s, seed=31, n_families=9, ragged=True)
        rows, n_eff = dense_rank_rows(H, N, s)
        dev = torch.device("cuda", rank)
        d_rows = torch.from_numpy(rows.view(np.int32)).to(dev); d_neff = torch.from_numpy(n_eff.view(np.int32)).to(dev)
        d_len = torch.from_numpy(L.view(np.int64)).to(dev)
        eng = mash_b200.Engine(device=rank)
        b, e = shard_bounds(n, world)[rank]
        job = eng.dist_open_encoded(d_rows.data_ptr(), d_neff.data_ptr(), d_len.data_ptr(), n, b, e - b, sketch_size=s, k=k,
                                    kmer_space=4.0 ** k, max_distance=0.3, keepalive=(d_rows, d_neff, d_len))
        f = job.spanning_forest()
        job.close()
        got = spanning_forest({k: torch.from_numpy(f[k].astype(np.int64) if f[k].dtype == np.uint32 else f[k]).to(dev) for k in KEYS})
        np.savez(os.path.join(tmp, f"f{rank}.npz"), **{k: v.cpu().numpy() for k, v in got.items()})
        eng.close()
        td.barrier()
    finally:
        td.destroy_process_group()


def test_multi_rank_nccl(gpu, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 or more GPUs")
    import torch.multiprocessing as mp
    from test_shard_gloo import _free_port
    world = min(torch.cuda.device_count(), 4)
    mp.spawn(_nccl_worker, args=(world, _free_port(), str(tmp_path)), nprocs=world, join=True)
    s, k, n = 300, 21, 200
    H, N, L = synth_sketches(n, s, seed=31, n_families=9, ragged=True)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.3)
    try:
        want = check_job(job)
    finally:
        job.close()
    for r in range(world):
        got = np.load(tmp_path / f"f{r}.npz")
        assert_same({k: got[k] for k in KEYS}, want)
