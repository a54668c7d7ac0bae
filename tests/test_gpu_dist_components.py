"""GPU tests of the connected components of dist (mashgpu_dist_components): the edges are the pairs of the lower triangle with
pass == 1 and numer > 0, and every sketch is labelled with the smallest index of its component.  The want is built from the dense
grid of DistJob.run on the same job (itself checked against the oracle) and scipy's connected components; labels and edge counts
must be equal.  The two largest input sets are shared with test_gpu_dist_forest.py: each is sketched and run once per session
(one_family_run, shuffled_path_run), and each module checks its own results of that run."""
import functools
import os

import numpy as np
import pytest
import torch

from fixtures import dense_rank_rows, mutate, synth_genome, synth_sketches
from test_gpu_dist_prefilter import mixed_sketches
from test_shard_components_gloo import min_labels

pytestmark = pytest.mark.gpu


def want_from_grid(grid, r0=0):
    """(labels, n_edges) from a dense grid of a self job (r0 = 0) or an encoded job whose references start at row r0"""
    n, n_ref = grid["numer"].shape
    hit = grid["pass"].astype(bool) & (grid["numer"] > 0)
    q, r = np.nonzero(hit)
    keep = r0 + r < q
    edges = np.stack([q[keep], r0 + r[keep]], 1)
    return min_labels(n, edges), len(edges)


def check_job(job, r0=0):
    grid = job.run(0, job.n_qry)
    labels, n_edges = job.components()
    want, want_edges = want_from_grid(grid, r0)
    assert labels.dtype == np.uint32 and labels.shape == (job.n_qry,)
    assert np.array_equal(labels, want)
    assert n_edges == want_edges
    return labels, n_edges


@pytest.mark.parametrize("s,k", [(1000, 21), (50, 11), (1, 21), (1034, 21), (1036, 21), (5000, 21)])
@pytest.mark.parametrize("prefilter", [0, 1])
def test_components_equal_the_grid_and_the_oracle(gpu, oracle, s, k, prefilter):
    H, N, L = synth_sketches(70, s, seed=3 + s, n_families=5, ragged=True)
    ks = 4.0 ** k
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=ks)
    try:
        job.set_prefilter(prefilter)
        labels, _ = check_job(job)
        job.set_triangle(True)                  # the job's own setting does not matter, and is left as it was
        assert np.array_equal(check_job(job)[0], labels)
        assert job.run(5, 1)["numer"][0, 5:].sum() == 0
    finally:
        job.close()
    want = oracle.compare_all(H, N, L, H, N, L, s, k, ks)
    assert np.array_equal(labels, want_from_grid(want)[0])


@pytest.mark.parametrize("pair_max", ["4", "0"])
def test_components_through_the_pair_list(gpu, monkeypatch, pair_max):
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
        labels, n_edges = check_job(job)
        if pair_max != "0":
            assert job.prefilter_stats()["pairs_from_lists"] > 0
        assert n_edges > 0 and 4 <= len(np.unique(labels[pos])) < 44
    finally:
        job.close()


@pytest.mark.parametrize("md,mp", [(1.0, 1.0), (0.1, 1.0), (1.0, 1e-10), (0.02, 1e-30)])
@pytest.mark.parametrize("ragged", [False, True])
def test_components_under_thresholds(gpu, md, mp, ragged):
    s, k = 500, 21
    H, N, L = synth_sketches(160, s, seed=7, n_families=6, ragged=ragged)
    if ragged:
        N[[3, 8, 40]] = 0                       # empty sketches: distance 0 to each other but no shared hash, never joined
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=md, max_pvalue=mp)
    try:
        labels, _ = check_job(job)
        if ragged:
            assert labels[3] == 3 and labels[8] == 8 and labels[40] == 40
    finally:
        job.close()


def test_small_sets_against_the_oracle(gpu, oracle):
    s, k = 200, 15
    for seed, md in ((1, 1.0), (2, 0.05), (3, 0.2)):
        H, N, L = synth_sketches(25, s, seed=seed, n_families=4, ragged=True)
        job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=md)
        try:
            labels, n_edges = job.components()
        finally:
            job.close()
        want = oracle.compare_all(H, N, L, H, N, L, s, k, 4.0 ** k)
        hit = (want["distance"] <= md) & (want["numer"] > 0)
        q, r = np.nonzero(np.tril(hit, -1))
        assert np.array_equal(labels, min_labels(25, np.stack([q, r], 1))) and n_edges == q.size


@functools.cache
def one_family_run(gpu):
    """20 000 sketches in which every member keeps the family's smallest s/2 hashes, so every pair shares a hash: components()
    and spanning_forest() twice each, the grid's distances at the forest's edges and at 50 of them run() one row at a time, and
    the sorted weights of Prim's algorithm over the dense distances on the device (every minimum spanning tree has the same)"""
    n, s, k = 20_000, 64, 21
    rng = np.random.Generator(np.random.PCG64(5))
    base = np.unique(rng.integers(0, 2 ** 60, 4 * s, dtype=np.uint64))
    H = np.empty((n, s), np.uint64)
    for i in range(n):
        H[i] = np.sort(np.concatenate([base[:s // 2], rng.choice(base[s // 2:], s // 2, replace=False)]))
    N = np.full(n, s, np.uint32)
    L = np.full(n, 5_000_000, np.uint64)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        out = {"n": n, "components": [job.components(), job.components()], "forests": [job.spanning_forest(), job.spanning_forest()]}
        f = out["forests"][0]
        d = torch.empty((n, n), dtype=torch.float64, device="cuda")
        job.run_dev(0, n, d_distance=d.data_ptr())
        torch.cuda.synchronize()
        sample = np.random.Generator(np.random.PCG64(6)).choice(n - 1, 50, replace=False)
        out["sample"] = [(e, job.run(int(f["row"][e]), 1), int(f["col"][e])) for e in sample]
    finally:
        job.close()
    out["grid_at_edges"] = d.cpu().numpy()[f["row"], f["col"]]
    inf = torch.tensor(float("inf"), dtype=torch.float64, device="cuda")
    key_d = d[0].clone()
    in_tree = torch.zeros(n, dtype=torch.bool, device="cuda")
    in_tree[0] = True
    weights = torch.empty(n - 1, dtype=torch.float64, device="cuda")
    for t in range(n - 1):
        masked = torch.where(in_tree, inf, key_d)
        v = torch.argmin(masked)
        weights[t] = masked[v]
        in_tree[v] = True
        key_d = torch.minimum(key_d, d[v])
    del d
    out["prim_weights"] = np.sort(weights.cpu().numpy())
    return out


def test_one_family_every_pair_an_edge(gpu):
    # every pair shares a hash: n (n - 1) / 2 edges, one component
    r = one_family_run(gpu)
    n, (first, second) = r["n"], r["components"]
    assert first[1] == second[1] == n * (n - 1) // 2
    assert not first[0].any() and np.array_equal(first[0], second[0])


def test_mutation_chain_is_a_path(gpu):
    # g_i = mutate(g_{i-1}) in shuffled order: at a cut-off between one step's and two steps' distance the edges form a path
    n, s, k = 400, 1000, 21
    g = [synth_genome(11, 60_000)]
    for i in range(1, n):
        g.append(mutate(g[-1], 0.004, 100 + i))
    perm = np.random.Generator(np.random.PCG64(12)).permutation(n)
    p = gpu.params(k=k, s=s)
    H, N, L = gpu.sketch([bytes(g[i]) for i in perm], p)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=p.kmer_space, max_distance=0.006)
    try:
        labels, n_edges = check_job(job)
        assert np.array_equal(job.components()[0], labels)
    finally:
        job.close()
    # mostly one step apart: long runs of the chain end up in one component
    assert n // 2 <= n_edges < 2 * n and len(np.unique(labels)) < n // 4


@functools.cache
def shuffled_path_run(gpu):
    """50 000 sketches: the host runs the queries in blocks of 2^31 / 50 000 = 42 949, so the union-find carries over from one block's
    runs to the next and unions join rows of both.  Sketch j of a chain holds the links {L_j, R_j} (small hashes, R_j == L_{j+1}
    except at a break) and two fresh large hashes: adjacent sketches share exactly one hash among the first s = 4 of their union,
    every other pair shares none.  In shuffled order the trees grow deep, which is what the read-only flatten has to walk.
    components() and spanning_forest() twice each, with the chains: chain position j is sketch perm[j], no link after a break."""
    n, s, k = 50_000, 4, 21
    rng = np.random.Generator(np.random.PCG64(77))
    breaks = np.zeros(n, bool)
    breaks[rng.choice(n - 1, 25, replace=False)] = True         # no link between chain positions j and j + 1
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
    perm = rng.permutation(n)                                   # chain position j is sketch perm[j]
    H = np.empty((n, s), np.uint64)
    H[perm] = np.sort(np.stack([left, right, fill[:n], fill[n:]], 1), axis=1)
    N = np.full(n, s, np.uint32)
    L = np.full(n, 5_000_000, np.uint64)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        assert (2 ** 31) // job.n_ref < n - 1                   # more than one block of queries
        return {"n": n, "perm": perm, "breaks": breaks, "components": [job.components(), job.components()],
                "forests": [job.spanning_forest(), job.spanning_forest()]}
    finally:
        job.close()


def test_shuffled_path_over_several_query_blocks(gpu):
    r = shuffled_path_run(gpu)
    n, perm, breaks = r["n"], r["perm"], r["breaks"]
    j = np.flatnonzero(~breaks[:-1])
    want = min_labels(n, np.stack([perm[j], perm[j + 1]], 1))
    for labels, n_edges in r["components"]:
        assert n_edges == j.size and np.array_equal(labels, want)
    assert len(np.unique(want)) == 26


@pytest.mark.parametrize("shards", [2, 3])
def test_encoded_shards_merge_to_the_self_job(gpu, shards):
    from mash_b200.shard import merge_component_labels, shard_bounds
    s, k, n = 300, 21, 150
    H, N, L = synth_sketches(n, s, seed=12 + shards, n_families=7, ragged=True)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.3)
    try:
        want, want_edges = check_job(job)
    finally:
        job.close()
    rows, n_eff = dense_rank_rows(H, N, s)
    d_rows = torch.from_numpy(rows.view(np.int32)).cuda(); d_neff = torch.from_numpy(n_eff.view(np.int32)).cuda()
    d_len = torch.from_numpy(L.view(np.int64)).cuda()
    parts, edges = [], 0
    for b, e in shard_bounds(n, shards):
        assert b > 0 or e < n
        job = gpu.dist_open_encoded(d_rows.data_ptr(), d_neff.data_ptr(), d_len.data_ptr(), n, b, e - b, sketch_size=s, k=k,
                                    kmer_space=4.0 ** k, max_distance=0.3, keepalive=(d_rows, d_neff, d_len))
        try:
            labels, n_edges = check_job(job, r0=b)
            d_lab = torch.empty(n, dtype=torch.int32, device="cuda")
            assert job.components_dev(d_lab.data_ptr()) == n_edges
            assert np.array_equal(d_lab.cpu().numpy().view(np.uint32), labels)
        finally:
            job.close()
        parts.append(torch.from_numpy(labels.astype(np.int64)).cuda())
        edges += n_edges
    got = merge_component_labels(parts)
    assert got.is_cuda and np.array_equal(got.cpu().numpy(), want) and edges == want_edges


def test_refusals_and_tiny_sets(gpu):
    import mash_b200
    s, k = 100, 21
    H, N, L = synth_sketches(9, s, seed=4, n_families=2)
    job = gpu.dist_open(H, N, L, H[:4], N[:4], L[:4], sketch_size=s, k=k, kmer_space=4.0 ** k)       # two sets
    try:
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.components()
        assert e.value.code == 1
    finally:
        job.close()
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        import ctypes as C
        n = C.c_uint64(0)
        assert gpu.lib.mashgpu_dist_components(job.h, None, C.byref(n)) == 1
        lab = np.zeros(9, np.uint32)
        assert gpu.lib.mashgpu_dist_components(job.h, lab.ctypes.data_as(C.POINTER(C.c_uint32)), None) == 1
        assert gpu.lib.mashgpu_dist_components_dev(job.h, None, C.byref(n), None) == 1
        check_job(job)
    finally:
        job.close()
    for m in (0, 1, 2):
        job = gpu.dist_open(H[:m], N[:m], L[:m], sketch_size=s, k=k, kmer_space=4.0 ** k)
        try:
            labels, n_edges = job.components()
            if m < 2:
                assert np.array_equal(labels, np.arange(m)) and n_edges == 0
            else:
                check_job(job)
        finally:
            job.close()
    H2 = np.stack([H[0], H[0]]); N2 = N[:2].copy(); N2[:] = N[0]
    job = gpu.dist_open(H2, N2, L[:2], sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        assert np.array_equal(job.components()[0], [0, 0]) and job.components()[1] == 1
    finally:
        job.close()


def _nccl_worker(rank, world, port, tmp):
    import torch.distributed as td
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    td.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        import mash_b200
        from mash_b200.shard import merge_components, shard_bounds
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
        labels, _ = job.components()
        job.close()
        got = merge_components(torch.from_numpy(labels.astype(np.int64)).to(dev))
        np.save(os.path.join(tmp, f"cc{rank}.npy"), got.cpu().numpy())
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
        want, _ = check_job(job)
    finally:
        job.close()
    for r in range(world):
        assert np.array_equal(np.load(tmp_path / f"cc{r}.npy"), want), r
