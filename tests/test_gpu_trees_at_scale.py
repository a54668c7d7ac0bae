"""GPU tests of neighbor joining and average / complete linkage at collection sizes, on Mash distance grids full of ties: runs
of 1.0 between unrelated sketches, 0 between duplicates, Jaccard values quantised in steps of 1/s.  Under ties the trees depend
only on the tie-break orders mashgpu.h fixes, and these sizes reach code the model-sized tests do not: many column compactions on
one matrix, rescan lists far longer than the rescan grid, and the job's matrix fill in several query blocks.  The NJ scan's
grid-stride loop (m / 2 above 64 warps per SM) is reached by the 20 000-leaf additive tree with real-valued branch lengths.

The want is tools/tree_ref.cpp (tests/tree_ref.py), a full scan of the live lower triangle at every step, itself pinned to the
numpy models by tests/test_tree_ref.py: parent, merges and sizes equal, lengths and heights equal as uint64.  The engine runs on
its own stream, so every torch fill and copy is waited for before an engine call."""
import os
import time

import numpy as np
import pytest
import torch

import tree_ref
from fixtures import on_device, synth_sketches
from linkage_model import METHODS
from nj_model import TreeMatrix, random_tree, splits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return tree_ref.build(tmp_path_factory.mktemp("tree_ref"))


def collection(kind, n, s):
    """families: synth_sketches families with ragged lengths, plus empty sketches and exact duplicates (distance 0).
    unrelated: no two sketches share a hash, so every off-diagonal distance is 1.0."""
    rng = np.random.Generator(np.random.PCG64(n * 7 + s))
    if kind == "unrelated":
        H = np.sort(rng.integers(0, 2**62, (n, s), dtype=np.uint64), axis=1)
        return H, np.full(n, s, np.uint32), np.full(n, 5_000_000, np.uint64)
    H, N, L = synth_sketches(n, s, seed=n + s, n_families=max(6, n // 400), ragged=True)
    N[rng.choice(n, 5, replace=False)] = 0
    src = rng.choice(n, 40, replace=False)
    dst = rng.choice(n, 40, replace=False)
    H[dst], N[dst], L[dst] = H[src], N[src], L[src]
    return H, N, L


# (kind, n, s): n never a multiple of 32; s = 100 quantises far more coarsely than s = 1000.  The reference is O(n^3): 8191
# sketches take it about 30 s per tree on 8 host threads, so a grid past the NJ scan's grid-stride threshold (m / 2 > 64 * SMs,
# m >= 16 898 on a 132-SM H100) would take it about ten times that; the additive trees below reach that loop instead.
CASES = [("families", 2001, 1000), ("families", 2001, 100), ("unrelated", 2001, 200),
         ("families", 4097, 1000), ("families", 4097, 100),
         ("families", 8191, 1000), ("families", 8191, 100)]


@pytest.mark.parametrize("kind,n,s", CASES, ids=[f"{k}-{n}-s{s}" for k, n, s in CASES])
def test_trees_equal_the_reference(gpu, exe, kind, n, s):
    H, N, L = collection(kind, n, s)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=21, kmer_space=4.0 ** 21)
    try:
        D = job.run(0, n, outputs=("distance",))["distance"]
        low = D[np.tril_indices(n, -1)]
        if kind == "unrelated":
            assert (low == 1.0).all()
        else:
            assert (low == 0.0).any() and (low == 1.0).any()
        t0 = time.perf_counter()
        want = tree_ref.trees(exe, D, ("nj",) + METHODS)
        print(f"\n{kind} n={n} s={s}: {np.unique(low).size} distinct distances; C++ reference (nj, average, complete) took "
              f"{time.perf_counter() - t0:.1f} s on {len(os.sched_getaffinity(0))} threads")
        tree_ref.assert_nj_bits(job.neighbor_joining(), want["nj"])
        rescans = {}
        for method in METHODS:
            got = job.linkage(method)
            tree_ref.assert_linkage_bits(got, want[method])
            rescans[method] = got["rows_rescanned"]
    finally:
        job.close()
    for ld in (n, n + 33):
        tree_ref.assert_nj_bits(gpu.neighbor_joining_matrix(on_device(D, ld), n), want["nj"])
        for method in METHODS:
            M = on_device(D, ld)
            got = gpu.linkage_matrix(M, n, method=method)
            tree_ref.assert_linkage_bits(got, want[method])
            assert got["rows_rescanned"] == rescans[method]
            assert torch.isnan(M[:, n:]).all()


def test_multi_block_fill(gpu):
    """A self job large enough that its matrix fill runs in several query blocks (2^31 / n < n - 1).  The grid is produced
    independently, in other blocks, by run_dev into a torch tensor; average linkage of the two must agree merge for merge, which
    holds only if every block of the fill lands at its own rows."""
    n, s = 46_400, 12
    assert (1 << 31) // n < n - 1
    torch.cuda.synchronize()
    torch.cuda.empty_cache()                        # the engine allocates with cudaMalloc, outside torch's cache
    free = torch.cuda.mem_get_info()[0]
    if free < 40e9:
        pytest.skip(f"needs about 2 x {8 * n * n / 1e9:.1f} GB of device memory, {free / 1e9:.1f} GB free")
    H, N, L = synth_sketches(n, s, seed=46, n_families=64, ragged=True)
    M = torch.empty((n, n), dtype=torch.float64, device="cuda")
    torch.cuda.synchronize()
    try:
        job = gpu.dist_open(H, N, L, sketch_size=s, k=21, kmer_space=4.0 ** 21)
        try:
            job.set_triangle(True)
            step = 10_000
            for q0 in range(0, n, step):
                job.run_dev(q0, min(step, n - q0), d_distance=M.data_ptr() + 8 * q0 * n)
            for q in (1, 9_999, 10_000, 46_282, 46_283, n - 1):
                # run() returns after the engine's stream has drained, run_dev's kernels included; only then is M read
                want_row = job.run(q, 1, outputs=("distance",))["distance"][0, :q]
                assert np.array_equal(M[q, :q].cpu().numpy(), want_row), q
            want = job.linkage("average")
        finally:
            job.close()
        got = gpu.linkage_matrix(M, n, method="average")
        tree_ref.assert_linkage_bits(got, want)
        assert got["rows_rescanned"] == want["rows_rescanned"]
    finally:
        del M
        torch.cuda.empty_cache()                    # 17 GB back to the device, not kept in torch's cache


@pytest.mark.parametrize("n", [2000, 20000])
def test_additive_tree_with_real_lengths(gpu, exe, n):
    """Branch lengths uniform in [0.01, 1]: rounding is everywhere, but NJ of an additive matrix must still return the true
    topology, and every length to within the drift of the definition's updated row sums, which the last joins divide by only
    2 (m - 2).  On these trees the C++ reference's own largest errors are 8.6e-12 (2000 leaves) and 2.4e-9 (20 000 leaves,
    row sums up to 4.5e6), and the device's are the same to the bit; the bounds leave a factor of about 4 over them.  A wrong
    pair or update is off by far more: no branch is shorter than 0.01.  20 000 leaves run the NJ scan's grid-stride loop for
    the first 3 000 joins on a 132-SM H100; at 2000 the tree also equals the reference bit for bit."""
    rng = np.random.Generator(np.random.PCG64(n + 1))
    parent, length = random_tree(n, "random", rng)
    length = rng.uniform(0.01, 1.0, len(length))
    length[-1] = 0.0
    tm = TreeMatrix(parent, length, n)
    M = torch.empty((n, n), dtype=torch.float64, device="cuda")
    for i0 in range(0, n, 1024):
        rows = np.stack([tm.row(a) for a in range(i0, min(n, i0 + 1024))])
        M[i0:i0 + len(rows)] = torch.from_numpy(rows).cuda()
    torch.cuda.synchronize()
    if n <= 2000:
        want_bits = tree_ref.run(exe, M.cpu().numpy(), "nj")
    got = gpu.neighbor_joining_matrix(M, n)
    if n <= 2000:
        tree_ref.assert_nj_bits(got, want_bits)
    have, want = splits(got["parent"], got["length"], n), splits(parent, length, n)
    assert have.keys() == want.keys()
    err = max(abs(have[k] - want[k]) for k in want)
    tol = {2000: 4e-11, 20000: 1e-8}[n]
    print(f"\nadditive tree n={n}: largest length error {err:.3g}, bound {tol:.3g}")
    assert err <= tol
