"""GPU tests of dist at the sizes where its fixed-size device queues fill up (mash_b200/csrc/dist.cu, DESIGN.md 3.2b-3.2d):
  * the pair list of dist_probe_kernel -> dist_pair_kernel, max(2^20, pairs / 16) entries: a (query, tile) combination whose
    reservation does not fit is merged as a whole tile, and only the slots written by the run are merged from the list;
  * the p-value queue of dist_emit -> dist_fix_kernel, max(2^20, pairs / 16) entries: beyond it the epilogue evaluates in place;
  * mashgpu_dist_run's output chunks of 2^27 pairs.
The sketch sets are built so that the number of related pairs is known: sketch g is in class g % m and holds the class's two
core hashes (the smallest hashes of every row), so each query has exactly 32 / m relatives in every 32-reference tile.  Within a
tile only the core hashes are held by several references (at most 3 exact confirmations per combination, DESIGN.md 3.2b); the
rest of a row is drawn from the family of its tile lane with partial overlap, so merges are not trivial.  Every case asserts
that its queue really overflowed.  The file takes about 40 s on an H100 80GB HBM3 (700 W power limit), 11-13 s of it in the
s' = 28152 case."""
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import msh_reader
from fixtures import fmt_g
from test_gpu_dist import check_against_oracle

pytestmark = pytest.mark.gpu

MASH = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mash_b200", "host", "mash")

K = 21
KS = 4.0 ** K
KEYS = ("numer", "denom", "distance", "pvalue", "pass")
PAD = np.uint64(0xFFFFFFFFFFFFFFFF)
CHUNK_PAIRS = 1 << 27           # pairs per device launch of mashgpu_dist_run


def queue_capacity(pairs):
    """Entries of the pair list and of the p-value queue for a run of `pairs` pairs."""
    return max(1 << 20, pairs // 16)


def class_sketches(n, s, m, seed, extra=20):
    """Self set of n sketches, rows of s + extra hashes (lists longer than the sketch size), ragged and empty rows mixed in."""
    rng = np.random.Generator(np.random.PCG64(seed))
    hi = 2 ** 64 * s // 5_000_000
    lo = 1 << 44                                    # core hashes lie below, everything else above
    cores = np.unique(rng.integers(1, 1 << 40, 4 * m, dtype=np.uint64))[:2 * m].reshape(m, 2)
    assert cores.size == 2 * m
    fams = [np.unique(rng.integers(lo, hi, 2 * s, dtype=np.uint64)) for _ in range(32)]
    W = s + extra
    H = np.full((n, W), PAD, np.uint64)
    N = np.zeros(n, np.uint32)
    for g in range(n):
        base = fams[g % 32]
        keep = rng.random(base.size) < rng.choice([1.0, 0.9, 0.6, 0.3])
        v = np.unique(np.concatenate([cores[g % m], np.where(keep, base, rng.integers(lo, hi, base.size, dtype=np.uint64))]))[:W]
        if g % 89 == 7:
            v = v[:0]                                       # empty row: related to nothing
        elif g % 7 == 3:
            v = v[:int(rng.integers(1, s))]                 # ragged row: still holds a core hash
        H[g, :v.size] = v
        N[g] = v.size
    L = rng.integers(4_000_000, 6_000_000, n).astype(np.uint64)
    return H, N, L


def related(N, m, q0, q1, triangle=False):
    """Pairs of rows [q0, q1) x all that share a hash, from the construction: same class, both rows non-empty."""
    q = np.arange(q0, q1)[:, None]
    r = np.arange(N.size)[None, :]
    rel = (q % m == r % m) & (N[q] > 0) & (N[r] > 0)
    return rel & (r < q) if triangle else rel


def check_rows(oracle, res, H, N, L, s, q0, **thresholds):
    """res (rows q0 ... of the self grid) against the oracle, in blocks of rows on all cores.  Returns the oracle's count of
    pairs with shared hashes."""
    nq = res["numer"].shape[0]
    step = 128
    starts = list(range(q0, q0 + nq, step))
    workers = max(1, min(16, os.cpu_count() or 1))
    shared = 0
    with ThreadPoolExecutor(workers) as ex:
        for w in range(0, len(starts), workers):
            futs = [(a, ex.submit(oracle.compare_all, H, N, L, H[a:a + step], N[a:a + step], L[a:a + step], s, K, KS, **thresholds))
                    for a in starts[w:w + workers]]
            for a, f in futs:
                want = f.result()
                b = a + want.shape[0]
                check_against_oracle({key: v[a - q0:b - q0] for key, v in res.items()}, want)
                shared += int((want["numer"] > 0).sum())
    return shared


def split_threshold(p):
    """A -v threshold near the median of the p-values p, far (relative 1e-6) from each of them: about half pass."""
    u = np.unique(p[p > 1e-300])                      # away from the denormals, whose last bits are not pinned
    i = u.size // 2
    while i + 1 < u.size and u[i + 1] <= u[i] * (1 + 1e-6):
        i += 1
    assert 0 < i + 1 < u.size
    return float(np.sqrt(u[i] * u[i + 1]))


class Job:
    """A dist job that keeps the capacity of its grow-only pair list and the pairs merged from it per run."""

    def __init__(self, gpu, H, N, L, s, prefilter=1, **thresholds):
        self.j = gpu.dist_open(H, N, L, sketch_size=s, k=K, kmer_space=KS, **thresholds)
        self.j.set_prefilter(prefilter)
        self.n = H.shape[0]
        self.pair_capacity = 0
        self.merged = 0

    def _before(self, q_count):
        self.pair_capacity = max(self.pair_capacity, queue_capacity(q_count * self.n))
        self._m0 = self.j.prefilter_stats()["pairs_from_lists"]

    def _after(self):
        self.merged = self.j.prefilter_stats()["pairs_from_lists"] - self._m0

    def run(self, q0, qc):
        self._before(qc)
        out = self.j.run(q0, qc)
        self._after()
        return out

    def run_list(self, q0, qc, capacity):
        self._before(qc)
        n_pass, lst = self.j.run_list(q0, qc, capacity)
        self._after()
        assert n_pass <= capacity and lst["index"].size == n_pass
        return lst

    def assert_list_overflowed(self, listed, pair_max):
        # more pairs to list than the list holds; with the fix the list is filled up to the first reservation that did not fit
        # (pair_max slots at most) and nothing beyond it is merged
        assert listed > self.pair_capacity, (listed, self.pair_capacity)
        assert self.pair_capacity - pair_max < self.merged <= self.pair_capacity, (self.merged, self.pair_capacity)

    def close(self):
        self.j.close()


def assert_list_equals_dense(lst, dense):
    flat = np.flatnonzero(dense["pass"].ravel())
    assert np.all(np.diff(lst["index"].astype(np.int64)) > 0)          # unique (sorted by pair index)
    assert np.array_equal(lst["index"], flat.astype(np.uint64))
    for key in ("numer", "denom", "distance", "pvalue"):
        assert np.array_equal(lst[key], dense[key].ravel()[flat]), key


def lower(q0, q1, n):
    return np.arange(n)[None, :] < np.arange(q0, q1)[:, None]


def assert_triangle(tri, full, q0):
    """tri: triangle run over rows q0 ... of a self grid; full: the full grid"""
    low = lower(q0, q0 + tri["numer"].shape[0], full["numer"].shape[1])
    for key in KEYS:
        assert np.array_equal(tri[key][low], full[key][q0:][low]), key
        assert not tri[key][~low].any(), key                        # above the diagonal: untouched (zero)


# m = 2 and MASHGPU_DIST_PAIR_MAX = 31: 16 candidates per tile, half of the grid is listed.  m = 8 with the default pair_max = 4:
# an eighth is listed.  The lower triangle of a self grid holds half as many related pairs; at m = 8 that is pairs / 16 over any
# range starting at row 0, exactly the list's capacity, so the triangle runs there cover rows [1536, 4608) (2^20 entries,
# 1.18 M related pairs).
@pytest.mark.parametrize("m,pair_max,n,tri_q0", [(2, 31, 2304, 0), (8, None, 4608, 1536)])
def test_pair_list_overflow(gpu, oracle, monkeypatch, m, pair_max, n, tri_q0):
    if pair_max is None:
        monkeypatch.delenv("MASHGPU_DIST_PAIR_MAX", raising=False)
        pair_max = 4
    else:
        monkeypatch.setenv("MASHGPU_DIST_PAIR_MAX", str(pair_max))
    s = 100
    assert 32 // m <= pair_max
    H, N, L = class_sketches(n, s, m, seed=100 + m)
    rel = related(N, m, 0, n)

    job = Job(gpu, H, N, L, s)
    try:
        full = job.run(0, n)
        job.assert_list_overflowed(int(rel.sum()), pair_max)
        assert check_rows(oracle, full, H, N, L, s, 0) == int(rel.sum())        # the related pairs are the construction's
        assert np.array_equal(full["numer"] > 0, rel)
        # the same job over a shifted query range: the list still holds the first run's entries, of queries outside this range
        q0 = n // 4
        part = job.run(q0, n - q0)
        job.assert_list_overflowed(int(rel[q0:].sum()), pair_max)
        for key in KEYS:
            assert np.array_equal(part[key], full[key][q0:]), key
    finally:
        job.close()
    rel_tri = int(related(N, m, tri_q0, n, triangle=True).sum())

    job = Job(gpu, H, N, L, s)
    try:
        job.j.set_triangle(True)
        tri = job.run(tri_q0, n - tri_q0)
        job.assert_list_overflowed(rel_tri, pair_max)
        assert_triangle(tri, full, tri_q0)
    finally:
        job.close()

    # -v alone (near the median p-value): every pair with shared hashes is queued for its p-value, more than the queue holds.
    # dist_kernel (the combinations that did not fit the list) runs before dist_pair_kernel on the stream and queues first, so at
    # least min(rel - queue capacity, related pairs from the list) of the list's pairs get their p-value, pass flag and pass-list
    # entry in place
    v = split_threshold(full["pvalue"][full["numer"] > 0])
    n_rel, fix_capacity = int(rel.sum()), queue_capacity(n * n)
    job = Job(gpu, H, N, L, s, max_pvalue=v)
    try:
        dense = job.run(0, n)
        job.assert_list_overflowed(n_rel, pair_max)
        assert n_rel - fix_capacity > job.merged // 5, (n_rel, fix_capacity, job.merged)
        check_rows(oracle, dense, H, N, L, s, 0, max_pvalue=v)
        assert 0.2 < dense["pass"][rel].mean() < 0.8
        lst = job.run_list(0, n, n_rel)
        job.assert_list_overflowed(n_rel, pair_max)
        assert_list_equals_dense(lst, dense)
    finally:
        job.close()

    # -d between the core-only pairs (distance 0.154) and closer relatives, with -v: dense, pass list, triangle pass list
    md = 0.15
    job = Job(gpu, H, N, L, s, max_distance=md, max_pvalue=v)
    try:
        dense = job.run(0, n)
        job.assert_list_overflowed(int(rel.sum()), pair_max)
        check_rows(oracle, dense, H, N, L, s, 0, max_distance=md, max_pvalue=v)
        assert 0 < dense["pass"].sum() < (dense["numer"] > 0).sum()
        lst = job.run_list(0, n, int(rel.sum()))           # only pairs with shared hashes can pass
        job.assert_list_overflowed(int(rel.sum()), pair_max)
        assert_list_equals_dense(lst, dense)
    finally:
        job.close()
    job = Job(gpu, H, N, L, s, max_distance=md, max_pvalue=v)
    try:
        job.j.set_triangle(True)
        lst = job.run_list(tri_q0, n - tri_q0, rel_tri)
        job.assert_list_overflowed(rel_tri, pair_max)
        low = lower(tri_q0, n, n)
        assert_list_equals_dense(lst, {key: np.where(low, val[tri_q0:], 0) for key, val in dense.items()})
    finally:
        job.close()


# One merge path per case, each with more than 2^20 pairs with shared hashes (more than 1/16 of the grid): the p-value queue
# overflows and the rest is evaluated in place.  The pair list's path is covered by the -v run of test_pair_list_overflow (2.6 M
# pairs with shared hashes against a queue of 2^20 or 1.33 M entries).
@pytest.mark.parametrize("path,s,prefilter", [("tiled", 100, 0), ("tiled_after_probe", 100, 1), ("warp_per_pair", 1035, -1),
                                              ("general", 28152, -1)])
def test_pvalue_queue_overflow(gpu, oracle, path, s, prefilter):
    n = 1100
    H, N, L = class_sketches(n, s, 1, seed=7 + s)
    rel = related(N, 1, 0, n)
    assert int(rel.sum()) > queue_capacity(n * n)
    small = [(0, 900), (900, 200)]                     # at most 2^20 pairs each: every p-value is deferred
    assert all(qc * n <= 1 << 20 for _, qc in small)

    job = Job(gpu, H, N, L, s, prefilter)
    try:
        full = job.run(0, n)
        assert job.j.prefilter_stats()["active"] == (prefilter == 1)
        assert np.array_equal(full["numer"] > 0, rel)                  # the queue overflowed
        parts = [job.run(q0, qc) for q0, qc in small]
    finally:
        job.close()
    for (q0, qc), part in zip(small, parts):
        for key in KEYS:
            assert np.array_equal(part[key], full[key][q0:q0 + qc]), key
    v = split_threshold(full["pvalue"][rel])
    job = Job(gpu, H, N, L, s, prefilter, max_pvalue=v)
    try:
        res = job.run(0, n)
        parts = [job.run(q0, qc) for q0, qc in small]
        lst = job.run_list(0, n, int(rel.sum()))
    finally:
        job.close()
    for key in ("numer", "denom", "distance", "pvalue"):
        assert np.array_equal(res[key], full[key]), key
    assert np.array_equal(res["pass"], full["pvalue"] <= v)
    assert 0.2 < res["pass"][rel].mean() < 0.8
    for (q0, qc), part in zip(small, parts):
        for key in KEYS:
            assert np.array_equal(part[key], res[key][q0:q0 + qc]), key
    assert_list_equals_dense(lst, res)
    if path != "general":              # the oracle's sequential merge takes too long at s' = 28152: the small runs stand in
        check_rows(oracle, res, H, N, L, s, 0, max_pvalue=v)


def test_output_chunks(gpu, oracle):
    # a self grid of 12 000 x 12 000 is cut into query chunks of 2^27 / 12 000 = 11 184 rows; numer and denom only (the other
    # outputs are passed as NULL), compared with runs over sub-ranges that fit one chunk and, around the boundary, the oracle.
    # With the prefilter off every chunk is one dist launch (the engine's dist_kernel_launches counter): the full run must take
    # two, the sub-range runs one each.
    n, s, m = 12_000, 24, 3
    chunk = CHUNK_PAIRS // n
    assert n * n > CHUNK_PAIRS and chunk < n
    H, N, L = class_sketches(n, s, m, seed=12)
    out = ("numer", "denom")
    job = gpu.dist_open(H, N, L, sketch_size=s, k=K, kmer_space=KS)

    def launches():
        return gpu.stats(reset=True)["dist_kernel_launches"]

    try:
        job.set_prefilter(0)
        for tri in (False, True):
            job.set_triangle(tri)
            launches()
            full = job.run(0, n, outputs=out)
            assert launches() == 2
            assert set(full) == set(out)
            for q0, qc in ((0, 6000), (6000, 6000)):
                part = job.run(q0, qc, outputs=out)
                assert launches() == 1
                for key in out:
                    assert np.array_equal(part[key], full[key][q0:q0 + qc]), (tri, key)
                del part
            rows = slice(chunk - 4, chunk + 4)
            want = oracle.compare_all(H, N, L, H[rows], N[rows], L[rows], s, K, KS)
            low = np.arange(n)[None, :] < np.arange(chunk - 4, chunk + 4)[:, None]
            keep = low if tri else np.ones_like(low)
            for key in out:
                assert np.array_equal(full[key][rows][keep], want[key][keep]), (tri, key)
                assert not full[key][rows][~keep].any(), (tri, key)
            del full
    finally:
        job.close()


def test_cli_runs_several_blocks_on_one_job(gpu, tmp_path):
    # `mash dist` and `mash triangle` run blocks of at most 2^24 pairs on one dist job (mash.cpp: 2^24 / n query rows per block),
    # so the pair list and the p-value queue are reused from block to block.  4160 sketches (`mash sketch -i -s 100`) of 10
    # species in mixed order make two blocks of each.  `mash dist -d` takes the pass-list path (capacity 2^22), `mash triangle -d`
    # prints the edge list of dense triangle runs; both must print what the C ABI's dense grid with the prefilter off -- no lists
    # at all -- gives, formatted as the reference prints a double.  Relatives of one species share hashes with each other, so a
    # query with several of them in a tile is mostly merged as a whole tile (more than 3 shared-slot confirmations): this case
    # need not overflow the pair list; the synthetic grids above do.
    n, n_species, glen, s, md = 4160, 10, 8000, 100, 0.01
    rows = (1 << 24) // n
    assert 1 + rows < n                                  # two blocks for dist (from row 0) and for triangle (from row 1)
    rng = np.random.Generator(np.random.PCG64(4160))
    acgt = np.frombuffer(b"ACGT", np.uint8)
    bases = [acgt[rng.integers(0, 4, glen)] for _ in range(n_species)]
    species = rng.permutation(np.arange(n) % n_species)
    # a few close members per species (pairs within -d), the rest 2-10 % diverged (far outside it)
    rate = np.where(rng.random(n) < 0.03, rng.uniform(0, 0.002, n), rng.uniform(0.02, 0.1, n))
    with open(tmp_path / "mixed.fa", "wb") as f:
        for g in range(n):
            seq = bases[species[g]].copy()
            mut = rng.random(glen) < rate[g]
            seq[mut] = acgt[rng.integers(0, 4, int(mut.sum()))]
            f.write(b">r%d species %d\n" % (g, species[g]) + seq.tobytes() + b"\n")
    assert os.path.exists(MASH), "build the host shim first (__graft_entry__.build())"
    subprocess.run([MASH, "sketch", "-i", "-s", str(s), "-o", "mixed", "mixed.fa"], cwd=tmp_path, check=True, capture_output=True)
    d = msh_reader.read_msh(str(tmp_path / "mixed.msh"))
    refs = d["references"]
    assert len(refs) == n and d["sketchSize"] == s
    names = [r["name"] for r in refs]
    H = np.full((n, s), PAD, np.uint64)
    N = np.zeros(n, np.uint32)
    for g, r in enumerate(refs):
        H[g, :len(r["hashes64"])] = r["hashes64"]
        N[g] = len(r["hashes64"])
    L = np.array([r["length"] for r in refs], np.uint64)
    assert N.min() > 0

    job = gpu.dist_open(H, N, L, sketch_size=s, k=K, kmer_space=KS, max_distance=md)
    try:
        job.set_prefilter(0)
        grid = job.run(0, n)
    finally:
        job.close()

    def line(a, b, i, j):
        return f"{names[a]}\t{names[b]}\t{fmt_g(grid['distance'][i, j])}\t{fmt_g(grid['pvalue'][i, j])}\t{grid['numer'][i, j]}/{grid['denom'][i, j]}"

    qi, rj = np.nonzero(grid["pass"])                    # query-major
    want = [line(j, i, i, j) for i, j in zip(qi, rj)]    # dist prints reference, query
    assert n < len(want) < 3 * n                         # the diagonal and the close pairs: a small output
    got = subprocess.run([MASH, "dist", "-d", str(md), "mixed.msh", "mixed.msh"], cwd=tmp_path, check=True, capture_output=True,
                         text=True).stdout.splitlines()
    assert got == want
    want = [line(i, j, i, j) for i, j in zip(qi, rj) if j < i]      # triangle prints row i, column j < i
    got = subprocess.run([MASH, "triangle", "-d", str(md), "mixed.msh"], cwd=tmp_path, check=True, capture_output=True,
                         text=True).stdout.splitlines()
    assert got == want
