"""GPU parity tests for hot path 2 (compareSketches / pValue), through the C ABI.
Bit-exact: numer (shared hashes), denom, pass.  Doubles: 1e-12 (relative for p-values, which span 300 decades: held down to
1e-305, i.e. the whole normal range of a double short of its last three decades; below that the oracle's and the device's
results must both be below 1e-305 -- the denormal behaviour of GSL / Boost is unpinned, SURVEY.md appendix C)."""
import numpy as np
import pytest

from fixtures import synth_sketches, fmt_g

pytestmark = pytest.mark.gpu

TOL = 1e-12


def check_against_oracle(res, want, max_distance=1.0):
    assert np.array_equal(res["pass"], want["pass"].astype(bool))
    filled = want["filled"].astype(bool)
    assert np.array_equal(res["numer"][filled], want["numer"][filled])
    assert np.array_equal(res["denom"][filled], want["denom"][filled])
    d_g, d_o = res["distance"][filled], want["distance"][filled]
    assert np.all(np.abs(d_g - d_o) <= TOL)
    p_g, p_o = res["pvalue"][filled], want["pvalue"][filled]
    big = p_o > 1e-305
    assert np.all(np.abs(p_g[big] - p_o[big]) <= TOL * p_o[big])
    assert np.all(p_g[~big] <= 1.0000001e-305)


def test_golden_dist_lines(gpu, oracle, golden):
    # BASELINE config 1: `mash dist genomes.msh reads.msh` -> test/ref/genomes.dist, plus the tutorial values
    p = gpu.params(k=21, s=1000)
    recs, uor = [], []
    for u, (_, rs) in enumerate(golden.genomes):
        for r in rs:
            recs.append(r[2]); uor.append(u)
    reads = golden.reads_round_robin()
    recs += reads; uor += [3] * len(reads)
    h, n, length = gpu.sketch(recs, p, unit_of_record=uor, n_units=4)
    length[3] = int(np.uint64(2.0 ** 64 * float(n[3]) / float(h[3, n[3] - 1])))      # -r: estimateSetSize
    res = gpu.dist(h[:3], n[:3], length[:3], h[3:], n[3:], length[3:], sketch_size=1000, k=21, kmer_space=p.kmer_space)
    for i, line in enumerate(golden.dist_lines):
        got = [fmt_g(res["distance"][0, i]), fmt_g(res["pvalue"][0, i]), f"{res['numer'][0, i]}/{res['denom'][0, i]}"]
        assert got == line[2:5]
    res = gpu.dist(h[:3], n[:3], length[:3], sketch_size=1000, k=21, kmer_space=p.kmer_space)   # genomes all-vs-all
    assert (fmt_g(res["distance"][1, 0]), fmt_g(res["pvalue"][1, 0]), res["numer"][1, 0], res["denom"][1, 0]) == ("0.0222766", "0", 456, 1000)
    assert (fmt_g(res["distance"][2, 0]), res["numer"][2, 0], res["denom"][2, 0]) == ("0", 1000, 1000)


@pytest.mark.parametrize("s,k", [(1000, 21), (400, 16), (50, 11), (1, 21), (1030, 32), (1036, 21), (5000, 21)])
def test_grid_matches_oracle(gpu, oracle, s, k):
    H, N, L = synth_sketches(70, s, seed=3 + s, n_families=3, ragged=True)
    Hq, Nq, Lq = synth_sketches(45, s, seed=99 + s, n_families=3, ragged=True)
    Hq[:10] = H[:10]; Nq[:10] = N[:10]          # some identical pairs
    ks = 4.0 ** k
    res = gpu.dist(H, N, L, Hq, Nq, Lq, sketch_size=s, k=k, kmer_space=ks)
    want = oracle.compare_all(H, N, L, Hq, Nq, Lq, s, k, ks)
    check_against_oracle(res, want)


def test_self_grid_and_row_ranges(gpu, oracle):
    H, N, L = synth_sketches(130, 1000, seed=5, n_families=5, ragged=True)
    ks = 4.0 ** 21
    want = oracle.compare_all(H, N, L, H, N, L, 1000, 21, ks)
    job = gpu.dist_open(H, N, L, sketch_size=1000, k=21, kmer_space=ks)
    try:
        full = job.run(0, 130)
        check_against_oracle(full, want)
        part = job.run(37, 50)                  # the reference's chunked `compare` jobs enumerate sub-ranges the same way
        for key in ("numer", "denom", "distance", "pvalue", "pass"):
            assert np.array_equal(part[key], full[key][37:87])
    finally:
        job.close()
    # symmetry + diagonal (size-independent properties)
    assert np.array_equal(full["numer"], full["numer"].T)
    full_rows = N == 1000
    assert np.all(np.diag(full["distance"])[N > 0] == 0)
    assert np.all(np.diag(full["numer"]) == np.minimum(N, 1000))


def test_thresholds(gpu, oracle):
    # -d / -v filters: pass flags identical; filtered-by-distance pairs are left "unset" by the reference
    H, N, L = synth_sketches(60, 500, seed=8, n_families=2)
    ks = 4.0 ** 21
    for md, mp in ((0.05, 1.0), (1.0, 1e-10), (0.2, 1e-3), (-1.0, -1.0)):
        res = gpu.dist(H, N, L, sketch_size=500, k=21, kmer_space=ks, max_distance=md, max_pvalue=mp)
        want = oracle.compare_all(H, N, L, H, N, L, 500, 21, ks, max_distance=md, max_pvalue=mp)
        check_against_oracle(res, want)


def test_sketch_size_smaller_than_lists(gpu, oracle):
    # query/ref sketched with different s: sketchSize = min (CommandDistance.cpp:313-315); lists longer than it
    H, N, L = synth_sketches(40, 1000, seed=21, n_families=2)
    ks = 4.0 ** 21
    res = gpu.dist(H, N, L, sketch_size=300, k=21, kmer_space=ks)
    want = oracle.compare_all(H, N, L, H, N, L, 300, 21, ks)
    check_against_oracle(res, want)


def test_empty_and_tiny_sets(gpu, oracle):
    ks = 4.0 ** 21
    H = np.full((3, 8), np.uint64(2**64 - 1)); N = np.array([0, 3, 8], np.uint32); L = np.array([1000, 2000, 3000], np.uint64)
    H[1, :3] = [5, 9, 100]
    H[2] = [1, 5, 7, 9, 11, 100, 200, 300]
    res = gpu.dist(H, N, L, sketch_size=8, k=21, kmer_space=ks)
    want = oracle.compare_all(H, N, L, H, N, L, 8, 21, ks)
    check_against_oracle(res, want)
    assert res["denom"][0, 0] == 0 and res["distance"][0, 0] == 0 and res["pvalue"][0, 0] == 1.0


def test_pvalue_device_vs_mpmath(gpu, golden):
    # the device binomial tail against the 50-digit fixtures, driven through dist with crafted sketches:
    # ref = {0..n-1}, qry shares exactly x of them -> numer = x, denom = n, r from the lengths
    cases = [c for c in golden.pvalue_cases if c["n"] <= 1030 and 1 <= c["x"] <= c["n"]]
    worst = 0.0
    for c in cases[::3]:
        n, x, r = c["n"], c["x"], float(c["r"])
        # lengths with pX = pY = p0: r = p0 / (2 - p0)  ->  p0 = 2r/(1+r);  L = K p0/(1-p0)
        k = 21; K = 4.0 ** k
        p0 = 2 * r / (1 + r)
        Lf = K * p0 / (1 - p0)
        if not (1 <= Lf < 2**62):
            continue
        Li = int(round(Lf))
        pX = 1. / (1. + K / Li)
        r_eff = pX * pX / (pX + pX - pX * pX)
        import mpmath as mp
        mp.mp.dps = 50
        truth = float(mp.betainc(x, n - x + 1, 0, mp.mpf(r_eff), regularized=True))
        ref = np.arange(0, 2 * n, 2, dtype=np.uint64)[None, :]            # even numbers
        q = ref.copy(); q[0, x:] += 1                                      # first x shared, the rest odd (distinct)
        q.sort(axis=1)
        res = gpu.dist(ref, [n], [Li], q, [n], [Li], sketch_size=n, k=k, kmer_space=K)
        if res["numer"][0, 0] != x or res["denom"][0, 0] != n:
            continue                                                       # merge stopped early: different x, skip
        got = res["pvalue"][0, 0]
        if truth > 1e-305:
            worst = max(worst, abs(got - truth) / truth)
            assert abs(got - truth) <= TOL * truth, (c, got, truth)
    assert worst < 1e-12


def test_full_size_symmetry_property(gpu, oracle):
    # BASELINE configs[2] size (100 000 sketches, s=1000): size-independent property instead of an oracle run --
    # rows of a random subset Q against everything must equal the columns of everything against Q (merge symmetry),
    # self pairs have numer == denom == s, distance 0, and every distance/p-value is in [0, 1].
    n, s = 100_000, 1000
    rng = np.random.Generator(np.random.PCG64(77))
    hi = np.uint64(2**64 * s // 5_000_000)
    base = np.sort(rng.integers(0, int(hi), (40, 2 * s), dtype=np.uint64), axis=1)
    H = np.empty((n, s), np.uint64)
    fam = rng.integers(0, 40, n)
    keep = rng.random((n, 1)) < 0.5
    for lo in range(0, n, 5000):
        sl = slice(lo, lo + 5000)
        fresh = rng.integers(0, int(hi), (5000, 2 * s), dtype=np.uint64)
        mask = rng.random((5000, 2 * s)) < rng.choice([1.0, 0.9, 0.5, 0.0], (5000, 1))
        v = np.sort(np.where(mask, base[fam[sl]], fresh), axis=1)
        dup = np.zeros_like(v, dtype=bool); dup[:, 1:] = v[:, 1:] <= v[:, :-1]
        v = v + np.cumsum(dup, axis=1, dtype=np.uint64)
        H[sl] = np.sort(v, axis=1)[:, :s]
    N = np.full(n, s, np.uint32); L = rng.integers(4_000_000, 6_000_000, n).astype(np.uint64)
    ks = 4.0 ** 21
    q = np.sort(rng.choice(n, 96, replace=False))
    job = gpu.dist_open(H, N, L, H[q], N[q], L[q], sketch_size=s, k=21, kmer_space=ks)
    rows = job.run(0, 96)                      # (96, n): query = Q[i], reference = all
    job.close()
    job = gpu.dist_open(H[q], N[q], L[q], H, N, L, sketch_size=s, k=21, kmer_space=ks)
    cols = job.run(0, n)                       # (n, 96): query = all, reference = Q[j]
    job.close()
    assert np.array_equal(rows["numer"], cols["numer"].T) and np.array_equal(rows["denom"], cols["denom"].T)
    assert np.array_equal(rows["distance"], cols["distance"].T)
    assert np.all(np.abs(rows["pvalue"] - cols["pvalue"].T) <= 1e-12 * np.maximum(rows["pvalue"], 1e-300))
    assert np.all(rows["numer"][np.arange(96), q] == s) and np.all(rows["distance"][np.arange(96), q] == 0)
    assert np.all((rows["distance"] >= 0) & (rows["distance"] <= 1)) and np.all((rows["pvalue"] >= 0) & (rows["pvalue"] <= 1))
    assert np.all(rows["denom"] == s)
    # 10^4 sampled pairs of the full-size grid against the oracle: the 96 query rows x random columns, weighted towards the
    # queries' own families (related pairs), plus the closed-form majority
    cand = []
    for i in range(96):
        same = np.flatnonzero(fam == fam[q[i]])
        cand.append(np.stack([np.full(60, i), rng.choice(same, 60)], axis=1))
        cand.append(np.stack([np.full(45, i), rng.integers(0, n, 45)], axis=1))
    cand = np.concatenate(cand)
    assert cand.shape[0] >= 10_000
    n_related = 0
    for i in range(96):
        cols_i = cand[cand[:, 0] == i, 1]
        want = oracle.compare_all(H[cols_i], N[cols_i], L[cols_i], H[q[i]:q[i] + 1], N[q[i]:q[i] + 1], L[q[i]:q[i] + 1], s, 21, ks)[0]
        got = {key: rows[key][i, cols_i] for key in ("numer", "denom", "distance", "pvalue", "pass")}
        assert np.array_equal(got["numer"], want["numer"]) and np.array_equal(got["denom"], want["denom"])
        assert np.all(np.abs(got["distance"] - want["distance"]) <= TOL)
        big = want["pvalue"] > 1e-305
        assert np.all(np.abs(got["pvalue"][big] - want["pvalue"][big]) <= TOL * want["pvalue"][big])
        assert np.all(got["pvalue"][~big] <= 1.0000001e-305)
        n_related += int((want["numer"] > 0).sum())
    assert n_related > 1000      # the sample really contains pairs that went through the merge


def test_pass_list_equals_dense_filter(gpu, oracle):
    # -d / -v filtered output as a compacted list in the reference's (query-major) order
    H, N, L = synth_sketches(90, 600, seed=31, n_families=3, ragged=True)
    ks = 4.0 ** 21
    for md, mp in ((0.1, 1.0), (1.0, 1e-20), (0.05, 1e-5)):
        job = gpu.dist_open(H, N, L, sketch_size=600, k=21, kmer_space=ks, max_distance=md, max_pvalue=mp)
        try:
            dense = job.run(10, 70)
            n_pass, lst = job.run_list(10, 70, 70 * 90)
            n_over, empty = job.run_list(10, 70, 3)
        finally:
            job.close()
        flat = np.flatnonzero(dense["pass"].ravel())
        assert n_pass == flat.size and np.array_equal(lst["index"], flat.astype(np.uint64))
        for key in ("numer", "denom", "distance", "pvalue"):
            assert np.array_equal(lst[key], dense[key].ravel()[flat])
        assert n_over == flat.size and (flat.size <= 3 or empty["index"].size == 0)
        want = oracle.compare_all(H, N, L, H, N, L, 600, 21, ks, max_distance=md, max_pvalue=mp, q_begin=10, q_end=80)[10:80]
        assert np.array_equal(np.flatnonzero(want["pass"].ravel()), flat)


def test_query_row_staging_at_every_row_alignment(gpu, oracle):
    # dist_kernel stages the query rows with cp.async.bulk (TMA engine, mbarrier completion): rows start at 4-byte aligned
    # addresses, so the copy covers the 16-byte aligned span and the merge starts `skew` bytes in.  Same results for every row
    # alignment (P odd and even, ragged rows, query ranges), up to s = 1034, the largest sketch size of the tiled merge.
    for s, nq in ((1000, 61), (999, 40), (37, 70), (1020, 33), (1034, 45)):
        H, N, L = synth_sketches(70, s, seed=300 + s, n_families=3, ragged=True)
        Hq, Nq, Lq = synth_sketches(nq, s, seed=400 + s, n_families=3, ragged=True)
        Hq[:7] = H[:7]; Nq[:7] = N[:7]
        ks = 4.0 ** 21
        for pf in (0, 1):
            job = gpu.dist_open(H, N, L, Hq, Nq, Lq, sketch_size=s, k=21, kmer_space=ks)
            try:
                job.set_prefilter(pf)
                res = job.run(3, nq - 5)
            finally:
                job.close()
            want = oracle.compare_all(H, N, L, Hq, Nq, Lq, s, 21, ks, q_begin=3, q_end=nq - 2)[3:nq - 2]
            check_against_oracle(res, want)
