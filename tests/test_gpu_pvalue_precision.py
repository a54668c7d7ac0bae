"""The device binomial tail (binom.cuh) against 60-digit truth (tests/binom_truth.py) at large sketch sizes, through dist
and screen, and the merge / reduce variants those sizes take.

Every p-value whose truth is above 1e-305 must be within 1e-12 relative of it; below that the device value must be
<= 1.0000001e-305, as in the parity tests.  The grid is n in {4096, 10000, 28151, 28152, 32768, 100000} (plus the tiled merge's
sizes), r from 1e-9 to 0.999, and x at 1, 2, n-1, n and the mean plus -3 .. 100 standard deviations."""
from fractions import Fraction

import numpy as np
import pytest

from binom_truth import GRID_N, GRID_R, grid_x, upper_tail
from fixtures import synth_genome, mutate, synth_sketches
from test_gpu_dist import check_against_oracle

pytestmark = pytest.mark.gpu

TOL = 1e-12
K21 = 4.0 ** 21


def pair_warps(S):
    """dist.cu: warps per CTA of the warp-per-pair merge; below 1 the job runs dist_kernel_general."""
    row_pitch = (S + 1 + 8 + 3) & ~3
    return min(8, (220 * 1024) // (row_pitch * 8))


GENERAL_MIN_S = next(S for S in range(20000, 40000) if pair_warps(S) < 1)


def _rnd(q):
    return float(q)            # Fraction -> nearest double (ties to even)


def device_r(L_ref, L_qry, K=K21):
    """r of mash_pvalue for these lengths, or None when it depends on whether the compiler fuses pX + pY - pX pY."""
    pX = 1.0 / (1.0 + K / float(L_ref))
    pY = 1.0 / (1.0 + K / float(L_qry))
    num = _rnd(Fraction(pX) * Fraction(pY))
    unfused = _rnd(Fraction(_rnd(Fraction(pX) + Fraction(pY))) - Fraction(num))
    fused = _rnd(Fraction(_rnd(Fraction(pX) + Fraction(pY))) - Fraction(pX) * Fraction(pY))
    r1, r2 = _rnd(Fraction(num) / Fraction(unfused)), _rnd(Fraction(num) / Fraction(fused))
    return r1 if r1 == r2 else None


L_REF = int(K21 * 9999)          # pX = 0.9999: every r < 0.9999 is reachable with a query length


def query_length(r):
    """(length, exact device r) of a query whose r against L_REF is within 1e-3 relative of the target r."""
    pX = 1.0 / (1.0 + K21 / float(L_REF))
    pY = 1.0 / (1.0 / r - 1.0 / pX + 1.0)
    L0 = int(round(K21 * pY / (1.0 - pY)))
    for d in range(0, 4000):
        for L in (L0 + d, L0 - d):
            if L >= 1:
                got = device_r(L_REF, L)
                if got is not None:
                    assert abs(got - r) <= 1e-3 * r, (r, got)
                    return L, got
    raise AssertionError(f"no length reaches r = {r}")


def check_p(got, truth, what):
    """got: device double; truth: mpf.  Returns the relative error (0 below 1e-305)."""
    if truth > 1e-305:
        err = float(abs(got - truth) / truth)
        assert err <= TOL, (what, got, float(truth), err)
        return err
    assert got <= 1.0000001e-305, (what, got, float(truth))
    return 0.0


def crafted_job(n, S):
    """One reference row of n even values and one query row per grid point (x, r).  S == n: the query holds x of the
    reference's values and n - x odd ones (denom = S, the table path).  S > n: the query is the first x of the reference's
    values, so the union has n < S elements (denom = n, the plain path)."""
    assert S >= n
    cases = []
    for r in GRID_R:
        L, r_dev = query_length(r)
        for x in grid_x(n, r):
            cases.append((x, L, r_dev))
    ref = np.arange(0, 2 * n, 2, dtype=np.uint64)
    H = np.full((1, S), np.uint64(2**64 - 1)); H[0, :n] = ref
    Hq = np.full((len(cases), S), np.uint64(2**64 - 1)); Nq = np.zeros(len(cases), np.uint32)
    for i, (x, _, _) in enumerate(cases):
        if S == n:
            q = ref.copy(); q[x:] += 1
            Hq[i, :n] = q; Nq[i] = n
        else:
            Hq[i, :x] = ref[:x]; Nq[i] = x
    Lq = np.array([c[1] for c in cases], np.uint64)
    return (H, np.array([n], np.uint32), np.array([L_REF], np.uint64), Hq, Nq, Lq), cases


def kernel_names(fn):
    """Names of the CUDA kernels fn() launches (CUPTI activity records through torch.profiler)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.init()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return {e.name for e in prof.events()}


def run_crafted(gpu, n, S, prefilter=None, expect_kernel=None):
    args, cases = crafted_job(n, S)
    H, N, L, Hq, Nq, Lq = args
    job = gpu.dist_open(H, N, L, Hq, Nq, Lq, sketch_size=S, k=21, kmer_space=K21)
    try:
        if prefilter is not None:
            job.set_prefilter(prefilter)
        if expect_kernel is None:
            res = job.run(0, len(cases))
        else:
            out = {}
            names = kernel_names(lambda: out.setdefault("res", job.run(0, len(cases))))
            assert any(expect_kernel in nm for nm in names), (n, S, sorted(names))
            res = out["res"]
        if prefilter:
            assert job.prefilter_stats()["active"]
    finally:
        job.close()
    truths = []
    worst = 0.0
    for i, (x, _, r) in enumerate(cases):
        assert res["numer"][i, 0] == x and res["denom"][i, 0] == n, (n, S, x)
        t = upper_tail(x, r, n)
        truths.append(t)
        worst = max(worst, check_p(res["pvalue"][i, 0], t, (n, S, x, r)))
    # -v: thresholds between neighbouring p-values decide the same pass flags as the truth
    tv = np.array([float(t) for t in truths])
    u = np.unique(tv[(tv > 1e-300) & (tv < 1.0)])
    gaps = [(u[j] * u[j + 1]) ** 0.5 for j in range(u.size - 1) if u[j + 1] > u[j] * (1 + 1e-9)]
    assert len(gaps) >= 4
    for thr in (gaps[len(gaps) // 4], gaps[(3 * len(gaps)) // 4]):
        job = gpu.dist_open(H, N, L, Hq, Nq, Lq, sketch_size=S, k=21, kmer_space=K21, max_pvalue=thr)
        try:
            res_v = job.run(0, len(cases))
        finally:
            job.close()
        assert np.array_equal(res_v["pass"][:, 0], tv <= thr), thr
    return worst


# (n, S, merge): S == n is the table path (denom == sketch size), S > n the plain path (rows shorter than the sketch size)
DIST_CASES = [
    (1034, 1034, "tiled"), (1000, 1034, "tiled"),
    (4096, 4096, "pair"), (10000, 10000, "pair"), (28151, 28151, "pair"),
    (4096, 28151, "pair"), (10000, 28151, "pair"), (28000, 28151, "pair"),
    (28152, 28152, "general"), (32768, 32768, "general"), (100000, 100000, "general"),
    (28151, 100001, "general"), (28152, 100001, "general"), (32768, 100001, "general"), (100000, 100001, "general"),
]


def test_general_merge_boundary():
    # dist_kernel_general takes over where a warp's two query rows no longer fit the warp-per-pair kernel's shared memory
    assert GENERAL_MIN_S == 28152 and pair_warps(28151) == 1
    assert all(n in GRID_N for n in (28151, 28152))


@pytest.mark.parametrize("n,S,merge", DIST_CASES)
def test_dist_pvalue_vs_truth(gpu, n, S, merge):
    assert (S >= GENERAL_MIN_S) == (merge == "general") and (S <= 1034) == (merge == "tiled")
    if merge == "tiled":
        worst = max(run_crafted(gpu, n, S, prefilter=pf) for pf in (0, 1))
    else:
        worst = run_crafted(gpu, n, S, expect_kernel="dist_kernel_general" if merge == "general" else "dist_pair_kernel")
    print(f"dist n={n} S={S} {merge}: worst relative error {worst:.2e}")


# ---- screen ------------------------------------------------------------------------------------------------------------

def _screen(gpu, ref, ref_n, p, chunks):
    job = gpu.screen_open(ref, ref_n, p)
    try:
        for c in chunks:
            job.feed(c)
        return job.finish()
    finally:
        job.close()


SCREEN_MIXES = [   # (k, noncanonical, mixture bases): r = set_size / 4^k from ~0.05 to ~0.85
    (12, False, 1_000_000), (12, False, 2_000_000), (11, False, 2_000_000), (10, False, 2_000_000), (10, True, 2_000_000),
]


@pytest.mark.parametrize("k,nonc,mix_len", SCREEN_MIXES)
def test_screen_pvalue_vs_truth(gpu, oracle, k, nonc, mix_len):
    s = 1000
    p = gpu.params(k=k, s=s, noncanonical=nonc)
    po = oracle.params(k=k, noncanonical=nonc)
    mix = [synth_genome(9000 + i, mix_len // 4) for i in range(4)]
    chunks = [b"".join(b"*" + bytes(g[a:a + 10_000]) for a in range(0, g.size, 10_000 - k + 1)) for g in mix]
    unrelated = [synth_genome(9100 + i, 120_000) for i in range(3)]
    related = [mutate(mix[i][:120_000], rate, 50 + i) for i, rate in enumerate((0.01, 0.04, 0.1))]
    genomes = unrelated + related
    worst = {}
    r_job = None
    for stride in (1000, 8192, 8193, 16384, 32768):
        ref = np.full((len(genomes), stride), np.uint64(2**64 - 1)); ref_n = np.zeros(len(genomes), np.uint32)
        for i, g in enumerate(genomes):
            h, _, _ = oracle.sketch_unit([bytes(g)], po, s=stride)
            ref[i, :h.size] = h; ref_n[i] = h.size
        assert ref_n.min() == stride
        res = _screen(gpu, ref, ref_n, p, chunks)
        want = oracle.screen(ref, ref_n, chunks, po, s=s)
        assert res["set_size"] == want["set_size"] and np.array_equal(res["mixture"], want["mixture"])
        assert np.array_equal(res["shared"], want["shared"]) and np.array_equal(res["median"], want["median"])
        assert np.all(np.abs(res["identity"] - want["identity"]) <= 1e-12)
        r = res["set_size"] / p.kmer_space
        r_job = r
        w = 0.0
        for i in range(len(genomes)):
            x = int(res["shared"][i])
            w = max(w, check_p(res["pvalue"][i], upper_tail(x, r, int(ref_n[i])), (k, nonc, stride, i, x, r)))
        worst[stride] = w
    print(f"screen k={k} noncanonical={nonc} r={r_job:.3f}: worst relative error per stride {worst}")


# ---- dist_kernel_general against the oracle -----------------------------------------------------------------------------

def test_general_merge_matches_oracle(gpu, oracle):
    # sketch sizes whose query rows do not fit the warp-per-pair kernel (S >= 28152): one thread per pair, rows from global
    # memory; same results as the reference's sequential merge, ragged and empty rows, the lower triangle and the pass list
    s = 30000
    assert s >= GENERAL_MIN_S
    H, N, L = synth_sketches(24, s, seed=41, n_families=3, ragged=True)
    Hq, Nq, Lq = synth_sketches(11, s, seed=42, n_families=3, ragged=True)
    Hq[:4] = H[:4]; Nq[:4] = N[:4]
    N[7] = 0; Nq[3] = 1
    res = {}
    names = kernel_names(lambda: res.setdefault("r", gpu.dist(H, N, L, Hq, Nq, Lq, sketch_size=s, k=21, kmer_space=K21)))
    assert any("dist_kernel_general" in nm for nm in names)
    check_against_oracle(res["r"], oracle.compare_all(H, N, L, Hq, Nq, Lq, s, 21, K21))
    # self comparison: the dense run, its lower triangle, and the pass list of a filtered run
    want = oracle.compare_all(H, N, L, H, N, L, s, 21, K21)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=21, kmer_space=K21)
    try:
        full = job.run(0, 24)
        check_against_oracle(full, want)
        job.set_triangle(1)
        tri = job.run(0, 24)
    finally:
        job.close()
    low = np.tril(np.ones((24, 24), bool), -1)
    for key in ("numer", "denom", "distance", "pvalue", "pass"):
        assert np.array_equal(tri[key][low], full[key][low])
    for md, mp in ((0.1, 1.0), (1.0, 1e-30)):
        job = gpu.dist_open(H, N, L, sketch_size=s, k=21, kmer_space=K21, max_distance=md, max_pvalue=mp)
        try:
            dense = job.run(2, 20)
            n_pass, lst = job.run_list(2, 20, 20 * 24)
        finally:
            job.close()
        flat = np.flatnonzero(dense["pass"].ravel())
        assert 0 < flat.size < dense["pass"].size
        assert n_pass == flat.size and np.array_equal(lst["index"], flat.astype(np.uint64))
        for key in ("numer", "denom", "distance", "pvalue"):
            assert np.array_equal(lst[key], dense[key].ravel()[flat])
        w = oracle.compare_all(H, N, L, H, N, L, s, 21, K21, max_distance=md, max_pvalue=mp, q_begin=2, q_end=22)[2:22]
        assert np.array_equal(np.flatnonzero(w["pass"].ravel()), flat)
