"""GPU tests of the dist tile prefilter (dist_probe_kernel): pairs that share no hash get the closed form of the merge
(CommandDistance.cpp:347-407 with an empty intersection) without being merged.  Every result must be identical to the
merge-everything path and to the oracle, bit for bit (the doubles included: both paths run the same epilogue)."""
import numpy as np
import pytest

from fixtures import synth_sketches
from test_gpu_dist import check_against_oracle

pytestmark = pytest.mark.gpu

KEYS = ("numer", "denom", "distance", "pvalue", "pass")


def mixed_sketches(n, s, seed, n_related=40, ragged=True):
    """Mostly unrelated sketches (every one its own random draw) with a few related families and ragged / empty rows mixed in,
    in shuffled order, so that reference tiles hold both kinds."""
    rng = np.random.Generator(np.random.PCG64(seed))
    hi = int(2 ** 64 * s / 5_000_000)
    H = np.full((n, s), np.uint64(0xFFFFFFFFFFFFFFFF), dtype=np.uint64)
    N = np.zeros(n, np.uint32)
    Hf, Nf, _ = synth_sketches(n_related, s, seed + 1, n_families=3, ragged=ragged)
    for g in range(n):
        if g < n_related:
            H[g], N[g] = Hf[g], Nf[g]
            continue
        m = s
        if ragged and g % 7 == 0:
            m = int(rng.integers(0, s + 1))
        v = np.unique(rng.integers(0, hi, s + 8, dtype=np.uint64))[:m]
        H[g, :v.size] = v
        N[g] = v.size
    perm = rng.permutation(n)
    L = rng.integers(4_000_000, 6_000_000, n).astype(np.uint64)
    return H[perm], N[perm], L


def run_modes(gpu, H, N, L, Hq=None, Nq=None, Lq=None, *, s, k, q_begin=0, q_count=None, **kw):
    out = {}
    stats = None
    for mode in (0, 1):
        job = gpu.dist_open(H, N, L, Hq, Nq, Lq, sketch_size=s, k=k, kmer_space=4.0 ** k, **kw)
        try:
            job.set_prefilter(mode)
            out[mode] = job.run(q_begin, job.n_qry - q_begin if q_count is None else q_count)
            if mode == 1:
                stats = job.prefilter_stats()
        finally:
            job.close()
    for key in KEYS:
        assert np.array_equal(out[0][key], out[1][key]), key
    return out[1], stats


@pytest.mark.parametrize("s,k", [(1000, 21), (200, 16), (13, 11), (1, 21)])
def test_prefilter_equals_merge_and_oracle(gpu, oracle, s, k):
    H, N, L = mixed_sketches(150, s, seed=11 + s)
    Hq, Nq, Lq = mixed_sketches(77, s, seed=500 + s, n_related=20)
    Hq[:5] = H[:5]; Nq[:5] = N[:5]
    res, st = run_modes(gpu, H, N, L, Hq, Nq, Lq, s=s, k=k)
    want = oracle.compare_all(H, N, L, Hq, Nq, Lq, s, k, 4.0 ** k)
    check_against_oracle(res, want)
    assert st["active"] and st["combos_probed"] == 77 * 5          # ceil(150 / 32) reference tiles
    if s >= 200:
        assert st["combos_flagged"] < st["combos_probed"]          # the closed form was exercised ...
        assert st["combos_flagged"] + st["pairs_from_lists"] > 0   # ... and so was a merge (whole combinations and / or listed pairs)


def test_prefilter_self_ranges_and_thresholds(gpu, oracle):
    s, k = 500, 21
    H, N, L = mixed_sketches(200, s, seed=7)
    for md, mp in ((1.0, 1.0), (0.1, 1.0), (1.0, 1e-10), (-1.0, -1.0)):
        res, _ = run_modes(gpu, H, N, L, s=s, k=k, q_begin=23, q_count=131, max_distance=md, max_pvalue=mp)
        want = oracle.compare_all(H, N, L, H, N, L, s, k, 4.0 ** k, max_distance=md, max_pvalue=mp, q_begin=23, q_end=154)[23:154]
        check_against_oracle(res, want)


def test_prefilter_lists_longer_than_sketch_size(gpu, oracle):
    # s' = 300 < list lengths: only the first 300 ranks of a row can take part in a merge, and in the filter
    H, N, L = mixed_sketches(120, 1000, seed=3)
    res, st = run_modes(gpu, H, N, L, s=300, k=21)
    want = oracle.compare_all(H, N, L, H, N, L, 300, 21, 4.0 ** 21)
    check_against_oracle(res, want)


def test_prefilter_pass_list(gpu):
    s, k = 600, 21
    H, N, L = mixed_sketches(180, s, seed=19)
    lists = {}
    for mode in (0, 1):
        job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.2, max_pvalue=1e-3)
        try:
            job.set_prefilter(mode)
            lists[mode] = job.run_list(0, 180, 180 * 180)
        finally:
            job.close()
    assert lists[0][0] == lists[1][0] > 0
    for key in ("index", "numer", "denom", "distance", "pvalue"):
        assert np.array_equal(lists[0][1][key], lists[1][1][key])


def test_auto_mode_switches_off_on_dense_sets(gpu):
    # every query shares hashes with every tile: after the first run the counters say so and later runs merge directly
    s, k = 400, 21
    H, N, L = synth_sketches(96, s, seed=2, n_families=1)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k)
    try:
        first = job.run(0, 96)
        st = job.prefilter_stats()
        assert st["combos_probed"] == 96 * 3 and st["combos_flagged"] == 96 * 3
        second = job.run(0, 96)
        st2 = job.prefilter_stats()
        assert not st2["active"] and st2["combos_probed"] == st["combos_probed"]
        for key in KEYS:
            assert np.array_equal(first[key], second[key])
    finally:
        job.close()


@pytest.mark.parametrize("mode", [0, 1])
def test_triangle_enumeration(gpu, mode):
    # `mash triangle` (CommandTriangle.cpp:200-214): row i against rows 0..i-1 -- pairs on or above the diagonal are not
    # computed; the lower triangle equals the full grid's
    s, k = 300, 21
    H, N, L = mixed_sketches(210, s, seed=41)
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.3, max_pvalue=1.0)
    try:
        job.set_prefilter(mode)
        full = job.run(0, 210)
        n_full, lst_full = job.run_list(0, 210, 210 * 210)
        job.set_triangle(True)
        tri = job.run(0, 210)            # host buffers start zeroed (see _capi.DistJob.run)
        n_tri, lst_tri = job.run_list(0, 210, 210 * 210)
        part = job.run(100, 60)
    finally:
        job.close()
    q, r = np.indices((210, 210))
    low = r < q
    for key in KEYS:
        assert np.array_equal(tri[key][low], full[key][low]), key
        assert np.array_equal(part[key][low[100:160]], full[key][100:160][low[100:160]]), key
    assert not tri["numer"][~low].any() and not tri["pass"][~low].any()      # untouched
    keep = low.ravel()[lst_full["index"].astype(np.int64)]
    assert n_tri == int(keep.sum()) and np.array_equal(lst_tri["index"], lst_full["index"][keep])
    for key in ("numer", "denom", "distance", "pvalue"):
        assert np.array_equal(lst_tri[key], lst_full[key][keep])


def test_triangle_needs_self_comparison(gpu):
    H, N, L = mixed_sketches(40, 100, seed=5)
    job = gpu.dist_open(H, N, L, H[:7], N[:7], L[:7], sketch_size=100, k=21, kmer_space=4.0 ** 21)
    try:
        with pytest.raises(Exception):
            job.set_triangle(True)
    finally:
        job.close()


@pytest.mark.parametrize("pair_max", ["4", "0", "31"])
def test_scattered_relatives_take_the_pair_list(gpu, oracle, monkeypatch, pair_max):
    # Related sketches scattered over the collection (one or two per reference tile): the probe kernel names the candidate
    # references of each (query, tile) combination and only those pairs are merged, one warp per pair (dist_pair_kernel).
    # MASHGPU_DIST_PAIR_MAX=0 switches the path off (whole combinations merged), 31 sends everything through it.
    monkeypatch.setenv("MASHGPU_DIST_PAIR_MAX", pair_max)
    s, k = 1000, 21
    n = 700
    rng = np.random.Generator(np.random.PCG64(2024))
    H, N, L = mixed_sketches(n, s, seed=91, n_related=0)
    Hf, Nf, _ = synth_sketches(44, s, 92, n_families=4, ragged=True)       # 4 families of 11, two ragged members, placed far apart
    pos = rng.choice(n, 44, replace=False)
    H[pos], N[pos] = Hf, Nf
    res, st = run_modes(gpu, H, N, L, s=s, k=k)
    want = oracle.compare_all(H, N, L, H, N, L, s, k, 4.0 ** k)
    check_against_oracle(res, want)
    if pair_max == "0":
        assert st["pairs_from_lists"] == 0 and st["combos_flagged"] > 0
    else:
        assert st["pairs_from_lists"] >= 44 * 10               # every related pair went through the list (plus a few false candidates)
    # filtered list output and the triangle enumeration through the same path
    job = gpu.dist_open(H, N, L, sketch_size=s, k=k, kmer_space=4.0 ** k, max_distance=0.3, max_pvalue=1.0)
    try:
        job.set_prefilter(1)
        job.set_triangle(True)
        n_pass, lst = job.run_list(0, n, n * n)
    finally:
        job.close()
    wf = oracle.compare_all(H, N, L, H, N, L, s, k, 4.0 ** k, max_distance=0.3, max_pvalue=1.0)
    lower = np.arange(n)[None, :] < np.arange(n)[:, None]
    flat = np.flatnonzero((wf["pass"].astype(bool) & lower).ravel())
    assert n_pass == flat.size and np.array_equal(lst["index"], flat.astype(np.uint64))
    assert np.array_equal(lst["numer"], wf["numer"].ravel()[flat])


def test_tiled_merge_ends_at_sketch_size_1034(gpu):
    # the prefilter runs in front of the tiled merge only: on at s = 1034, the largest sketch size whose 32-reference tile and
    # query buffers fit shared memory, off at s = 1035, which takes the warp-per-pair merge
    for s, tiled in ((1034, True), (1035, False)):
        H, N, L = synth_sketches(40, s, seed=s)
        job = gpu.dist_open(H, N, L, sketch_size=s, k=21, kmer_space=4.0 ** 21)
        try:
            assert job.prefilter_stats()["active"] == tiled, s
        finally:
            job.close()


@pytest.mark.parametrize("s", [1035, 1036, 2500, 10000])
def test_large_sketch_sizes_use_the_warp_per_pair_merge(gpu, oracle, s):
    # `mash sketch -s 10000` is a documented setting: sketches whose 32-reference tile does not fit shared memory are compared one
    # warp per pair (zooming union count) -- same results as the reference's sequential merge, ragged and empty rows included
    H, N, L = synth_sketches(48, s, seed=5 + s, n_families=3, ragged=True)
    Hq, Nq, Lq = synth_sketches(21, s, seed=77 + s, n_families=3, ragged=True)
    Hq[:6] = H[:6]; Nq[:6] = N[:6]
    N[7] = 0; Nq[3] = 1
    ks = 4.0 ** 21
    res = gpu.dist(H, N, L, Hq, Nq, Lq, sketch_size=s, k=21, kmer_space=ks)
    want = oracle.compare_all(H, N, L, Hq, Nq, Lq, s, 21, ks)
    check_against_oracle(res, want)
    # a smaller sketch_size than the lists hold: only the first s' elements of a row can matter
    res2 = gpu.dist(H, N, L, Hq, Nq, Lq, sketch_size=s - 500, k=21, kmer_space=ks)
    check_against_oracle(res2, oracle.compare_all(H, N, L, Hq, Nq, Lq, s - 500, 21, ks))
