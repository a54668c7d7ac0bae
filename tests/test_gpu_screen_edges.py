"""Screen (hot path 3) at its edges, compared with the oracle hash by hash: the per-hash hit counters next to the per-sketch
aggregates, sketch sizes up to the 8192 limit, tables whose presence bitmap reaches its 2^27-bit cap, linear-probe runs that wrap
past the last slot, the multi-rank merge entry points on one GPU, two jobs sharing one context, and the reference sets
mashgpu_screen_open refuses (each followed by an ordinary screen on the same context).

Every comparison is exact except identity (1e-12 absolute) and p-value (1e-12 relative above 1e-305), as in test_gpu_screen."""
import numpy as np
import pytest

import mash_b200
from mash_b200._capi import _Set
from fixtures import synth_genome, mutate
from test_gpu_screen import check

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = 1, 3
EMPTY = 2**64 - 1
GOLDEN_RATIO_64 = 0x9E3779B97F4A7C15          # slot_hash multiplier (scan.cuh)


# ---- helpers -------------------------------------------------------------------------------------------------------

class _Cai:
    """A library-owned device buffer seen by torch without a copy (CUDA array interface), as mash_b200/shard.py does."""

    def __init__(self, ptr, n, typestr):
        self.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 3}


def _dev_view(ptr, n, typestr):
    import torch
    return torch.as_tensor(_Cai(ptr, n, typestr), device="cuda:0")


def counters(job):
    """The job's per-hash hit counters, ascending-key order (the oracle's `counts`), copied to the host."""
    ptr, n = job.counters()
    if n == 0:
        return np.zeros(0, np.uint32)
    return _dev_view(ptr, n, "<i4").cpu().numpy().view(np.uint32).copy()


def feed_dev(job, chunk):
    """One kernel pass over a chunk already in device memory (readable up to its length rounded up to 16)."""
    import torch
    b = np.frombuffer(chunk, np.uint8)
    t = torch.zeros(((b.size + 15) // 16) * 16, dtype=torch.uint8, device="cuda:0")
    t[:b.size] = torch.from_numpy(b.copy()).to("cuda:0")
    torch.cuda.synchronize()
    job.feed_dev(t.data_ptr(), b.size)


def run(gpu, ref, ref_n, p, chunks, feed="host", winner=False, ref_len=None):
    job = gpu.screen_open(ref, ref_n, p, ref_len=ref_len)
    try:
        for c in chunks:
            if feed == "dev":
                feed_dev(job, c)
            else:
                job.feed(c)
        if winner:
            job.set_winner(True)
        res = job.finish()
        return res, counters(job)
    finally:
        job.close()


def check_all(res, cnt, want):
    check(res, want)
    assert cnt.size == want["keys"].size
    assert np.array_equal(cnt, want["counts"])


def sketch_rows(oracle, po, genomes, s, stride=None):
    stride = stride or s
    ref = np.full((len(genomes), stride), np.uint64(EMPTY)); ref_n = np.zeros(len(genomes), np.uint32)
    for i, g in enumerate(genomes):
        h, _, _ = oracle.sketch_unit([bytes(g)], po, s=s)
        ref[i, :h.size] = h; ref_n[i] = h.size
    return ref, ref_n


def make_reads(genomes, n_reads, seed, max_len=300, lower=0.1):
    """Reads of 1..max_len bases (so read boundaries fall at every position modulo 32 and some reads are shorter than k),
    one in ten with an N, a fraction with a lower-case stretch."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for _ in range(n_reads):
        g = genomes[int(rng.integers(0, len(genomes)))]
        L = int(rng.integers(1, max_len + 1))
        a = int(rng.integers(0, max(1, g.size - L)))
        r = g[a:a + L].copy()
        if rng.random() < 0.1:
            r[int(rng.integers(0, r.size))] = ord("N")
        if rng.random() < lower:
            i = int(rng.integers(0, r.size))
            r[i:i + int(rng.integers(1, 80))] |= 0x20
        out.append(bytes(r))
    return out


def join(reads, per):
    return [b"".join(b"*" + r for r in reads[i:i + per]) for i in range(0, len(reads), per)]


def clean_context_screen(gpu, oracle):
    """An ordinary screen on the same context matches the oracle: no device error was left behind."""
    p = gpu.params(k=21, s=200); po = oracle.params(k=21)
    genomes = [synth_genome(900 + i, 40_000) for i in range(2)]
    ref, ref_n = sketch_rows(oracle, po, genomes, 200)
    chunks = join(make_reads(genomes, 1500, seed=901), 500)
    want = oracle.screen(ref, ref_n, chunks, po, s=200)
    res, cnt = run(gpu, ref, ref_n, p, chunks)
    check_all(res, cnt, want)
    assert want["shared"].min() > 0


def ceil_log2(x):
    return max(0, (x - 1).bit_length())


def bits_log2(n_distinct):
    return min(27, max(20, ceil_log2(4 * n_distinct)))      # presence bitmap size (screen.cu, mashgpu_screen_open)


# ---- 1. per-hash counters ------------------------------------------------------------------------------------------

@pytest.mark.parametrize("mode", ["canonical", "noncanonical", "preserve_case"])
@pytest.mark.parametrize("k", [9, 12, 16, 17, 21, 32])
def test_counters_match_oracle(gpu, oracle, k, mode):
    # 32-bit (k <= 16) and 64-bit hashes, the window-validity word loop up to k = 32; lower-case stretches are bases without
    # preserve_case and separators with it
    nc, pc = mode == "noncanonical", mode == "preserve_case"
    s = 400
    p = gpu.params(k=k, s=s, noncanonical=nc, preserve_case=pc); po = oracle.params(k=k, noncanonical=nc, preserve_case=pc)
    genomes = [synth_genome(300 + i, 80_000) for i in range(3)]
    genomes.append(mutate(genomes[0], 0.03, 301))
    ref, ref_n = sketch_rows(oracle, po, genomes, s)
    chunks = join(make_reads(genomes[:2], 8000, seed=310 + k), 2000)
    stars = np.concatenate([np.flatnonzero(np.frombuffer(c, np.uint8) == ord("*")) for c in chunks])
    assert np.unique(stars % 32).size == 32
    want = oracle.screen(ref, ref_n, chunks, po, s=s)
    res, cnt = run(gpu, ref, ref_n, p, chunks)
    check_all(res, cnt, want)
    assert (want["counts"] > 1).sum() > 100


def _whole_range_refs(oracle, po, k, s):
    genomes = [synth_genome(340 + i, 100_000) for i in range(2)]
    tiny = [synth_genome(760 + i, 150 + 37 * i) for i in range(6)]          # fewer k-mers than s: every k-mer is in the sketch
    ref, ref_n = sketch_rows(oracle, po, genomes + tiny, s)
    return genomes, tiny, ref, ref_n


@pytest.mark.parametrize("bitmap", ["1", "0"])
@pytest.mark.parametrize("k", [12, 21])
def test_counters_whole_hash_range_table(gpu, oracle, monkeypatch, k, bitmap):
    monkeypatch.setenv("MASHGPU_SCREEN_BITMAP", bitmap)
    s = 300
    p = gpu.params(k=k, s=s); po = oracle.params(k=k)
    genomes, tiny, ref, ref_n = _whole_range_refs(oracle, po, k, s)
    top = 2**32 if k <= 16 else 2**64
    assert int(ref[np.arange(ref.shape[0]), ref_n - 1].max()) > top // 2        # the table spans the whole hash range
    chunks = join(make_reads(genomes + tiny[:3], 6000, seed=350 + k), 1500)
    want = oracle.screen(ref, ref_n, chunks, po, s=s)
    res, cnt = run(gpu, ref, ref_n, p, chunks)
    check_all(res, cnt, want)
    assert want["shared"][2] > 0
    if k > 16:
        assert want["shared"][-1] == 0


_BIG = {}


def _big_chunks():
    """Four chunks of 4.3-4.5 MB (above the 4 MiB joining threshold: one kernel pass each, through the two-buffer pipeline)."""
    if "chunks" not in _BIG:
        genomes = [synth_genome(400 + i, 200_000) for i in range(3)]
        reads = make_reads(genomes, 4 * 29_000, seed=401)
        _BIG["genomes"] = genomes
        _BIG["chunks"] = join(reads, 29_000)
    assert min(len(c) for c in _BIG["chunks"]) >= 4 << 20
    return _BIG["genomes"], _BIG["chunks"]


def _big_case(oracle, k, s, which):
    key = (k, s, which)
    if key not in _BIG:
        genomes, chunks = _big_chunks()
        po = oracle.params(k=k)
        ref, ref_n = sketch_rows(oracle, po, genomes + [mutate(genomes[1], 0.05, 402)], s)
        mine = [chunks[i] for i in which]
        _BIG[key] = (ref, ref_n, mine, oracle.screen(ref, ref_n, mine, po, s=s))
    return _BIG[key]


@pytest.mark.parametrize("path", ["ascii", "packed", "dev"])
@pytest.mark.parametrize("k", [12, 21])
def test_counters_large_chunks_every_feed_path(gpu, oracle, monkeypatch, k, path):
    # host chunks >= 4 MiB uploaded as ASCII or 2-bit packed on the host, and device chunks through feed_dev on a nucleotide job
    monkeypatch.setenv("MASHGPU_SCREEN_HOST_PACK", "1" if path == "packed" else "0")
    s = 500
    ref, ref_n, chunks, want = _big_case(oracle, k, s, (0, 1))
    res, cnt = run(gpu, ref, ref_n, gpu.params(k=k, s=s), chunks, feed="dev" if path == "dev" else "host")
    check_all(res, cnt, want)


def test_exact_rerun_does_not_count_twice(gpu, oracle):
    # a mixture of few distinct k-mers: the chunk's threshold pass holds fewer than s hashes and the chunk is re-run exactly;
    # the table hits were counted in the first pass only
    k, s = 21, 1000
    p = gpu.params(k=k, s=s); po = oracle.params(k=k)
    rep = synth_genome(5, 3000)
    ref, ref_n = sketch_rows(oracle, po, [rep, synth_genome(6, 50_000)], s)
    chunk = b"*" + bytes(np.tile(rep, 200))                  # 600 kbp, ~3000 distinct k-mers, one kernel pass
    want = oracle.screen(ref, ref_n, [chunk], po, s=s)
    before = gpu.stats()["exact_reruns"]
    res, cnt = run(gpu, ref, ref_n, p, [chunk])
    assert gpu.stats()["exact_reruns"] > before
    check_all(res, cnt, want)
    assert want["counts"].max() >= 200


# ---- 2. sketch sizes -----------------------------------------------------------------------------------------------

_SIZES = {}


@pytest.mark.parametrize("s", [1, 2, 999, 1001, 2048, 4095, 4096, 4097, 8191, 8192])
def test_sketch_sizes_up_to_the_limit(gpu, oracle, s):
    # ~750 000 distinct k-mers in four device chunks (four kernel passes): from the second pass on, each chunk's threshold is
    # capped at the running s-th smallest hash (t_cap), and the merge sorts up to 2 s = 16384 keys in shared memory
    k = 21
    p = gpu.params(k=k, s=s); po = oracle.params(k=k)
    if not _SIZES:
        genomes = [synth_genome(500 + i, 400_000) for i in range(2)]
        _SIZES["genomes"] = genomes + [mutate(genomes[0], 0.02, 502), synth_genome(503, 100_000)]
        _SIZES["chunks"] = join(make_reads(genomes, 20_000, seed=504, lower=0.0), 5000)
    chunks = _SIZES["chunks"]
    assert len(chunks) == 4
    ref, ref_n = sketch_rows(oracle, po, _SIZES["genomes"], s)
    want = oracle.screen(ref, ref_n, chunks, po, s=s)
    assert want["mixture"].size == s
    res, cnt = run(gpu, ref, ref_n, p, chunks, feed="dev")
    check_all(res, cnt, want)


def test_sketch_size_above_8192_is_refused(gpu, oracle):
    ref = np.arange(1, 11, dtype=np.uint64)[None, :] << np.uint64(40)
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.screen_open(ref, np.array([10], np.uint32), gpu.params(k=21, s=8193))
    assert e.value.code == ERR_UNSUPPORTED
    clean_context_screen(gpu, oracle)


# ---- 3. table scale, probe runs, reference shapes ------------------------------------------------------------------

def graded_rows(n, s, seed):
    """n full sketches of genomes of 0.3-10 Mbp (log-uniform): sorted distinct draws below 2^64 s / L, so the density of
    the rows grades like a real collection's."""
    rng = np.random.Generator(np.random.PCG64(seed))
    L = np.exp(rng.uniform(np.log(3e5), np.log(1e7), n))
    hi = (2.0**64 * s / L).astype(np.uint64)
    H = rng.integers(0, hi[:, None], size=(n, s), dtype=np.uint64)
    H.sort(axis=1)
    return H


def _scale_case(oracle, po, n_graded, seed):
    s = 1000
    genomes = [synth_genome(600 + i, 100_000) for i in range(3)]
    tiny = [synth_genome(610 + i, 200 + 50 * i) for i in range(4)]         # hashes up to ~2^64: every k-mer meets the bitmap
    ref_g, n_g = sketch_rows(oracle, po, genomes + tiny, s)
    ref = np.concatenate([graded_rows(n_graded, s, seed), ref_g])
    ref_n = np.concatenate([np.full(n_graded, s, np.uint32), n_g])
    chunks = join(make_reads(genomes + tiny[:2], 4000, seed=seed + 1), 1000)
    return ref, ref_n, chunks, oracle.screen(ref, ref_n, chunks, po, s=s)


@pytest.mark.parametrize("n_graded,bits", [(400, 21), (800, 22)])
def test_table_scale_bitmap_sizes(gpu, oracle, n_graded, bits):
    p = gpu.params(k=21, s=1000); po = oracle.params(k=21)
    ref, ref_n, chunks, want = _scale_case(oracle, po, n_graded, seed=620 + bits)
    assert bits_log2(want["keys"].size) == bits
    res, cnt = run(gpu, ref, ref_n, p, chunks)
    check_all(res, cnt, want)
    assert want["shared"][-7:-4].min() > 0


@pytest.fixture(scope="module")
def capped_table(oracle):
    """>= 2^25 distinct keys (270 MB of rows): the presence bitmap at its 2^27-bit cap, a table of 2^27 slots."""
    po = oracle.params(k=21)
    return _scale_case(oracle, po, 33_560, seed=640)


@pytest.mark.parametrize("bitmap", ["1", "0"])
def test_table_scale_bitmap_at_its_cap(gpu, oracle, monkeypatch, capped_table, bitmap):
    monkeypatch.setenv("MASHGPU_SCREEN_BITMAP", bitmap)
    ref, ref_n, chunks, want = capped_table
    assert want["keys"].size >= 2**25 and bits_log2(want["keys"].size) == 27
    assert ceil_log2(2 * ref.size + 2) >= 26
    res, cnt = run(gpu, ref, ref_n, gpu.params(k=21, s=1000), chunks)
    check_all(res, cnt, want)
    assert want["shared"][-7:-4].min() > 0


def home_slot(key, log2cap):
    return ((key * GOLDEN_RATIO_64) % 2**64) >> (64 - log2cap)


def key_with_home(slot, log2cap, j):
    """slot_hash is invertible: the key whose product with the multiplier is (slot << (64 - log2cap)) + j."""
    inv = pow(GOLDEN_RATIO_64, -1, 2**64)
    return (inv * ((slot << (64 - log2cap)) + j)) % 2**64


@pytest.mark.parametrize("bitmap,winner", [("1", False), ("0", False), ("0", True)])
def test_probe_run_wrapping_past_the_last_slot(gpu, oracle, monkeypatch, bitmap, winner):
    # 1000 synthetic keys on consecutive slots [cap - 500, cap) + [0, 500): real reference hashes whose home slot lies in the
    # run are inserted behind it, so their hits need probes that wrap through the last slot, in the scan (screen_probe_lanes),
    # the reduce and the winner kernel; misses homed in the run walk to its end (without the bitmap every k-mer probes)
    monkeypatch.setenv("MASHGPU_SCREEN_BITMAP", bitmap)
    k, s = 21, 1000
    p = gpu.params(k=k, s=s); po = oracle.params(k=k)
    genomes = [synth_genome(700 + i, 150_000) for i in range(3)]
    genomes.append(mutate(genomes[0], 0.03, 703))
    real, real_n = sketch_rows(oracle, po, genomes, s)
    ref = np.concatenate([real, np.zeros((1, s), np.uint64)]); ref_n = np.concatenate([real_n, [s]]).astype(np.uint32)
    log2cap = max(4, ceil_log2(2 * ref.size + 2))
    cap = 1 << log2cap
    run_slots = [(cap - 500 + i) % cap for i in range(1000)]
    rng = np.random.Generator(np.random.PCG64(704))
    taken = set(int(x) for x in real[real != np.uint64(EMPTY)])
    synth = []
    for sl in run_slots:
        while True:
            key = key_with_home(sl, log2cap, int(rng.integers(0, 1 << (64 - log2cap))))
            if key != EMPTY and key not in taken:
                break
        assert home_slot(key, log2cap) == sl
        synth.append(key)
    ref[-1] = np.sort(np.array(synth, np.uint64))
    lengths = np.array([150_000, 150_001, 150_002, 150_003, 1], np.uint64)
    chunks = join(make_reads(genomes[:2], 6000, seed=705), 2000)
    want = oracle.screen(ref, ref_n, chunks, po, s=s, winner=winner, ref_len=lengths)
    in_run = set(run_slots)
    behind = [i for i, key in enumerate(want["keys"]) if int(key) in taken and home_slot(int(key), log2cap) in in_run]
    assert sum(1 for i in behind if want["counts"][i] > 0) >= 20
    assert any(home_slot(int(want["keys"][i]), log2cap) >= cap - 500 for i in behind if want["counts"][i] > 0)
    res, cnt = run(gpu, ref, ref_n, p, chunks, winner=winner, ref_len=lengths)
    check_all(res, cnt, want)


_SHAPES = {}


def _shape_data(oracle, po):
    if not _SHAPES:
        genomes = [synth_genome(800 + i, 150_000) for i in range(3)]
        _SHAPES["genomes"] = genomes
        _SHAPES["pool"] = np.unique(np.concatenate([oracle.sketch_unit([bytes(g)], po, s=1000)[0] for g in genomes]))
        _SHAPES["chunks"] = join(make_reads(genomes, 20_000, seed=810, lower=0.0), 5000)
    return _SHAPES["genomes"], _SHAPES["pool"], _SHAPES["chunks"]


def reference_shape(name, oracle, po):
    genomes, pool, _ = _shape_data(oracle, po)
    rng = np.random.Generator(np.random.PCG64(820))
    if name == "no_sketches":
        return np.zeros((0, 100), np.uint64), np.zeros(0, np.uint32)
    if name == "all_rows_empty":
        return np.full((5, 100), np.uint64(EMPTY)), np.zeros(5, np.uint32)
    if name == "ragged":
        ref, ref_n = sketch_rows(oracle, po, genomes * 3, 1000)
        ref_n[:] = [0, 1, 2, 17, 1000, 999, 0, 1, 500]
        return ref, ref_n
    if name in ("one_hash_in_5000_rows", "20000_rows_of_50"):
        n, w = (5000, 20) if name == "one_hash_in_5000_rows" else (20_000, 50)
        ref = np.full((n, w), np.uint64(EMPTY)); ref_n = np.zeros(n, np.uint32)
        common = pool[len(pool) // 2]
        for r in range(n):
            v = np.concatenate([rng.choice(pool, w // 2, replace=False), rng.integers(0, 2**63, w - w // 2, dtype=np.uint64)])
            if name == "one_hash_in_5000_rows":
                v[0] = common
            v = np.unique(v)
            ref[r, :v.size] = v; ref_n[r] = v.size
        return ref, ref_n
    if name in ("rows_of_32768", "stride_40000"):
        stride = 32768 if name == "rows_of_32768" else 40_000
        ref, ref_n = sketch_rows(oracle, po, genomes[:2] + [mutate(genomes[2], 0.02, 821)], 32768, stride=stride)
        assert (ref_n == 32768).all()
        if name == "stride_40000":
            ref_n[2] = 20_000
        return ref, ref_n
    raise ValueError(name)


@pytest.mark.parametrize("name", ["no_sketches", "all_rows_empty", "ragged", "one_hash_in_5000_rows", "20000_rows_of_50",
                                  "rows_of_32768", "stride_40000"])
def test_reference_shapes(gpu, oracle, name):
    # rows of 32768 hashes sort up to 32768 depths in 128 KB of shared memory; a stride of 40000 with shorter rows is accepted
    # (the reduce is sized by the largest row); 20 000 rows make a reduce grid of 20 000 CTAs
    s = 1000
    p = gpu.params(k=21, s=s); po = oracle.params(k=21)
    _, _, chunks = _shape_data(oracle, po)
    ref, ref_n = reference_shape(name, oracle, po)
    want = oracle.screen(ref, ref_n, chunks, po, s=s)
    res, cnt = run(gpu, ref, ref_n, p, chunks)
    check_all(res, cnt, want)
    if name == "one_hash_in_5000_rows":
        assert want["shared"].min() > 0
    if name in ("rows_of_32768", "stride_40000"):
        assert want["shared"].min() > 10_000


# ---- 4. multi-rank merge on one GPU --------------------------------------------------------------------------------

_MULTI = {}


def _multi_case(oracle, s):
    """Reference sketches at 1000, and 60 chunks of 1..150 reads; chunk 0 (one read of 150 bases, 130 k-mers) is the only
    input of one job, so mixture counts are ragged."""
    po = oracle.params(k=21)
    if "chunks" not in _MULTI:
        genomes = [synth_genome(1000 + i, 200_000) for i in range(3)]
        reads = make_reads(genomes[:2], 5000, seed=1003, lower=0.0)
        sizes = [(i * 37) % 150 + 1 for i in range(1, 60)]
        bounds = np.cumsum([0] + sizes)
        _MULTI["chunks"] = [b"*" + bytes(genomes[0][5000:5150])] + \
            [b"".join(b"*" + r for r in reads[bounds[i]:bounds[i + 1]]) for i in range(59)]
        _MULTI["refs"] = sketch_rows(oracle, po, genomes + [mutate(genomes[0], 0.02, 1004)], 1000)
    if s not in _MULTI:
        ref, ref_n = _MULTI["refs"]
        _MULTI[s] = oracle.screen(ref, ref_n, _MULTI["chunks"], po, s=s)
    return _MULTI["refs"] + (_MULTI["chunks"], _MULTI[s])


def _sharded_jobs(gpu, ref, ref_n, p, chunks, W):
    """W jobs on one context; chunk 0 goes to job W-2 alone, the others round robin to jobs 0..W-3; job W-1 gets nothing.
    Their counters are summed into every job."""
    import torch
    jobs = [gpu.screen_open(ref, ref_n, p) for _ in range(W)]
    feed_dev(jobs[W - 2], chunks[0])
    for i, c in enumerate(chunks[1:]):
        feed_dev(jobs[i % (W - 2)], c)
    views = [_dev_view(*j.counters(), "<i4") for j in jobs]
    total = torch.stack(views).sum(0, dtype=torch.int32)
    for v in views:
        v.copy_(total)
    torch.cuda.synchronize()
    return jobs


@pytest.mark.parametrize("s,W", [(1, 70), (200, 70), (1000, 20), (8192, 3)])
def test_merge_mixtures_dev_over_many_jobs(gpu, oracle, s, W):
    # W lists in more launches than one (per_launch = min(64, 2^14 / s - 1) lists), stride > s, ragged and zero counts
    import torch
    ref, ref_n, chunks, want = _multi_case(oracle, s)
    jobs = _sharded_jobs(gpu, ref, ref_n, gpu.params(k=21, s=s), chunks, W)
    try:
        stride = s + 3
        lists = torch.zeros((W, stride), dtype=torch.int64, device="cuda:0")
        counts = torch.zeros(W, dtype=torch.int32, device="cuda:0")
        for w, j in enumerate(jobs):
            mp, mnp = j.mixture_dev()
            lists[w, :s] = _dev_view(mp, s, "<i8")
            counts[w] = _dev_view(mnp, 1, "<i4")[0]
        torch.cuda.synchronize()
        c = counts.cpu().numpy()
        assert c[-1] == 0 and c.max() == s
        if s > 1:
            assert 0 < c[-2] < s
        for j in jobs:
            j.merge_mixtures_dev(lists.data_ptr(), counts.data_ptr(), W, stride)
        for j in jobs:
            check_all(j.finish(), counters(j), want)
    finally:
        for j in jobs:
            j.close()


def test_merge_mixture_host_lists(gpu, oracle):
    # the host entry point: every job folds in every list, its own (fully overlapping) and the empty one (n = 0) included
    import torch
    s, W = 200, 5
    ref, ref_n, chunks, want = _multi_case(oracle, s)
    jobs = _sharded_jobs(gpu, ref, ref_n, gpu.params(k=21, s=s), chunks, W)
    try:
        lists = []
        for j in jobs:
            mp, mnp = j.mixture_dev()
            n = int(_dev_view(mnp, 1, "<i4")[0])
            lists.append(_dev_view(mp, s, "<i8")[:n].cpu().numpy().view(np.uint64).copy())
        assert lists[-1].size == 0 and 0 < lists[-2].size < s
        for j in jobs:
            for lst in lists:
                j.merge_mixture(lst)
        for j in jobs:
            check_all(j.finish(), counters(j), want)
        with pytest.raises(mash_b200.MashGpuError) as e:
            jobs[0].merge_mixture(np.arange(1, s + 2, dtype=np.uint64))
        assert e.value.code == ERR_INVALID
        short = torch.zeros((1, s - 1), dtype=torch.int64, device="cuda:0")
        one = torch.ones(1, dtype=torch.int32, device="cuda:0")
        torch.cuda.synchronize()
        with pytest.raises(mash_b200.MashGpuError) as e:
            jobs[0].merge_mixtures_dev(short.data_ptr(), one.data_ptr(), 1, s - 1)
        assert e.value.code == ERR_INVALID
        check_all(jobs[0].finish(), counters(jobs[0]), want)         # the refused calls changed nothing
    finally:
        for j in jobs:
            j.close()


@pytest.mark.parametrize("s,W", [(1, 70), (7, 200), (1000, 40), (8192, 5)])
def test_merge_kernel_against_numpy(gpu, s, W):
    # random ascending lists drawn from a shared pool (so they overlap), lengths 0..s, folded twice into one running list
    import torch
    rng = np.random.Generator(np.random.PCG64(1100 + s))
    pool = np.unique(rng.integers(0, 2**64 - 1, 3 * s + 10, dtype=np.uint64))
    job = gpu.screen_open(np.ones((1, 1), np.uint64), np.ones(1, np.uint32), gpu.params(k=21, s=s))
    try:
        seen = []
        for _ in range(2):
            stride = s + 1
            host = np.zeros((W, stride), np.uint64); n = np.zeros(W, np.int32)
            for w in range(W):
                m = int(rng.integers(0, s + 1)) if w % 7 else (0 if w % 14 else s)
                v = np.sort(rng.choice(pool, m, replace=False))
                host[w, :m] = v; n[w] = m
                seen.append(v)
            lists = torch.from_numpy(host.view(np.int64)).to("cuda:0"); counts = torch.from_numpy(n).to("cuda:0")
            torch.cuda.synchronize()
            job.merge_mixtures_dev(lists.data_ptr(), counts.data_ptr(), W, stride)
            assert np.array_equal(job.mixture(), np.unique(np.concatenate(seen))[:s])
    finally:
        job.close()


# ---- 5. job lifecycle on one context -------------------------------------------------------------------------------

@pytest.mark.parametrize("host_pack", ["0", "1"])
def test_two_jobs_alternate_on_one_context(gpu, oracle, monkeypatch, host_pack):
    # job A (k=21, s=1000) takes the context's staging pair at its first feed, job B (k=12, s=300) allocates its own; A is
    # closed while B is mid-stream, and B's next chunks take over the context's pair
    monkeypatch.setenv("MASHGPU_SCREEN_HOST_PACK", host_pack)
    ref_a, n_a, _, want_a = _big_case(oracle, 21, 1000, (0, 2))
    ref_b, n_b, chunks_b, want_b = _big_case(oracle, 12, 300, (1, 3, 0, 2))
    idle = gpu.screen_open(ref_a, n_a, gpu.params(k=21, s=1000))
    idle.close()                                               # opened and closed without a feed
    a = gpu.screen_open(ref_a, n_a, gpu.params(k=21, s=1000))
    b = gpu.screen_open(ref_b, n_b, gpu.params(k=12, s=300))
    try:
        _, chunks = _big_chunks()
        a.feed(chunks[0]); b.feed(chunks[1]); a.feed(chunks[2]); b.feed(chunks[3])
        assert np.array_equal(counters(a), want_a["counts"])         # before finish
        res = a.finish()
        check(res, want_a)
        check(a.finish(), want_a)                                    # finish is repeatable
        a.close()
        b.feed(chunks[0]); b.feed(chunks[2])
        assert np.array_equal(counters(b), want_b["counts"])
        check_all(b.finish(), counters(b), want_b)
    finally:
        a.close(); b.close()


# ---- 6. refusals, each followed by an ordinary screen on the same context ------------------------------------------

def _refused_set(name, gpu, oracle, keep):
    if name in ("hash_above_2_32_dna", "hash_above_2_32_bytes"):
        if name == "hash_above_2_32_dna":
            p, po = gpu.params(k=12, s=100), oracle.params(k=12)
            h, _, _ = oracle.sketch_unit([bytes(synth_genome(1200, 20_000))], po, s=100)
        else:
            p = gpu.params(k=10, s=100, alphabet="ABCDEFGH", noncanonical=True)      # 8^10 = 2^30 k-mers: 32-bit hashes
            h = np.arange(1, 100, dtype=np.uint64) << np.uint64(20)
        assert p.use64 == 0
        row = np.sort(np.append(h[:-1], np.uint64(2**32 + 5)))
        return p, _Set(row[None, :], np.array([row.size], np.uint32)), ERR_INVALID
    if name == "n_hashes_above_stride_host":
        ref = np.arange(1, 101, dtype=np.uint64).reshape(2, 50) << np.uint64(40)
        return gpu.params(k=21, s=100), _Set(ref, np.array([50, 51], np.uint32)), ERR_INVALID
    if name == "n_hashes_above_stride_device":
        import torch
        h = (torch.arange(1, 101, dtype=torch.int64) << 40).reshape(2, 50).to("cuda:0")
        n = torch.tensor([51, 50], dtype=torch.int32, device="cuda:0")
        torch.cuda.synchronize()
        keep += [h, n]
        return gpu.params(k=21, s=100), _Set(h.data_ptr(), n.data_ptr(), None, on_device=True, n=2, stride=50), ERR_INVALID
    if name in ("row_of_32769_k12", "row_of_32769_k21"):
        k = 12 if name.endswith("k12") else 21
        rng = np.random.Generator(np.random.PCG64(1201))
        row = np.unique(rng.integers(0, 2**32 if k == 12 else 2**63, 40_000, dtype=np.uint64))[:32769]
        return gpu.params(k=k, s=1000), _Set(row[None, :], np.array([32769], np.uint32)), ERR_UNSUPPORTED
    raise ValueError(name)


@pytest.mark.parametrize("name", ["hash_above_2_32_dna", "hash_above_2_32_bytes", "n_hashes_above_stride_host",
                                  "n_hashes_above_stride_device", "row_of_32769_k12", "row_of_32769_k21"])
def test_open_refuses_before_building_the_table(gpu, oracle, name):
    keep = []
    p, refs, code = _refused_set(name, gpu, oracle, keep)
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.screen_open(refs, None, p)
    assert e.value.code == code
    clean_context_screen(gpu, oracle)


def test_32bit_job_accepts_the_largest_32bit_hash(gpu, oracle):
    # the bound of the refusal above: 2^32 - 1 is a valid key of a k <= 16 job (the bitmap's last bit)
    s = 300
    p = gpu.params(k=12, s=s); po = oracle.params(k=12)
    genomes = [synth_genome(1300 + i, 60_000) for i in range(2)]
    ref, ref_n = sketch_rows(oracle, po, genomes, s, stride=s + 1)
    ref[1, ref_n[1]] = 2**32 - 1; ref_n[1] += 1
    chunks = join(make_reads(genomes, 3000, seed=1302), 1000)
    want = oracle.screen(ref, ref_n, chunks, po, s=s)
    res, cnt = run(gpu, ref, ref_n, p, chunks)
    check_all(res, cnt, want)
