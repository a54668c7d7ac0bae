"""GPU tests for the block tables of the filter-word scan kernels (k = 17..32, mash_b200/csrc/scan.cuh: CodeTables,
fill_code_tables, code_filter_word).  The fast path takes the first multiply of every MurmurHash3 block lane from shared
memory tables indexed by one byte of 2-bit codes, that is by one 4-base group of the canonical k-mer; a wrong entry would
make the filter drop windows whose hash belongs in the sketch.  So the thresholds here are selective, the input is half
clean and half dirty (N runs, single IUPAC bytes, lower case), and each case checks, with a numpy restatement of
MurmurHash3 on the k-mers the sketch keeps, that every one of the 256 group values occurs in each of the four byte
positions of block 0 among them, and every value the tail's groups can take, so that each table entry the kernel reads is
one a kept hash depends on."""
import numpy as np
import pytest

from fixtures import synth_genome

pytestmark = pytest.mark.gpu

C1, C2 = np.uint64(0x87c37b91114253d5), np.uint64(0x4cf5ad432745937f)
ASCII = np.frombuffer(b"ACGT", np.uint8)


def _rotl(x, r):
    return (x << np.uint64(r)) | (x >> np.uint64(64 - r))


def _fmix(k):
    k ^= k >> np.uint64(33)
    k *= np.uint64(0xff51afd7ed558ccd)
    k ^= k >> np.uint64(33)
    k *= np.uint64(0xc4ceb9fe1a85ec53)
    k ^= k >> np.uint64(33)
    return k


def _lane(keys, lo, hi):
    # little-endian 64-bit word of key bytes lo..hi-1 (zero bytes past the key)
    w = np.zeros(keys.shape[0], np.uint64)
    for i in range(lo, min(hi, keys.shape[1])):
        w |= keys[:, i].astype(np.uint64) << np.uint64(8 * (i - lo))
    return w


def murmur3_h1(keys, seed=42):
    """h1 of MurmurHash3_x64_128 of every row of `keys` (uint8, one k-mer per row), vectorised."""
    n = keys.shape[1]
    with np.errstate(over="ignore"):
        h1 = np.full(keys.shape[0], seed, np.uint64)
        h2 = h1.copy()
        for b in range(n // 16):
            h1 ^= _rotl(_lane(keys, 16 * b, 16 * b + 8) * C1, 31) * C2
            h1 = (_rotl(h1, 27) + h2) * np.uint64(5) + np.uint64(0x52dce729)
            h2 ^= _rotl(_lane(keys, 16 * b + 8, 16 * b + 16) * C2, 33) * C1
            h2 = (_rotl(h2, 31) + h1) * np.uint64(5) + np.uint64(0x38495ab5)
        t = 16 * (n // 16)
        if n - t > 8:
            h2 ^= _rotl(_lane(keys, t + 8, n) * C2, 33) * C1
        if n > t:
            h1 ^= _rotl(_lane(keys, t, min(n, t + 8)) * C1, 31) * C2
        h1 ^= np.uint64(n)
        h2 ^= np.uint64(n)
        h1 += h2
        h2 += h1
        return _fmix(h1) + _fmix(h2)


def _canonical(win):
    rc = (3 - win)[:, ::-1]
    # memcmp order of the ASCII k-mers = order of the base-4 numbers, first base most significant
    weights = np.uint64(4) ** np.arange(win.shape[1] - 1, -1, -1, dtype=np.uint64)
    fwd_v = (win.astype(np.uint64) * weights).sum(axis=1, dtype=np.uint64)
    rc_v = (rc.astype(np.uint64) * weights).sum(axis=1, dtype=np.uint64)
    return np.where((rc_v < fwd_v)[:, None], rc, win)


def canonical_kmers(seq, k):
    """Codes (one row per window, k columns) of the canonical k-mer of every window in the alphabet, upper-cased."""
    u = seq & 0xDF
    code = np.full(seq.size, 255, np.uint8)
    for c, ch in enumerate(b"ACGT"):
        code[u == ch] = c
    win = np.lib.stride_tricks.sliding_window_view(code, k)
    return _canonical(win[(win != 255).all(axis=1)])


def _crafted(k, missing, below, seed):
    """One k-mer per (group start, value) whose canonical form has that value there and whose hash is below `below`: the
    group and its mirror image are reverse complements of each other, so both strands carry the value (random input
    rarely has a canonical k-mer that starts with T or ends with A)."""
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for st, v in missing:
        cand = rng.integers(0, 4, (8192, k)).astype(np.uint8)
        for i in range(min(4, k - st)):
            cand[:, st + i] = (v >> (2 * i)) & 3
            cand[:, k - 1 - st - i] = 3 - ((v >> (2 * i)) & 3)
        h = murmur3_h1(ASCII[_canonical(cand)])
        j = int(np.argmin(h))
        assert h[j] < below, (st, v)
        out.append(ASCII[cand[j]])
    return out


def _dirty(seed, n):
    # the first half is ACGT alone (the kernels' code-only staging of clean tiles), the second half has N runs, single IUPAC
    # bytes and lower case (staging with the validity test)
    g = synth_genome(seed, n, n_runs=2, lower_frac=0.1)
    g[:n // 2] = synth_genome(seed + 2, n // 2)
    rng = np.random.Generator(np.random.PCG64(seed + 1))
    pos = rng.integers(n // 2, n, n // 422)
    g[pos] = np.frombuffer(b"NnRY", np.uint8)[rng.integers(0, 4, pos.size)]
    return g


def _group_values(codes, start, k):
    # byte of 2-bit codes of bases start..start+3 (base start at bits 0-1), bases past k absent
    v = np.zeros(codes.shape[0], np.int64)
    for i in range(start, min(start + 4, k)):
        v |= codes[:, i].astype(np.int64) << (2 * (i - start))
    return v


def _missing(kmers, k):
    return [(st, v) for st in range(0, k, 4)
            for v in np.setdiff1d(np.arange(4 ** min(4, k - st)), _group_values(kmers, st, k))]


@pytest.mark.parametrize("k", list(range(17, 33)))
def test_block_tables_every_group_value(gpu, oracle, k):
    s = 6000
    g = _dirty(4242 + k, 600_000)
    po = oracle.params(k=k)
    # random input leaves some values of the first and last groups out of the kept k-mers: add a window for each, separated
    # by N, with a hash well inside the sketch (values are counted as present only with a margin of 64 places below the
    # threshold, which the added windows cannot take away)
    oh, _, _ = oracle.sketch_unit([bytes(g)], po, s=s)
    kmers = canonical_kmers(g, k)
    missing = _missing(kmers[murmur3_h1(ASCII[kmers]) <= oh[-65]], k)
    assert len(missing) < 64
    extra = _crafted(k, missing, oh[-1] // np.uint64(4), 99 + k)
    g = np.concatenate([g] + [np.concatenate([np.frombuffer(b"N", np.uint8), x]) for x in extra])

    p = gpu.params(k=k, s=s)
    out = gpu.sketch([bytes(g)], p, unit_of_record=[0], n_units=1)
    oh, _, _ = oracle.sketch_unit([bytes(g)], po, s=s)
    assert oh.size == s, "the threshold must be selective"
    assert out[1][0] == oh.size and np.array_equal(out[0][0, :out[1][0]], oh)

    # the same sketch from the packed source
    codes, runs, starts = gpu.host_pack([bytes(g)], p, threads=2)
    unit_start = np.array([0, starts[-1]], np.uint64)
    h, n, _ = gpu.sketch_packed(codes, int(starts[-1]), runs, unit_start, p, counts=True)
    assert n[0] == oh.size and np.array_equal(h[0, :n[0]], oh)

    # the kept k-mers: the restated hash reproduces the oracle's sketch, and among them every value of every 4-base group
    # occurs (block 0: all 256 in each of the four byte positions; the tail's groups: every value they can take)
    kmers = canonical_kmers(g, k)
    hashes = murmur3_h1(ASCII[kmers])
    kept = hashes <= oh[-1]
    assert np.array_equal(np.unique(hashes[kept]), oh)
    assert _missing(kmers[kept], k) == []
