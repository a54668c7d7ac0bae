"""GPU tests of the clean-tile staging of the filter-word scan kernels (k = 17..32, ASCII source): a warp tile whose 1024
bytes and 64 halo bytes are all A/C/G/T (or a/c/g/t, upper-cased) is converted to codes only and checked with one vote; a
tile with any other byte is converted again with the per-byte validity test.  Each case puts a single dirty byte where
the check has to see it -- the tile's first byte, its last body byte, the first and the last byte of each halo word --
in otherwise clean tiles, and compares every window with the oracle (keep-all, through hash_windows) and keep-all
sketches of the device stream path."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

KS = [17, 21, 24, 25, 32]
TILE = 1024          # window starts per warp tile
HALO = 64            # halo bytes staged past a warp tile (8 words of 8 bytes)
ACGT = np.frombuffer(b"ACGT", np.uint8)
# tile offsets of the single dirty byte: the first byte, the last body byte, the first and last byte of each halo word
# (a halo byte of tile t is byte offset - 1024 of tile t + 1, so it is checked once in each)
OFFSETS = [0, TILE - 1] + [TILE + 8 * w for w in range(8)] + [TILE + 8 * w + 7 for w in range(8)]
DIRTY = b"NnR*.\x00\x80\xff"


def _clean(seed, n):
    rng = np.random.Generator(np.random.PCG64(seed))
    return ACGT[rng.integers(0, 4, n)]


def _one_dirty_byte_per_tile(seed, lower=False):
    """Two clean tiles around every dirty tile: each offset in OFFSETS gets its own tile, and each byte of DIRTY is used."""
    g = _clean(seed, (3 * len(OFFSETS) + 2) * TILE)
    for i, off in enumerate(OFFSETS):
        g[3 * (i + 1) * TILE + off - (TILE if off >= TILE else 0)] = DIRTY[i % len(DIRTY)]
    if lower:
        g = np.where((g >= 65) & (g <= 90), g + 32, g).astype(np.uint8)
    return g


def _check_windows(gpu, oracle, seq, p, po):
    h, v = gpu.hash_windows(seq, p)
    want = oracle.all_hashes(bytes(seq), po)
    assert int(v.sum()) == want.size and np.array_equal(h[v], want)


def _sketch_dev(gpu, p, s, flat, unit_start):
    # device stream followed by 256 valid bases: a byte past the end read as a base changes the last unit's sketch
    import torch
    pad = ACGT[np.arange(256) % 4]
    dev = torch.from_numpy(np.concatenate([flat, pad])).cuda()
    n_units = len(unit_start) - 1
    d_h = torch.zeros((n_units, s), dtype=torch.int64, device="cuda")
    d_n = torch.zeros(n_units, dtype=torch.int32, device="cuda")
    gpu.sketch_stream_dev(p, dev.data_ptr(), np.asarray(unit_start, np.uint64), d_h.data_ptr(), d_n.data_ptr())
    torch.cuda.synchronize()
    return d_h.cpu().numpy().view(np.uint64), d_n.cpu().numpy()


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
def test_one_dirty_byte_in_clean_tiles(gpu, oracle, k, noncanonical):
    p = gpu.params(k=k, noncanonical=noncanonical)
    po = oracle.params(k=k, noncanonical=noncanonical)
    _check_windows(gpu, oracle, _one_dirty_byte_per_tile(40 + k), p, po)
    _check_windows(gpu, oracle, _clean(41 + k, 9 * TILE + HALO), p, po)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
@pytest.mark.parametrize("preserve_case", [False, True])
def test_lower_case_tiles(gpu, oracle, k, noncanonical, preserve_case):
    # all lower case: clean after upper-casing, every byte outside the alphabet under preserve_case; plus tiles that mix the
    # cases, and the single dirty bytes in lower-case tiles
    p = gpu.params(k=k, noncanonical=noncanonical, preserve_case=preserve_case)
    po = oracle.params(k=k, noncanonical=noncanonical, preserve_case=preserve_case)
    low = _clean(60 + k, 6 * TILE + 100) + 32
    _check_windows(gpu, oracle, low, p, po)
    mixed = _clean(61 + k, 6 * TILE + 100)
    mixed[2 * TILE:3 * TILE] += 32              # one lower-case tile between upper-case ones
    mixed[4 * TILE + 500] += 32                 # one lower-case byte
    _check_windows(gpu, oracle, mixed, p, po)
    _check_windows(gpu, oracle, _one_dirty_byte_per_tile(62 + k, lower=True), p, po)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
def test_separators_and_stream_ends_in_the_halo(gpu, oracle, k, noncanonical):
    # keep-all units of clean bases back to back, each ended by a separator, with unit boundaries and separators at a tile's
    # first byte, its last body byte and inside the halo; then streams whose end falls inside the last tile's halo
    s = 6000
    p = gpu.params(k=k, s=s, noncanonical=noncanonical)
    po = oracle.params(k=k, noncanonical=noncanonical)
    ends = [TILE, 2 * TILE + TILE - 1, 3 * TILE + TILE + 5, 5 * TILE + TILE + HALO - 1, 7 * TILE + 1, 9 * TILE + 333]
    starts = [0] + ends[:-1]
    seqs = [_clean(700 * k + u, e - b) for u, (b, e) in enumerate(zip(starts, ends))]
    for q in seqs:
        q[-1] = ord("*")
    h, n = _sketch_dev(gpu, p, s, np.concatenate(seqs), starts + [ends[-1]])
    for u, q in enumerate(seqs):
        oh, _, _ = oracle.sketch_unit([bytes(q)], po, s=s)
        assert n[u] == oh.size and np.array_equal(h[u, :n[u]], oh), u
    g = _clean(800 + k, 5 * TILE + HALO)
    for n_end in [4 * TILE, 4 * TILE + 1, 4 * TILE + 8, 4 * TILE + 31, 4 * TILE + HALO - 1, 4 * TILE - 1]:
        h, cnt = _sketch_dev(gpu, p, s, g[:n_end], [0, n_end])
        oh, _, _ = oracle.sketch_unit([bytes(g[:n_end])], po, s=s)
        assert cnt[0] == oh.size and np.array_equal(h[0, :cnt[0]], oh), n_end
    _check_windows(gpu, oracle, g[:4 * TILE + 37], p, po)
