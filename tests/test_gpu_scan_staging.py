"""GPU tests aimed at the staging of the filter-word scan kernels (k = 17..32, ASCII source): a warp tile's 1024 window
starts plus its 8 halo words (bytes 1024..1087 of the tile, converted 8 bytes at a time), the guard-free conversion of
tiles that lie wholly before the end of the stream, and the guarded conversion of the last tile of a launch.  Every byte
class goes through the halo: A/C/G/T, a/c/g/t with and without preserve_case, N, separators and bytes >= 0x80.  Everything
is checked bit-exact against the oracle."""
import numpy as np
import pytest

from fixtures import synth_genome

pytestmark = pytest.mark.gpu

KS = [17, 21, 24, 25, 32]
TILE = 1024          # window starts per warp tile
HALO = 64            # halo bytes staged past a warp tile
JUNK = np.frombuffer(b"NnRYacgt*-.\x00\x80\xff\xc3\x41\x7f", np.uint8)


def _halo_dirty(seed, n):
    """A genome with every byte class placed at the halo offsets (position mod 1024 < 64) and nowhere else."""
    g = synth_genome(seed, n)
    rng = np.random.Generator(np.random.PCG64(seed))
    pos = np.arange(n)
    halo = pos[(pos % TILE) < HALO]
    pick = halo[rng.random(halo.size) < 0.15]
    g[pick] = JUNK[rng.integers(0, JUNK.size, pick.size)]
    lower = halo[rng.random(halo.size) < 0.2]
    g[lower] = np.where((g[lower] >= 65) & (g[lower] <= 90), g[lower] + 32, g[lower])
    for t in range(0, n - TILE, 3 * TILE):        # an N run across a halo every third tile
        g[t + TILE - 5:t + TILE + 9] = ord("N")
    return g


def _check_windows(gpu, oracle, seq, p, po):
    h, v = gpu.hash_windows(seq, p)
    want = oracle.all_hashes(bytes(seq), po)
    assert int(v.sum()) == want.size and np.array_equal(h[v], want)


def _sketch_dev(gpu, p, s, flat, unit_start):
    # device stream followed by 256 valid bases: a byte past the end read as a base changes the last unit's sketch
    import torch
    pad = np.frombuffer(b"ACGT", np.uint8)[np.arange(256) % 4]
    dev = torch.from_numpy(np.concatenate([flat, pad])).cuda()
    n_units = len(unit_start) - 1
    d_h = torch.zeros((n_units, s), dtype=torch.int64, device="cuda")
    d_n = torch.zeros(n_units, dtype=torch.int32, device="cuda")
    gpu.sketch_stream_dev(p, dev.data_ptr(), np.asarray(unit_start, np.uint64), d_h.data_ptr(), d_n.data_ptr())
    torch.cuda.synchronize()
    return d_h.cpu().numpy().view(np.uint64), d_n.cpu().numpy()


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
def test_stream_end_at_every_halo_offset(gpu, oracle, k, noncanonical):
    # a keep-all unit whose stream ends in the last full tile's halo, at each offset 0..15 of a halo vector and in each of
    # its 4 vectors, and around the tile's own boundary: the guarded conversion must make every byte at or past the end a
    # separator, and the tiles before it take the guard-free path
    s = 6000
    p = gpu.params(k=k, s=s, noncanonical=noncanonical)
    po = oracle.params(k=k, noncanonical=noncanonical)
    g = synth_genome(7000 + k, 5 * TILE + HALO)
    lens = [4 * TILE + 16 * vec + off for vec in range(4) for off in range(16)]
    lens += [4 * TILE - 1, 3 * TILE + k - 1, 3 * TILE + k]
    for n in lens:
        h, cnt = _sketch_dev(gpu, p, s, g[:n], [0, n])
        oh, _, _ = oracle.sketch_unit([bytes(g[:n])], po, s=s)
        assert cnt[0] == oh.size and np.array_equal(h[0, :cnt[0]], oh), n
    _check_windows(gpu, oracle, g[:4 * TILE + 37], p, po)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("preserve_case", [False, True])
def test_byte_classes_inside_the_halo(gpu, oracle, k, preserve_case):
    # every byte class at the halo offsets of each tile, read once as a halo and once as the next tile's own bytes
    p = gpu.params(k=k, preserve_case=preserve_case)
    po = oracle.params(k=k, preserve_case=preserve_case)
    seq = _halo_dirty(100 + k, 40 * TILE + 333)
    _check_windows(gpu, oracle, seq, p, po)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
def test_units_ending_in_the_last_halo_word(gpu, oracle, k, noncanonical):
    # device stream, keep-all units (s above their k-mer count): unit boundaries at a tile's first window, and units whose
    # last k-mer starts at the tile's last window start, so that it ends in the last halo word any window reads
    s = 4000
    p = gpu.params(k=k, s=s, noncanonical=noncanonical)
    po = oracle.params(k=k, noncanonical=noncanonical)
    ends = [TILE, 3 * TILE + TILE - 1 + k, 5 * TILE, 7 * TILE + TILE - 1 + k, 8 * TILE + TILE - 1 + k, 10 * TILE]
    starts = [0] + ends[:-1]
    seqs = [_halo_dirty(300 * k + u, e - b) for u, (b, e) in enumerate(zip(starts, ends))]
    for q in seqs:
        q[-1] = ord("*")      # a separator ends each dirty unit (windows that span two dirty units are not compared here)
    h, n = _sketch_dev(gpu, p, s, np.concatenate(seqs), starts + [ends[-1]])
    n_units = len(seqs)
    for u in range(n_units):
        oh, _, _ = oracle.sketch_unit([bytes(seqs[u])], po, s=s)
        assert n[u] == oh.size and np.array_equal(h[u, :n[u]], oh), u


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
def test_ascii_and_packed_sources_agree(gpu, oracle, k, noncanonical):
    # the same dirty units through the ASCII staging and the packed staging, against the oracle; keep-all (s above every
    # unit's k-mer count), so that one wrong window changes a sketch
    s = 4000
    p = gpu.params(k=k, s=s, noncanonical=noncanonical)
    po = oracle.params(k=k, noncanonical=noncanonical)
    recs = [bytes(_halo_dirty(500 * k + u, n)) for u, n in enumerate((TILE - 1, TILE + HALO, 3 * TILE + 17, 1500))]
    units = list(range(len(recs)))
    codes, runs, rstart = gpu.host_pack(recs, p, threads=2)
    unit_start = np.array(list(rstart[:-1]) + [rstart[-1]], np.uint64)
    hp, n_p, _ = gpu.sketch_packed(codes, int(rstart[-1]), runs, unit_start, p, counts=True)
    ha = gpu.sketch(recs, p, unit_of_record=units, n_units=len(recs))
    assert np.array_equal(n_p, ha[1]) and np.array_equal(hp, ha[0])
    for u, r in enumerate(recs):
        oh, _, _ = oracle.sketch_unit([r], po, s=s)
        assert ha[1][u] == oh.size and np.array_equal(ha[0][u, :ha[1][u]], oh), u
