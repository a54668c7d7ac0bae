"""GPU tests aimed at the staging of the byte-alphabet scan kernel (scan_bytes_kernel: protein `-a` and custom `-z`
alphabets): a warp tile's 1024 window starts plus its 64 halo bytes, staged as 68 vectors of 16 through the alphabet table,
with a per-byte guard that turns every byte at or past the end of the stream into a non-alphabet byte.  Junk bytes of
every class go through the halo, and keep-all sketches end the stream at every byte of the last tile's halo.  Everything
is checked bit-exact against the oracle."""
import numpy as np
import pytest

from fixtures import synth_genome
from oracle.pyoracle import ALPHABET_PROTEIN

pytestmark = pytest.mark.gpu

TILE = 1024          # window starts per warp tile
HALO = 64            # halo bytes staged past a warp tile
# outside both alphabets, lower case of their letters (alphabet bytes unless preserve_case), separators, bytes >= 0x80
JUNK = np.frombuffer(b"BJOUXZbjouxzRYacdefgnwy*-.\x00\x80\xff\xc3\x7f", np.uint8)
CASES = [(k, ALPHABET_PROTEIN) for k in (1, 2, 6, 9, 14, 16, 17, 30, 31, 32)] + [(13, "ACGTN"), (14, "ACGTN")]
IDS = [f"{'protein' if a == ALPHABET_PROTEIN else a}-k{k}" for k, a in CASES]


def _letters(alphabet, seed, n):
    return synth_genome(seed, n, alphabet=alphabet.encode())


def _halo_dirty(alphabet, seed, n):
    """Alphabet letters with every junk class placed at the halo offsets (position mod 1024 < 64) and nowhere else."""
    g = _letters(alphabet, seed, n)
    rng = np.random.Generator(np.random.PCG64(seed))
    pos = np.arange(n)
    halo = pos[(pos % TILE) < HALO]
    pick = halo[rng.random(halo.size) < 0.15]
    g[pick] = JUNK[rng.integers(0, JUNK.size, pick.size)]
    lower = halo[rng.random(halo.size) < 0.2]
    g[lower] = np.where((g[lower] >= 65) & (g[lower] <= 90), g[lower] + 32, g[lower])
    for t in range(0, n - TILE, 3 * TILE):        # a junk run across a halo every third tile
        g[t + TILE - 5:t + TILE + 9] = ord("*")
    return g


def _params(gpu, oracle, k, alphabet, s=100, preserve_case=False):
    p = gpu.params(k=k, s=s, alphabet=alphabet, noncanonical=True, preserve_case=preserve_case)
    po = oracle.params(k=k, alphabet=alphabet, noncanonical=True, preserve_case=preserve_case)
    assert p.use64 == po.use64 and bytes(p.alphabet) == bytes(po.alphabet)
    return p, po


def _check_windows(gpu, oracle, seq, p, po):
    h, v = gpu.hash_windows(seq, p)
    want = oracle.all_hashes(bytes(seq), po)
    assert int(v.sum()) == want.size and np.array_equal(h[v], want)


def _sketch_dev(gpu, p, s, flat, unit_start, pad):
    # device stream followed by 256 alphabet bytes: a byte past the end read as a letter changes the last unit's sketch
    import torch
    dev = torch.from_numpy(np.concatenate([flat, pad[np.arange(256) % pad.size]])).cuda()
    n_units = len(unit_start) - 1
    d_h = torch.zeros((n_units, s), dtype=torch.int64, device="cuda")
    d_n = torch.zeros(n_units, dtype=torch.int32, device="cuda")
    gpu.sketch_stream_dev(p, dev.data_ptr(), np.asarray(unit_start, np.uint64), d_h.data_ptr(), d_n.data_ptr())
    torch.cuda.synchronize()
    return d_h.cpu().numpy().view(np.uint64), d_n.cpu().numpy()


@pytest.mark.parametrize("k,alphabet", CASES, ids=IDS)
@pytest.mark.parametrize("preserve_case", [False, True])
def test_byte_classes_inside_the_halo(gpu, oracle, k, alphabet, preserve_case):
    # every junk class at the halo offsets of each tile, read once as a halo and once as the next tile's own bytes
    p, po = _params(gpu, oracle, k, alphabet, preserve_case=preserve_case)
    seq = _halo_dirty(alphabet, 100 + k, 40 * TILE + 333)
    _check_windows(gpu, oracle, seq, p, po)


@pytest.mark.parametrize("k,alphabet", CASES, ids=IDS)
def test_stream_end_at_every_halo_byte(gpu, oracle, k, alphabet):
    # a keep-all unit whose stream ends at each byte of the last full tile's halo (the guard is per byte), and around the
    # tile's own boundary; the 256 alphabet bytes after the end must not be read as part of the stream
    s = 6000
    p, po = _params(gpu, oracle, k, alphabet, s=s)
    g = _letters(alphabet, 7000 + k, 5 * TILE + HALO)
    pad = np.frombuffer(alphabet.encode(), np.uint8)
    lens = [4 * TILE + off for off in range(HALO)]
    lens += [4 * TILE - 1, 4 * TILE - k, 4 * TILE - k + 1, 3 * TILE + k - 1, 3 * TILE + k, 4 * TILE + HALO, 4 * TILE + HALO + 1]
    lens += [n for n in range(1, 2 * k + 3)]                          # streams shorter than one vector, and than k
    for n in lens:
        h, cnt = _sketch_dev(gpu, p, s, g[:n], [0, n], pad)
        oh, _, _ = oracle.sketch_unit([bytes(g[:n])], po, s=s)
        assert cnt[0] == oh.size and np.array_equal(h[0, :cnt[0]], oh), n
    _check_windows(gpu, oracle, g[:4 * TILE + 37], p, po)


@pytest.mark.parametrize("k,alphabet", CASES, ids=IDS)
def test_units_ending_in_the_last_halo_byte(gpu, oracle, k, alphabet):
    # device stream, keep-all units: unit boundaries at a tile's first window, and units whose last k-mer starts at the
    # tile's last window start, so that it ends in the last halo bytes any window reads
    s = 4000
    p, po = _params(gpu, oracle, k, alphabet, s=s)
    ends = [TILE, 3 * TILE + TILE - 1 + k, 5 * TILE, 7 * TILE + TILE - 1 + k, 8 * TILE + TILE - 1 + k, 10 * TILE]
    starts = [0] + ends[:-1]
    seqs = [_halo_dirty(alphabet, 300 * k + u, e - b) for u, (b, e) in enumerate(zip(starts, ends))]
    for q in seqs:
        q[-1] = ord("*")      # a separator ends each dirty unit (windows that span two units are not compared here)
    h, n = _sketch_dev(gpu, p, s, np.concatenate(seqs), starts + [ends[-1]], np.frombuffer(alphabet.encode(), np.uint8))
    for u in range(len(seqs)):
        oh, _, _ = oracle.sketch_unit([bytes(seqs[u])], po, s=s)
        assert n[u] == oh.size and np.array_equal(h[u, :n[u]], oh), u
