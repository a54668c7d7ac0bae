"""GPU tests aimed at the filter-word scan kernels (k = 17..32): per-lane pass masks resolved once per warp tile, and the
next tile prefetched into a shared landing buffer.  The cases are the ones where the mask is dense, where its
bit <-> window mapping (bit 8 i + j = window 8 (lane + 32 i) + j of the 1024-window warp tile) could go wrong, and where the
prefetch meets the end of the stream.  Everything is checked bit-exact against the oracle."""
import numpy as np
import pytest

from fixtures import synth_genome

pytestmark = pytest.mark.gpu

KS = [17, 21, 24, 25, 32]


def _units_recs(units):
    recs, uor = [], []
    for u, rs in enumerate(units):
        recs += rs
        uor += [u] * len(rs)
    return recs, uor


def _check_batch(gpu, oracle, units, p, po, s, counts=True):
    recs, uor = _units_recs(units)
    out = gpu.sketch(recs, p, unit_of_record=uor, n_units=len(units), counts=counts)
    for u, rs in enumerate(units):
        oh, oc, olen = oracle.sketch_unit(rs, po, s=s, counts=counts)
        assert out[2][u] == olen, u
        assert out[1][u] == oh.size and np.array_equal(out[0][u, :out[1][u]], oh), u
        if counts:
            assert np.array_equal(out[3][u, :out[1][u]], oc), u
    return out


def _dirty(seed, n):
    # N runs, lower case and bytes outside the alphabet: windows that hold them are hashed by the fast path anyway, and
    # when the threshold keeps everything they all pass the filter and must be rejected by the exact rebuild
    g = synth_genome(seed, n, n_runs=3, lower_frac=0.1)
    if n == 0:
        return g
    rng = np.random.Generator(np.random.PCG64(seed + 7))
    junk = np.frombuffer(b"*-.RYKMSWnx\x00\xff", np.uint8)
    pos = rng.integers(0, n, max(1, n // 500))
    g[pos] = junk[rng.integers(0, junk.size, pos.size)]
    return g


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
def test_keep_all_units_dense_masks(gpu, oracle, k, noncanonical):
    # span <= 6 s: the unit threshold is 2^64 - 1, so every window of these units passes the filter -- every lane's mask is
    # full, and a warp tile's ~1000 survivors overflow the 64-entry queue into direct scan_emit
    s = 1000
    p = gpu.params(k=k, s=s, noncanonical=noncanonical)
    po = oracle.params(k=k, noncanonical=noncanonical)
    units = [[bytes(synth_genome(10 * k + u, 2500 + 517 * u))] for u in range(6)]
    units += [[bytes(_dirty(20 * k + u, 4000 + 311 * u))] for u in range(6)]
    units.append([bytes(synth_genome(5 * k, 300_000, n_runs=4, lower_frac=0.05))])      # a unit with a coarse threshold after them
    _check_batch(gpu, oracle, units, p, po, s)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
def test_tiny_units_across_lane_and_tile_boundaries(gpu, oracle, k, noncanonical):
    # hundreds of units of 0..300 bases (some shorter than k, some multi-record): unit starts and ends fall inside one
    # lane's 32 windows and across warp-tile (1024) and SCAN_TILE (8192) boundaries
    s = 50
    p = gpu.params(k=k, s=s, noncanonical=noncanonical)
    po = oracle.params(k=k, noncanonical=noncanonical)
    rng = np.random.Generator(np.random.PCG64(1000 + k))
    units = []
    for u in range(400):
        n_rec = 1 + (u % 5 == 0)
        units.append([bytes(_dirty(100_000 * k + 10 * u + r, int(rng.integers(0, 301)))) if u % 3 == 0
                      else bytes(synth_genome(100_000 * k + 10 * u + r, int(rng.integers(0, 301)))) for r in range(n_rec)])
    units.append([bytes(synth_genome(77 * k, 40_000))])
    _check_batch(gpu, oracle, units, p, po, s)


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("preserve_case", [False, True])
def test_lower_case_and_invalid_windows(gpu, oracle, k, preserve_case):
    s = 400
    p = gpu.params(k=k, s=s, preserve_case=preserve_case)
    po = oracle.params(k=k, preserve_case=preserve_case)
    units = [[bytes(_dirty(3 * k, 250_000))], [bytes(synth_genome(4 * k, 2000, lower_frac=0.5))],
             [bytes(_dirty(5 * k, 60_000)), b"acgtn" * 40, bytes(synth_genome(6 * k, 9000, n_runs=2, lower_frac=0.3))]]
    _check_batch(gpu, oracle, units, p, po, s)
    # every window hash (SCAN_DUMP) on the same kind of input
    seq = _dirty(7 * k, 20_000)
    h, v = gpu.hash_windows(seq, p)
    want = oracle.all_hashes(bytes(seq), po)
    assert int(v.sum()) == want.size and np.array_equal(h[v], want)


@pytest.mark.parametrize("k", KS)
def test_packed_source_matches_ascii_and_oracle(gpu, oracle, k):
    # mashgpu_sketch_batch_packed: the packed source is staged from the landing buffer too (codes and invalid bits)
    s = 300
    p = gpu.params(k=k, s=s)
    po = oracle.params(k=k)
    units = [[bytes(_dirty(40 * k + u, 30_000 + 7919 * u))] for u in range(4)]
    units += [[bytes(synth_genome(50 * k + u, 1200 + 61 * u))] for u in range(8)]                  # keep-all, dense masks
    units += [[bytes(synth_genome(60 * k + u, int(n))) for n in (5, 100, 37)] for u in range(6)]   # tiny records
    recs, uor = _units_recs(units)
    codes, runs, starts = gpu.host_pack(recs, p, threads=2)
    unit_first = [uor.index(u) for u in range(len(units))]
    unit_start = np.array([starts[i] for i in unit_first] + [starts[-1]], np.uint64)
    h, n, c = gpu.sketch_packed(codes, int(starts[-1]), runs, unit_start, p, counts=True)
    ref = gpu.sketch(recs, p, unit_of_record=uor, n_units=len(units), counts=True)
    assert np.array_equal(n, ref[1]) and np.array_equal(h, ref[0]) and np.array_equal(c, ref[3])
    for u, rs in enumerate(units):
        oh, _, _ = oracle.sketch_unit(rs, po, s=s)
        assert np.array_equal(h[u, :n[u]], oh), u


@pytest.mark.parametrize("k,s", [(21, 200), (17, 100), (32, 300)])
def test_counts_quirk_and_min_copies(gpu, oracle, k, s):
    # multiplicities (SCAN_COUNT and the top-of-heap quirk) and `-m 2` (positions per slot) through the resolved masks
    p = gpu.params(k=k, s=s)
    po = oracle.params(k=k)
    g = synth_genome(900 + k, 40_000)
    rng = np.random.Generator(np.random.PCG64(k))
    reads = [bytes(g[a:a + 150]) for a in rng.integers(0, g.size - 150, 1500)]
    units = [reads, [bytes(np.tile(g[:5000], 8))]]
    _check_batch(gpu, oracle, units, p, po, s)
    pm = gpu.params(k=k, s=s, min_copies=2)
    out = gpu.sketch(reads, pm, unit_of_record=[0] * len(reads), n_units=1, counts=True)
    oh, oc, _ = oracle.sketch_unit_m(reads, po, s=s, min_copies=2, counts=True)
    assert np.array_equal(out[0][0, :out[1][0]], oh) and np.array_equal(out[3][0, :out[1][0]], oc)


@pytest.mark.parametrize("k", [21, 25])
def test_target_coverage_events(gpu, oracle, k):
    # `-c`: the SCAN_EVENTS pass appends every survivor of its position bands as an event; events are sorted by position
    # before replay, so resolving a tile's survivors at its end cannot change the stop
    s = 200
    p = gpu.params(k=k, s=s, min_copies=2, target_cov=3.0)
    po = oracle.params(k=k)
    g = synth_genome(4321 + k, 150_000)
    rng = np.random.Generator(np.random.PCG64(99 + k))
    reads = []
    for a in rng.integers(0, g.size - 120, 20_000):
        r = g[a:a + 120].copy()
        if rng.random() < 0.05:
            r[int(rng.integers(0, 120))] = ord("N")
        reads.append(bytes(r))
    h, cnt, used = gpu.sketch_reads(reads, p, counts=True)
    oh, oc, _, ou = oracle.sketch_unit_mc(reads, po, s=s, min_copies=2, target_cov=3.0, counts=True)
    assert used == ou and 0 < used < len(reads) - 1
    assert np.array_equal(h, oh) and np.array_equal(cnt, oc)


def test_exact_rerun_only_unit(gpu, oracle):
    # a highly repetitive unit next to normal ones: its exact re-run scans the whole stream with only_unit set, so the
    # other units' survivors are resolved and then dropped
    p = gpu.params(k=24, s=1000)
    po = oracle.params(k=24)
    units = [[bytes(synth_genome(11, 70_000))], [bytes(np.tile(synth_genome(12, 2500), 150))], [bytes(_dirty(13, 90_000))]]
    before = gpu.stats()["exact_reruns"]
    _check_batch(gpu, oracle, units, p, po, 1000, counts=False)
    assert gpu.stats()["exact_reruns"] > before


@pytest.mark.parametrize("k", [21, 32])
@pytest.mark.parametrize("tail", [1087, 1088, 1089, 1103, 9])
def test_device_stream_ragged_end(gpu, oracle, k, tail):
    # a device-resident stream whose length is not a multiple of 16 (except tail 1088: the last warp tile's 1088 bytes end
    # exactly at the end).  Tiles that reach past stream_len are loaded with guarded loads, the others by cp.async; bytes
    # past stream_len are valid bases here, so reading them as bases would change the last unit's sketch.
    import torch
    s = 500
    p = gpu.params(k=k, s=s)
    po = oracle.params(k=k)
    n_units = 3
    lens = [70_001, 1024 * 37 + 13, 0]
    lens[2] = 1024 * 60 + tail - (lens[0] + lens[1]) % 1024
    seqs = [synth_genome(2024 + 10 * u + k, n) for u, n in enumerate(lens)]
    flat = np.concatenate(seqs)
    total = flat.size
    for exact in (True, False):
        if exact:
            dev = torch.from_numpy(flat.copy()).cuda()
        else:
            pad = np.frombuffer(b"ACGT", np.uint8)[np.arange(256) % 4]
            dev = torch.from_numpy(np.concatenate([flat, pad])).cuda()
        unit_start = np.array([0, lens[0], lens[0] + lens[1], total], np.uint64)
        d_h = torch.zeros((n_units, s), dtype=torch.int64, device="cuda")
        d_n = torch.zeros(n_units, dtype=torch.int32, device="cuda")
        gpu.sketch_stream_dev(p, dev.data_ptr(), unit_start, d_h.data_ptr(), d_n.data_ptr())
        torch.cuda.synchronize()
        h = d_h.cpu().numpy().view(np.uint64)
        n = d_n.cpu().numpy()
        for u in range(n_units):
            oh, _, _ = oracle.sketch_unit([bytes(seqs[u])], po, s=s)
            assert n[u] == oh.size and np.array_equal(h[u, :n[u]], oh), (exact, u)
