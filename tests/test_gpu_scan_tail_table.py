"""GPU tests for the filter-word scan kernels' tail table (k = 17..21) and the one-op padding of the last k-mer word
(every k).  For k = 17..21 the fast path takes the tail block's k1 from a shared-memory table indexed by the canonical
k-mer's last nibble word; a wrong entry or index would make the filter drop windows whose hash belongs in the sketch.  So
the units here are long enough that the thresholds are selective, and k = 22, 25 and 32 (no table) run the same cases.
Everything is checked bit-exact against the oracle."""
import numpy as np
import pytest

from fixtures import synth_genome

pytestmark = pytest.mark.gpu

TABLE_KS = [17, 18, 19, 20, 21]
KS = TABLE_KS + [22, 25, 32]


def _tail_dirty(seed, n, lower_frac=0.25):
    # N runs, single Ns and lower case every few bases, so that they land inside the tail bases (16..k-1) of many windows
    g = synth_genome(seed, n, n_runs=3, lower_frac=lower_frac)
    rng = np.random.Generator(np.random.PCG64(seed + 3))
    pos = rng.integers(0, n, max(1, n // 97))
    g[pos] = np.frombuffer(b"NnRx", np.uint8)[rng.integers(0, 4, pos.size)]
    return g


def _units(k, seed):
    # unit lengths that are not multiples of 8 (units end inside a lane's block of 8 windows) and thresholds that keep a
    # small share of the windows
    return [[bytes(synth_genome(seed + 1, 150_001))], [bytes(_tail_dirty(seed + 2, 80_003))],
            [bytes(synth_genome(seed + 3, 33_333, lower_frac=0.4))],
            [bytes(_tail_dirty(seed + 4, 20_000)), bytes(synth_genome(seed + 5, 12_345)), b"acgtN" * 50],
            [bytes(_tail_dirty(seed + 6, 250_007, lower_frac=0.05))]]


def _check_batch(gpu, oracle, units, p, po, s, counts=True):
    recs, uor = [], []
    for u, rs in enumerate(units):
        recs += rs
        uor += [u] * len(rs)
    out = gpu.sketch(recs, p, unit_of_record=uor, n_units=len(units), counts=counts)
    for u, rs in enumerate(units):
        oh, oc, olen = oracle.sketch_unit(rs, po, s=s, counts=counts)
        assert out[2][u] == olen, u
        assert out[1][u] == oh.size and np.array_equal(out[0][u, :out[1][u]], oh), u
        if counts:
            assert np.array_equal(out[3][u, :out[1][u]], oc), u
    return out, recs, uor


@pytest.mark.parametrize("k", KS)
@pytest.mark.parametrize("noncanonical", [False, True])
def test_sketch_ascii_and_packed(gpu, oracle, k, noncanonical):
    s = 500
    p = gpu.params(k=k, s=s, noncanonical=noncanonical)
    po = oracle.params(k=k, noncanonical=noncanonical)
    units = _units(k, 1000 * k + 7 * noncanonical)
    out, recs, uor = _check_batch(gpu, oracle, units, p, po, s)
    codes, runs, starts = gpu.host_pack(recs, p, threads=2)
    unit_first = [uor.index(u) for u in range(len(units))]
    unit_start = np.array([starts[i] for i in unit_first] + [starts[-1]], np.uint64)
    h, n, c = gpu.sketch_packed(codes, int(starts[-1]), runs, unit_start, p, counts=True)
    assert np.array_equal(n, out[1]) and np.array_equal(h, out[0]) and np.array_equal(c, out[3])


@pytest.mark.parametrize("k", [17, 19, 21, 22])
def test_preserve_case(gpu, oracle, k):
    # with -Z lower-case bases are outside the alphabet: windows with one in their tail must be rejected
    s = 400
    p = gpu.params(k=k, s=s, preserve_case=True)
    po = oracle.params(k=k, preserve_case=True)
    _check_batch(gpu, oracle, _units(k, 77 * k), p, po, s)


@pytest.mark.parametrize("k", [17, 18, 21, 22])
@pytest.mark.parametrize("tail", [1089, 9])
def test_device_stream_ragged_end(gpu, oracle, k, tail):
    # the units lie back to back; each but the last ends with a byte outside the alphabet, so that no window spans two units
    import torch
    s = 500
    p = gpu.params(k=k, s=s)
    po = oracle.params(k=k)
    lens = [90_001, 1024 * 41 + 5, 0]
    lens[2] = 1024 * 70 + tail - (lens[0] + lens[1]) % 1024
    seqs = [_tail_dirty(3030 + 10 * u + k, n) for u, n in enumerate(lens)]
    seqs[0][-1] = seqs[1][-1] = ord("*")
    flat = np.concatenate(seqs)
    dev = torch.from_numpy(flat.copy()).cuda()
    unit_start = np.array([0, lens[0], lens[0] + lens[1], flat.size], np.uint64)
    d_h = torch.zeros((3, s), dtype=torch.int64, device="cuda")
    d_n = torch.zeros(3, dtype=torch.int32, device="cuda")
    gpu.sketch_stream_dev(p, dev.data_ptr(), unit_start, d_h.data_ptr(), d_n.data_ptr())
    torch.cuda.synchronize()
    h = d_h.cpu().numpy().view(np.uint64)
    n = d_n.cpu().numpy()
    for u in range(3):
        oh, _, _ = oracle.sketch_unit([bytes(seqs[u])], po, s=s)
        assert n[u] == oh.size and np.array_equal(h[u, :n[u]], oh), u


@pytest.mark.parametrize("k", [18, 21])
def test_min_copies_and_target_coverage(gpu, oracle, k):
    s = 200
    g = synth_genome(5150 + k, 120_000)
    rng = np.random.Generator(np.random.PCG64(k))
    reads = []
    for a in rng.integers(0, g.size - 120, 15_000):
        r = g[a:a + 120].copy()
        if rng.random() < 0.1:
            r[int(rng.integers(0, 120))] = ord("N")
        reads.append(bytes(r))
    po = oracle.params(k=k)
    pm = gpu.params(k=k, s=s, min_copies=2)
    out = gpu.sketch(reads, pm, unit_of_record=[0] * len(reads), n_units=1, counts=True)
    oh, oc, _ = oracle.sketch_unit_m(reads, po, s=s, min_copies=2, counts=True)
    assert np.array_equal(out[0][0, :out[1][0]], oh) and np.array_equal(out[3][0, :out[1][0]], oc)
    pc = gpu.params(k=k, s=s, min_copies=2, target_cov=3.0)
    h, cnt, used = gpu.sketch_reads(reads, pc, counts=True)
    oh, oc, _, ou = oracle.sketch_unit_mc(reads, po, s=s, min_copies=2, target_cov=3.0, counts=True)
    assert used == ou and np.array_equal(h, oh) and np.array_equal(cnt, oc)


def test_exact_rerun(gpu, oracle):
    p = gpu.params(k=21, s=1000)
    po = oracle.params(k=21)
    units = [[bytes(synth_genome(21, 70_000))], [bytes(np.tile(synth_genome(22, 2500), 150))], [bytes(_tail_dirty(23, 90_000))]]
    before = gpu.stats()["exact_reruns"]
    _check_batch(gpu, oracle, units, p, po, 1000, counts=False)
    assert gpu.stats()["exact_reruns"] > before
