"""GPU tests of the streaming unit job (mashgpu_unit_*): one unit of any size sketched stage by stage must equal the same unit through
mashgpu_sketch_batch and the checker (oracle.sketch_unit), counts included, for any feed split and with records longer than a stage;
device memory fixed by the parameters; the routing of large units and read sets to the job; refusals."""
import numpy as np
import pytest

import mash_b200
import reads_stream_model as M
from fixtures import synth_genome

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = 1, 3
STAGE = "50000"                      # 50 kB stages: long records cross stages


def _job(gpu, p, feeds, counts=True):
    job = gpu.unit_open(p)
    try:
        for f in feeds:
            job.feed(f)
        return job.finish(counts=counts)
    finally:
        job.close()


def _splits(recs, seed):
    rng = np.random.default_rng(seed)
    cuts = sorted(set(rng.integers(1, len(recs), 6).tolist())) if len(recs) > 1 else []
    return [recs[a:b] for a, b in zip([0] + cuts, cuts + [len(recs)])]


def _unit(seed, n_rec=12, short=True):
    """Records from 30 bp to 180 kb with N runs and soft-masked (lower-case) bases; a few shorter than any k."""
    rng = np.random.default_rng(seed)
    recs = []
    for i in range(n_rec):
        n = int(rng.choice([30, 900, 20_000, 70_000, 180_000]))
        recs.append(bytes(synth_genome(seed * 100 + i, n, n_runs=2, lower_frac=0.05)))
    if short:
        recs[1] = b"ACG"
        recs.append(b"")
    return recs


def _batch(gpu, p, recs, counts=True):
    out = gpu.sketch(recs, p, unit_of_record=[0] * len(recs), n_units=1, counts=counts)
    n = int(out[1][0])
    return out[0][0, :n], (out[3][0, :n] if counts else None), int(out[2][0])


def _check_all_feeds(gpu, oracle, p, po, recs, s, counts=True):
    bh, bc, blen = _batch(gpu, p, recs, counts)
    oh, oc, olen = oracle.sketch_unit(recs, po, s=s, counts=counts)
    assert np.array_equal(bh, oh) and blen == olen
    if counts:
        assert np.array_equal(bc, oc)
    kept = sum(1 for r in recs if len(r) >= p.kmer_size)
    for feeds in ([recs], [[r] for r in recs], _splits(recs, s + p.kmer_size)):
        h, c, length, n_rec = _job(gpu, p, feeds, counts)
        assert np.array_equal(h, oh) and length == olen and n_rec == kept
        if counts:
            assert np.array_equal(c, oc)
        else:
            assert c is None


@pytest.mark.parametrize("k", [9, 16, 17, 21, 32])
@pytest.mark.parametrize("noncanonical", [False, True])
@pytest.mark.parametrize("preserve_case", [False, True])
def test_job_equals_batch_and_checker(gpu, oracle, monkeypatch, k, noncanonical, preserve_case):
    monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", STAGE)
    recs = _unit(k + 3 * noncanonical + 7 * preserve_case)
    for s, counts in ((200, True), (1000, False)):
        p = gpu.params(k=k, s=s, noncanonical=noncanonical, preserve_case=preserve_case)
        po = oracle.params(k=k, noncanonical=noncanonical, preserve_case=preserve_case)
        _check_all_feeds(gpu, oracle, p, po, recs, s, counts)


@pytest.mark.parametrize("s", [1, 10_000])
@pytest.mark.parametrize("counts", [True, False])
def test_sketch_sizes(gpu, oracle, monkeypatch, s, counts):
    monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", STAGE)
    recs = _unit(50 + s)
    _check_all_feeds(gpu, oracle, gpu.params(k=21, s=s), oracle.params(k=21), recs, s, counts)


def test_golden_genomes(gpu, oracle, golden, monkeypatch):
    monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", STAGE)
    p, po = gpu.params(k=21, s=1000), oracle.params(k=21)
    for i, (_, rs) in enumerate(golden.genomes):
        recs = [r[2] for r in rs]
        gh, glen, _, _ = golden.golden_sketch(i)
        h, c, length, _ = _job(gpu, p, [recs])
        assert np.array_equal(h, gh) and length == glen
        _check_all_feeds(gpu, oracle, p, po, recs, 1000)


@pytest.mark.parametrize("alphabet", [mash_b200.ALPHABET_PROTEIN, "ACDEGHIKLM"])
def test_byte_alphabets(gpu, oracle, monkeypatch, alphabet):
    monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", STAGE)
    recs = [bytes(synth_genome(900 + i, n, alphabet=alphabet.encode(), lower_frac=0.03)) for i, n in enumerate([60_000, 5, 130_000, 900])]
    p = gpu.params(k=9, s=500, alphabet=alphabet, noncanonical=True)
    po = oracle.params(k=9, alphabet=alphabet, noncanonical=True)
    _check_all_feeds(gpu, oracle, p, po, recs, 500)


@pytest.mark.parametrize("stage", ["50000", "2000000"])
def test_top_counted_up_to_tstar(gpu, oracle, monkeypatch, stage):
    # a 30 kb genome repeated 20 times: the bottom-s settles in the first copy, so the final top keeps occurring after t* -- across
    # stages with 50 kB stages, inside one stage with 2 MB stages -- and counts only its occurrences up to t*
    monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", stage)
    g = bytes(synth_genome(31, 30_000))
    recs = [g * 20, g[:5000] * 3]
    p, po = gpu.params(k=21, s=1000), oracle.params(k=21)
    oh, oc, _ = oracle.sketch_unit(recs, po, s=1000, counts=True)
    assert oc[-1] < oc[:-1].max()                     # the quirk is visible
    _check_all_feeds(gpu, oracle, p, po, recs, 1000)


def test_repetitive_first_stage_trips_the_guard(gpu, oracle, monkeypatch):
    # the first stage holds few distinct k-mers: fewer than s survive its planned threshold, and it is re-run while resident
    monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", STAGE)
    recs = [b"ACGTTGCAAC" * 4000, bytes(synth_genome(5, 200_000))]
    p, po = gpu.params(k=21, s=1000), oracle.params(k=21)
    gpu.stats(reset=True)
    h, c, _, _ = _job(gpu, p, [recs])
    assert gpu.stats()["exact_reruns"] > 0
    _check_all_feeds(gpu, oracle, p, po, recs, 1000)


def test_edge_inputs(gpu, oracle):
    p = gpu.params(k=21, s=100)
    assert [x.size for x in _job(gpu, p, [[b"ACGT", b"", b"A" * 20]])[:2]] == [0, 0]
    assert _job(gpu, p, [[b"ACGT", b"A" * 20]])[2:] == (0, 0)
    assert _job(gpu, p, [])[2:] == (0, 0) and _job(gpu, p, [])[0].size == 0
    recs = _unit(3)
    h, c, length, n = _job(gpu, p, [[], recs[:4], [], recs[4:], []])
    oh, oc, olen = oracle.sketch_unit(recs, oracle.params(k=21), s=100, counts=True)
    assert np.array_equal(h, oh) and np.array_equal(c, oc) and length == olen


def test_device_memory_is_fixed_by_the_parameters(gpu, monkeypatch):
    monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", "1000000")
    recs = _unit(9, short=False)
    peak, stages = [], []
    for feeds in ([recs], [recs] * 8):
        gpu.stats(reset=True)
        _job(gpu, gpu.params(k=21, s=1000), feeds)
        st = gpu.stats()
        peak.append(st["unit_peak_device_bytes"])
        stages.append(st["unit_stages"])
    assert peak[0] == peak[1] > 0
    assert stages[1] > stages[0] > 1


def test_sketch_batch_streams_a_large_unit_among_small_ones(gpu, monkeypatch):
    big = _unit(11, short=False)
    recs, uor = [], []
    for u, rs in enumerate([[b"ACGTACGTAC" * 30], big, [bytes(synth_genome(2, 5000))], big[:3], [b"ACG"]]):
        recs += rs
        uor += [u] * len(rs)
    for counts in (True, False):
        p = gpu.params(k=21, s=500)
        base = gpu.sketch(recs, p, unit_of_record=uor, n_units=5, counts=counts)
        monkeypatch.setenv("MASHGPU_UNIT_STREAM_BYTES", "100000")
        monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", STAGE)
        gpu.stats(reset=True)
        got = gpu.sketch(recs, p, unit_of_record=uor, n_units=5, counts=counts)
        assert gpu.stats()["unit_stages"] > 0
        monkeypatch.delenv("MASHGPU_UNIT_STREAM_BYTES")
        assert np.array_equal(got[1], base[1]) and np.array_equal(got[2], base[2])
        for u in range(5):
            n = int(base[1][u])
            assert np.array_equal(got[0][u, :n], base[0][u, :n])
            if counts:
                assert np.array_equal(got[3][u, :n], base[3][u, :n])


def test_sketch_reads_streams_plain_read_sets_through_the_job(gpu, oracle, monkeypatch):
    reads = M.synth_reads(21, 30_000, 4000)
    reads[7] = b"ACGT"
    p = gpu.params(k=21, s=500)
    rj = gpu.reads_open(p)
    try:
        rj.feed(reads)
        jh, jc, ju = rj.finish()
    finally:
        rj.close()
    monkeypatch.setenv("MASHGPU_UNIT_STREAM_BYTES", "1000")
    monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", STAGE)
    gpu.stats(reset=True)
    h, c, used = gpu.sketch_reads(reads, p, counts=True)
    st = gpu.stats()
    assert st["reads_events"] == 0 and st["unit_stages"] > 1
    want = M.sketch_reads_reference(M.record_hashes(oracle, reads, oracle.params(k=21)), 500)
    assert used == ju == want[2] == len(reads) - 1
    assert np.array_equal(h, jh) and np.array_equal(c, jc)
    assert np.array_equal(h, want[0]) and np.array_equal(c, want[1])


def test_refusals(gpu):
    for kw in ({"min_copies": 2}, {"target_cov": 2.0}, {"bloom_bytes": 1000}):
        with pytest.raises(mash_b200.MashGpuError) as e:
            gpu.unit_open(gpu.params(k=21, s=100, **kw))
        assert e.value.code == ERR_UNSUPPORTED
    L = gpu.lib
    import ctypes as C
    assert L.mashgpu_unit_open(None, None, None) == ERR_INVALID
    assert L.mashgpu_unit_open(gpu.h, None, C.byref(C.c_void_p())) == ERR_INVALID
    assert L.mashgpu_unit_feed(None, 0, None, None) == ERR_INVALID
    assert L.mashgpu_unit_finish(None, None, None, None, None, None) == ERR_INVALID
    job = gpu.unit_open(gpu.params(k=21, s=100))
    try:
        assert L.mashgpu_unit_feed(job.h, 1, None, None) == ERR_INVALID
        assert L.mashgpu_unit_finish(job.h, None, None, None, None, None) == ERR_INVALID
        job.feed([b"ACGT" * 40])
        h, _, _, _ = job.finish()
        with pytest.raises(mash_b200.MashGpuError) as e:
            job.feed([b"ACGT" * 40])
        assert e.value.code == ERR_INVALID
        h2, _, _, _ = job.finish()
        assert np.array_equal(h, h2)
    finally:
        job.close()
    assert L.mashgpu_unit_close(None) == 0
