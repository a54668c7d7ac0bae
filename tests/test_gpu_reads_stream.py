"""GPU tests of the streaming reads job (`mash sketch -r [-m] [-c] [-b]`, mashgpu_reads_*): results against the heap model
(tests/reads_stream_model.py, pinned to the reference's object code by test_reads_stream_model.py) and the checker, independent of
how the records are split into feeds, of the staging size and of event-buffer overflows; bounded device memory; refusals."""
import numpy as np
import pytest

import mash_b200
import reads_stream_model as M

pytestmark = pytest.mark.gpu

ERR_INVALID, ERR_UNSUPPORTED = 1, 3


def _job(gpu, p, feeds):
    job = gpu.reads_open(p)
    try:
        flags = [job.feed(f) for f in feeds]
        h, c, used = job.finish()
    finally:
        job.close()
    return h, c, used, flags[-1] if flags else False


def _splits(reads, seed):
    rng = np.random.default_rng(seed)
    cuts = sorted(set(rng.integers(1, len(reads), 12).tolist()))
    return [reads[a:b] for a, b in zip([0] + cuts, cuts + [len(reads)])]


def _reads(seed, glen, n):
    reads = M.synth_reads(seed, glen, n)
    reads[3] = b"ACGT"                      # shorter than k: skipped, not counted as used
    return reads


# (m, bloom_bytes, c): c = 0 (off), 2.0 (an early stop), 6.0 (a late stop or none), 1e9 (never reached)
CASES = [(m, 0, c) for m in (1, 2, 3) for c in (0.0, 2.0, 6.0, 1e9)] + \
        [(1, b, c) for b in (1000, 65_536, 16 << 20) for c in (0.0, 2.0, 1e9)]


@pytest.mark.parametrize("k", [15, 21, 32])
@pytest.mark.parametrize("m,b,c", CASES)
def test_job_matches_the_reference_heap_for_any_feed_split(gpu, oracle, monkeypatch, k, m, b, c):
    monkeypatch.setenv("MASHGPU_READS_STAGE_BYTES", "50000")             # many stages, and stretches inside them
    reads = _reads(1000 + k + 10 * m + b % 97, 20_000, 2500)
    po = oracle.params(k=k)
    want = M.sketch_reads_reference(M.record_hashes(oracle, reads, po), 200, m=m, bloom_bytes=b, target_cov=c, use64=bool(po.use64))
    p = gpu.params(k=k, s=200, min_copies=m, target_cov=c, bloom_bytes=b)
    runs = [_job(gpu, p, [reads]), _job(gpu, p, [[r] for r in reads]), _job(gpu, p, _splits(reads, k + m))]
    for h, cnt, used, stopped in runs:
        assert used == want[2]
        assert np.array_equal(h, want[0]) and np.array_equal(cnt, want[1])
        assert stopped == runs[0][3]
    if b == 0:
        oh, oc, _, ou = oracle.sketch_unit_mc(reads, po, s=200, min_copies=m, target_cov=c, counts=True)
        assert ou == want[2] and np.array_equal(oh, want[0]) and np.array_equal(oc, want[1])
    if c == 2.0:
        assert runs[0][3] and 0 < want[2] < len(reads) - 1
    elif c != 6.0:                                                        # 6.0 stops late or not at all, depending on m and k
        assert not runs[0][3] and want[2] == len(reads) - 1


def test_sketch_reads_is_the_job_fed_once(gpu, oracle):
    reads = _reads(77, 30_000, 3000)
    p = gpu.params(k=21, s=300, min_copies=2, target_cov=4.0)
    h, c, used = gpu.sketch_reads(reads, p, counts=True)
    jh, jc, ju, _ = _job(gpu, p, _splits(reads, 5))
    assert used == ju and np.array_equal(h, jh) and np.array_equal(c, jc)


@pytest.mark.parametrize("b", [0, 1000])
def test_records_longer_than_the_stage(gpu, oracle, monkeypatch, b):
    # a record split across stages with a (k-1)-base overlap: every window counted once
    monkeypatch.setenv("MASHGPU_READS_STAGE_BYTES", "10000")
    rng = np.random.default_rng(5)
    acgt = np.frombuffer(b"ACGT", np.uint8)
    g = acgt[rng.integers(0, 4, 40_000)]
    recs = [bytes(g[:33_333]), bytes(g[1000:1150]), bytes(g[5000:40_000]), bytes(g[:9_999]), bytes(g[:10_000]), bytes(g[7:10_001])]
    po = oracle.params(k=21)
    want = M.sketch_reads_reference(M.record_hashes(oracle, recs, po), 500, bloom_bytes=b)
    p = gpu.params(k=21, s=500, bloom_bytes=b)
    for feeds in ([recs], [[r] for r in recs]):
        h, c, used, _ = _job(gpu, p, feeds)
        assert used == len(recs) and np.array_equal(h, want[0]) and np.array_equal(c, want[1])


@pytest.mark.parametrize("m,b,c", [(1, 0, 3.0), (2, 0, 0.0), (1, 1000, 0.0)])
def test_event_buffer_overflow_splits_stretches(gpu, oracle, monkeypatch, m, b, c):
    reads = _reads(91 + m, 40_000, 4000)
    p = gpu.params(k=21, s=500, min_copies=m, target_cov=c, bloom_bytes=b)
    base = _job(gpu, p, [reads])
    monkeypatch.setenv("MASHGPU_READS_EVENT_CAP", "8192")               # one tile: the first stretches overflow and split
    monkeypatch.setenv("MASHGPU_READS_STAGE_BYTES", "300000")
    gpu.stats(reset=True)
    small = _job(gpu, p, _splits(reads, 3))
    assert small[2] == base[2] and np.array_equal(small[0], base[0]) and np.array_equal(small[1], base[1])
    po = oracle.params(k=21)
    want = M.sketch_reads_reference(M.record_hashes(oracle, reads, po), 500, m=m, bloom_bytes=b, target_cov=c)
    assert base[2] == want[2] and np.array_equal(base[0], want[0]) and np.array_equal(base[1], want[1])
    assert gpu.stats()["reads_events"] > 0


def test_slow_filling_heap_completes(gpu, oracle, monkeypatch):
    # -m 3 at low coverage: the heap stays open for most of the stream, so nearly every k-mer (~2.6 M) is an event, stretches overflow
    # the event buffer again and again, and the pending tables grow on the device far beyond their initial size
    monkeypatch.setenv("MASHGPU_READS_EVENT_CAP", "65536")
    reads = M.synth_reads(123, 3_000_000, 20_000, err=0.002)
    p = gpu.params(k=21, s=2000, min_copies=3)
    h, c, used, _ = _job(gpu, p, _splits(reads, 9))
    po = oracle.params(k=21)
    oh, oc, _, ou = oracle.sketch_unit_mc(reads, po, s=2000, min_copies=3, counts=True)
    assert used == ou and np.array_equal(h, oh) and np.array_equal(c, oc)


@pytest.mark.parametrize("m,b", [(2, 0), (3, 0), (1, 1 << 20)])
def test_device_memory_does_not_grow_with_the_read_set(gpu, monkeypatch, m, b):
    # -m > 1 is the configuration whose pending tables grow during the job
    monkeypatch.setenv("MASHGPU_READS_STAGE_BYTES", "1000000")
    reads = M.synth_reads(8, 200_000, 20_000)
    peak = []
    for feeds in ([reads], [reads] * 8):
        _job(gpu, gpu.params(k=21, s=1000, min_copies=m, bloom_bytes=b), feeds)
        peak.append(gpu.stats()["reads_peak_device_bytes"])
    assert peak[0] == peak[1] > 0


def test_timing_reports_replay_time(gpu):
    gpu.set_timing(True)
    try:
        gpu.stats(reset=True)
        _job(gpu, gpu.params(k=21, s=1000), [M.synth_reads(9, 100_000, 5000)])
        st = gpu.stats(reset=True)
    finally:
        gpu.set_timing(False)
    assert st["reads_events"] > 0 and st["reads_replay_ms"] > 0


def test_bloom_bytes_is_refused_outside_reads_mode(gpu):
    p = gpu.params(k=21, s=100, bloom_bytes=1000)
    recs = [b"ACGT" * 50]
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.sketch(recs, p)
    assert e.value.code == ERR_UNSUPPORTED
    codes, runs, starts = gpu.host_pack(recs, gpu.params(k=21, s=100))
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.sketch_packed(codes, int(starts[-1]), runs, np.array([0, starts[-1]], np.uint64), p)
    assert e.value.code == ERR_UNSUPPORTED
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.sketch_stream_dev(p, None, [0, 0], None, None)
    assert e.value.code == ERR_UNSUPPORTED
    ref = np.arange(1, 101, dtype=np.uint64)[None, :]
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.screen_open(ref, np.array([100], np.uint32), p)
    assert e.value.code == ERR_UNSUPPORTED
    both = gpu.params(k=21, s=100, bloom_bytes=1000, min_copies=2)
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.reads_open(both)
    assert e.value.code == ERR_INVALID
    with pytest.raises(mash_b200.MashGpuError) as e:
        gpu.sketch_reads(recs, both)
    assert e.value.code == ERR_INVALID


def test_feeds_after_the_stop_are_ignored(gpu):
    reads = _reads(31, 20_000, 3000)
    p = gpu.params(k=21, s=200, target_cov=2.0)
    job = gpu.reads_open(p)
    try:
        assert job.feed(reads)
        h, c, used = job.finish()
    finally:
        job.close()
    job = gpu.reads_open(p)
    try:
        assert job.feed(reads)
        assert job.feed(M.synth_reads(32, 20_000, 3000))
        h2, c2, used2 = job.finish()
    finally:
        job.close()
    assert used2 == used and np.array_equal(h2, h) and np.array_equal(c2, c)


@pytest.mark.parametrize("m", [1, 2, 3])
def test_whole_set_path_equals_the_job(gpu, m):
    # without -c and -b mashgpu_sketch_reads sketches a read set that fits on the device in one parallel pass; the job's replay
    # gives the same heap
    reads = _reads(600 + m, 50_000, 6000)
    p = gpu.params(k=21, s=500, min_copies=m)
    h, c, used = gpu.sketch_reads(reads, p, counts=True)
    jh, jc, ju, _ = _job(gpu, p, _splits(reads, m))
    assert used == ju == len(reads) - 1 and np.array_equal(h, jh) and np.array_equal(c, jc)
