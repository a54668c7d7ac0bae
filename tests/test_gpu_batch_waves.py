"""GPU tests of mashgpu_sketch_batch's routing around its waves, and of the context's grow-only pinned buffers: a batch of one unit
per record whose large records stream through the unit job, and one context whose feed buffers grow call after call."""
import numpy as np
import pytest

import mash_b200
from fixtures import synth_genome

pytestmark = pytest.mark.gpu


def assert_same_sketches(got, want):
    """(hashes, n, length[, counts]) equal wherever a sketch has entries."""
    assert np.array_equal(got[1], want[1]) and np.array_equal(got[2], want[2])
    held = np.arange(got[0].shape[1]) < got[1][:, None].astype(np.int64)
    for i in range(0, len(want), 3):               # hashes, then counts if present
        assert np.array_equal(got[i][held], want[i][held])


def test_one_unit_per_record_streams_large_records(gpu, monkeypatch):
    # unit_of_record = NULL: record r is unit r.  Records above MASHGPU_UNIT_STREAM_BYTES go through the unit job; the runs of
    # records around them (at the start, between two of them, at the end) go through the waves
    lens = [5000, 180_000, 30, 2000, 150_000, 160_000, 900, 70_000, 3]
    recs = [bytes(synth_genome(4000 + i, n, n_runs=1, lower_frac=0.05)) for i, n in enumerate(lens)]
    p = gpu.params(k=21, s=400)
    for counts in (True, False):
        base = gpu.sketch(recs, p, counts=counts)
        monkeypatch.setenv("MASHGPU_UNIT_STREAM_BYTES", "100000")
        monkeypatch.setenv("MASHGPU_UNIT_STAGE_BYTES", "50000")
        gpu.stats(reset=True)
        got = gpu.sketch(recs, p, counts=counts)
        assert gpu.stats()["unit_stages"] > 0
        monkeypatch.delenv("MASHGPU_UNIT_STREAM_BYTES")
        assert_same_sketches(got, base)


def test_pinned_buffers_grow_on_one_context(gpu, monkeypatch):
    # Rounds of calls, each round twice the size of the one before, on one context: more units per batch (unit flags), larger
    # waves through the ASCII feed alone (staging of small records, separator list of a record copied straight from the
    # caller's buffer) and the packed feed alone (host codes), larger chunks through screen's packed host feed.  So every
    # pinned buffer of the context is reallocated between rounds; each call must give what it gives on a fresh context.
    p = gpu.params(k=21, s=300)
    genomes = [synth_genome(5000 + i, 200_000) for i in range(3)]
    ref = gpu.sketch([bytes(g) for g in genomes], p)
    windows = np.lib.stride_tricks.sliding_window_view(np.concatenate(genomes[:2]), 150)
    rng = np.random.Generator(np.random.PCG64(5))

    def batch_of_units(f):
        recs = [bytes(synth_genome(6000 + 1000 * f + i, 2000 + 37 * i)) for i in range(40 * f)]
        return lambda eng: eng.sketch(recs, p, counts=True)

    def waves(f):
        recs, uor = [], []
        for u in range(6):
            for r in range(2):
                recs.append(bytes(synth_genome(7000 + 100 * f + 10 * u + r, 20_000 * f + 97 * u + r)))
                uor.append(u)
        recs.append(bytes(synth_genome(8000 + f, 300_000 * f)))          # at least 2^18 bytes: copied straight, not staged
        uor.append(5)
        return lambda eng: eng.sketch(recs, p, unit_of_record=uor, n_units=6, counts=True)

    def screen(f):
        n = 28_000 * f                                                   # 151 B per read: chunks above 4 MiB are fed whole
        reads = windows[rng.integers(0, windows.shape[0], 2 * n)]
        stream = np.concatenate([np.full((2 * n, 1), ord("*"), np.uint8), reads], axis=1).ravel()
        chunks = [bytes(stream[:n * 151]), bytes(stream[n * 151:])]

        def run(eng):
            job = eng.screen_open(ref[0], ref[1], p)
            try:
                for c in chunks:
                    job.feed(c)
                return job.finish()
            finally:
                job.close()
        return run

    eng = mash_b200.Engine(device=0)
    try:
        for f in (1, 2, 4):
            for env, run in (({}, batch_of_units(f)),
                             ({"MASHGPU_HOST_PACK": "0", "MASHGPU_WAVE_UNITS": "2"}, waves(f)),
                             ({"MASHGPU_HOST_PACK": "1", "MASHGPU_WAVE_UNITS": "2"}, waves(f)),
                             ({"MASHGPU_SCREEN_HOST_PACK": "1"}, screen(f))):
                with monkeypatch.context() as m:
                    for name, value in env.items():
                        m.setenv(name, value)
                    got = run(eng)
                    fresh = mash_b200.Engine(device=0)
                    try:
                        want = run(fresh)
                    finally:
                        fresh.close()
                if isinstance(want, dict):
                    assert want["shared"][:2].min() > 0           # the reads come from the first two references
                    for key in want:
                        assert np.array_equal(got[key], want[key]), (f, key)
                else:
                    assert want[1].min() == p.sketch_size
                    assert_same_sketches(got, want)
    finally:
        eng.close()
