"""GPU tests of screening samples one after another on one job (mashgpu_screen_reset, mashgpu_screen_finish_hits), through the
C ABI: every sample's finish() and finish_hits() equal, bit for bit, a fresh job's finish() over the same chunks, and the oracle."""
import numpy as np
import pytest

import screen_samples_model as ssm
import translated_screen_oracle as tso
from fixtures import synth_genome, mutate
from oracle.pyoracle import ALPHABET_PROTEIN
from test_gpu_screen import check
from test_gpu_screen_translated import joined, protein_refs, reads_from

pytestmark = pytest.mark.gpu

FIELDS = ("shared", "median", "identity", "pvalue")


def reads_of(genomes, n, seed, length=150):
    rng = np.random.Generator(np.random.PCG64(seed))
    out = []
    for _ in range(n):
        g = genomes[int(rng.integers(0, len(genomes)))]
        a = int(rng.integers(0, max(1, g.size - length)))
        r = g[a:a + length].copy()
        if rng.random() < 0.05:
            r[int(rng.integers(0, r.size))] = ord("N")
        out.append(bytes(r))
    return out


def nucleotide_refs(oracle, po, s, genomes, stride=None):
    stride = stride or s
    ref = np.full((len(genomes), stride), np.uint64(2**64 - 1)); ref_n = np.zeros(len(genomes), np.uint32)
    for i, g in enumerate(genomes):
        h, _, _ = oracle.sketch_unit([bytes(g)], po, s=s)
        ref[i, :h.size] = h; ref_n[i] = h.size
    return ref, ref_n


def nucleotide_samples(genomes, seed):
    """(how, chunks) per sample: an empty sample, one without a hit, large pipelined host chunks, many small joined chunks,
    device chunks, and two ordinary ones."""
    other = [synth_genome(seed + 900, 50_000)]
    return [
        ("host", joined(reads_of(genomes[:2], 4000, seed + 1), 1000)),
        ("host", []),
        ("host", joined(reads_of(other, 3000, seed + 2), 1000)),
        ("host", joined(reads_of(genomes, 90_000, seed + 3), 30_000)),
        ("host", joined(reads_of(genomes[1:], 3000, seed + 4), 7)),
        ("dev", joined(reads_of(genomes[:1], 3000, seed + 5), 1000)),
        ("host", joined(reads_of(genomes[-2:], 5000, seed + 6), 2500)),
    ]


def feed(job, how, chunks):
    if how == "host":
        for c in chunks:
            job.feed(c)
        return
    import torch
    for c in chunks:
        dev = torch.from_numpy(np.frombuffer(c, np.uint8).copy()).cuda()
        torch.cuda.synchronize()
        job.feed_dev(dev.data_ptr(), len(c))
        del dev


def fresh_finish(gpu, ref, ref_n, p, how, chunks, winner, lengths):
    job = gpu.screen_open(ref, ref_n, p, ref_len=lengths)
    try:
        job.set_winner(winner)
        feed(job, how, chunks)
        return job.finish()
    finally:
        job.close()


def same(a, b):
    for f in FIELDS:
        assert a[f].dtype == b[f].dtype and np.array_equal(a[f], b[f]), f        # floats compared with ==
    assert a["set_size"] == b["set_size"]


def same_rows(hits, want):
    rows = np.flatnonzero(want["shared"] >= 1)
    assert np.array_equal(hits["ref"], rows.astype(np.uint32))
    for f in FIELDS:
        assert np.array_equal(hits[f], want[f][rows]), f
    assert hits["set_size"] == want["set_size"]
    # the closed form of the rows left out
    rest = np.flatnonzero(want["shared"] == 0)
    assert np.all(want["median"][rest] == 0) and np.all(want["pvalue"][rest] == 1.0)


def run_samples(gpu, ref, ref_n, p, samples, winner=False, lengths=None, want_of=None):
    """Feeds the samples one after another on one job with reset() between them; checks each against a fresh job and, when
    want_of is given, against want_of(chunks).  Returns [(finish, finish_hits, hits_stats)]."""
    out = []
    job = gpu.screen_open(ref, ref_n, p, ref_len=lengths)
    try:
        job.set_winner(winner)
        for how, chunks in samples:
            feed(job, how, chunks)
            hits = job.finish_hits()
            stats = job.hits_stats()
            fin = job.finish()
            same_rows(job.finish_hits(), fin)                 # twice in a row, and finish() in between, change nothing
            same(job.finish(), fin)
            fresh = fresh_finish(gpu, ref, ref_n, p, how, chunks, winner, lengths)
            same(fin, fresh)
            assert np.array_equal(fin["mixture"], fresh["mixture"])
            same_rows(hits, fresh)
            if want_of is not None and chunks:
                check(fin, want_of(chunks))
            out.append((fin, hits, stats))
            job.reset()
    finally:
        job.close()
    return out


def model_stats(ref, ref_n, counts, keys, winner=False):
    index = ssm.build_index(ref, ref_n)
    cnt = np.zeros(index["distinct"].size, np.int64)
    cnt[np.searchsorted(index["distinct"], keys)] = counts[:keys.size]
    return ssm.sparse(index, cnt, ref_n, winner=winner)[1]


@pytest.mark.parametrize("k,s", [(21, 1000), (15, 400)])
def test_samples_match_fresh_jobs_and_the_oracle(gpu, oracle, k, s):
    p = gpu.params(k=k, s=s)
    po = oracle.params(k=k)
    assert bool(p.use64) == (k > 16)
    genomes = [synth_genome(140 + i, 120_000) for i in range(3)]
    genomes.append(mutate(genomes[0], 0.02, 5))
    ref, ref_n = nucleotide_refs(oracle, po, s, genomes)
    samples = nucleotide_samples(genomes, 10 * k)
    res = run_samples(gpu, ref, ref_n, p, samples, want_of=lambda ch: oracle.screen(ref, ref_n, ch, po, s=s))
    assert res[1][1]["ref"].size == 0 and res[1][0]["set_size"] == 0           # the empty sample
    assert res[2][0]["set_size"] > 0                                           # an unrelated genome's reads: no hit at k=21
    if k == 21:
        assert res[2][1]["ref"].size == 0
    assert all(r[1]["ref"].size > 0 for i, r in enumerate(res) if i not in (1, 2))
    for (how, chunks), (_, _, stats) in zip(samples, res):
        if chunks:
            want = oracle.screen(ref, ref_n, chunks, po, s=s)
            st = model_stats(ref, ref_n, want["counts"], want["keys"])
            assert (stats["hit_hashes"], stats["hit_pairs"]) == (st["hit_hashes"], st["hit_pairs"])
    assert res[0][2]["index_ms"] > 0


def test_winner_samples(gpu, oracle):
    from test_oracle_screen_winner import build
    po, ref, ref_n, lengths, chunks = build(oracle)
    p = gpu.params(k=21, s=400)
    other = joined(reads_of([synth_genome(4, 120_000)], 2000, 31), 500)
    samples = [("host", chunks), ("host", []), ("host", other), ("host", chunks[:1]), ("dev", chunks[1:])]
    want_of = lambda ch: oracle.screen(ref, ref_n, ch, po, s=400, winner=True, ref_len=lengths)
    res = run_samples(gpu, ref, ref_n, p, samples, winner=True, lengths=lengths, want_of=want_of)
    plain = oracle.screen(ref, ref_n, chunks, po, s=400)
    assert not np.array_equal(res[0][0]["shared"], plain["shared"])             # the reallocation changed the counts
    want = oracle.screen(ref, ref_n, chunks, po, s=400, winner=True, ref_len=lengths)
    st = model_stats(ref, ref_n, want["counts"], want["keys"], winner=True)
    assert (res[0][2]["hit_hashes"], res[0][2]["hit_pairs"]) == (st["hit_hashes"], st["hit_pairs"])


@pytest.mark.parametrize("bitmap", ["1", "0"])
def test_whole_range_table_samples(gpu, oracle, monkeypatch, bitmap):
    monkeypatch.setenv("MASHGPU_SCREEN_BITMAP", bitmap)
    s = 300
    p = gpu.params(k=21, s=s); po = oracle.params(k=21)
    genomes = [synth_genome(140 + i, 120_000) for i in range(3)]
    tiny = [synth_genome(700 + i, 150 + 37 * i) for i in range(6)]
    ref, ref_n = nucleotide_refs(oracle, po, s, genomes + tiny)
    assert ref[np.arange(ref.shape[0]), ref_n - 1].max() > np.uint64(2**63)
    samples = [("host", joined(reads_of(genomes[:2] + tiny[:2], 5000, 40 + i), 1000)) for i in range(3)]
    samples.insert(1, ("host", joined(reads_of(tiny[2:4], 500, 44), 100)))
    zeros = np.zeros(ref_n.size, np.uint64)
    for winner in (False, True):
        run_samples(gpu, ref, ref_n, p, samples, winner=winner,
                    want_of=lambda ch: oracle.screen(ref, ref_n, ch, po, s=s, winner=winner, ref_len=zeros))


def test_protein_samples(gpu, oracle):
    s = 1000
    p = gpu.params(k=9, s=s, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    po = oracle.params(k=9, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    ref, ref_n, lengths = protein_refs(oracle, po, s)
    samples = [("host", joined(reads_from(1200 + i, 3000), 1000)) for i in range(3)]
    samples.insert(1, ("host", []))
    samples.append(("dev", joined(reads_from(1300, 2000), 500)))
    for winner in (False, True):
        run_samples(gpu, ref, ref_n, p, samples, winner=winner, lengths=lengths,
                    want_of=lambda ch: tso.screen(oracle, ref, ref_n, ch, po, s=s, winner=winner, ref_len=lengths))


def test_custom_alphabet_samples(gpu, oracle):
    s = 500
    p = gpu.params(k=15, s=s, alphabet="ACGTN", noncanonical=True)
    po = oracle.params(k=15, alphabet="ACGTN", noncanonical=True)
    genomes = [synth_genome(300 + i, 60_000) for i in range(3)]
    ref, ref_n = nucleotide_refs(oracle, po, s, [g[:30_000] for g in genomes])
    samples = [("host", joined(reads_of([g[:30_000] for g in genomes[:2]], 3000, 50 + i), 600)) for i in range(3)]
    run_samples(gpu, ref, ref_n, p, samples, want_of=lambda ch: oracle.screen(ref, ref_n, ch, po, s=s))


def test_sketches_of_32768_hashes(gpu, oracle):
    s = 1000
    p = gpu.params(k=21, s=s); po = oracle.params(k=21)
    genomes = [synth_genome(810 + i, 200_000) for i in range(2)]
    genomes.append(mutate(genomes[1], 0.02, 821))
    ref, ref_n = nucleotide_refs(oracle, po, 32768, genomes)
    assert (ref_n == 32768).all()
    samples = [("host", joined(reads_of(genomes, 40_000, 60 + i), 10_000)) for i in range(2)]
    zeros = np.zeros(ref_n.size, np.uint64)
    for winner in (False, True):
        res = run_samples(gpu, ref, ref_n, p, samples, winner=winner,
                          want_of=lambda ch: oracle.screen(ref, ref_n, ch, po, s=s, winner=winner, ref_len=zeros))
        assert res[0][1]["shared"].max() > 10_000


def test_5000_identical_sketches(gpu, oracle):
    # every hash is held by 5000 sketches (warp segments); under -w ties in the estimate go to the longest genome, then the
    # lowest index
    s = 500
    p = gpu.params(k=21, s=s); po = oracle.params(k=21)
    g = synth_genome(900, 80_000)
    h, _, _ = oracle.sketch_unit([bytes(g)], po, s=s)
    n = 5000
    ref = np.tile(h, (n, 1)); ref_n = np.full(n, h.size, np.uint32)
    ref_n[::5] = h.size // 2                                     # a prefix: a different estimate for the same hashes
    lengths = (np.arange(n) % 3).astype(np.uint64)
    samples = [("host", joined(reads_of([g], 3000, 70 + i), 1000)) for i in range(2)]
    for winner in (False, True):
        res = run_samples(gpu, ref, ref_n, p, samples, winner=winner, lengths=lengths,
                          want_of=lambda ch: oracle.screen(ref, ref_n, ch, po, s=s, winner=winner, ref_len=lengths))
        if winner:
            assert res[0][1]["ref"].size >= 1


def test_taxonomy_after_reset_equals_a_fresh_job(gpu, oracle):
    s = 400
    p = gpu.params(k=21, s=s); po = oracle.params(k=21)
    genomes = [synth_genome(140 + i, 120_000) for i in range(3)]
    ref, ref_n = nucleotide_refs(oracle, po, s, genomes)
    first, second = joined(reads_of(genomes[:1], 3000, 80), 1000), joined(reads_of(genomes[1:], 3000, 81), 1000)
    parent = np.array([0, 0, 0, 1, 1], np.uint32)
    taxid = np.array([1, 2, 3, 10, 11], np.uint64)
    tax = gpu.taxonomy_open(parent, taxid)
    code = np.array([3, 4, 2], np.uint32)
    try:
        job = gpu.screen_open(ref, ref_n, p)
        try:
            for c in first:
                job.feed(c)
            job.finish_hits()
            job.reset()
            for c in second:
                job.feed(c)
            got = job.taxonomy(tax, code, hash_taxid=True)
        finally:
            job.close()
        job = gpu.screen_open(ref, ref_n, p)
        try:
            for c in second:
                job.feed(c)
            want = job.taxonomy(tax, code, hash_taxid=True)
        finally:
            job.close()
    finally:
        tax.close()
    assert np.array_equal(got["rows"], want["rows"]) and np.array_equal(got["hash_taxid"], want["hash_taxid"])
    assert got["total_count"] == want["total_count"] and got["total_count"] > 0
