"""GPU parity tests for the translated screen (protein sketches: six-frame translation of the mixture) and for the
byte-alphabet screen (custom `-z` alphabets, untranslated), through the C ABI, against the oracle's hash, heap and reduce
(the translated path restated in tests/translated_screen_oracle.py)."""
import numpy as np
import pytest

from fixtures import synth_genome
import translated_screen_oracle as tso
from oracle.pyoracle import ALPHABET_PROTEIN
from test_gpu_screen import check, run_screen
from test_translate_model import revcomp, translate

pytestmark = pytest.mark.gpu

SEG = 30_000          # bases of each source genome that are translated into a reference protein and sampled by the reads


def _genomes():
    return [synth_genome(300 + i, 60_000) for i in range(3)]


def protein_refs(oracle, po, s):
    """Protein sketches: genome 0's frame-0 translation, genome 1's reverse-strand translation, an unrelated genome's
    translation, a random protein, and a short peptide with fewer k-mers than s.  Returns (ref, ref_n, lengths)."""
    g = _genomes()
    prots = [translate(bytes(g[0][:SEG])),
             translate(revcomp(bytes(g[1][:SEG]))),
             translate(bytes(g[2][:SEG])),
             bytes(synth_genome(77, 8000, alphabet=ALPHABET_PROTEIN.encode())),
             bytes(synth_genome(78, 120, alphabet=ALPHABET_PROTEIN.encode()))]
    ref = np.full((len(prots), s), np.uint64(2**64 - 1)); ref_n = np.zeros(len(prots), np.uint32)
    lengths = np.zeros(len(prots), np.uint64)
    for i, prot in enumerate(prots):
        h, _, ln = oracle.sketch_unit([prot], po, s=s)     # '*' (stops) is outside the alphabet: windows never span one
        ref[i, :h.size] = h; ref_n[i] = h.size; lengths[i] = ln
    assert ref_n[-1] < s
    return ref, ref_n, lengths


def reads_from(seed, n, lower=False):
    """150 bp reads of genomes 0 and 1 (first SEG bases), from both strands, with N / U / lower case, and short reads."""
    g = _genomes()
    rng = np.random.Generator(np.random.PCG64(seed))
    reads = []
    for i in range(n):
        src = g[int(rng.integers(0, 2))]
        a = int(rng.integers(0, SEG - 150))
        r = bytearray(src[a:a + 150].tobytes())
        if rng.random() < 0.5:
            r = bytearray(revcomp(bytes(r)))
        u = rng.random()
        if u < 0.05:
            r[int(rng.integers(0, 150))] = ord("N")
        elif u < 0.10:
            r[int(rng.integers(0, 150))] = ord("U")          # a stop on the forward strand, 'A' on the reverse strand
        elif u < 0.12:
            r[int(rng.integers(0, 150))] = ord("R")
        if lower and i % 9 == 0:
            r = bytearray(bytes(r).lower())
        if i % 40 == 0:
            r = r[:int(rng.integers(1, 40))]                # shorter than 3k sometimes
        reads.append(bytes(r))
    return reads


def joined(reads, per):
    return [b"".join(b"*" + r for r in reads[i:i + per]) for i in range(0, len(reads), per)]


@pytest.mark.parametrize("k,s,preserve_case", [(9, 1000, False), (7, 200, True), (9, 200, False), (7, 1000, False)])
def test_translated_screen_matches_oracle(gpu, oracle, k, s, preserve_case):
    p = gpu.params(k=k, s=s, alphabet=ALPHABET_PROTEIN, noncanonical=True, preserve_case=preserve_case)
    po = oracle.params(k=k, alphabet=ALPHABET_PROTEIN, noncanonical=True, preserve_case=preserve_case)
    assert bool(p.use64) == (k == 9)
    ref, ref_n, _ = protein_refs(oracle, po, s)
    reads = reads_from(500 + k, 6000, lower=True)
    one = joined(reads, len(reads))
    want = tso.screen(oracle, ref, ref_n, one, po, s=s)
    # the source proteins are found, on both strands; the unrelated ones are not
    assert want["shared"][0] > 0 and want["shared"][1] > 0
    assert want["identity"][0] > 0.9 and want["identity"][1] > 0.9
    assert want["shared"][3] == 0
    check(run_screen(gpu, ref, ref_n, p, one), want)
    # many small host chunks (joined inside the library with 0 bytes); the answer does not depend on the cut
    check(run_screen(gpu, ref, ref_n, p, joined(reads, 7)), want)
    assert tso.screen(oracle, ref, ref_n, joined(reads, 7), po, s=s)["counts"].tolist() == want["counts"].tolist()


def test_translated_large_chunks_ignore_host_pack(gpu, oracle, monkeypatch):
    # chunks above the joining threshold go through the two-buffer pipeline; the 2-bit host packer cannot carry 'U', so a
    # translated job uploads ASCII whatever MASHGPU_SCREEN_HOST_PACK says
    monkeypatch.setenv("MASHGPU_SCREEN_HOST_PACK", "1")
    s = 1000
    p = gpu.params(k=9, s=s, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    po = oracle.params(k=9, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    ref, ref_n, _ = protein_refs(oracle, po, s)
    reads = reads_from(600, 90_000)
    chunks = joined(reads, 30_000)
    chunks[1] = chunks[1] + b"*ACGUACGTACGTACGTACGTACGTACGTACGTAC"          # a length that is not a multiple of 3, 16 or 32
    assert min(len(c) for c in chunks) >= 4 << 20
    want = tso.screen(oracle, ref, ref_n, chunks, po, s=s)
    job = gpu.screen_open(ref, ref_n, p)
    try:
        for c in chunks:
            buf = bytearray(c)
            job.feed(bytes(buf))
            buf[:] = b"N" * len(buf)          # the caller may reuse its buffer as soon as feed() returns
        res = job.finish()
    finally:
        job.close()
    check(res, want)


@pytest.mark.parametrize("offset", [0, 1, 5])
def test_translated_feed_dev(gpu, oracle, offset):
    # device-resident chunks, also at addresses that are not 16-byte aligned (the translation kernel's byte-load path)
    import torch
    s = 200
    p = gpu.params(k=9, s=s, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    po = oracle.params(k=9, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    ref, ref_n, _ = protein_refs(oracle, po, s)
    chunks = joined(reads_from(700, 4000), 1000)
    want = tso.screen(oracle, ref, ref_n, chunks, po, s=s)
    job = gpu.screen_open(ref, ref_n, p)
    try:
        for c in chunks:
            host = np.zeros(offset + len(c) + 16, np.uint8)
            host[offset:offset + len(c)] = np.frombuffer(c, np.uint8)
            dev = torch.from_numpy(host).cuda()
            torch.cuda.synchronize()
            job.feed_dev(dev.data_ptr() + offset, len(c))
            del dev
        res = job.finish()
    finally:
        job.close()
    check(res, want)


@pytest.mark.parametrize("bitmap", ["1", "0"])
def test_translated_table_spanning_the_whole_hash_range(gpu, oracle, monkeypatch, bitmap):
    # short peptides: each sketch is every k-mer, hashes up to ~2^64, so every amino-acid k-mer of the mixture probes the table
    monkeypatch.setenv("MASHGPU_SCREEN_BITMAP", bitmap)
    s = 300
    p = gpu.params(k=9, s=s, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    po = oracle.params(k=9, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    g = _genomes()
    prots = [translate(bytes(g[0][a:a + 600])) for a in range(0, 6000, 600)] + [translate(revcomp(bytes(g[1][:900])))]
    prots += [bytes(synth_genome(900 + i, 150, alphabet=ALPHABET_PROTEIN.encode())) for i in range(4)]
    ref = np.full((len(prots), s), np.uint64(2**64 - 1)); ref_n = np.zeros(len(prots), np.uint32)
    for i, prot in enumerate(prots):
        h, _, _ = oracle.sketch_unit([prot], po, s=s)
        ref[i, :h.size] = h; ref_n[i] = h.size
    assert ref[np.arange(ref.shape[0]), ref_n - 1].max() > np.uint64(2**63)
    chunks = joined(reads_from(800, 5000), 1000)
    want = tso.screen(oracle, ref, ref_n, chunks, po, s=s)
    assert want["shared"][0] > 0 and want["shared"][10] > 0 and want["shared"][-1] == 0
    check(run_screen(gpu, ref, ref_n, p, chunks), want)


def test_translated_repetitive_mixture_takes_the_exact_rerun(gpu, oracle):
    # poly-A reads translate to poly-K / poly-F (and a few other repeats): a chunk holds far fewer distinct k-mers than s,
    # so the first pass cannot fill its candidate list and the chunk is re-run exactly
    s = 1000
    p = gpu.params(k=9, s=s, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    po = oracle.params(k=9, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    ref, ref_n, _ = protein_refs(oracle, po, s)
    ref[-1, :2] = np.sort(np.array([oracle.get_hash(b"K" * 9), oracle.get_hash(b"F" * 9)], np.uint64))
    ref_n[-1] = 2
    reads = [b"A" * 150] * 3000 + [b"AAC" * 50] * 500 + [b"aaaaaaaaaaaaaaaaaaaaaaaaaaaaaaNAAAAAAAAAAAAAAAAAAAAAAAAAAAAUA"] * 100
    chunks = joined(reads, 800)
    want = tso.screen(oracle, ref, ref_n, chunks, po, s=s)
    assert want["mixture"].size < s and want["shared"][-1] == 2
    before = gpu.stats()["exact_reruns"]
    check(run_screen(gpu, ref, ref_n, p, chunks), want)
    assert gpu.stats()["exact_reruns"] > before


def test_translated_winner_take_all(gpu, oracle):
    # `-w` on a translated job: genome 0's protein is also held, in part, by a second sketch
    s = 400
    p = gpu.params(k=9, s=s, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    po = oracle.params(k=9, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    g = _genomes()
    prots = [translate(bytes(g[0][:SEG])), translate(bytes(g[0][:SEG // 3])), translate(revcomp(bytes(g[1][:SEG])))]
    ref = np.full((len(prots), s), np.uint64(2**64 - 1)); ref_n = np.zeros(len(prots), np.uint32)
    lengths = np.zeros(len(prots), np.uint64)
    for i, prot in enumerate(prots):
        h, _, ln = oracle.sketch_unit([prot], po, s=s)
        ref[i, :h.size] = h; ref_n[i] = h.size; lengths[i] = ln
    chunks = joined(reads_from(1000, 4000), 1000)
    want_plain = tso.screen(oracle, ref, ref_n, chunks, po, s=s)
    want = tso.screen(oracle, ref, ref_n, chunks, po, s=s, winner=True, ref_len=lengths)
    assert not np.array_equal(want["shared"], want_plain["shared"])
    job = gpu.screen_open(ref, ref_n, p, ref_len=lengths)
    try:
        for c in chunks:
            job.feed(c)
        check(job.finish(), want_plain)
        job.set_winner(True)
        res = job.finish()
    finally:
        job.close()
    check(res, want)


def test_custom_alphabet_screen_is_untranslated(gpu, oracle):
    # `-z ACGTN`: a non-nucleotide, non-protein alphabet screens byte k-mers of the reads as they stand (CommandScreen.cpp:541)
    s = 500
    p = gpu.params(k=15, s=s, alphabet="ACGTN", noncanonical=True)
    po = oracle.params(k=15, alphabet="ACGTN", noncanonical=True)
    assert not tso.is_translated(po)
    g = _genomes()
    ref = np.full((3, s), np.uint64(2**64 - 1)); ref_n = np.zeros(3, np.uint32)
    for i in range(3):
        h, _, _ = oracle.sketch_unit([bytes(g[i][:SEG])], po, s=s)
        ref[i, :h.size] = h; ref_n[i] = h.size
    reads = [r.replace(b"U", b"A") for r in reads_from(1100, 5000)]
    chunks = joined(reads, 1000)
    want = oracle.screen(ref, ref_n, chunks, po, s=s)
    assert want["shared"][0] > 0 and want["shared"][2] == 0
    check(run_screen(gpu, ref, ref_n, p, chunks), want)
    check(run_screen(gpu, ref, ref_n, p, joined(reads, 5)), want)
