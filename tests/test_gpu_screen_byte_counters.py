"""Per-hash hit counters of the translated screen (protein sketches) and of the byte-alphabet screen (`-z`), against the
checkers: translated_screen_oracle.screen(...)["counts"] and oracle.screen(...)["counts"].  The reference tables are dense
(each sketch holds every k-mer of a short protein or letter string), so one wrong amino acid or letter anywhere in the
mixture moves a counter; the aggregates (shared, median, identity, p-value, mixture) can stay the same.  Every feed path
runs: small host chunks joined inside the library, host chunks of at least 4 MiB (the two-buffer pipeline), and device
chunks at offsets 0 (the translation kernel's vector loads) and 1 and 5 (its byte loads)."""
import numpy as np
import pytest

from fixtures import synth_genome
import translated_screen_oracle as tso
from oracle.pyoracle import ALPHABET_PROTEIN
from test_gpu_screen import check
from test_translate_model import revcomp, translate

LARGE = 4 << 20       # host chunks from this size on are fed through the pipeline, not joined
S = 300               # above the k-mer count of every reference: each sketch is all its k-mers
CASES = [(ALPHABET_PROTEIN, 7, False), (ALPHABET_PROTEIN, 7, True), (ALPHABET_PROTEIN, 9, False), (ALPHABET_PROTEIN, 9, True),
         ("ABCDEFGH", 10, False), ("ACGTN", 15, False)]
IDS = ["protein-k7", "protein-k7-preserve_case", "protein-k9", "protein-k9-preserve_case", "ABCDEFGH-k10", "ACGTN-k15"]
FEEDS = ["host", "large", "dev0", "dev1", "dev5"]


def _sources(alphabet):
    """Source strings the reads are cut from: nucleotide genomes for the translated screen, letter strings otherwise."""
    if alphabet == ALPHABET_PROTEIN:
        return [synth_genome(400 + i, 8000) for i in range(2)]
    return [synth_genome(420 + i, 8000, alphabet=alphabet.encode()) for i in range(2)]


def dense_refs(oracle, po, alphabet):
    """Sketches of every k-mer of short proteins (both strands, all three frames of a source) or of short letter strings,
    and one unrelated sketch."""
    g = _sources(alphabet)
    if alphabet == ALPHABET_PROTEIN:
        prots = [translate(bytes(g[0][a + a // 600 % 3:a + 600])) for a in range(0, 6000, 600)]
        prots += [translate(revcomp(bytes(g[1][a:a + 900]))) for a in (0, 901, 1802)]
        prots += [bytes(synth_genome(440, 150, alphabet=ALPHABET_PROTEIN.encode()))]
    else:
        prots = [bytes(g[0][a:a + 200]) for a in range(0, 6000, 200)] + [bytes(g[1][a:a + 250]) for a in (0, 251, 502)]
        prots += [bytes(synth_genome(441, 150, alphabet=alphabet.encode()))]
    ref = np.full((len(prots), S), np.uint64(2**64 - 1)); ref_n = np.zeros(len(prots), np.uint32)
    for i, prot in enumerate(prots):
        h, _, _ = oracle.sketch_unit([prot], po, s=S)
        assert 0 < h.size < S
        ref[i, :h.size] = h; ref_n[i] = h.size
    return ref, ref_n


def make_reads(alphabet, seed, total):
    """Reads of 1..300 bytes, both strands for nucleotides, cut mostly from the regions the references cover, with N, U, R,
    junk bytes and lower-case stretches, until `total` bytes."""
    g = _sources(alphabet)
    rng = np.random.Generator(np.random.PCG64(seed))
    junk = np.frombuffer(b"NURnu*X\x00\x80", np.uint8)
    reads, size = [], 0
    while size < total:
        src = g[int(rng.integers(0, 2))]
        n = int(rng.integers(1, 301))
        hi = 6600 if rng.random() < 0.9 else src.size
        a = int(rng.integers(0, max(1, min(hi, src.size) - n)))
        r = src[a:a + n].copy()
        u = rng.random()
        if u < 0.1:
            r[int(rng.integers(0, r.size))] = junk[int(rng.integers(0, junk.size))]
        elif u < 0.2:
            i = int(rng.integers(0, r.size))
            r[i:i + int(rng.integers(1, 40))] |= 0x20
        r = bytes(r)
        if alphabet == ALPHABET_PROTEIN and rng.random() < 0.5:
            r = revcomp(r)
        reads.append(r)
        size += len(r) + 1
    return reads


def chunked(reads, size):
    """'*'-joined chunks of at least `size` bytes (the reads left over join the last one); chunk i is padded to a length
    = i (mod 3) with a read too short to hold a k-mer, so that chunk lengths take every value mod 3."""
    chunks, cur, n = [], [], 0
    for r in reads:
        cur.append(b"*" + r); n += len(r) + 1
        if n >= size:
            chunks.append(b"".join(cur)); cur, n = [], 0
    if cur:
        tail = b"".join(cur)
        if chunks:
            chunks[-1] += tail
        else:
            chunks.append(tail)
    return [c + b"*" + b"A" * ((i - len(c) - 1) % 3) for i, c in enumerate(chunks)]


def read_starts(chunks):
    return np.concatenate([np.flatnonzero(np.frombuffer(c, np.uint8) == ord("*")) + 1 for c in chunks])


_DATA = {}


def case_data(oracle, alphabet, k, preserve_case):
    key = (alphabet, k, preserve_case)
    if key not in _DATA:
        po = oracle.params(k=k, alphabet=alphabet, noncanonical=True, preserve_case=preserve_case)
        ref, ref_n = dense_refs(oracle, po, alphabet)
        reads = make_reads(alphabet, 500 + k + 7 * preserve_case, 3 * LARGE + 3 * 300_000)
        feeds = {"host": chunked(reads, 150_000), "large": chunked(reads, LARGE), "dev": chunked(reads, 1 << 20)}
        assert min(len(c) for c in feeds["large"]) >= LARGE
        for name, chunks in feeds.items():
            assert np.unique(read_starts(chunks) % 48).size == 48, name
            assert {len(c) % 3 for c in chunks} == {0, 1, 2}, name
        if alphabet == ALPHABET_PROTEIN:
            assert tso.is_translated(po)
            want = tso.screen(oracle, ref, ref_n, feeds["host"], po, s=S)
        else:
            assert not tso.is_translated(po)
            want = oracle.screen(ref, ref_n, feeds["host"], po, s=S)
        assert (want["counts"] > 0).sum() > 0.5 * want["counts"].size and want["counts"].max() > 20
        _DATA[key] = (ref, ref_n, feeds, want)
    return _DATA[key]


def _counters(job):
    import torch
    ptr, n = job.counters()

    class Cai:
        __cuda_array_interface__ = {"shape": (n,), "typestr": "<i4", "data": (ptr, False), "version": 3}
    return torch.as_tensor(Cai(), device="cuda:0").cpu().numpy().view(np.uint32).copy()


def _feed_dev(job, chunk, offset):
    # the chunk at `offset` bytes past a 512-byte aligned allocation, readable up to its end rounded up to 16
    import torch
    host = np.zeros(offset + len(chunk) + 16, np.uint8)
    host[offset:offset + len(chunk)] = np.frombuffer(chunk, np.uint8)
    dev = torch.from_numpy(host).cuda()
    torch.cuda.synchronize()
    job.feed_dev(dev.data_ptr() + offset, len(chunk))


@pytest.mark.gpu
@pytest.mark.parametrize("feed", FEEDS)
@pytest.mark.parametrize("alphabet,k,preserve_case", CASES, ids=IDS)
def test_counters_match_checker(gpu, oracle, alphabet, k, preserve_case, feed):
    ref, ref_n, feeds, want = case_data(oracle, alphabet, k, preserve_case)
    p = gpu.params(k=k, s=S, alphabet=alphabet, noncanonical=True, preserve_case=preserve_case)
    assert bool(p.use64) == (k in (9, 15))
    job = gpu.screen_open(ref, ref_n, p)
    try:
        for c in feeds["dev" if feed.startswith("dev") else feed]:
            if feed.startswith("dev"):
                _feed_dev(job, c, int(feed[3:]))
            else:
                job.feed(c)
        res = job.finish()
        cnt = _counters(job)
    finally:
        job.close()
    assert cnt.size == want["keys"].size
    if not np.array_equal(cnt, want["counts"]):
        bad = np.flatnonzero(cnt != want["counts"])
        pytest.fail(f"{bad.size} of {cnt.size} counters differ, e.g. key {want['keys'][bad[0]]:#x}: got {cnt[bad[0]]}, want "
                    f"{want['counts'][bad[0]]}")
    check(res, want)


def test_checker_sees_one_amino_acid(oracle):
    # one codon changed in one read (to another amino acid, not a stop) changes the checker's counters: a kernel that
    # mistranslated a single codon of the mixture would fail the comparison above
    k = 9
    po = oracle.params(k=k, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    ref, ref_n = dense_refs(oracle, po, ALPHABET_PROTEIN)
    g = _sources(ALPHABET_PROTEIN)
    reads = [bytes(g[0][a:a + 150]) for a in range(0, 6000, 97)]
    base = tso.screen(oracle, ref, ref_n, [b"".join(b"*" + r for r in reads)], po, s=S)["counts"]
    assert base.sum() > 1000
    r = bytearray(reads[20])                            # bases 1940..2089 of the source, inside the protein translated from 1800
    at = 75 + (1800 - 1940) % 3                         # a codon in that protein's frame, in the middle of the read
    old = tso.aa_from_codon(bytes(r[at:at + 3]))
    r[at:at + 3] = next(c for c in (b"TGG", b"ATG", b"GCC") if tso.aa_from_codon(c) != old)
    mutated = reads[:20] + [bytes(r)] + reads[21:]
    got = tso.screen(oracle, ref, ref_n, [b"".join(b"*" + q for q in mutated)], po, s=S)["counts"]
    assert not np.array_equal(got, base)
    assert (got < base).any()                          # the k-mers over the old amino acid lost a hit
