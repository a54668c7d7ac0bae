"""CPU model of the translated screen (protein sketches, `mash screen` with trans == true).

tests/translated_screen_oracle.py restates the reference's hashSequence literally: six frame translations of each whole
'*'-joined chunk and the lastGood window walk.  The GPU engine relies on a property of that computation: it does not depend on how the reads are cut
into chunks.  Per record, every nucleotide window W of length 3k yields translate(W) and translate(revcomp(W)), each kept when
it holds no stop or invalid codon.  These tests pin that equivalence and the codon table, independently of the reference.
"""
import collections

import numpy as np
import pytest

import translated_screen_oracle as tso
from oracle.pyoracle import ALPHABET_PROTEIN

# NCBI translation table 1 (the standard code), codons in TCAG order
NCBI_TABLE_1 = "FFLLSSSSYY**CC*WLLLLPPPPHHQQRRRRIIIMTTTTNNKKSSRRVVVVAAAADDEEGGGG"


def standard_code():
    bases = "TCAG"
    return {(a + b + c).encode(): NCBI_TABLE_1[16 * i + 4 * j + m].encode()
            for i, a in enumerate(bases) for j, b in enumerate(bases) for m, c in enumerate(bases)}


CODE = standard_code()
# complement of the bases only ('U' pairs with 'A'); every other byte complements to a non-base
COMPLEMENT = {ord("A"): ord("T"), ord("C"): ord("G"), ord("G"): ord("C"), ord("T"): ord("A"), ord("U"): ord("A")}


def translate(nt: bytes) -> bytes:
    """Codons over {A,C,G,T} by the standard code; anything else (stops, other bytes) as '*'."""
    return b"".join(CODE.get(nt[i:i + 3], b"*") for i in range(0, len(nt) - 2, 3))


def revcomp(nt: bytes) -> bytes:
    return bytes(COMPLEMENT.get(c, ord("N")) for c in reversed(nt))


def fold(rec: bytes, preserve_case: bool) -> bytes:
    return rec if preserve_case else bytes(c - 32 if 96 < c < 123 else c for c in rec)


def model_peptides(records, k, preserve_case):
    """Per record, sliding 3k windows: the amino-acid k-mers of both strands that hold no '*'."""
    for rec in records:
        r = fold(rec, preserve_case)
        for i in range(len(r) - 3 * k + 1):
            w = r[i:i + 3 * k]
            for pep in (translate(w), translate(revcomp(w))):
                if b"*" not in pep:
                    yield pep


def model_counts(oracle, records, k, preserve_case, p):
    return collections.Counter(oracle.get_hash(pep, p.seed, bool(p.use64)) for pep in model_peptides(records, k, preserve_case))


def literal_counts(oracle, chunks, want, p):
    """The literal restatement over `chunks`: (distinct hashes it saw, counts of the model's hashes)."""
    keys = np.array(sorted(want), dtype=np.uint64)
    counts = np.zeros(max(1, keys.size), np.uint32)

    def run(heap):
        for ch in chunks:
            tso.hash_sequence_literal(oracle, heap, keys, counts, ch, p)
    seen = tso.heap_list(oracle, p, run, keys.size + 64)
    return seen, counts[:keys.size]


def fast_counts(oracle, chunks, want, p):
    """The checker's fast form (per-frame window scan) over `chunks`, in the same shape as literal_counts."""
    hashes = np.concatenate([tso.window_hashes(oracle, ch, p) for ch in chunks])
    uniq, mult = np.unique(hashes, return_counts=True)
    keys = np.array(sorted(want), dtype=np.uint64)
    at = np.minimum(np.searchsorted(uniq, keys), uniq.size - 1)
    return uniq, np.where(uniq[at] == keys, mult[at], 0).astype(np.uint32)


def fuzz_records(seed, n):
    rng = np.random.Generator(np.random.PCG64(seed))
    letters = np.frombuffer(b"ACGTACGTACGTACGTACGTACGTacgtNUuRYKMSWBDHVn", np.uint8)
    recs = []
    for i in range(n):
        ln = int(rng.integers(0, 140)) if i % 4 else int(rng.integers(0, 30))     # many shorter than 3k
        ln += i % 3                                                                # every length mod 3
        p = np.where(rng.random(ln) < 0.93, np.frombuffer(b"ACGT", np.uint8)[rng.integers(0, 4, ln)], letters[rng.integers(0, letters.size, ln)])
        if i % 11 == 0:
            p = np.frombuffer(bytes(p).lower(), np.uint8)
        recs.append(bytes(p.astype(np.uint8)))
    return recs


def test_codon_table_is_the_standard_code():
    for codon, aa in CODE.items():
        assert tso.aa_from_codon(codon) == aa, codon
        assert tso.six_frames(codon, False)[0].tobytes() == aa, codon
    assert len(CODE) == 64 and sum(v == b"*" for v in CODE.values()) == 3
    for bad in (b"NAA", b"AUG", b"ATU", b"aaa", b"AC*", b"A\x00G", b"RYK"):
        assert tso.aa_from_codon(bad) == b"*", bad
    # the translation kernel carries the same table (a copy: the library cannot import the checker)
    import os
    src = open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "mash_b200", "csrc", "translate.cu")).read()
    assert '"' + tso.CODON_AA.decode() + '"' in src


def test_model_translation_basics():
    assert translate(b"ATGGCCTAA") == b"MA*"
    assert translate(b"ATGGC") == b"M"
    assert revcomp(b"AUGC") == b"GCAT"
    assert revcomp(b"ACGTNRa*") == b"NNNNACGT"


@pytest.mark.parametrize("k", [9, 7])
@pytest.mark.parametrize("preserve_case", [False, True])
def test_translated_hash_sequence_is_chunk_independent(oracle, k, preserve_case):
    p = oracle.params(k=k, alphabet=ALPHABET_PROTEIN, noncanonical=True, preserve_case=preserve_case)
    assert bool(p.use64) == (k == 9)
    assert tso.is_translated(p)
    records = fuzz_records(100 + k + 7 * preserve_case, 400)
    want = model_counts(oracle, records, k, preserve_case, p)
    assert sum(want.values()) > 1000
    expect_keys = np.array(sorted(want), dtype=np.uint64)
    expect_counts = np.array([want[h] for h in sorted(want)], dtype=np.uint32)
    cuts = {
        "one chunk": [b"".join(b"*" + r for r in records)],
        "chunks of 37": [b"".join(b"*" + r for r in records[i:i + 37]) for i in range(0, len(records), 37)],
        "one record each": [b"*" + r for r in records],
        "zero-joined": [b"".join(b"\0" + r for r in records[i:i + 50]) for i in range(0, len(records), 50)],
    }
    for name, chunks in cuts.items():
        for form, fn in (("literal", literal_counts), ("fast", fast_counts)):
            got_keys, got_counts = fn(oracle, chunks, want, p)
            assert np.array_equal(got_keys, expect_keys), (name, form)
            assert np.array_equal(got_counts, expect_counts), (name, form)


def test_translated_screen_selects_trans_path(oracle):
    # a record of poly-A translates to poly-K on the forward strand and poly-F on the reverse strand
    p = oracle.params(k=9, alphabet=ALPHABET_PROTEIN, noncanonical=True)
    h_k = oracle.get_hash(b"K" * 9, 42, True)
    h_f = oracle.get_hash(b"F" * 9, 42, True)
    ref = np.array([[min(h_k, h_f), max(h_k, h_f)]], dtype=np.uint64)
    res = tso.screen(oracle, ref, np.array([2], np.uint32), [b"*" + b"A" * 40], p, s=100)
    # 40 bases hold 40 - 27 + 1 = 14 windows of 9 codons, on each strand
    assert sorted(res["counts"].tolist()) == [14, 14]
    assert res["shared"][0] == 2
    # not translated: a nucleotide sketch screens the same chunk as nucleotide k-mers
    assert not tso.is_translated(oracle.params(k=9))
    assert not tso.is_translated(oracle.params(k=9, alphabet="ACDEFGHIKLMNPQRSTVW", noncanonical=True))


@pytest.mark.parametrize("k,s,preserve_case", [(9, 50, False), (7, 200, True)])
def test_translated_screen_fast_form_equals_literal_form(oracle, k, s, preserve_case):
    # the whole screen (table, heap, reduce) through the literal hashSequence and through the fast form used by the GPU tests
    p = oracle.params(k=k, alphabet=ALPHABET_PROTEIN, noncanonical=True, preserve_case=preserve_case)
    records = fuzz_records(300 + k, 300)
    chunks = [b"".join(b"*" + r for r in records[i:i + 60]) for i in range(0, len(records), 60)]
    peps = sorted(set(model_peptides(records, k, preserve_case)))
    rng = np.random.Generator(np.random.PCG64(k))
    sel = [peps[int(i)] for i in rng.choice(len(peps), 40, replace=False)]
    rows = [sorted({oracle.get_hash(q, p.seed, bool(p.use64)) for q in sel[i::4]}) for i in range(4)]
    ref = np.full((5, 16), np.uint64(2**64 - 1)); ref_n = np.zeros(5, np.uint32)
    for i, r in enumerate(rows + [[oracle.get_hash(b"W" * k, p.seed, bool(p.use64))]]):
        ref[i, :len(r)] = r; ref_n[i] = len(r)
    lens = np.arange(5, dtype=np.uint64) + 100
    for winner in (False, True):
        a = tso.screen(oracle, ref, ref_n, chunks, p, s=s, winner=winner, ref_len=lens, literal=True)
        b = tso.screen(oracle, ref, ref_n, chunks, p, s=s, winner=winner, ref_len=lens)
        assert a["set_size"] == b["set_size"] and a["set_size"] > 0
        for key in ("mixture", "counts", "shared", "median", "identity", "pvalue"):
            assert np.array_equal(a[key], b[key]), (key, winner)
    assert a["shared"][:4].min() > 0
