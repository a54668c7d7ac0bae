"""Checker for the translated screen (protein sketches; TEST INFRASTRUCTURE, never imported by the product).

`mash screen` with a protein sketch runs hashSequence with trans == true (reference CommandScreen.cpp:120, 484-599): each
'*'-joined chunk is upper-cased unless preserveCase (:500-506), seqRev = reverseComplement of the whole chunk
(Sketch.cpp:1071-1106), every frame f = 0..2 of (rev ? seqRev : seq) is translated into (l - f) / 3 amino acids
(translate / aaFromCodon, :617-809), and every window of k amino acids without a '*' is hashed as it stands, inserted into
the chunk's MinHashHeap and counted if it is a reference hash.  This module restates that path twice, on top of the
oracle's hash, heap, table and reduce (oracle/pyoracle.py):

  hash_sequence_literal   the reference's own structure: frame loop, per-chunk translation, the lastGood walk and its
                          '*' test, one getHash / tryInsert per window.  Slow; used on small inputs.
  screen                  the same chunk translation, each frame's windows hashed by the oracle's window scan
                          (mo_all_hashes: every window of alphabet bytes; '*' lies outside the protein alphabet), then the
                          oracle's table, heap and reduce.  tests/test_translate_model.py pins it to the literal form.

Where the reference is undefined: reverseComplement indexes complement[c - 'A'] out of range for bytes outside 'A'..'Z'
(the '*' separators, lower case under preserveCase); here they complement to 'N', a non-base.  Inside 'A'..'Z' the
reference's table maps A, C, G, T, U to T, G, C, A, A and every other letter outside {A,C,G,T}, which is all translation
can tell apart, so the other letters are written as 'N' too.  The lastGood loop reads seqTrans[length] one past the end when
lastGood reaches length; by then j > length - k whatever that byte is, so the loop ends either way: bounds-checked here.
"""
import ctypes as C

import numpy as np

from oracle.pyoracle import ALPHABET_PROTEIN, _ptr, f64p, u32p, u64p

# aaFromCodon as a table: index 16 b0 + 4 b1 + b2 with A0 C1 G2 T3 ('*' = stop)
CODON_AA = b"KNKNTTTTRSRSIIMIQHQHPPPPRRRRLLLLEDEDAAAAGGGGVVVV*Y*YSSSS*CWCLFLF"
_BASE = np.full(256, 4, np.int64)
for _i, _c in enumerate(b"ACGT"):
    _BASE[_c] = _i
_AA = np.frombuffer(CODON_AA + b"*", np.uint8)            # index 64: a codon with a byte outside {A,C,G,T}
_COMPLEMENT = np.full(256, ord("N"), np.uint8)
for _a, _b in zip(b"ACGTU", b"TGCAA"):
    _COMPLEMENT[_a] = _b


def is_translated(p):
    """CommandScreen.cpp:120: a protein sketch (alphabet == alphabetProtein) switches screen to translated mode."""
    return [i for i in range(256) if p.alphabet[i]] == sorted(ALPHABET_PROTEIN.encode())


def aa_from_codon(codon: bytes) -> bytes:
    if len(codon) != 3 or any(_BASE[c] == 4 for c in codon):
        return b"*"
    return bytes([CODON_AA[16 * _BASE[codon[0]] + 4 * _BASE[codon[1]] + _BASE[codon[2]]]])


def _as_u8(chunk):
    return np.frombuffer(chunk, np.uint8) if isinstance(chunk, (bytes, bytearray)) else np.ascontiguousarray(chunk, np.uint8)


def fold_and_reverse(chunk, preserve_case):
    """(seq, seqRev) of one chunk: upper-cased unless preserve_case (:500-506), and its reverse complement."""
    seq = _as_u8(chunk).copy()
    if not preserve_case:
        low = (seq > 96) & (seq < 123)
        seq[low] -= 32
    return seq, _COMPLEMENT[seq[::-1]]


def six_frames(chunk, preserve_case):
    """translate((rev ? seqRev : seq) + frame, (l - frame) / 3) for the six (frame, rev) of :516-530, in that order."""
    seq, rev = fold_and_reverse(chunk, preserve_case)
    out = []
    for i in range(6):
        frame, src = i % 3, (rev if i > 2 else seq)
        n = max(0, src.size - frame) // 3                   # C division of a non-negative length, 0 when l < frame
        codons = _BASE[src[frame:frame + 3 * n].reshape(n, 3)]
        idx = np.where((codons == 4).any(axis=1), 64, codons[:, 0] * 16 + codons[:, 1] * 4 + codons[:, 2])
        out.append(_AA[idx])
    return out


def hash_sequence_literal(oracle, heap, keys, counts, chunk, p):
    """hashSequence, trans == true, with the reference's loop structure (:516-599)."""
    k = p.kmer_size
    for seq_trans in six_frames(chunk, bool(p.preserve_case)):
        st = seq_trans.tobytes()
        length = len(st)
        last_good = -1
        j = 0
        while j < length - k + 1:
            while last_good < j + k - 1 and last_good < length:
                last_good += 1
                if last_good < length and st[last_good] == ord("*"):
                    j = last_good + 1
            if j > length - k:
                break
            h = oracle.get_hash(st[j:j + k], p.seed, bool(p.use64))
            if heap is not None:
                oracle.lib.mo_heap_try_insert(heap, h)
            at = np.searchsorted(keys, np.uint64(h))
            if at < keys.size and keys[at] == np.uint64(h):
                counts[at] += 1
            j += 1


def window_hashes(oracle, chunk, p):
    """Every kept amino-acid k-mer hash of one chunk (six frames; each frame's windows without a '*')."""
    hs = [oracle.all_hashes(f.tobytes(), p) for f in six_frames(chunk, bool(p.preserve_case))]
    return np.concatenate(hs) if hs else np.zeros(0, np.uint64)


def screen(oracle, ref, ref_n, chunks, p, s=1000, winner=False, ref_len=None, literal=False):
    """Translated counterpart of Oracle.screen (same inputs, same dict): the reference table, the chunks' hits and bottom-s
    heap, then the oracle's reduce (mo_screen_finish / mo_screen_finish_winner)."""
    L = oracle.lib
    ref = np.ascontiguousarray(ref, np.uint64); ref_n = np.ascontiguousarray(ref_n, np.uint32)
    nr, stride = ref.shape
    keys = np.empty(max(1, int(ref_n.sum())), dtype=np.uint64)
    nk = L.mo_screen_build_table(_ptr(ref, u64p), _ptr(ref_n, u32p), nr, stride, _ptr(keys, u64p))
    keys = keys[:nk].copy()
    counts = np.zeros(max(1, nk), dtype=np.uint32)
    heap = L.mo_heap_new(int(p.use64), s)
    if literal:
        for ch in chunks:
            hash_sequence_literal(oracle, heap, keys, counts, ch, p)
    else:
        hashes = np.concatenate([window_hashes(oracle, ch, p) for ch in chunks] + [np.zeros(0, np.uint64)])
        uniq, mult = np.unique(hashes, return_counts=True)
        at = np.searchsorted(uniq, keys)
        hit = at < uniq.size
        hit[hit] = uniq[at[hit]] == keys[hit]
        counts[:nk][hit] = mult[at[hit]]
        for h in uniq[:s]:                                  # the heap keeps the s smallest distinct hashes in any order
            L.mo_heap_try_insert(heap, int(h))
    set_size = int(np.uint64(L.mo_heap_estimate_set_size(heap))) if L.mo_heap_size(heap) else 0
    mix = np.empty(s, dtype=np.uint64)
    nm = L.mo_heap_to_list(heap, _ptr(mix, u64p), None)
    L.mo_heap_free(heap)
    shared = np.zeros(nr, np.uint64); median = np.zeros(nr, np.uint64)
    ident = np.zeros(nr, np.float64); pv = np.zeros(nr, np.float64)
    if winner:
        ref_len = np.ascontiguousarray(ref_len, np.uint64)
        L.mo_screen_finish_winner(_ptr(ref, u64p), _ptr(ref_n, u32p), _ptr(ref_len, u64p), nr, stride, _ptr(keys, u64p), _ptr(counts, u32p), nk,
                                  set_size, p.kmer_size, oracle.kmer_space(p), _ptr(shared, u64p), _ptr(median, u64p),
                                  _ptr(ident, f64p), _ptr(pv, f64p))
    else:
        L.mo_screen_finish(_ptr(ref, u64p), _ptr(ref_n, u32p), nr, stride, _ptr(keys, u64p), _ptr(counts, u32p), nk,
                           set_size, p.kmer_size, oracle.kmer_space(p), _ptr(shared, u64p), _ptr(median, u64p),
                           _ptr(ident, f64p), _ptr(pv, f64p))
    return dict(shared=shared, median=median, identity=ident, pvalue=pv, set_size=set_size,
                counts=counts[:nk], keys=keys, mixture=mix[:nm].copy())


def heap_list(oracle, p, hashes_by_chunk_fn, cap):
    """Distinct hashes a fresh heap of `cap` holds after hashes_by_chunk_fn(heap) has run (helper of the model tests)."""
    L = oracle.lib
    heap = L.mo_heap_new(int(p.use64), cap)
    try:
        hashes_by_chunk_fn(heap)
        out = np.empty(cap, np.uint64)
        n = L.mo_heap_to_list(heap, out.ctypes.data_as(C.POINTER(C.c_uint64)), None)
    finally:
        L.mo_heap_free(heap)
    return out[:n]
