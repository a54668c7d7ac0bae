"""CPU model of the scan kernel's tail table (mash_b200/csrc/scan.cuh: TAIL_IDX_MUL, tail_index, fill_tail_table, and the
TAIL_TABLE branch of scan_window_filter).

For 17 <= k <= 21 the filter-word kernels do not hash the tail block (bases 16..k-1) of the canonical k-mer: they look up
its k1 = rotl31(t * c1) * c2 in a 1024-entry table, indexed by the k-mer's last nibble word with the two code bits of every
nibble kept.  This restates MurmurHash3_x64_128 in Python, fills the table as the kernel does (with the index constants read
from scan.cuh), and checks, for every 1..5-base tail, that the lookup is the tail step of the published algorithm.
"""
import itertools
import os
import re

import pytest

M64 = (1 << 64) - 1
C1, C2 = 0x87c37b91114253d5, 0x4cf5ad432745937f
SCAN_CUH = os.path.join(os.path.dirname(__file__), "..", "mash_b200", "csrc", "scan.cuh")
CODE = {ord("A"): 0, ord("C"): 1, ord("G"): 2, ord("T"): 3}


def rotl64(x, r):
    return ((x << r) | (x >> (64 - r))) & M64


def fmix64(k):
    k ^= k >> 33
    k = (k * 0xff51afd7ed558ccd) & M64
    k ^= k >> 33
    k = (k * 0xc4ceb9fe1a85ec53) & M64
    k ^= k >> 33
    return k


def tail_k1(t):
    """k1 of a tail of at most 8 bytes (murmur3.cuh murmur3_tail_k1)."""
    return (rotl64((t * C1) & M64, 31) * C2) & M64


def murmur3_h1(key, seed, k1_tail=None):
    """h1 of MurmurHash3_x64_128; with k1_tail given (tails of 1..8 bytes) the tail's k1 is taken from it."""
    n = len(key)
    h1 = h2 = seed
    nb = n // 16
    for b in range(nb):
        k1 = int.from_bytes(key[16 * b:16 * b + 8], "little")
        k2 = int.from_bytes(key[16 * b + 8:16 * b + 16], "little")
        h1 ^= tail_k1(k1)
        h1 = (rotl64(h1, 27) + h2) & M64
        h1 = (h1 * 5 + 0x52dce729) & M64
        h2 ^= (rotl64((k2 * C2) & M64, 33) * C1) & M64
        h2 = (rotl64(h2, 31) + h1) & M64
        h2 = (h2 * 5 + 0x38495ab5) & M64
    tail = key[16 * nb:]
    if len(tail) > 8:
        h2 ^= (rotl64((int.from_bytes(tail[8:], "little") * C2) & M64, 33) * C1) & M64
    if tail:
        if k1_tail is None:
            k1_tail = tail_k1(int.from_bytes(tail[:8], "little"))
        h1 ^= k1_tail
    h1 ^= n
    h2 ^= n
    h1 = (h1 + h2) & M64
    h2 = (h2 + h1) & M64
    h1 = fmix64(h1)
    h2 = fmix64(h2)
    return (h1 + h2) & M64


def scan_constants():
    src = open(SCAN_CUH).read()

    def get(name):
        m = re.search(r"constexpr\s+\w+\s+" + name + r"\s*=\s*(0x[0-9a-fA-F]+|\d+)u?;", src)
        assert m, name
        return int(m.group(1), 0)
    return get("TAIL_IDX_MUL"), get("TAIL_IDX_SHIFT"), get("TAIL_TAB_SIZE")


MUL, SHIFT, SIZE = scan_constants()


def tail_index(w):
    return ((w * MUL) & 0xFFFFFFFF) >> SHIFT


def last_word(tail):
    """The kernel's index word: the tail's codes at bits 0, 4, .. (the last nibble word masked with LAST_MASK & 0x33333333)."""
    return sum(CODE[c] << (4 * i) for i, c in enumerate(tail))


def fill_table(k):
    """fill_tail_table<K>: all 4^5 code words, the codes past k ignored."""
    tab = [None] * SIZE
    for v in range(4 ** 5):
        codes = [(v >> (2 * i)) & 3 for i in range(5)]
        w = sum(c << (4 * i) for i, c in enumerate(codes))
        t = int.from_bytes(bytes(b"ACGT"[c] for c in codes[:k - 16]), "little")
        tab[tail_index(w)] = tail_k1(t)
    return tab


def test_python_murmur_matches_known_answers(golden):
    n = 0
    for c in golden.murmur_kat:
        if not c["use64"]:
            continue
        assert murmur3_h1(c["kmer"].encode(), c["seed"]) == int(c["hash"]), c["kmer"]
        n += 1
    assert n > 0


def test_index_is_a_bijection_onto_the_table():
    idx = {tail_index(sum(c << (4 * i) for i, c in enumerate(codes))) for codes in itertools.product(range(4), repeat=5)}
    assert len(idx) == 4 ** 5 == SIZE and max(idx) < SIZE


@pytest.mark.parametrize("k", [17, 18, 19, 20, 21])
def test_table_is_the_murmur_tail_step(k):
    tab = fill_table(k)
    assert all(e is not None for e in tab)
    prefixes = [b"ACGTTGCAACGTTGCA", b"TTTTTTTTTTTTTTTT", b"GATTACAGATTACAGA"]
    for tail in itertools.product(b"ACGT", repeat=k - 16):
        tail = bytes(tail)
        want_k1 = tail_k1(int.from_bytes(tail, "little"))
        assert tab[tail_index(last_word(tail))] == want_k1, tail
        for seed, prefix in zip((42, 0, 0x9E3779B9), prefixes):
            key = prefix + tail
            assert murmur3_h1(key, seed, tab[tail_index(last_word(tail))]) == murmur3_h1(key, seed)
