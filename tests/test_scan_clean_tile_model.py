"""CPU model of the clean-tile check of the filter-word scan kernels' staging (mash_b200/csrc/scan.cuh,
ascii8_to_code_word): each byte's code is ((u >> 1) ^ (u >> 2)) & 3, the ACGT byte of that code is rebuilt by PRMT from
the pool "ACGT", and the byte is clean when it equals that rebuild after the case fold (0xDF, or 0xFF under
preserve_case).  A tile is staged from the codes alone only when every byte is clean, so "clean" must mean exactly "in
the alphabet under that fold", and the codes of clean bytes must be what the validity-testing conversion
(ascii4_to_codes) gives them."""
import numpy as np
import pytest

POOL = np.frombuffer(b"ACGT", np.uint8)


def code(u):
    return ((u >> 1) ^ (u >> 2)) & 3                         # ascii8_to_code_word, from the raw byte


def clean(u, fold):
    return (u & fold) == POOL[code(u)]                       # prmt(pool, 0, codes) ^ (bytes & fold) == 0


def ascii4_to_codes(w, fold):
    """scan.cuh's ascii4_to_codes on one 32-bit word, as the kernel computes it (the conversion with the validity test)."""
    M = 0xFFFFFFFF
    u = w & fold
    t = (u >> 2) & ~(u >> 1) & 0x01010101
    expect = (0x41414141 | (u & 0x06060606)) ^ ((t * 0x11) & M)
    bad = u ^ expect
    nz = ((((bad & 0x7F7F7F7F) + 0x7F7F7F7F) & M) | bad) & 0x80808080
    return (((u >> 1) ^ (u >> 2)) & 0x03030303) | (nz >> 4)


@pytest.mark.parametrize("preserve_case", [False, True])
def test_clean_exactly_when_in_the_alphabet(preserve_case):
    fold = 0xFF if preserve_case else 0xDF
    alphabet = set(b"ACGT") if preserve_case else set(b"ACGTacgt")
    for b in range(256):
        assert bool(clean(np.uint8(b), fold)) == (b in alphabet), hex(b)


@pytest.mark.parametrize("preserve_case", [False, True])
def test_codes_of_clean_bytes_match_the_checked_conversion(preserve_case):
    # every byte value in each lane of a word: clean bytes get the code the validity-testing conversion gives (bit 3 clear),
    # and a byte the check calls dirty is one that conversion marks outside the alphabet (bit 3 set)
    fold8 = 0xFF if preserve_case else 0xDF
    fold = 0xFFFFFFFF if preserve_case else 0xDFDFDFDF
    for lane in range(4):
        for b in range(256):
            other = [0x41, 0x63, 0x47, 0x74]
            bs = other[:lane] + [b] + other[lane + 1:]
            w = int.from_bytes(bytes(bs), "little")
            x = (ascii4_to_codes(w, fold) >> (8 * lane)) & 0xFF
            if clean(np.uint8(b), fold8):
                assert x == code(b), (lane, hex(b))
            else:
                assert x & 8, (lane, hex(b))


def test_nibble_gather_and_rebuild():
    # 8 bytes -> one nibble word (two byte_perm and a shift-or), and the PRMT rebuild of both halves from it
    rng = np.random.Generator(np.random.PCG64(3))
    for _ in range(2000):
        bs = POOL[rng.integers(0, 4, 8)]
        c = [int(code(x)) for x in bs]
        x0 = sum(c[i] << (8 * i) for i in range(4))
        x1 = sum(c[4 + i] << (8 * i) for i in range(4))
        even = (x0 & 0xFF) | ((x0 >> 16 & 0xFF) << 8) | ((x1 & 0xFF) << 16) | ((x1 >> 16 & 0xFF) << 24)        # 0x6420
        odd = (x0 >> 8 & 0xFF) | ((x0 >> 24) << 8) | ((x1 >> 8 & 0xFF) << 16) | ((x1 >> 24) << 24)             # 0x7531
        w = even | (odd << 4)
        assert all((w >> (4 * i)) & 0xF == c[i] for i in range(8))
        rebuilt = bytes(int(POOL[(w >> (4 * i)) & 0xF]) for i in range(8))                                    # prmt(pool, 0, w), w >> 16
        assert rebuilt == bytes(bs)
