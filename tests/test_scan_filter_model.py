"""CPU model of the scan kernel's filter word (mash_b200/csrc/murmur3.cuh, murmur3_h1_filter / filter_threshold).

For k > 16 the fast path of scan_kernel does not finish MurmurHash3: of h1 = fmix(a) + fmix(b) it computes only
X = hi(fmix(a)) + hi(fmix(b)) + 1 (mod 2^32) -- the carry out of the low words is never formed -- and lets a window through
when X <= filter_threshold(tmax >> 32).  The slow path then recomputes the exact hash and applies the exact `<= tmax`.
So the filter may let extra hashes through but must never reject one whose exact high word is <= tmax >> 32.  The sketch
parity tests would not notice a filter that drops boundary hashes (the per-unit thresholds keep 3x headroom), hence this model.
"""
import numpy as np
import pytest

M32 = 0xFFFFFFFF
M64 = (1 << 64) - 1


def fmix64(k):
    k ^= k >> 33
    k = (k * 0xff51afd7ed558ccd) & M64
    k ^= k >> 33
    k = (k * 0xc4ceb9fe1a85ec53) & M64
    k ^= k >> 33
    return k


# Each function below restates one piece of mash_b200/csrc (keep them in step with it):
#   fmix_hi_model    murmur3.cuh  fmix_hi(k, add) with add = 0
#   filter_threshold murmur3.cuh  filter_threshold(t_hi):           t_hi + (t_hi != 0xFFFFFFFFu ? 1u : 0u)
#   filter_word      murmur3.cuh  murmur3_h1_filter:                fmix_hi(h2, fmix_hi(h1, one)), one = 1
#   passes           scan.cuh     scan_group_filter: `x[J] <= tf`,  tf = filter_threshold((uint32_t)(tmax >> 32)) in scan_kernel

def fmix_hi_model(k):
    """fmix_hi as the kernel computes it: 32-bit halves, the last multiply's high word only."""
    lo, hi = k & M32, k >> 32
    lo ^= hi >> 1                                            # k.lo ^= shr1(k.hi)        (k ^= k >> 33 on the halves)
    k = (((hi << 32) | lo) * 0xff51afd7ed558ccd) & M64      # k = mul_const(k, 0xff51afd7ed558ccdULL)
    lo, hi = k & M32, k >> 32
    lo ^= hi >> 1                                            # k.lo ^= shr1(k.hi)
    c = 0xc4ceb9fe1a85ec53
    # mad.hi.u32(k.lo, c_lo, add) + k.lo * c_hi + k.hi * c_lo
    return (((lo * (c & M32)) >> 32) + lo * (c >> 32) + hi * (c & M32)) & M32


def filter_threshold(t_hi):
    return t_hi + (1 if t_hi != M32 else 0)                  # the saturation at 2^32 - 1


def filter_word(fa_hi, fb_hi):
    return (fa_hi + fb_hi + 1) & M32                         # the `one` addend: the carry of the low words replaced by 1


def passes(fa, fb, t_hi):
    return filter_word(fa >> 32, fb >> 32) <= filter_threshold(t_hi)


def exact_hi(fa, fb):
    return ((fa + fb) & M64) >> 32


def test_fmix_hi_is_the_high_word_of_fmix():
    rng = np.random.Generator(np.random.PCG64(7))
    vals = [int(x) for x in rng.integers(0, 1 << 63, 20000, dtype=np.uint64)] + [0, 1, M32, M32 + 1, M64, M64 - 1, 1 << 63]
    vals += [int(x) | (1 << 63) for x in vals[:5000]]
    for k in vals:
        assert fmix_hi_model(k) == fmix64(k) >> 32


EDGE_LO = [0, 1, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, M32]
EDGE_HI = [0, 1, 2, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFE, M32]
EDGE_T = [0, 1, 2, 0x7FFFFFFF, 0x80000000, 0xFFFFFFFD, 0xFFFFFFFE, M32]


def test_never_rejects_a_hash_at_or_below_the_threshold_edges():
    """Every combination of edge halves: carries out of the low words, high words summing to 2^32 - 1 (the exact high word
    wraps to 0 when the low words carry), and thresholds 0 .. 2^32 - 1."""
    for alo in EDGE_LO:
        for blo in EDGE_LO:
            for ahi in EDGE_HI:
                for bhi in EDGE_HI + [(M32 - ahi) & M32, (M32 - ahi - 1) & M32, (-ahi) & M32]:
                    fa, fb = (ahi << 32) | alo, (bhi << 32) | blo
                    H = exact_hi(fa, fb)
                    for t in EDGE_T + [H, (H - 1) & M32, (H + 1) & M32]:
                        if H <= t:
                            assert passes(fa, fb, t), (hex(fa), hex(fb), hex(t))


@pytest.mark.parametrize("seed", [1, 2, 3])
def test_never_rejects_random_and_boundary_thresholds(seed):
    rng = np.random.Generator(np.random.PCG64(seed))
    n = 20000
    fa = [int(x) for x in rng.integers(0, M64, n, dtype=np.uint64, endpoint=True)]
    fb = [int(x) for x in rng.integers(0, M64, n, dtype=np.uint64, endpoint=True)]
    ts = [int(x) for x in rng.integers(0, M32, n, dtype=np.uint64, endpoint=True)]
    for a, b, t in zip(fa, fb, ts):
        H = exact_hi(a, b)
        for tt in (t, H, (H - 1) & M32, M32, 0):
            if H <= tt:
                assert passes(a, b, tt)


def test_extra_passes_are_only_the_next_high_word_or_the_wrap():
    """What gets through besides the exact passes: the one high word T + 1 (carry 1) or filter word 0 (high words summing to
    2^32 - 1 without a carry) -- the slow path's exact test removes them."""
    rng = np.random.Generator(np.random.PCG64(11))
    n = 50000
    hits = 0
    for _ in range(n):
        a = int(rng.integers(0, M64, dtype=np.uint64, endpoint=True))
        b = int(rng.integers(0, M64, dtype=np.uint64, endpoint=True))
        H = exact_hi(a, b)
        t = (H - int(rng.integers(0, 3))) & M32
        if passes(a, b, t) and H > t:
            hits += 1
            assert H == t + 1 or filter_word(a >> 32, b >> 32) == 0
    assert hits > 0


def test_threshold_at_the_top_lets_everything_through():
    for a, b in [(0, 0), (M64, M64), (M64, 1), (0xFFFFFFFF00000000, 0xFFFFFFFF00000000)]:
        assert passes(a, b, M32)
