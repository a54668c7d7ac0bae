// murmur3.cuh -- MurmurHash3_x64_128 (first 64 bits) for k-mers of compile-time length K <= 32,
// fed from ASCII words held in registers.  Follows the published algorithm the reference uses
// (reference MurmurHash3.cpp:255-332, fmix64 :81-90; getHash hash.cpp:10-38 keeps h1 only).
#pragma once
#include <cstdint>

namespace mashgpu {

// 64-bit values are carried as two 32-bit halves so that every operation maps onto one SASS instruction:
//   x * const  -> IMAD.WIDE.U32 + 2 IMAD          rotl -> 2 SHF (funnel)        add -> IADD3 + IADD3.X
struct u64x2 { uint32_t lo, hi; };

// The hot loop is bound by the ALU pipe (SHF/LOP3/IADD3/PRMT).  Moving 64-bit adds, shifts, rotates or the PRMT selector
// shift onto the FMA pipe through opaque power-of-two IMADs made the k=21 scan slower on B200 and on H100 (IMAD.WIDE/IMAD.HI
// cost more issue slots than the SHF/IADD3 they replace); the scan uses the FMA pipe only where an add can ride on a
// multiply-add that is there anyway (fmix_hi).

__device__ __forceinline__ u64x2 mul_const(u64x2 a, uint64_t c)
{
    const uint32_t clo = (uint32_t)c, chi = (uint32_t)(c >> 32);
    u64x2 r;
    asm("{\n\t.reg .u64 t;\n\tmul.wide.u32 t, %2, %4;\n\tmov.b64 {%0, %1}, t;\n\t"
        "mad.lo.u32 %1, %2, %5, %1;\n\tmad.lo.u32 %1, %3, %4, %1;\n\t}"
        : "=r"(r.lo), "=&r"(r.hi) : "r"(a.lo), "r"(a.hi), "r"(clo), "r"(chi));
    return r;
}

template <int R>
__device__ __forceinline__ u64x2 rotl(u64x2 a)
{
    u64x2 r;
    if constexpr (R == 32) { r.lo = a.hi; r.hi = a.lo; }
    else if constexpr (R < 32) { r.hi = __funnelshift_l(a.lo, a.hi, R); r.lo = __funnelshift_l(a.hi, a.lo, R); }
    else { r.hi = __funnelshift_l(a.hi, a.lo, R - 32); r.lo = __funnelshift_l(a.lo, a.hi, R - 32); }
    return r;
}

__device__ __forceinline__ u64x2 add64(u64x2 a, u64x2 b)
{
    u64x2 r;
    asm("add.cc.u32 %0, %2, %4;\n\taddc.u32 %1, %3, %5;" : "=r"(r.lo), "=r"(r.hi) : "r"(a.lo), "r"(a.hi), "r"(b.lo), "r"(b.hi));
    return r;
}

__device__ __forceinline__ u64x2 xor64(u64x2 a, u64x2 b) { return u64x2{a.lo ^ b.lo, a.hi ^ b.hi}; }

// a * 5 + c
__device__ __forceinline__ u64x2 mul5_add(u64x2 a, uint32_t c)
{
    u64x2 r;
    asm("{\n\t.reg .u64 t, cc;\n\tcvt.u64.u32 cc, %3;\n\tmad.wide.u32 t, %2, 5, cc;\n\tmov.b64 {%0, %1}, t;\n\t}"
        : "=r"(r.lo), "=r"(r.hi) : "r"(a.lo), "r"(c));
    r.hi = a.hi * 5u + r.hi;
    return r;
}

__device__ __forceinline__ uint32_t shr1(uint32_t x) { return x >> 1; }

__device__ __forceinline__ u64x2 fmix(u64x2 k)
{
    k.lo ^= shr1(k.hi);                      // k ^= k >> 33
    k = mul_const(k, 0xff51afd7ed558ccdULL);
    k.lo ^= shr1(k.hi);
    k = mul_const(k, 0xc4ceb9fe1a85ec53ULL);
    k.lo ^= shr1(k.hi);
    return k;
}

// high word of fmix(k), plus `add` (the final `k ^= k >> 33` only changes the low word).  The addend enters the first
// multiply-add (IMAD.HI), so summing two of these and a constant stays on the FMA pipe.
__device__ __forceinline__ uint32_t fmix_hi(u64x2 k, uint32_t add)
{
    k.lo ^= shr1(k.hi);
    k = mul_const(k, 0xff51afd7ed558ccdULL);
    k.lo ^= shr1(k.hi);
    constexpr uint64_t c = 0xc4ceb9fe1a85ec53ULL;
    uint32_t r;
    asm("mad.hi.u32 %0, %1, %2, %3;" : "=r"(r) : "r"(k.lo), "n"((uint32_t)c), "r"(add));
    return r + k.lo * (uint32_t)(c >> 32) + k.hi * (uint32_t)c;
}

// k1 of the tail block, rotl31(t * c1) * c2, where t holds the tail's (at most 8) bytes; when the tail has 8 bytes or fewer,
// h1 ^= this is all the tail does
__host__ __device__ __forceinline__ uint64_t murmur3_tail_k1(uint64_t t)
{
    t *= 0x87c37b91114253d5ULL;
    t = (t << 31) | (t >> 33);
    return t * 0x4cf5ad432745937fULL;
}

// The body of MurmurHash3_x64_128 up to the finalisation: h1, h2 after the length xor and the two cross adds.
// K1_GIVEN (tails of 1..8 bytes only): the tail's k1 is `k1_tail` (murmur3_tail_k1, e.g. from a table) and the tail words of
// `a` are not read.
template <int K, int NA, bool K1_GIVEN = false>
__device__ __forceinline__ void murmur3_body(const uint32_t (&a)[NA], uint32_t seed, u64x2 &h1_out, u64x2 &h2_out,
                                             u64x2 k1_tail = u64x2{0u, 0u})
{
    constexpr uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
    constexpr int NB = K / 16, TAIL = K & 15;
    u64x2 h1{seed, 0u}, h2{seed, 0u};
#pragma unroll
    for (int b = 0; b < NB; b++) {
        u64x2 k1{a[4 * b], a[4 * b + 1]}, k2{a[4 * b + 2], a[4 * b + 3]};
        k1 = mul_const(k1, c1); k1 = rotl<31>(k1); k1 = mul_const(k1, c2); h1 = xor64(h1, k1);
        h1 = rotl<27>(h1); h1 = add64(h1, h2); h1 = mul5_add(h1, 0x52dce729u);
        k2 = mul_const(k2, c2); k2 = rotl<33>(k2); k2 = mul_const(k2, c1); h2 = xor64(h2, k2);
        h2 = rotl<31>(h2); h2 = add64(h2, h1); h2 = mul5_add(h2, 0x38495ab5u);
    }
    if constexpr (TAIL > 8) {
        u64x2 k2{a[4 * NB + 2], a[4 * NB + 3]};
        k2 = mul_const(k2, c2); k2 = rotl<33>(k2); k2 = mul_const(k2, c1); h2 = xor64(h2, k2);
    }
    static_assert(!K1_GIVEN || (TAIL > 0 && TAIL <= 8), "a given k1 replaces the whole tail");
    if constexpr (K1_GIVEN) {
        h1 = xor64(h1, k1_tail);
    } else if constexpr (TAIL > 0) {
        u64x2 k1{a[4 * NB], a[4 * NB + 1]};
        k1 = mul_const(k1, c1); k1 = rotl<31>(k1); k1 = mul_const(k1, c2); h1 = xor64(h1, k1);
    }
    h1.lo ^= (uint32_t)K; h2.lo ^= (uint32_t)K;
    h1 = add64(h1, h2); h2 = add64(h2, h1);
    h1_out = h1; h2_out = h2;
}

// a[i] = ASCII bytes 4i..4i+3 of the k-mer (little endian, byte 0 = first base), bytes >= K zeroed.
// NA = 2*ceil(K/8) words.  Returns h1 (the first 8 bytes of the 128-bit digest).
template <int K, int NA>
__device__ __forceinline__ u64x2 murmur3_h1(const uint32_t (&a)[NA], uint32_t seed)
{
    u64x2 h1, h2;
    murmur3_body<K, NA>(a, seed, h1, h2);
    h1 = fmix(h1); h2 = fmix(h2);
    h1 = add64(h1, h2);
    return h1;
}

// Filter word of h1 for the scan's fast path: X = hi(fmix(h1)) + hi(fmix(h2)) + 1 (mod 2^32), the high word of h1 with
// the carry out of the low words (never computed) replaced by 1.  With H the exact high word of h1 and T < 2^32 - 1,
//   H <= T  implies  X <= T + 1
// (carry 0: X = H + 1 <= T + 1;  carry 1: X = H), so `X <= T + 1` (or anything, when T = 2^32 - 1) never rejects a hash
// whose high word is <= T.  It lets through at most the one extra high word T + 1 and X = 0 (high words summing to
// 2^32 - 1); the slow path recomputes the exact hash.  tests/test_scan_filter_model.py models this predicate.
template <int K, int NA, bool K1_GIVEN = false>
__device__ __forceinline__ uint32_t murmur3_h1_filter(const uint32_t (&a)[NA], uint32_t seed, u64x2 k1_tail = u64x2{0u, 0u})
{
    u64x2 h1, h2;
    murmur3_body<K, NA, K1_GIVEN>(a, seed, h1, h2, k1_tail);
    uint32_t one;    // opaque, so that ptxas keeps the +1 as the IMAD.HI addend rather than a separate add on the ALU pipe
    asm("mov.u32 %0, 1;" : "=r"(one));
    return fmix_hi(h2, fmix_hi(h1, one));
}

// threshold for murmur3_h1_filter's word, from the exact high-word threshold T = tmax >> 32: T + 1, saturated at 2^32 - 1
__host__ __device__ __forceinline__ uint32_t filter_threshold(uint32_t t_hi)
{
    return t_hi + (t_hi != 0xFFFFFFFFu ? 1u : 0u);
}

}  // namespace mashgpu
