// dist_filter.cuh -- partial-key cuckoo filter over the 32-bit dictionary ranks of one reference tile.
//
// Used by dist_probe_kernel (dist.cu): before any (query, reference) pair of a 32-reference tile is merged, the query's
// ranks are looked up in a filter that holds every rank of the tile.  A query none of whose ranks is in the filter shares
// no hash with any of the 32 references, so the reference's merge loop (CommandDistance.cpp:347-365) would end with
// common == 0 for all 32 pairs and only the closed form is written.  The filter has no false negatives; a positive is
// confirmed by an exact binary search before the tile is handed to the merge kernel.
//
// Layout: 2^15 buckets of two 16-bit fingerprints (one 32-bit word per bucket, 128 KB of shared memory), 0 = free slot.
// h = rank * odd constant is a bijection of the 32-bit rank: bucket = low 15 bits (a bijection of the rank's low 15 bits,
// which are uniform for dictionary ranks), fingerprint = 14 of the bits 15..29 of h; the alternate bucket is
// bucket ^ f(fingerprint) (partial-key cuckoo hashing), so a lookup is exactly two shared-memory loads and no loop.
// The bit assignment is chosen for the lookup's instruction count (the probe kernel is bound by the ALU pipe): the byte
// offset of the bucket is (h << 2) & mask and the alternate one an xor-and of a product, one ALU instruction each; and a
// fingerprint always has bit 14 clear and bit 0 set, which makes it, read as an IEEE half, a finite non-zero number --
// so "is fp in this bucket" is ONE half2 compare (HSETP2, two predicates) instead of the xor / subtract / and-not
// zero-halfword test, and the free slot 0x0000 (+0.0) never compares equal.
// 32 references x 1000 ranks fill 49 % of the slots (two-slot buckets work up to ~84 %).
//
// The functions compile for the host too (tests/test_dist_filter.py drives them through tools/cf_host_test.cpp) --
// there the "atomic" is a plain compare-and-swap.
#pragma once
#include <cstdint>

#if defined(__CUDACC__)
#define MG_HD __host__ __device__ __forceinline__
#else
#define MG_HD inline
#endif

namespace mashgpu {

constexpr uint32_t CF_LOG2_BUCKETS = 15;
constexpr uint32_t CF_BUCKETS = 1u << CF_LOG2_BUCKETS;
constexpr uint32_t CF_MAX_KICKS = 256;

MG_HD uint32_t cf_hash(uint32_t code) { return code * 0x9E3779B1u; }
MG_HD uint32_t cf_fp(uint32_t h) { return ((h >> 14) & 0xBFFEu) + 1u; }       // bits 15..27 and 29 of h, bit 0 set, bit 14 clear
MG_HD uint32_t cf_bucket(uint32_t h) { return h & (CF_BUCKETS - 1u); }
MG_HD uint32_t cf_alt(uint32_t bucket, uint32_t fp) { return bucket ^ ((fp * 0x5BD1E995u) & (CF_BUCKETS - 1u)); }

// does one of the two 16-bit halves of w equal fp (fp != 0)
MG_HD bool cf_word_has(uint32_t w, uint32_t fp)
{
    const uint32_t x = w ^ (fp * 0x00010001u);
    return ((x - 0x00010001u) & ~x & 0x80008000u) != 0;
}

MG_HD uint32_t cf_cas(uint32_t *addr, uint32_t expect, uint32_t value)
{
#if defined(__CUDA_ARCH__)
    return atomicCAS(addr, expect, value);
#else
    const uint32_t old = *addr;
    if (old == expect) *addr = value;
    return old;
#endif
}

MG_HD uint32_t cf_read(const uint32_t *addr)
{
#if defined(__CUDA_ARCH__)
    return *reinterpret_cast<const volatile uint32_t *>(addr);
#else
    return *addr;
#endif
}

// true when fp is (now) in bucket b; false when the bucket is full of other fingerprints
MG_HD bool cf_try_place(uint32_t *tab, uint32_t b, uint32_t fp)
{
    uint32_t w = cf_read(tab + b);
    for (;;) {
        if (cf_word_has(w, fp)) return true;
        uint32_t nw;
        if ((w & 0xFFFFu) == 0) nw = w | fp;
        else if ((w >> 16) == 0) nw = w | (fp << 16);
        else return false;
        const uint32_t old = cf_cas(tab + b, w, nw);
        if (old == w) return true;
        w = old;
    }
}

// Concurrent insert (shared-memory atomics on the device).  Returns false when the random walk gives up; the caller
// then treats the whole tile as "may share" (correct, only slower).
MG_HD bool cf_insert(uint32_t *tab, uint32_t code, uint32_t salt)
{
    const uint32_t h = cf_hash(code);
    uint32_t fp = cf_fp(h);
    const uint32_t b1 = cf_bucket(h), b2 = cf_alt(b1, fp);
    if (cf_try_place(tab, b1, fp)) return true;
    if (cf_try_place(tab, b2, fp)) return true;
    uint32_t rnd = salt * 747796405u + 2891336453u;
    uint32_t b = (rnd >> 31) ? b1 : b2;
    for (uint32_t kick = 0; kick < CF_MAX_KICKS; kick++) {
        rnd = rnd * 1664525u + 1013904223u;
        const uint32_t sh = (rnd >> 31) * 16u;
        uint32_t w = cf_read(tab + b), victim;
        for (;;) {
            if (cf_word_has(w, fp)) return true;           // the same fingerprint arrived by another route
            victim = (w >> sh) & 0xFFFFu;
            const uint32_t nw = (w & ~(0xFFFFu << sh)) | (fp << sh);
            const uint32_t old = cf_cas(tab + b, w, nw);
            if (old == w) break;
            w = old;
        }
        if (victim == 0) return true;                       // the slot had been freed: nothing to move on
        fp = victim;
        b = cf_alt(b, fp);
        if (cf_try_place(tab, b, fp)) return true;
    }
    return false;
}

MG_HD bool cf_lookup(const uint32_t *tab, uint32_t code)
{
    const uint32_t h = cf_hash(code);
    const uint32_t fp = cf_fp(h);
    const uint32_t w1 = tab[cf_bucket(h)], w2 = tab[cf_alt(cf_bucket(h), fp)];
    return cf_word_has(w1, fp) || cf_word_has(w2, fp);
}

// ---- which reference does a fingerprint belong to?  One byte per slot (2 slots per bucket), filled after the filter is built:
// the reference index 0..31 when every rank that owns this slot's fingerprint comes from one reference of the tile, CF_ID_MULTI
// when several do.  A filter hit then names the one reference the query may share the rank with -- no search -- and only
// CF_ID_MULTI hits need the exact confirmation.  (A rank's fingerprint may sit in either of its two buckets, and another rank
// with the same fingerprint and bucket pair shares the entry: every slot that shows the fingerprint is marked.)
// The byte also carries 3 more bits of the rank (a second hash, values 0..6) above the 5-bit reference index: a query rank that
// merely collides with the slot's 16-bit fingerprint is rejected 6 times out of 7 before it costs a spurious pair merge.
constexpr uint32_t CF_ID_NONE = 0xFFu, CF_ID_MULTI = 0xFEu;

MG_HD uint32_t cf_tag(uint32_t code)
{
    const uint32_t v = (code * 0x85EBCA6Bu) >> 29;
    return v > 6u ? 6u : v;
}

MG_HD void cf_mark_slot(uint8_t *ids, uint32_t slot, uint32_t value)
{
    const uint32_t old = ids[slot];
    ids[slot] = (uint8_t)((old == CF_ID_NONE || old == value) ? value : CF_ID_MULTI);
}

// marks the slots holding the fingerprint of `code` with reference r.  Calls for different r must not run concurrently
// (the probe kernel processes one reference per phase); concurrent calls for the same r are fine.
MG_HD void cf_mark_ids(const uint32_t *tab, uint8_t *ids, uint32_t code, uint32_t r)
{
    const uint32_t h = cf_hash(code);
    const uint32_t fp = cf_fp(h);
    const uint32_t b1 = cf_bucket(h), b2 = cf_alt(b1, fp);
    const uint32_t w1 = tab[b1], w2 = tab[b2];
    const uint32_t value = (cf_tag(code) << 5) | r;
    if ((w1 & 0xFFFFu) == fp) cf_mark_slot(ids, 2 * b1, value);
    if ((w1 >> 16) == fp) cf_mark_slot(ids, 2 * b1 + 1, value);
    if ((w2 & 0xFFFFu) == fp) cf_mark_slot(ids, 2 * b2, value);
    if ((w2 >> 16) == fp) cf_mark_slot(ids, 2 * b2 + 1, value);
}

// references that may hold `code`: bit r for every slot that shows its fingerprint and names reference r; *multi is set when
// a matching slot is shared by several references.  0 / false: the code is not in the filter.
MG_HD uint32_t cf_owner_bits(const uint32_t *tab, const uint8_t *ids, uint32_t code, bool *multi)
{
    const uint32_t h = cf_hash(code);
    const uint32_t fp = cf_fp(h);
    const uint32_t b1 = cf_bucket(h), b2 = cf_alt(b1, fp);
    const uint32_t w1 = tab[b1], w2 = tab[b2];
    uint32_t bits = 0;
    bool m = false;
    const uint32_t slot[4] = {2 * b1, 2 * b1 + 1, 2 * b2, 2 * b2 + 1};
    const bool hit[4] = {(w1 & 0xFFFFu) == fp, (w1 >> 16) == fp, (w2 & 0xFFFFu) == fp, (w2 >> 16) == fp};
    const uint32_t tag = cf_tag(code);
    for (int i = 0; i < 4; i++)
        if (hit[i]) {
            const uint32_t id = ids[slot[i]];
            if (id >= CF_ID_MULTI) m = true;              // shared slot (CF_ID_NONE: ids not built -- the caller confirms every hit)
            else if ((id >> 5) == tag) bits |= 1u << (id & 31u);
        }
    *multi = m;
    return bits;
}

// The probe kernel's form of the lookup: everything derives from ONE product h4 = rank * (C << 2) = h << 2:
//   byte offset of bucket 1 = h4 & mask;  x = (h4 >> 16) & 0xBFFE = fp - 1;  offset 2 = offset 1 ^ ((x * K + K) & mask)
//   with K = (alt multiplier << 2);  f2 = x * 0x10001 + 0x10001 = fp in both halves.
// Returns the two bucket words and f2; the comparison is done for a whole group by cf_group_any.
struct CfProbe { uint32_t w1, w2, f2; };
MG_HD void cf_offsets(uint32_t code, uint32_t &o1, uint32_t &o2, uint32_t &f2)
{
    constexpr uint32_t OFF_MASK = 4u * CF_BUCKETS - 4u;
    const uint32_t h4 = code * (0x9E3779B1u << 2);
    o1 = h4 & OFF_MASK;
    const uint32_t x = (h4 >> 16) & 0xBFFEu;
    o2 = o1 ^ ((x * (0x5BD1E995u << 2) + (0x5BD1E995u << 2)) & OFF_MASK);
    f2 = x * 0x00010001u + 0x00010001u;
}
MG_HD CfProbe cf_fetch(const uint32_t *tab, uint32_t code)
{
    uint32_t o1, o2;
    CfProbe r;
    cf_offsets(code, o1, o2, r.f2);
    r.w1 = *reinterpret_cast<const uint32_t *>(reinterpret_cast<const char *>(tab) + o1);
    r.w2 = *reinterpret_cast<const uint32_t *>(reinterpret_cast<const char *>(tab) + o2);
    return r;
}

#if defined(__CUDACC__)

// Device form of the probe: `tab_s` is the 32-bit shared-memory address of the table.  Both buckets are loaded by every lane,
// because loading the second only where the first is full costs more ALU-pipe predicate logic than the shared-memory
// wavefronts it saves.
__device__ __forceinline__ CfProbe cf_fetch_s(uint32_t tab_s, uint32_t code)
{
    uint32_t o1, o2;
    CfProbe r;
    cf_offsets(code, o1, o2, r.f2);
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r.w1) : "r"(tab_s + o1));
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(r.w2) : "r"(tab_s + o2));
    return r;
}

// Does any lane of the warp have a fingerprint match in any of its four probes?  8 half2 compares (a fingerprint is a
// finite non-zero half, the free slot is +0.0), predicate ors and one vote.  An f2 of 0x7E007E00 (NaN) never matches.
__device__ __forceinline__ bool cf_group_any(const CfProbe &a, const CfProbe &b, const CfProbe &c, const CfProbe &d)
{
    uint32_t any;
    asm volatile("{\n\t.reg .pred p0, p1, p2, p3, p4, p5, p6, p7, q;\n\t"
                 "setp.eq.f16x2 p0|p1, %1, %3;\n\t"
                 "setp.eq.f16x2 p2|p3, %2, %3;\n\t"
                 "setp.eq.f16x2 p4|p5, %4, %6;\n\t"
                 "setp.eq.f16x2 p6|p7, %5, %6;\n\t"
                 "or.pred p0, p0, p1;\n\tor.pred p2, p2, p3;\n\tor.pred p4, p4, p5;\n\tor.pred p6, p6, p7;\n\t"
                 "or.pred p0, p0, p2;\n\tor.pred p4, p4, p6;\n\tor.pred q, p0, p4;\n\t"
                 "setp.eq.f16x2 p0|p1, %7, %9;\n\t"
                 "setp.eq.f16x2 p2|p3, %8, %9;\n\t"
                 "setp.eq.f16x2 p4|p5, %10, %12;\n\t"
                 "setp.eq.f16x2 p6|p7, %11, %12;\n\t"
                 "or.pred p0, p0, p1;\n\tor.pred p2, p2, p3;\n\tor.pred p4, p4, p5;\n\tor.pred p6, p6, p7;\n\t"
                 "or.pred p0, p0, p2;\n\tor.pred p4, p4, p6;\n\tor.pred p0, p0, p4;\n\tor.pred q, q, p0;\n\t"
                 "vote.sync.any.pred q, q, 0xffffffff;\n\t"
                 "selp.u32 %0, 1, 0, q;\n\t}"
                 : "=r"(any)
                 : "r"(a.w1), "r"(a.w2), "r"(a.f2), "r"(b.w1), "r"(b.w2), "r"(b.f2),
                   "r"(c.w1), "r"(c.w2), "r"(c.f2), "r"(d.w1), "r"(d.w2), "r"(d.f2));
    return any != 0;
}
#endif

}  // namespace mashgpu
