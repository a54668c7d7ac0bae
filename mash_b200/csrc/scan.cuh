// scan.cuh -- the k-mer scan + hash + filter kernel (K1 of DESIGN.md), shared by sketch and screen.
//
// Replaces the per-base loop of addMinHashes (reference Sketch.cpp:512-583) and hashSequence
// (CommandScreen.cpp:484-599):  upper-case -> alphabet check -> canonical k-mer -> getHash -> tryInsert.
//
// Layout.  The input is one flat byte stream in HBM (units back to back, records separated by a byte
// outside the alphabet).  A CTA processes TILE window-start positions at a time: the tile's ASCII bytes
// are read once with 128-bit loads, converted to 4-bit codes (A,C,G,T -> 0,1,2,3, anything else -> 8)
// and staged in shared memory as nibble words (8 bases per 32-bit word).  A thread takes a block of 8
// consecutive window starts: it loads the BW words that cover them, builds the reverse-complement block
// in registers (nibble reversal + xor 3), and for each of the 8 windows extracts the forward and the
// reverse-complement k-mer with funnel shifts, picks the canonical one by an integer compare of the
// little-endian nibble words (equivalent to the reference's memcmp because complementing reverses the
// base order, see DESIGN.md), expands it to ASCII with one PRMT per 4 bases and runs MurmurHash3_x64_128.
// Only hashes at or below the tile's coarse threshold leave the fast path.
#pragma once
#include <cstdint>
#include <utility>
#include "murmur3.cuh"

namespace mashgpu {

constexpr int SCAN_THREADS = 256;
constexpr int SCAN_TILE = 8192;              // window starts per tile
constexpr int SCAN_HALO_WORDS = 8;           // extra nibble words (64 bases) staged past the tile
constexpr int SCAN_WORDS = SCAN_TILE / 8 + SCAN_HALO_WORDS;
constexpr int SCAN_WARPS = SCAN_THREADS / 32;
constexpr int SCAN_WARP_TILE = 1024;         // window starts per warp tile (32 lanes x 4 blocks x 8)
constexpr int SCAN_WARP_WORDS = SCAN_WARP_TILE / 8 + SCAN_HALO_WORDS;   // 136 nibble words
constexpr int SCAN_WARP_VECS = SCAN_WARP_WORDS / 2;                     // 68 16-byte vectors
constexpr uint64_t EMPTY_KEY = 0xFFFFFFFFFFFFFFFFULL;

enum ScanMode : int { SCAN_SKETCH = 0, SCAN_SCREEN = 1, SCAN_DUMP = 2, SCAN_COUNT = 3, SCAN_EVENTS = 4 };

struct ScanArgs {
    const uint8_t *stream;        // flat byte stream (ASCII source; NULL when the packed source is used)
    const uint64_t *codes;        // packed source: 2-bit codes, 32 positions per word (A0 C1 G2 T3), see pack.cpp
    const uint32_t *inval;        // packed source: 1 bit per position, set = not in the alphabet / separator / past the end
    uint64_t stream_len;          // positions >= stream_len are treated as separators
    uint64_t tile_begin, tile_end;
    const uint64_t *tile_tmax;    // per-tile coarse threshold (indexed by absolute tile id); NULL -> coarse_t
    const uint32_t *tile_unit;    // per-tile first unit: last u with unit_start[u] <= the tile's first position (absolute
                                  //   tile id); NULL -> the slow path binary-searches unit_start
    uint64_t coarse_t;
    uint32_t seed;
    int use64;
    int preserve_case;
    int mode;
    // candidate tables (sketch units / the screen mixture): open addressing, keys EMPTY_KEY when free
    const uint64_t *unit_start;   // n_units + 1 stream offsets
    uint32_t n_units;
    const uint64_t *unit_t;       // per-unit threshold: keep hash <= unit_t[u]
    const uint64_t *tab_off;      // per-unit slot offset into tab_keys / tab_cnt
    const uint32_t *tab_log2;     // per-unit log2(capacity)
    uint64_t *tab_keys;
    uint32_t *tab_cnt;
    uint64_t *tab_first;          // optional (multiplicity counts): stream position of the first / last occurrence per slot,
    uint64_t *tab_last;           //   needed to reproduce MinHashHeap's top-of-heap counting quirk (sketch.cu, quirk_kernel)
    uint32_t *unit_flags;         // bit0: table overflow
    uint32_t *unit_maxhash;       // occurrences of the hash value 2^64-1 (cannot be a table key)
    int64_t only_unit;            // >= 0: ignore every other unit (exact re-run)
    uint32_t min_copies;          // `-m` (>= 1): tab_first holds min_copies positions per slot, the smallest stream positions of the key
    // screen: reference hash table (distinct keys, EMPTY_KEY when free) with u32 hit counters
    const uint64_t *ref_keys;
    const uint32_t *ref_idx;      // slot -> index of the key in the sorted distinct key list (deterministic across ranks)
    uint32_t *ref_cnt;            // hit counters, indexed by that key index
    uint32_t ref_log2;
    uint64_t ref_hmax;            // largest reference hash (probe prefilter)
    const uint32_t *ref_bitmap;   // optional second prefilter: bit (hash >> ref_bitmap_shift) is set iff some reference hash has these
    uint32_t ref_bitmap_shift;    //   top bits (indexed by value, not hashed: reference hashes crowd the low end of the range)
    uint64_t screen_mix_t;        // screen: largest unit threshold -- only hashes at or below it can enter the mixture's bottom-s
    // dump
    uint64_t *out_hash;
    uint8_t *out_valid;
    // byte-alphabet kernels (any alphabet, non-canonical): byte -> itself (upper-cased unless preserve_case) if it is in
    // the alphabet, else 0
    uint8_t byte_lut[256];
    // SCAN_COUNT: occurrences of one hash at stream positions [count_lo, count_hi]
    uint64_t count_target, count_lo, count_hi;
    uint32_t *count_out;
    // SCAN_EVENTS (`-c`): every k-mer whose hash is at or below the threshold of its position band (the "units" of this pass)
    // is appended as an event {position, hash}; sketch.cu replays the events in stream order through the heap
    uint64_t *ev_pos, *ev_hash;
    unsigned long long *ev_count;
    uint64_t ev_capacity;
};

__device__ __forceinline__ uint32_t slot_hash(uint64_t key, uint32_t log2cap)
{
    return (uint32_t)((key * 0x9E3779B97F4A7C15ULL) >> (64 - log2cap));
}

// Insert-or-count into an open-addressing table. Returns the slot, or -1 when the table is full.
__device__ __forceinline__ int64_t table_add(uint64_t *keys, uint32_t *cnt, uint32_t log2cap, uint64_t key)
{
    const uint32_t mask = (1u << log2cap) - 1;
    uint32_t slot = slot_hash(key, log2cap);
    for (uint32_t probes = 0; probes <= mask; probes++) {
        unsigned long long prev = atomicCAS((unsigned long long *)&keys[slot], (unsigned long long)EMPTY_KEY, (unsigned long long)key);
        if (prev == EMPTY_KEY || prev == key) {
            atomicAdd(&cnt[slot], 1u);
            return slot;
        }
        slot = (slot + 1) & mask;
    }
    return -1;
}

// Slow path: a hash passed the tile's coarse threshold.
static __device__ __noinline__ void scan_emit(const ScanArgs &a, uint32_t hash_lo, uint32_t hash_hi, uint64_t tile_base, uint32_t local_pos)
{
    const uint64_t hash = ((uint64_t)hash_hi << 32) | hash_lo;
    const uint64_t pos = tile_base + local_pos;
    if (a.mode == SCAN_DUMP) {
        a.out_hash[pos] = hash;
        a.out_valid[pos] = 1;
        return;
    }
    if (a.mode == SCAN_COUNT) {
        if (hash == a.count_target && pos >= a.count_lo && pos <= a.count_hi) atomicAdd(a.count_out, 1u);
        return;
    }
    // (screen: the reference table was probed by screen_probe_lanes before the survivors were serialised)
    // unit of this position: last u with unit_start[u] <= pos -- from the tile's first unit a tile rarely spans more than one
    // or two units, so a forward scan of a load or two replaces a binary search of ~log2(n_units) dependent loads
    uint32_t u;
    if (a.tile_unit) {
        u = a.tile_unit[pos / SCAN_TILE];
        while (u + 1 < a.n_units && a.unit_start[u + 1] <= pos) u++;
    } else {
        uint32_t lo = 0, hi = a.n_units;
        while (hi - lo > 1) {
            uint32_t mid = (lo + hi) >> 1;
            if (a.unit_start[mid] <= pos) lo = mid; else hi = mid;
        }
        u = lo;
    }
    if (a.only_unit >= 0 && (int64_t)u != a.only_unit) return;
    if (hash > a.unit_t[u]) return;
    if (a.mode == SCAN_EVENTS) {
        const unsigned long long at = atomicAdd(a.ev_count, 1ull);
        if (at < a.ev_capacity) { a.ev_pos[at] = pos; a.ev_hash[at] = hash; }
        return;
    }
    if (hash == EMPTY_KEY) { atomicAdd(&a.unit_maxhash[u], 1u); return; }
    const int64_t slot = table_add(a.tab_keys + a.tab_off[u], a.tab_cnt + a.tab_off[u], a.tab_log2[u], hash);
    if (slot < 0) { atomicOr(&a.unit_flags[u], 1u); return; }
    if (a.tab_first) {
        // the m smallest positions of the key, ascending: a cascade of atomic minima -- level i ends up with the (i+1)-th smallest
        // position whatever the arrival order, because every value that reaches a level is either its final minimum or is passed
        // on exactly once.  Level m-1 is the position at which MinHashHeap promotes the hash (MinHashHeap.cpp:96-100); m = 1: the
        // first occurrence.
        unsigned long long *f = (unsigned long long *)a.tab_first + (a.tab_off[u] + (uint64_t)slot) * a.min_copies;
        unsigned long long x = pos;
        for (uint32_t i = 0; i < a.min_copies; i++) {
            const unsigned long long old = atomicMin(&f[i], x);
            if (old == EMPTY_KEY) break;            // the level was empty: nothing to pass on
            if (old > x) x = old;
        }
        atomicMax((unsigned long long *)&a.tab_last[a.tab_off[u] + slot], (unsigned long long)pos);
    }
}

// Warp-uniform wrapper around the slow path.  The hot loop never branches on a per-lane condition: a window's pass
// flag is voted, and when any lane has a survivor the whole warp enters here and serialises the survivors with
// ballot/shuffle (lane 0 does the table work).  Keeping the main loop free of divergent branches matters: with a
// per-lane `if (pass) emit()` the warp kept running split into sub-warps between emits (ncu: 19 active lanes on
// average, 1.6x the warp instructions).
// The fast path does not even test window validity (2 instructions per k-mer saved): hashes of windows that contain
// a non-alphabet byte are garbage, and the few that slip under the threshold are rejected here by re-reading the
// window's nibbles from the warp's shared-memory tile.  The fast-path filter only compares the high word (k > 16)
// or the low word (k <= 16) of the hash with the tile threshold; the exact 64-bit test is in scan_emit.
// window validity from the warp's tile: DNA kernels keep nibbles (bit 3 = outside the alphabet), byte kernels bytes (0 = outside)
__device__ __forceinline__ bool window_valid(const uint32_t *sm_tile, uint32_t lp, int k)
{
    if (k > 0) {   // bit 3 of the window's k nibbles, a word (8 nibbles) at a time
        const uint32_t w = lp >> 3, sh = 4 * (lp & 7);
        uint32_t bad = 0;
        for (int i = 0; 8 * i < k; i++) {
            uint32_t x = __funnelshift_r(sm_tile[w + i], sm_tile[w + i + 1], sh);
            if (k - 8 * i < 8) x &= (1u << (4 * (k - 8 * i))) - 1u;
            bad |= x;
        }
        return !(bad & 0x88888888u);
    }
    const uint8_t *bytes = reinterpret_cast<const uint8_t *>(sm_tile);
    bool ok = true;
    for (int i = 0; i < -k; i++) ok &= bytes[lp + i] != 0;
    return ok;
}

// Screen: hashCounts[key]++ iff key is a reference hash (CommandScreen.cpp:571-575).  Every lane probes for its own window --
// with a reference set that spans the whole hash range (small genomes, plasmids, viruses in the .msh: their bottom-s reaches
// up to 2^64 s / L) EVERY k-mer of the mixture is a candidate, so this cannot go through the serialised survivor path.
// Order: largest reference hash -> value-indexed bitmap (L2 resident, rejects the sparse upper range without touching the
// table) -> open-addressing table in HBM -> on a hit only, the window's validity (the fast path hashes invalid windows too).
static __device__ __noinline__ void screen_probe_lanes(const ScanArgs &a, bool pass, uint32_t hash_lo, uint32_t hash_hi,
                                                       uint32_t local_pos, const uint32_t *sm_tile, int k)
{
    const uint64_t hash = ((uint64_t)hash_hi << 32) | hash_lo;
    bool go = pass && hash <= a.ref_hmax;
    if (go && a.ref_bitmap) {
        const uint64_t b = hash >> a.ref_bitmap_shift;
        go = (__ldg(a.ref_bitmap + (b >> 5)) >> (b & 31)) & 1u;
    }
    if (!go) return;
    const uint32_t mask = (1u << a.ref_log2) - 1;
    uint32_t slot = slot_hash(hash, a.ref_log2);
    for (;;) {
        const uint64_t key = __ldg(a.ref_keys + slot);
        if (key == hash) {
            if (window_valid(sm_tile, local_pos, k)) atomicAdd(&a.ref_cnt[a.ref_idx[slot]], 1u);
            return;
        }
        if (key == EMPTY_KEY) return;
        slot = (slot + 1) & mask;
    }
}

static __device__ __noinline__ void scan_emit_warp(const ScanArgs &a, bool pass, uint32_t hash_lo, uint32_t hash_hi,
                                                   uint64_t tile_base, uint32_t local_pos, const uint32_t *sm_tile, int k,
                                                   uint64_t tmax)
{
    if (a.mode == SCAN_SCREEN) {
        screen_probe_lanes(a, pass, hash_lo, hash_hi, local_pos, sm_tile, k);
        __syncwarp();
        pass = pass && ((((uint64_t)hash_hi) << 32) | hash_lo) <= a.screen_mix_t;      // the rest is about the mixture's bottom-s only
    }
    unsigned m = __ballot_sync(0xFFFFFFFFu, pass);
    const int lane = threadIdx.x & 31;
    while (m) {
        const int src = __ffs(m) - 1;
        m &= m - 1;
        const uint32_t lo = __shfl_sync(0xFFFFFFFFu, hash_lo, src);
        const uint32_t hi = __shfl_sync(0xFFFFFFFFu, hash_hi, src);
        const uint32_t lp = __shfl_sync(0xFFFFFFFFu, local_pos, src);
        if (lane == 0) {
            if (window_valid(sm_tile, lp, k) && ((((uint64_t)hi) << 32) | lo) <= tmax) scan_emit(a, lo, hi, tile_base, lp);
        }
        __syncwarp();
    }
}

// 4 ASCII bytes -> 4 nibbles (in the low 16 bits).  Codes: A=0 C=1 G=2 T=3 (order preserving, complement = xor 3),
// anything else 8.  `fold` = 0xDFDFDFDF to upper-case first (a..z -> A..Z is the only effect that matters), or ~0.
__device__ __forceinline__ uint32_t ascii4_to_nibbles(uint32_t w, uint32_t fold)
{
    const uint32_t u = w & fold;
    const uint32_t t = (u >> 2) & ~(u >> 1) & 0x01010101u;                    // bit2 & ~bit1: 'T'
    const uint32_t expect = (0x41414141u | (u & 0x06060606u)) ^ (t * 0x11u);  // the ACGT byte with these bits 1,2
    const uint32_t bad = u ^ expect;
    const uint32_t nz = (((bad & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | bad) & 0x80808080u;  // bit7 set where byte != 0
    const uint32_t c = (u >> 1) & 0x03030303u;                                // A0 C1 T2 G3
    const uint32_t code = c ^ ((c >> 1) & 0x01010101u);                       // A0 C1 G2 T3
    uint32_t x = code | (nz >> 4);
    x = (x | (x >> 4)) & 0x00FF00FFu;
    x = (x | (x >> 8)) & 0x0000FFFFu;
    return x;
}

// PRMT in its native 4-bit-selector form (bit 3 of a selector nibble = sign replicate; never set for valid codes)
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel)
{
    uint32_t d;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(sel));
    return d;
}

__device__ __forceinline__ uint32_t nibble_reverse(uint32_t x)
{
    x = __byte_perm(x, 0, 0x0123);
    return ((x & 0x0F0F0F0Fu) << 4) | ((x >> 4) & 0x0F0F0F0Fu);
}

// word i of (block >> 4*OFF nibbles), block = BW little-endian words
template <int OFF, int BW>
__device__ __forceinline__ uint32_t block_word(const uint32_t (&b)[BW], int i)
{
    constexpr int WS = OFF / 8, SH = 4 * (OFF % 8);
    const int lo_i = i + WS, hi_i = i + WS + 1;
    const uint32_t lo = lo_i < BW ? b[lo_i < BW ? lo_i : 0] : 0u;
    if (SH == 0) return lo;
    const uint32_t hi = hi_i < BW ? b[hi_i < BW ? hi_i : 0] : 0u;
    return __funnelshift_r(lo, hi, SH);
}

template <int K>
struct KmerShape {
    static constexpr int NW = (K + 7) / 8;           // nibble words per k-mer
    static constexpr int BW = (K + 7 + 7) / 8;       // nibble words per block of 8 window starts
    static constexpr int NA = 2 * NW;                // ASCII words per k-mer
    static constexpr uint32_t LAST_MASK = (K % 8) ? ((1u << (4 * (K % 8))) - 1u) : 0xFFFFFFFFu;
    // the nibbles of the last word past the k-mer hold 0xF: as a PRMT selector that is the sign-replicate of byte 7 of
    // {0, pool}, a 0x00 byte, which is what MurmurHash3 reads past the key.  The pad is the complement of the mask, so
    // masking and padding are one OR.  Both strands carry the same padding in their most significant nibbles, so the
    // canonical compare is decided by the k-mer's own nibbles.
    static constexpr uint32_t LAST_PAD = ~LAST_MASK;
    // 17 <= K <= 21 (a tail block of 1..5 bases): the filter-word kernels take the tail's k1 from a table (TailTable)
    static constexpr bool TAIL_TABLE = K >= 17 && K <= 21;
};

// Tail block by table.  For 17 <= K <= 21 the tail block of MurmurHash3 is bases 16..K-1 of the canonical k-mer, and its k1
// (murmur3_tail_k1 of their ASCII bytes) takes at most 4^5 values and does not depend on the seed.  The filter-word kernels
// keep the 1024 values in shared memory and replace the tail's two PRMT, two multiplies and rotate by one IMAD, one shift
// and one 8-byte LDS.  The index is computed from the canonical k-mer's last nibble word with bit 3 and bit 2 of every
// nibble cleared (codes c0..c4 at bits 0, 4, 8, 12, 16): w * (2^10 + 1) puts c0, c3, c1, c4, c2 side by side at bits
// 10..19 without overlap and without a carry, and the shift keeps those ten bits.  Windows with a base outside the
// alphabet read some entry and are rejected by the exact rebuild, as before.
constexpr uint32_t TAIL_IDX_MUL = 0x401000u;   // (2^10 + 1) << 12
constexpr int TAIL_IDX_SHIFT = 22;
constexpr int TAIL_TAB_SIZE = 1024;
__host__ __device__ __forceinline__ uint32_t tail_index(uint32_t w) { return (w * TAIL_IDX_MUL) >> TAIL_IDX_SHIFT; }

// nibble words (codes 0..3, padded with 0xF past K) -> ASCII words, bytes >= K zeroed
template <int K>
__device__ __forceinline__ void expand_ascii(const uint32_t (&c)[KmerShape<K>::NW], uint32_t (&a)[KmerShape<K>::NA], uint32_t POOL)
{
#pragma unroll
    for (int i = 0; i < KmerShape<K>::NW; i++) {
        a[2 * i] = prmt(POOL, 0, c[i]);
        a[2 * i + 1] = K - 8 * i - 4 <= 0 ? 0u : prmt(POOL, 0, c[i] >> 16);   // no base left for word 2i+1: zero
    }
}

// canonical k-mer of a window: c = rc when rc < fwd as little-endian multi-word integers  <=>  memcmp(fwd, rc, k) > 0
// (Sketch.cpp:569-571): borrow out of rc - fwd.  m = all-ones when the reverse complement is the canonical k-mer.
template <int K>
__device__ __forceinline__ void canonical_words(const uint32_t (&f)[KmerShape<K>::NW], const uint32_t (&r)[KmerShape<K>::NW],
                                                uint32_t (&c)[KmerShape<K>::NW])
{
    using S = KmerShape<K>;
    uint32_t m;
    if (S::NW == 1) {
        asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\tsubc.u32 %0, 0, 0;\n\t}" : "=r"(m) : "r"(r[0]), "r"(f[0]));
    } else if (S::NW == 2) {
        asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\tsubc.cc.u32 t, %3, %4;\n\tsubc.u32 %0, 0, 0;\n\t}"
            : "=r"(m) : "r"(r[0]), "r"(f[0]), "r"(r[S::NW > 1 ? 1 : 0]), "r"(f[S::NW > 1 ? 1 : 0]));
    } else if (S::NW == 3) {
        asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\tsubc.cc.u32 t, %3, %4;\n\tsubc.cc.u32 t, %5, %6;\n\tsubc.u32 %0, 0, 0;\n\t}"
            : "=r"(m) : "r"(r[0]), "r"(f[0]), "r"(r[S::NW > 1 ? 1 : 0]), "r"(f[S::NW > 1 ? 1 : 0]), "r"(r[S::NW > 2 ? 2 : 0]), "r"(f[S::NW > 2 ? 2 : 0]));
    } else {
        asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\tsubc.cc.u32 t, %3, %4;\n\tsubc.cc.u32 t, %5, %6;\n\tsubc.cc.u32 t, %7, %8;\n\tsubc.u32 %0, 0, 0;\n\t}"
            : "=r"(m) : "r"(r[0]), "r"(f[0]), "r"(r[S::NW > 1 ? 1 : 0]), "r"(f[S::NW > 1 ? 1 : 0]), "r"(r[S::NW > 2 ? 2 : 0]), "r"(f[S::NW > 2 ? 2 : 0]),
              "r"(r[S::NW > 3 ? 3 : 0]), "r"(f[S::NW > 3 ? 3 : 0]));
    }
#pragma unroll
    for (int i = 0; i < S::NW; i++) c[i] = (f[i] & ~m) | (r[i] & m);
}

__device__ __forceinline__ uint32_t lds_u32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}
__device__ __forceinline__ uint64_t lds_u64(uint32_t addr)
{
    uint64_t v;
    asm volatile("ld.shared.u64 %0, [%1];" : "=l"(v) : "r"(addr));
    return v;
}

// Exact hash of the window at nibble `lp` of a warp tile (shared-memory address sm_addr), rebuilt from the tile's nibble
// words alone: forward words by funnel shifts, reverse complement by nibble reversal of those.  Returns false when the
// window holds a base outside the alphabet (bit 3 of a nibble).
template <int K, bool CANON>
__device__ __forceinline__ bool window_hash(const ScanArgs &a, uint32_t sm_addr, uint32_t lp, uint64_t &hash)
{
    using S = KmerShape<K>;
    uint32_t x[S::NW + 1], f[S::NW], c[S::NW];
    const uint32_t w = sm_addr + 4 * (lp >> 3), sh = 4 * (lp & 7);
#pragma unroll
    for (int i = 0; i <= S::NW; i++) x[i] = lds_u32(w + 4 * i);     // word index <= 127 + 4 < SCAN_WARP_WORDS
    uint32_t bad = 0;
#pragma unroll
    for (int i = 0; i < S::NW; i++) {
        f[i] = __funnelshift_r(x[i], x[i + 1], sh);
        if (i == S::NW - 1) f[i] = (f[i] & S::LAST_MASK) | S::LAST_PAD;
        bad |= i == S::NW - 1 ? f[i] & S::LAST_MASK : f[i];
    }
    if (CANON) {
        // rr = the 8 NW nibbles of f reversed and complemented; the reverse complement starts P = 8 NW - K nibbles in
        constexpr int P = 8 * S::NW - K;
        uint32_t rr[S::NW + 1], r[S::NW];
#pragma unroll
        for (int i = 0; i < S::NW; i++) rr[i] = nibble_reverse(f[S::NW - 1 - i]) ^ 0x33333333u;
        rr[S::NW] = 0;
#pragma unroll
        for (int i = 0; i < S::NW; i++) {
            r[i] = P ? __funnelshift_r(rr[i], rr[i + 1], 4 * P) : rr[i];
            if (i == S::NW - 1) r[i] = (r[i] & S::LAST_MASK) | S::LAST_PAD;
        }
        canonical_words<K>(f, r, c);
    } else {
#pragma unroll
        for (int i = 0; i < S::NW; i++) c[i] = f[i];
    }
    uint32_t pool;
    asm("mov.u32 %0, 0x54474341;" : "=r"(pool));
    uint32_t asc[S::NA];
    expand_ascii<K>(c, asc, pool);
    const u64x2 h = murmur3_h1<K, S::NA>(asc, a.seed);
    hash = K <= 16 ? (uint64_t)h.lo : (((uint64_t)h.hi << 32) | h.lo);
    return !(bad & 0x88888888u);
}

// Survivor queue of the filter-word kernels: per warp, up to SCAN_SQ exact survivors {hash, stream position} waiting for
// their table work.  scan_emit's work is a chain of dependent global loads and atomics (unit lookup, threshold, table
// insert) of a few thousand cycles; done where the survivor is found, the whole warp waits for it once per survivor (about
// one vote group in 25 at the sketch's thresholds), which was 12.7 % of the k=21 kernel's time (DESIGN.md §2.4).  Queued,
// it is done by scan_sq_flush between tiles, 32 survivors at a time, one per lane, so the warp waits once per 32.  Every
// effect of scan_emit is an order-independent atomic or a write to the survivor's own position (SCAN_EVENTS' events are
// sorted by position before they are replayed), so the results do not depend on when it runs.
constexpr int SCAN_SQ = 64;          // queue capacity per warp; a survivor that finds it full does its table work at once
constexpr int SCAN_SQ_FLUSH = 32;    // scan_kernel flushes the queue after a tile that leaves at least this many entries
__shared__ uint64_t scan_sq_hash[SCAN_WARPS][SCAN_SQ];
__shared__ uint64_t scan_sq_pos[SCAN_WARPS][SCAN_SQ];
__shared__ uint32_t scan_sq_n[SCAN_WARPS];   // entries appended since the last flush (may exceed SCAN_SQ: those went direct)

// Slow path of the filter-word kernels, once per warp tile that has a survivor.  A lane's pass mask covers its 32 windows of
// the tile: bit 8 i + j = window j of the lane's block i (window start 8 (lane + 32 i) + j) passed the fast-path filter.  The
// lanes walk their set bits together (a lane with none left idles), rebuild the exact hash of each passing window from the
// tile, and queue the valid ones at or below the tile threshold for their table work.
#ifndef SCAN_RESOLVE_INLINE
#define SCAN_RESOLVE_INLINE 0   // 1: inline the per-tile resolution into scan_kernel (tools/scan_microbench.cu compares both)
#endif
template <int K, bool CANON>
static __device__ __forceinline__ void scan_resolve_body(const ScanArgs &a, uint32_t pm, uint32_t sm_addr, uint64_t tile_base, uint64_t tmax)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    while (__any_sync(0xFFFFFFFFu, pm != 0)) {
        if (pm) {
            const uint32_t bit = __ffs(pm) - 1;
            pm &= pm - 1;
            const uint32_t lp = 8 * (lane + 32 * (bit >> 3)) + (bit & 7);
            uint64_t hash;
            if (window_hash<K, CANON>(a, sm_addr, lp, hash) && hash <= tmax) {
                const uint32_t at = atomicAdd(&scan_sq_n[warp], 1u);
                if (at < SCAN_SQ) {
                    scan_sq_hash[warp][at] = hash;
                    scan_sq_pos[warp][at] = tile_base + lp;
                } else {
                    scan_emit(a, (uint32_t)hash, (uint32_t)(hash >> 32), tile_base, lp);
                }
            }
        }
    }
}
template <int K, bool CANON>
static __device__ __noinline__ void scan_resolve_call(const ScanArgs &a, uint32_t pm, uint32_t sm_addr, uint64_t tile_base, uint64_t tmax)
{
    scan_resolve_body<K, CANON>(a, pm, sm_addr, tile_base, tmax);
}
template <int K, bool CANON>
__device__ __forceinline__ void scan_resolve(const ScanArgs &a, uint32_t pm, uint32_t sm_addr, uint64_t tile_base, uint64_t tmax)
{
    if (SCAN_RESOLVE_INLINE) scan_resolve_body<K, CANON>(a, pm, sm_addr, tile_base, tmax);
    else scan_resolve_call<K, CANON>(a, pm, sm_addr, tile_base, tmax);
}

// Table work of the queued survivors of this warp, one per lane; warp-uniform call, leaves the queue empty
static __device__ __noinline__ void scan_sq_flush(const ScanArgs &a)
{
    const uint32_t warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncwarp();
    const uint32_t n = min(scan_sq_n[warp], (uint32_t)SCAN_SQ);
    for (uint32_t i = lane; i < n; i += 32) {
        const uint64_t hash = scan_sq_hash[warp][i];
        scan_emit(a, (uint32_t)hash, (uint32_t)(hash >> 32), scan_sq_pos[warp][i], 0);
    }
    __syncwarp();
    if (lane == 0) scan_sq_n[warp] = 0;
    __syncwarp();
}

// Cost-accounting switches for tools/scan_microbench.cu (0 in the library; see DESIGN.md §2.4).  Each takes one part of
// the kernel out or measures it; the kernel's results are not what the library needs when one of them is set.
//   SCAN_MB_NO_SURVIVORS: (filter-word kernels) no per-tile resolution of the pass masks; each tile's mask is xor-ed into a
//                         per-lane accumulator that is stored once at the end (a.out_hash[global thread]), so the hash and
//                         the compare stay live.
//   SCAN_MB_STAGE_ONCE:   each warp stages its first tile only and hashes it again in place of every later tile: no
//                         staging and no global prefetch after the first.
//   SCAN_MB_CLOCK:        clock64() around each tile's hot loop; lane 0 stores the warp's total cycles at
//                         a.out_hash[gridDim.x * SCAN_THREADS + global warp].
#ifndef SCAN_MB_NO_SURVIVORS
#define SCAN_MB_NO_SURVIVORS 0
#endif
#ifndef SCAN_MB_STAGE_ONCE
#define SCAN_MB_STAGE_ONCE 0
#endif
#ifndef SCAN_MB_CLOCK
#define SCAN_MB_CLOCK 0
#endif
#ifndef SCAN_VOTE_GROUP
#define SCAN_VOTE_GROUP 2      // FULL kernels only: windows hashed back to back before one warp vote (1, 2, 4 or 8); see
                               // scan_group.  The filter-word kernels do not vote in the hot loop (per-lane pass masks,
                               // resolved once per tile).  On H100 2 beat 4 and 8 (filter-word kernel, before the masks)
#endif
#ifndef SCAN_PREFETCH_SMEM
#define SCAN_PREFETCH_SMEM 1   // filter-word kernels: 1 = the next tile is prefetched by cp.async into a per-warp shared landing
                               // buffer, 0 = into registers (as the FULL kernels do); tools/scan_microbench.cu compares them
#endif

// Nibble words of the canonical k-mer of window J of the block (b = forward words, rb = reverse-complement words); the last
// word of each strand becomes (w & LM) | LP before the compare
template <int K, bool CANON, int J, uint32_t LM, uint32_t LP>
__device__ __forceinline__ void window_words(const uint32_t (&b)[KmerShape<K>::BW], const uint32_t (&rb)[KmerShape<K>::BW],
                                             uint32_t (&c)[KmerShape<K>::NW])
{
    using S = KmerShape<K>;
    uint32_t f[S::NW];
#pragma unroll
    for (int i = 0; i < S::NW; i++) {
        f[i] = block_word<J, S::BW>(b, i);
        if (i == S::NW - 1) f[i] = (f[i] & LM) | LP;
    }
    if (CANON) {
        constexpr int RO = 8 * S::BW - K - J;   // nibble offset of the reverse-complement window
        uint32_t r[S::NW];
#pragma unroll
        for (int i = 0; i < S::NW; i++) {
            r[i] = block_word<RO, S::BW>(rb, i);
            if (i == S::NW - 1) r[i] = (r[i] & LM) | LP;
        }
        canonical_words<K>(f, r, c);
    } else {
#pragma unroll
        for (int i = 0; i < S::NW; i++) c[i] = f[i];
    }
}

// ASCII words of the canonical k-mer of window J of the block
template <int K, bool CANON, int J>
__device__ __forceinline__ void window_ascii(const uint32_t (&b)[KmerShape<K>::BW], const uint32_t (&rb)[KmerShape<K>::BW], uint32_t pool,
                                             uint32_t (&asc)[KmerShape<K>::NA])
{
    using S = KmerShape<K>;
    uint32_t c[S::NW];
    window_words<K, CANON, J, S::LAST_MASK, S::LAST_PAD>(b, rb, c);
    expand_ascii<K>(c, asc, pool);
}

// Cost accounting (tools/scan_microbench.cu, DESIGN.md §2.4): SCAN_MB_EXTRA_FMA = n adds a chain of n dependent IMADs to
// every window's filter word, SCAN_MB_EXTRA_ALU = n a chain of n dependent ALU instructions (LOP3 and IADD3 in turn: a
// chain of LOP3 alone over fewer than four inputs would fold into one).  Their operands are kernel parameters, which ptxas
// cannot fold, and the chain enters the word as `x | (y & preserve_case)`, which the microbenchmark leaves 0, so its
// results do not change.  The slope of the kernel's time over n tells which pipe binds the hot loop.
#ifndef SCAN_MB_EXTRA_FMA
#define SCAN_MB_EXTRA_FMA 0
#endif
#ifndef SCAN_MB_EXTRA_ALU
#define SCAN_MB_EXTRA_ALU 0
#endif
__device__ __forceinline__ uint32_t scan_mb_extra(const ScanArgs &a, uint32_t x)
{
    if (SCAN_MB_EXTRA_FMA == 0 && SCAN_MB_EXTRA_ALU == 0) return x;
    uint32_t y = x;
#pragma unroll
    for (int i = 0; i < SCAN_MB_EXTRA_FMA; i++) y = y * (uint32_t)a.coarse_t + a.seed;
#pragma unroll
    for (int i = 0; i < SCAN_MB_EXTRA_ALU; i++) y = (i & 1) ? y + a.seed : y ^ (uint32_t)a.coarse_t;
    return x | (y & (uint32_t)a.preserve_case);
}

// Full-hash fast path (k <= 16, and the screen's probing kernels: every lane probes the reference table with its own hash)
template <int K, bool CANON, int J>
__device__ __forceinline__ bool scan_window(const ScanArgs &a, const uint32_t (&b)[KmerShape<K>::BW],
                                            const uint32_t (&rb)[KmerShape<K>::BW], uint64_t tmax, uint32_t pool, u64x2 &h_out)
{
    using S = KmerShape<K>;
    uint32_t asc[S::NA];
    window_ascii<K, CANON, J>(b, rb, pool, asc);
    u64x2 h = murmur3_h1<K, S::NA>(asc, a.seed);
    if (K <= 16) h.hi = 0;        // 32-bit hashes: |{A,C,G,T}|^k <= 2^32 (reference Sketch.cpp:1136, hash.cpp:31-35)
    // coarse filter on one 32-bit word; validity and the exact threshold are checked in the slow path
    h_out = h;
    return (K <= 16) ? (h.lo <= (uint32_t)tmax) : (h.hi <= (uint32_t)(tmax >> 32));
}

// Filter-word fast path (k > 16): only murmur3_h1_filter's word, to be tested against filter_threshold(tmax >> 32)
// (tail_tab: the CTA's tail table in shared memory, used when KmerShape<K>::TAIL_TABLE)
template <int K, bool CANON, int J>
__device__ __forceinline__ uint32_t scan_window_filter(const ScanArgs &a, const uint32_t (&b)[KmerShape<K>::BW],
                                                       const uint32_t (&rb)[KmerShape<K>::BW], uint32_t pool, const uint64_t *tail_tab)
{
    using S = KmerShape<K>;
    uint32_t x;
    if constexpr (S::TAIL_TABLE) {
        // the last word keeps the two code bits of the tail's nibbles (both strands alike, so the compare is unchanged for
        // windows in the alphabet); it becomes the table index instead of ASCII words
        uint32_t c[S::NW], asc[S::NA - 2];
        window_words<K, CANON, J, S::LAST_MASK & 0x33333333u, 0u>(b, rb, c);
#pragma unroll
        for (int i = 0; i < S::NW - 1; i++) {
            asc[2 * i] = prmt(pool, 0, c[i]);
            asc[2 * i + 1] = prmt(pool, 0, c[i] >> 16);
        }
        uint32_t at;   // base + 8 index as one IMAD: written in C, ptxas makes it a shift, a mask and an add
        asm("mad.lo.u32 %0, %1, 8, %2;" : "=r"(at) : "r"(tail_index(c[S::NW - 1])), "r"((uint32_t)__cvta_generic_to_shared(tail_tab)));
        const uint64_t k1 = lds_u64(at);
        x = murmur3_h1_filter<K, S::NA - 2, true>(asc, a.seed, u64x2{(uint32_t)k1, (uint32_t)(k1 >> 32)});
    } else {
        uint32_t asc[S::NA];
        window_ascii<K, CANON, J>(b, rb, pool, asc);
        x = murmur3_h1_filter<K, S::NA>(asc, a.seed);
    }
    return scan_mb_extra(a, x);
}

// The 8 windows of a block hashed back to back (independent multiply chains that ptxas can interleave), their pass flags
// at bits 24..31 of the result (bit 24 + j = window j).  No vote and no branch: the hot loop shifts the block's flags into
// the lane's pass mask, and the mask is resolved once per tile (scan_resolve).
template <int K, bool CANON, int... J>
__device__ __forceinline__ uint32_t scan_block_filter(const ScanArgs &a, const uint32_t (&b)[KmerShape<K>::BW], const uint32_t (&rb)[KmerShape<K>::BW],
                                                      uint32_t tf, uint32_t pool, const uint64_t *tail_tab, std::integer_sequence<int, J...>)
{
    return (((scan_window_filter<K, CANON, J>(a, b, rb, pool, tail_tab) <= tf ? 1u : 0u) << (24 + J)) | ...);
}

// Fill the CTA's tail table (KmerShape<K>::TAIL_TABLE): entry tail_index(w) = murmur3_tail_k1 of the ASCII bytes of bases
// 16..K-1 whose codes w holds at bits 0, 4, .. (all 4^5 code words, the codes past K ignored).
template <int K>
__device__ __forceinline__ void fill_tail_table(uint64_t *tab)
{
    for (uint32_t v = threadIdx.x; v < TAIL_TAB_SIZE; v += blockDim.x) {
        uint32_t w = 0;
        uint64_t t = 0;
#pragma unroll
        for (int i = 0; i < 5; i++) {
            const uint32_t code = (v >> (2 * i)) & 3u;
            w |= code << (4 * i);
            if (i < K - 16) t |= (uint64_t)((0x54474341u >> (8 * code)) & 0xFFu) << (8 * i);   // 'A' 'C' 'G' 'T'
        }
        tab[tail_index(w)] = murmur3_tail_k1(t);
    }
}

// Full-hash variant of the group: G windows, one warp vote, then the survivors of each window serialised by scan_emit_warp.
template <int K, bool CANON, int J0, int G>
__device__ __forceinline__ void scan_group(const ScanArgs &a, const uint32_t (&b)[KmerShape<K>::BW], const uint32_t (&rb)[KmerShape<K>::BW],
                                           uint64_t tile_base, uint32_t local0, uint64_t tmax, uint32_t pool, const uint32_t *sm_tile)
{
    u64x2 h[G];
    bool pass[G];
    bool any = false;
    pass[0] = scan_window<K, CANON, J0>(a, b, rb, tmax, pool, h[0]);
    if constexpr (G > 1) pass[1] = scan_window<K, CANON, J0 + (G > 1 ? 1 : 0)>(a, b, rb, tmax, pool, h[G > 1 ? 1 : 0]);
    if constexpr (G > 2) {
        pass[2] = scan_window<K, CANON, J0 + (G > 2 ? 2 : 0)>(a, b, rb, tmax, pool, h[G > 2 ? 2 : 0]);
        pass[3] = scan_window<K, CANON, J0 + (G > 2 ? 3 : 0)>(a, b, rb, tmax, pool, h[G > 2 ? 3 : 0]);
    }
    if constexpr (G > 4) {
        pass[4] = scan_window<K, CANON, J0 + (G > 4 ? 4 : 0)>(a, b, rb, tmax, pool, h[G > 4 ? 4 : 0]);
        pass[5] = scan_window<K, CANON, J0 + (G > 4 ? 5 : 0)>(a, b, rb, tmax, pool, h[G > 4 ? 5 : 0]);
        pass[6] = scan_window<K, CANON, J0 + (G > 4 ? 6 : 0)>(a, b, rb, tmax, pool, h[G > 4 ? 6 : 0]);
        pass[7] = scan_window<K, CANON, J0 + (G > 4 ? 7 : 0)>(a, b, rb, tmax, pool, h[G > 4 ? 7 : 0]);
    }
#pragma unroll
    for (int j = 0; j < G; j++) any |= pass[j];
    if (__any_sync(0xFFFFFFFFu, any)) {
#pragma unroll
        for (int j = 0; j < G; j++)
            if (__any_sync(0xFFFFFFFFu, pass[j])) scan_emit_warp(a, pass[j], h[j].lo, h[j].hi, tile_base, local0 + J0 + j, sm_tile, K, tmax);
    }
}

// 16 ASCII bytes at stream offset `off` -> two nibble words (bytes at or past stream_len become separators)
__device__ __forceinline__ uint2 stage16(const uint4 q, uint64_t off, uint64_t stream_len, uint32_t fold)
{
    uint32_t w0 = 0x88888888u, w1 = 0x88888888u;
    if (off < stream_len) {
        w0 = ascii4_to_nibbles(q.x, fold) | (ascii4_to_nibbles(q.y, fold) << 16);
        w1 = ascii4_to_nibbles(q.z, fold) | (ascii4_to_nibbles(q.w, fold) << 16);
        if (off + 16 > stream_len) {   // ragged end
            const int keep = (int)(stream_len - off);   // 1..15
            if (keep < 8) { w0 |= 0x88888888u << (4 * keep); w1 = 0x88888888u; }
            else if (keep > 8) w1 |= 0x88888888u << (4 * (keep - 8));
            else w1 = 0x88888888u;
        }
    }
    return make_uint2(w0, w1);
}

__device__ __forceinline__ uint4 load16(const uint8_t *stream, uint64_t off, uint64_t stream_len)
{
    if (off < stream_len) return __ldg(reinterpret_cast<const uint4 *>(stream + off));
    return make_uint4(0, 0, 0, 0);
}

// asynchronous global -> shared copies (cp.async, completed by cp_async_wait_all) of 16, 8 or 4 bytes
template <int N>
__device__ __forceinline__ void cp_async(uint32_t dst, const void *src)
{
    if (N == 16) asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" :: "r"(dst), "l"(src) : "memory");
    else asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" :: "r"(dst), "l"(src), "n"(N) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all()
{
    asm volatile("cp.async.wait_all;" ::: "memory");
}

__device__ __forceinline__ uint4 lds_u128(uint32_t addr)
{
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(addr));
    return v;
}
__device__ __forceinline__ void sts_u128(uint32_t addr, uint4 v)
{
    asm volatile("st.shared.v4.u32 [%0], {%1, %2, %3, %4};" :: "r"(addr), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// Prefetch of warp tile `wt` into the warp's landing buffer (shared address `land`), filter-word kernels.  ASCII source: the
// tile's 68 16-byte vectors, lanes taking vectors lane, lane + 32 and (lanes 0-3) 64 + lane.  A tile that lies wholly
// before stream_len goes by cp.async; one that reaches past it (the last tile of a launch) is loaded with load16 and stored
// by the lanes themselves, so no copy touches memory past the caller's buffer.  Packed source: groups lane and (lanes
// 0, 1) 32 + lane, the 64-bit codes at byte 8 g and the invalid bits at byte 8 * 34 + 4 g -- the words the register
// prefetch reads.
constexpr int SCAN_LAND_INVAL = 8 * 34;
template <bool PACKED>
__device__ __forceinline__ void scan_prefetch_land(const ScanArgs &a, uint64_t wt, uint32_t land, int lane)
{
    if (PACKED) {
        const uint64_t g0 = wt * (uint64_t)(SCAN_WARP_TILE / 32);
        cp_async<8>(land + 8 * lane, a.codes + g0 + lane);
        cp_async<4>(land + SCAN_LAND_INVAL + 4 * lane, a.inval + g0 + lane);
        if (lane < 2) {
            cp_async<8>(land + 8 * (32 + lane), a.codes + g0 + 32 + lane);
            cp_async<4>(land + SCAN_LAND_INVAL + 4 * (32 + lane), a.inval + g0 + 32 + lane);
        }
        return;
    }
    const uint64_t base = wt * (uint64_t)SCAN_WARP_TILE;
    if (base + 16ull * SCAN_WARP_VECS <= a.stream_len) {
        cp_async<16>(land + 16 * lane, a.stream + base + 16ull * lane);
        cp_async<16>(land + 16 * (lane + 32), a.stream + base + 16ull * (lane + 32));
        if (lane < 4) cp_async<16>(land + 16 * (64 + lane), a.stream + base + 16ull * (64 + lane));
    } else {
        sts_u128(land + 16 * lane, load16(a.stream, base + 16ull * lane, a.stream_len));
        sts_u128(land + 16 * (lane + 32), load16(a.stream, base + 16ull * (lane + 32), a.stream_len));
        if (lane < 4) sts_u128(land + 16 * (64 + lane), load16(a.stream, base + 16ull * (64 + lane), a.stream_len));
    }
}

// 32 packed positions (2-bit codes + invalid bits) -> 4 nibble words
__device__ __forceinline__ uint32_t spread_codes8(uint32_t x)   // 8 two-bit codes (16 bits) -> 8 nibbles
{
    x = (x | (x << 8)) & 0x00FF00FFu;
    x = (x | (x << 4)) & 0x0F0F0F0Fu;
    x = (x | (x << 2)) & 0x33333333u;
    return x;
}
__device__ __forceinline__ uint32_t spread_bits8(uint32_t y)    // 8 bits -> bit 3 of 8 nibbles
{
    y = (y | (y << 12)) & 0x000F000Fu;
    y = (y | (y << 6)) & 0x03030303u;
    y = (y | (y << 3)) & 0x11111111u;
    return y << 3;
}
__device__ __forceinline__ uint4 expand32(uint64_t c, uint32_t m)
{
    const uint32_t lo = (uint32_t)c, hi = (uint32_t)(c >> 32);
    uint4 r;
    r.x = spread_codes8(lo & 0xFFFFu) | spread_bits8(m & 0xFFu);
    r.y = spread_codes8(lo >> 16) | spread_bits8((m >> 8) & 0xFFu);
    r.z = spread_codes8(hi & 0xFFFFu) | spread_bits8((m >> 16) & 0xFFu);
    r.w = spread_codes8(hi >> 16) | spread_bits8(m >> 24);
    return r;
}

// Warp-private tiles: every warp owns WARP_TILE window starts at a time, staged in its own slice of shared memory,
// so the only synchronisation is __syncwarp().  The next tile's bytes are prefetched before the current tile is hashed
// (global latency hidden behind ~4000 instructions of work per lane): by the FULL kernels into registers, by the
// filter-word kernels into a per-warp shared landing buffer (SCAN_PREFETCH_SMEM), which keeps those registers free
// through the hot loop.
#ifndef SCAN_MIN_BLOCKS
#define SCAN_MIN_BLOCKS 4      // filter-word kernels: resident CTAs per SM requested from ptxas (4 => 64 registers, no spills
                               // since the hot loop holds neither a survivor call nor prefetch registers; 3 => 80 registers, 1 %
                               // slower); tools/scan_microbench.cu compares the settings (-DSCAN_MIN_BLOCKS=n)
#endif
#ifndef SCAN_MIN_BLOCKS_FULL
#define SCAN_MIN_BLOCKS_FULL 3 // FULL kernels (=> 80 registers, no spills; 4 => 64 registers and spills)
#endif
// FULL: the fast path computes the whole 64-bit hash (k <= 16, where the filter is on the low word, and SCAN_SCREEN, where
// every lane probes the reference table with it); otherwise only murmur3_h1_filter's word and the slow path recomputes.
template <int K, bool CANON, bool PACKED, bool FULL>
__global__ void __launch_bounds__(SCAN_THREADS, FULL ? ((K > 24 && SCAN_MIN_BLOCKS_FULL > 3) ? 3 : SCAN_MIN_BLOCKS_FULL) : SCAN_MIN_BLOCKS)
scan_kernel(const __grid_constant__ ScanArgs a)
{
    using S = KmerShape<K>;
    static_assert(FULL || K > 16, "the filter word is the high word of the hash");
    __shared__ __align__(16) uint32_t sm_all[SCAN_WARPS][SCAN_WARP_WORDS];
    // reverse-complement image of the tile (word i = nibble-reversed, complemented word NW-1-i), written once at staging so
    // that a block's reverse-complement words are 4 more LDS (the LSU is idle) instead of ~16 ALU instructions per block
    __shared__ __align__(16) uint32_t smr_all[CANON ? SCAN_WARPS : 1][SCAN_WARP_WORDS];
    constexpr bool LAND = !FULL && SCAN_PREFETCH_SMEM;
    __shared__ __align__(16) uint4 land_all[LAND ? SCAN_WARPS : 1][LAND ? SCAN_WARP_VECS : 1];   // next tile's raw bytes
    constexpr bool TAB = !FULL && S::TAIL_TABLE;
    __shared__ __align__(16) uint64_t tail_tab[TAB ? TAIL_TAB_SIZE : 1];
    if (TAB) {
        fill_tail_table<K>(tail_tab);
        __syncthreads();
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t *sm = sm_all[warp];
    uint32_t *smr = smr_all[CANON ? warp : 0];
    // the hot loop and the slow path address the tiles as 32-bit shared-memory addresses, passed through a shuffle (they are
    // warp-uniform) so that ptxas keeps them in registers: it otherwise re-derives them (S2R SR_CgaCtaId, LEA, IMAD) on every
    // iteration of the hot loop to save a register
    const uint32_t sm_addr = __shfl_sync(0xFFFFFFFFu, (uint32_t)__cvta_generic_to_shared(sm), 0);
    const uint32_t smr_addr = __shfl_sync(0xFFFFFFFFu, (uint32_t)__cvta_generic_to_shared(smr), 0);
    const uint32_t land = (uint32_t)__cvta_generic_to_shared(land_all[LAND ? warp : 0]);
    const uint32_t fold = a.preserve_case ? 0xFFFFFFFFu : 0xDFDFDFDFu;
    uint32_t pool;   // bytes 'A','C','G','T' for PRMT; opaque to the compiler so that it stays in one register
    asm volatile("mov.u32 %0, 0x54474341;" : "=r"(pool));

    const uint64_t wt_begin = a.tile_begin * (SCAN_TILE / SCAN_WARP_TILE);
    const uint64_t wt_end = a.tile_end * (SCAN_TILE / SCAN_WARP_TILE);
    const uint64_t wt_stride = (uint64_t)gridDim.x * SCAN_WARPS;
    uint64_t wt = wt_begin + (uint64_t)blockIdx.x * SCAN_WARPS + warp;
    if (wt >= wt_end) return;

    // each lane stages vectors lane, lane+32 and one of the 4 halo vectors (64 + lane%4: eight lanes write the same
    // words with the same values -- no lane-dependent branch, the warp never splits): 16 bytes -> 2 words each
    static_assert(SCAN_WARP_VECS - 64 == 4, "halo = 4 vectors");
    const int v2 = 64 + (lane & 3);
    uint4 q0, q1, q2;                      // ASCII source: three 16-byte vectors per lane
    uint64_t pc0 = 0, pc1 = 0;             // packed source: group (lane) and one of the 2 halo groups (32 + lane%2)
    uint32_t pm0 = 0, pm1 = 0;
    const int hg = 32 + (lane & 1);
    if (LAND) {
        scan_prefetch_land<PACKED>(a, wt, land, lane);
    } else if (PACKED) {
        const uint64_t g0 = wt * (uint64_t)(SCAN_WARP_TILE / 32);
        pc0 = __ldg(a.codes + g0 + lane); pm0 = __ldg(a.inval + g0 + lane);
        pc1 = __ldg(a.codes + g0 + hg);   pm1 = __ldg(a.inval + g0 + hg);
    } else {
        const uint64_t base = wt * (uint64_t)SCAN_WARP_TILE;
        q0 = load16(a.stream, base + 16ull * lane, a.stream_len);
        q1 = load16(a.stream, base + 16ull * (lane + 32), a.stream_len);
        q2 = load16(a.stream, base + 16ull * v2, a.stream_len);
    }
    if (!FULL) {
        if (lane == 0) scan_sq_n[warp] = 0;
        __syncwarp();
    }
    uint32_t mb_acc = 0;
    long long mb_cycles = 0;
    const uint64_t wt_first = wt;
    for (; wt < wt_end; wt += wt_stride) {
        const uint64_t base = wt * (uint64_t)SCAN_WARP_TILE;
        if (LAND && !(SCAN_MB_STAGE_ONCE && wt != wt_first)) {   // this tile's bytes, copied in during the previous tile
            cp_async_wait_all();
            __syncwarp();
            if (PACKED) {
                pc0 = lds_u64(land + 8 * lane); pm0 = lds_u32(land + SCAN_LAND_INVAL + 4 * lane);
                pc1 = lds_u64(land + 8 * hg);   pm1 = lds_u32(land + SCAN_LAND_INVAL + 4 * hg);
            } else {
                q0 = lds_u128(land + 16 * lane);
                q1 = lds_u128(land + 16 * (lane + 32));
                q2 = lds_u128(land + 16 * v2);
            }
        }
        if (SCAN_MB_STAGE_ONCE && wt != wt_first) {
            // microbenchmark only: hash the first tile again
        } else if (PACKED) {
            const uint4 e0 = expand32(pc0, pm0), e1 = expand32(pc1, pm1);
            *reinterpret_cast<uint4 *>(sm + 4 * lane) = e0;
            *reinterpret_cast<uint4 *>(sm + 4 * hg) = e1;
            if (CANON) {
                *reinterpret_cast<uint4 *>(smr + (SCAN_WARP_WORDS - 4 - 4 * lane)) =
                    make_uint4(nibble_reverse(e0.w) ^ 0x33333333u, nibble_reverse(e0.z) ^ 0x33333333u, nibble_reverse(e0.y) ^ 0x33333333u, nibble_reverse(e0.x) ^ 0x33333333u);
                *reinterpret_cast<uint4 *>(smr + (SCAN_WARP_WORDS - 4 - 4 * hg)) =
                    make_uint4(nibble_reverse(e1.w) ^ 0x33333333u, nibble_reverse(e1.z) ^ 0x33333333u, nibble_reverse(e1.y) ^ 0x33333333u, nibble_reverse(e1.x) ^ 0x33333333u);
            }
        } else {
            const uint2 s0 = stage16(q0, base + 16ull * lane, a.stream_len, fold);
            const uint2 s1 = stage16(q1, base + 16ull * (lane + 32), a.stream_len, fold);
            const uint2 s2 = stage16(q2, base + 16ull * v2, a.stream_len, fold);
            *reinterpret_cast<uint2 *>(sm + 2 * lane) = s0;
            *reinterpret_cast<uint2 *>(sm + 2 * (lane + 32)) = s1;
            *reinterpret_cast<uint2 *>(sm + 2 * v2) = s2;
            if (CANON) {
                *reinterpret_cast<uint2 *>(smr + (SCAN_WARP_WORDS - 2 - 2 * lane)) = make_uint2(nibble_reverse(s0.y) ^ 0x33333333u, nibble_reverse(s0.x) ^ 0x33333333u);
                *reinterpret_cast<uint2 *>(smr + (SCAN_WARP_WORDS - 2 - 2 * (lane + 32))) = make_uint2(nibble_reverse(s1.y) ^ 0x33333333u, nibble_reverse(s1.x) ^ 0x33333333u);
                *reinterpret_cast<uint2 *>(smr + (SCAN_WARP_WORDS - 2 - 2 * v2)) = make_uint2(nibble_reverse(s2.y) ^ 0x33333333u, nibble_reverse(s2.x) ^ 0x33333333u);
            }
        }
        __syncwarp();
        const uint64_t next = wt + wt_stride;
        if (!SCAN_MB_STAGE_ONCE && next < wt_end) {   // prefetch
            if (LAND) {
                scan_prefetch_land<PACKED>(a, next, land, lane);
            } else if (PACKED) {
                const uint64_t g0 = next * (uint64_t)(SCAN_WARP_TILE / 32);
                pc0 = __ldg(a.codes + g0 + lane); pm0 = __ldg(a.inval + g0 + lane);
                pc1 = __ldg(a.codes + g0 + hg);   pm1 = __ldg(a.inval + g0 + hg);
            } else {
                const uint64_t nb = next * (uint64_t)SCAN_WARP_TILE;
                q0 = load16(a.stream, nb + 16ull * lane, a.stream_len);
                q1 = load16(a.stream, nb + 16ull * (lane + 32), a.stream_len);
                q2 = load16(a.stream, nb + 16ull * v2, a.stream_len);
            }
        }
        __syncwarp();
        const uint64_t tmax = a.tile_tmax ? a.tile_tmax[base / SCAN_TILE] : a.coarse_t;
        const uint32_t tf = filter_threshold((uint32_t)(tmax >> 32));
        const long long c0 = SCAN_MB_CLOCK ? clock64() : 0;
        static_assert(SCAN_WARP_TILE / 8 == 4 * 32, "a lane's pass mask holds 4 blocks of 8 windows");
        uint32_t pmask = 0;   // filter-word kernels: the lane's pass flags of this tile, see scan_resolve
#pragma unroll 1
        for (int g = lane; g < SCAN_WARP_TILE / 8; g += 32) {
            uint32_t b[S::BW], rb[S::BW];
#pragma unroll
            for (int i = 0; i < S::BW; i++) b[i] = lds_u32(sm_addr + 4u * (g + i));
            if (CANON) {
#pragma unroll
                for (int i = 0; i < S::BW; i++) rb[i] = lds_u32(smr_addr + 4u * (SCAN_WARP_WORDS - S::BW - g + i));
            }
            const uint32_t local0 = 8u * g;
            constexpr int G = SCAN_VOTE_GROUP;
            if constexpr (!FULL) {
                // block i = (g - lane) / 32 ends at bits 8 i .. 8 i + 7 after the tile's 4 trips
                pmask = (pmask >> 8) | scan_block_filter<K, CANON>(a, b, rb, tf, pool, tail_tab, std::make_integer_sequence<int, 8>());
            } else {
                scan_group<K, CANON, 0, G>(a, b, rb, base, local0, tmax, pool, sm);
                if constexpr (G < 8) scan_group<K, CANON, (G < 8 ? G : 0), G>(a, b, rb, base, local0, tmax, pool, sm);
                if constexpr (G < 4) {
                    scan_group<K, CANON, (G < 4 ? 2 * G : 0), G>(a, b, rb, base, local0, tmax, pool, sm);
                    scan_group<K, CANON, (G < 4 ? 3 * G : 0), G>(a, b, rb, base, local0, tmax, pool, sm);
                }
                if constexpr (G < 2) {
                    scan_group<K, CANON, 4, 1>(a, b, rb, base, local0, tmax, pool, sm);
                    scan_group<K, CANON, 5, 1>(a, b, rb, base, local0, tmax, pool, sm);
                    scan_group<K, CANON, 6, 1>(a, b, rb, base, local0, tmax, pool, sm);
                    scan_group<K, CANON, 7, 1>(a, b, rb, base, local0, tmax, pool, sm);
                }
            }
        }
        if (SCAN_MB_CLOCK) mb_cycles += clock64() - c0;
        if (!FULL) {
            if (SCAN_MB_NO_SURVIVORS) mb_acc ^= pmask;
            else if (__any_sync(0xFFFFFFFFu, pmask != 0)) scan_resolve<K, CANON>(a, pmask, sm_addr, base, tmax);
        }
        __syncwarp();
        if (!FULL && scan_sq_n[warp] >= SCAN_SQ_FLUSH) scan_sq_flush(a);
    }
    if (!FULL && scan_sq_n[warp] > 0) scan_sq_flush(a);
    if (SCAN_MB_NO_SURVIVORS) a.out_hash[(uint64_t)blockIdx.x * SCAN_THREADS + threadIdx.x] = mb_acc;
    if (SCAN_MB_CLOCK && lane == 0) a.out_hash[(uint64_t)gridDim.x * SCAN_THREADS + (uint64_t)blockIdx.x * SCAN_WARPS + warp] = (uint64_t)mb_cycles;
}

// ---------------------------------------------------------------------------------------------------------------
// Byte-alphabet kernel: any alphabet (protein, custom -z), k-mers hashed as they stand (the reference makes every
// non-nucleotide alphabet non-canonical, sketchParameterSetup.cpp:79-95).  Same warp-private tiling; the tile is kept
// as bytes (alphabet bytes, 0 = outside the alphabet), a lane takes 4 consecutive window starts per block and builds each
// window with PRMT byte funnels.  Validity, exact threshold and table work stay in the shared slow path.
// ---------------------------------------------------------------------------------------------------------------
constexpr int GEN_WARP_WORDS = SCAN_WARP_TILE / 4 + 16;     // 1024 + 64 bytes

template <int K>
__global__ void __launch_bounds__(SCAN_THREADS) scan_bytes_kernel(const __grid_constant__ ScanArgs a)
{
    constexpr int NWB = (K + 3) / 4;              // words per k-mer
    constexpr int BWB = (K + 3 + 3) / 4;          // words per block of 4 window starts
    constexpr int NA = 2 * ((K + 7) / 8);         // words murmur3_h1 expects
    __shared__ __align__(16) uint32_t sm_all[SCAN_WARPS][GEN_WARP_WORDS];
    __shared__ uint8_t lut[256];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t *sm = sm_all[warp];
    for (int i = threadIdx.x; i < 256; i += SCAN_THREADS) lut[i] = a.byte_lut[i];
    __syncthreads();

    const uint64_t wt_begin = a.tile_begin * (SCAN_TILE / SCAN_WARP_TILE), wt_end = a.tile_end * (SCAN_TILE / SCAN_WARP_TILE);
    const uint64_t wt_stride = (uint64_t)gridDim.x * SCAN_WARPS;
    for (uint64_t wt = wt_begin + (uint64_t)blockIdx.x * SCAN_WARPS + warp; wt < wt_end; wt += wt_stride) {
        const uint64_t base = wt * (uint64_t)SCAN_WARP_TILE;
        // stage 1088 bytes = 68 vectors of 16: lanes take vectors lane, lane+32, 64 + lane%4
        const int vec[3] = {lane, lane + 32, 64 + (lane & 3)};
#pragma unroll
        for (int t = 0; t < 3; t++) {
            const uint64_t off = base + 16ull * vec[t];
            uint4 q = load16(a.stream, off, a.stream_len);
            uint32_t w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                uint32_t o = 0;
#pragma unroll
                for (int b = 0; b < 4; b++) {
                    const uint64_t pos = off + 4 * j + b;
                    const uint32_t c = pos < a.stream_len ? lut[(w[j] >> (8 * b)) & 0xFFu] : 0u;
                    o |= c << (8 * b);
                }
                w[j] = o;
            }
            *reinterpret_cast<uint4 *>(sm + 4 * vec[t]) = make_uint4(w[0], w[1], w[2], w[3]);
        }
        __syncwarp();
        const uint64_t tmax = a.tile_tmax ? a.tile_tmax[base / SCAN_TILE] : a.coarse_t;
#pragma unroll 1
        for (int g = lane; g < SCAN_WARP_TILE / 4; g += 32) {
            uint32_t b[BWB];
#pragma unroll
            for (int i = 0; i < BWB; i++) b[i] = sm[g + i];
#pragma unroll
            for (int j = 0; j < 4; j++) {
                uint32_t asc[NA];
#pragma unroll
                for (int i = 0; i < NA; i++) {
                    uint32_t v = 0;
                    if (i < NWB) {
                        const uint32_t lo = b[i], hi = (i + 1 < BWB) ? b[i + 1] : 0u;
                        v = j == 0 ? lo : __funnelshift_r(lo, hi, 8 * j);
                        const int rem = K - 4 * i;
                        if (rem < 4) v &= (1u << (8 * rem)) - 1u;
                    }
                    asc[i] = v;
                }
                u64x2 h = murmur3_h1<K, NA>(asc, a.seed);
                if (!a.use64) h.hi = 0;
                const bool pass = a.use64 ? (h.hi <= (uint32_t)(tmax >> 32)) : (h.lo <= (uint32_t)tmax);
                if (__any_sync(0xFFFFFFFFu, pass)) scan_emit_warp(a, pass, h.lo, h.hi, base, 4u * g + j, sm, -K, tmax);
            }
        }
        __syncwarp();
    }
}

// Host-side launcher table (defined in scan_inst_*.cu)
typedef void (*scan_launch_fn)(const ScanArgs &a, int grid, cudaStream_t stream);
typedef int (*scan_occupancy_fn)();
scan_launch_fn get_scan_launcher(int k, bool canonical, bool packed);
scan_launch_fn get_bytes_launcher(int k);

}  // namespace mashgpu
