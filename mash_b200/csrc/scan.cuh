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
// Only hashes at or below the tile's coarse threshold leave the fast path.  That is the layout of the FULL kernels
// (k <= 16 and the screen's probing kernels); the filter-word kernels (k = 17..32) stage 2-bit codes instead and take the
// first multiplies of MurmurHash3 from tables indexed by bytes of the canonical k-mer (CodeTables below), building no
// ASCII in the fast path.
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

// word i of (block >> BITS*OFF), block = BW little-endian words of BITS-bit digits (nibbles, or 2-bit codes)
template <int OFF, int BW, int BITS = 4>
__device__ __forceinline__ uint32_t block_word(const uint32_t (&b)[BW], int i)
{
    constexpr int DIGITS = 32 / BITS;
    constexpr int WS = OFF / DIGITS, SH = BITS * (OFF % DIGITS);
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
    // 17 <= K <= 21 (a tail block of 1..5 bases): the FULL kernels take the tail's k1 from a table (TailTable)
    static constexpr bool TAIL_TABLE = K >= 17 && K <= 21;
};

// Tail block by table.  For 17 <= K <= 21 the tail block of MurmurHash3 is bases 16..K-1 of the canonical k-mer, and its k1
// (murmur3_tail_k1 of their ASCII bytes) takes at most 4^5 values and does not depend on the seed.  The FULL kernels (the
// screen's probing kernels at these k) keep the 1024 values in shared memory and replace the tail's two PRMT, two multiplies and rotate by one IMAD, one shift
// and one 8-byte LDS.  The index is computed from the canonical k-mer's last nibble word with bit 3 and bit 2 of every
// nibble cleared (codes c0..c4 at bits 0, 4, 8, 12, 16): w * (2^10 + 1) puts c0, c3, c1, c4, c2 side by side at bits
// 10..19 without overlap and without a carry, and the shift keeps those ten bits.  Windows with a base outside the
// alphabet read some entry and are rejected by the slow path's validity test.
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
// (Sketch.cpp:569-571): borrow out of rc - fwd.  m = all-ones when the reverse complement is the canonical k-mer.  The
// argument (DESIGN.md §2.2) holds for any digit width, so N words of nibbles or of 2-bit codes.
template <int N>
__device__ __forceinline__ void canonical_words(const uint32_t (&f)[N], const uint32_t (&r)[N], uint32_t (&c)[N])
{
    uint32_t m;
    if (N == 1) {
        asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\tsubc.u32 %0, 0, 0;\n\t}" : "=r"(m) : "r"(r[0]), "r"(f[0]));
    } else if (N == 2) {
        asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\tsubc.cc.u32 t, %3, %4;\n\tsubc.u32 %0, 0, 0;\n\t}"
            : "=r"(m) : "r"(r[0]), "r"(f[0]), "r"(r[N > 1 ? 1 : 0]), "r"(f[N > 1 ? 1 : 0]));
    } else if (N == 3) {
        asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\tsubc.cc.u32 t, %3, %4;\n\tsubc.cc.u32 t, %5, %6;\n\tsubc.u32 %0, 0, 0;\n\t}"
            : "=r"(m) : "r"(r[0]), "r"(f[0]), "r"(r[N > 1 ? 1 : 0]), "r"(f[N > 1 ? 1 : 0]), "r"(r[N > 2 ? 2 : 0]), "r"(f[N > 2 ? 2 : 0]));
    } else {
        asm("{\n\t.reg .u32 t;\n\tsub.cc.u32 t, %1, %2;\n\tsubc.cc.u32 t, %3, %4;\n\tsubc.cc.u32 t, %5, %6;\n\tsubc.cc.u32 t, %7, %8;\n\tsubc.u32 %0, 0, 0;\n\t}"
            : "=r"(m) : "r"(r[0]), "r"(f[0]), "r"(r[N > 1 ? 1 : 0]), "r"(f[N > 1 ? 1 : 0]), "r"(r[N > 2 ? 2 : 0]), "r"(f[N > 2 ? 2 : 0]),
              "r"(r[N > 3 ? 3 : 0]), "r"(f[N > 3 ? 3 : 0]));
    }
#pragma unroll
    for (int i = 0; i < N; i++) c[i] = (f[i] & ~m) | (r[i] & m);
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

// ---------------------------------------------------------------------------------------------------------------
// 2-bit tiles of the filter-word kernels.  A warp tile's 1088 bases (1024 window starts + 64 halo) are staged as 68 words
// of 16 bases (base i of a word at bits 2i, codes A0 C1 G2 T3 as the packed source has them), beside a reverse-complement
// image (word j = word 67 - j with its codes in reverse order and complemented, so reverse-complement base q is the
// complement of forward base 1087 - q) and a validity bitmap (1 bit per base, set = outside the alphabet) that only the
// slow path reads.  A k-mer (17 <= k <= 32) is 2 words per strand; the first multiply of every MurmurHash3 block lane
// comes from tables indexed by single bytes of those words (CodeTables), so the fast path builds no ASCII.
// ---------------------------------------------------------------------------------------------------------------
constexpr int SCAN_C2_IMAGE = 68;      // code words per warp tile image
constexpr int SCAN_C2_WORDS = 72;      // padded: a block's reverse-complement load of an even lane reads word 68 (unused bits)
constexpr int SCAN_INV_WORDS = 36;     // 34 validity words, padded

template <int K>
struct CodeShape {
    static_assert(K > 16 && K <= 32, "2-bit tiles serve the filter-word kernels");
    static constexpr int NB = (K + 7 + 15) / 16;     // normalised code words per block of 8 window starts: 2 (k <= 25) or 3
    static constexpr uint32_t M1 = K == 32 ? 0xFFFFFFFFu : (1u << (2 * (K - 16) & 31)) - 1u;   // bases 16..K-1 of word 1
    // tail block (bases 16..K-1): k = 17..21 take its k1 whole from a 1024-entry table indexed by word 1 (TAIL_TABLE).  For
    // k = 22..31 its whole 4-base groups use the block tables, and the one group that K cuts short, starting at base GS,
    // has a K-specific table of 256 products with zero bytes past K: an H-lane group (bases 4..7 of a lane: GS = 20, 28)
    // or an L-lane group (GS = 24).
    static constexpr bool TAIL_TABLE = K <= 21;
    static constexpr int GS = (K <= 21 || K % 4 == 0) ? 0 : K / 4 * 4;
    static constexpr int TAIL_SIZE = TAIL_TABLE ? TAIL_TAB_SIZE : GS ? 256 : 1;
};

// First multiplies of a MurmurHash3 block lane.  A lane (k1 or k2) is 8 ASCII bytes, L + H 2^32 with L the bytes of its
// bases 0..3 and H of bases 4..7, so lane * c mod 2^64 = L c + ((H c_lo) mod 2^32) 2^32: a 64-bit value that depends on
// 4 bases and a 32-bit one that depends on 4 others, 256 values each, indexed by the byte of 2-bit codes of those bases.
// They depend neither on the seed nor on k.  a/b: k1 (c1), c/d: k2 (c2); tail: CodeShape<K>'s tail table.  One object, so
// that the hot loop addresses every table from one register with immediate offsets.
template <int K>
struct CodeTables {
    uint64_t a[256], c[256], tail[CodeShape<K>::TAIL_SIZE];
    uint32_t b[256], d[256];
    static constexpr uint32_t A = 0, C = 8 * 256, TAIL = 16 * 256, B = TAIL + 8 * CodeShape<K>::TAIL_SIZE, D = B + 4 * 256;
};

// ASCII bytes of the first n codes of v (2 bits each), zero bytes after
__device__ __forceinline__ uint64_t codes_ascii(uint32_t v, int n)
{
    uint64_t t = 0;
    for (int i = 0; i < n; i++) t |= (uint64_t)((0x54474341u >> (8 * ((v >> (2 * i)) & 3u))) & 0xFFu) << (8 * i);   // A C G T
    return t;
}

// Fill the CTA's tables (CodeShape<K>); the caller synchronises
template <int K>
__device__ __forceinline__ void fill_code_tables(CodeTables<K> &t)
{
    using C = CodeShape<K>;
    constexpr uint64_t c1 = 0x87c37b91114253d5ULL, c2 = 0x4cf5ad432745937fULL;
    for (uint32_t v = threadIdx.x; v < 256; v += blockDim.x) {
        const uint64_t l = codes_ascii(v, 4);
        t.a[v] = l * c1;
        t.c[v] = l * c2;
        t.b[v] = (uint32_t)l * (uint32_t)c1;
        t.d[v] = (uint32_t)l * (uint32_t)c2;
    }
    if (C::TAIL_TABLE) {
        for (uint32_t v = threadIdx.x; v < TAIL_TAB_SIZE; v += blockDim.x) t.tail[v] = murmur3_tail_k1(codes_ascii(v, K - 16));
    } else if (C::GS) {
        const uint64_t c = C::GS < 24 ? c1 : c2;
        for (uint32_t v = threadIdx.x; v < 256; v += blockDim.x) {
            const uint64_t l = codes_ascii(v, K - C::GS);
            t.tail[v] = C::GS % 8 == 4 ? (uint64_t)((uint32_t)l * (uint32_t)c) : l * c;
        }
    }
}

// Table lookups: the address idx * SCALE + tab is one IMAD (written in C, ptxas makes each a shift and a mask on the ALU
// pipe), and the table's offset in CodeTables is the LDS immediate
template <uint32_t OFF>
__device__ __forceinline__ uint64_t tab_u64(uint32_t tab, uint32_t idx)
{
    uint32_t at;
    uint64_t v;
    asm("mad.lo.u32 %0, %1, 8, %2;" : "=r"(at) : "r"(idx), "r"(tab));
    asm("ld.shared.u64 %0, [%1+%2];" : "=l"(v) : "r"(at), "n"(OFF));
    return v;
}
template <uint32_t OFF>
__device__ __forceinline__ uint32_t tab_u32(uint32_t tab, uint32_t idx)
{
    uint32_t at, v;
    asm("mad.lo.u32 %0, %1, 4, %2;" : "=r"(at) : "r"(idx), "r"(tab));
    asm("ld.shared.u32 %0, [%1+%2];" : "=r"(v) : "r"(at), "n"(OFF));
    return v;
}
// one byte of a word, as one ALU instruction
template <int I>
__device__ __forceinline__ uint32_t byte_of(uint32_t x)
{
    if (I == 0) return x & 0xFFu;
    if (I == 3) return x >> 24;
    return __byte_perm(x, 0u, 0x4440u + I);
}
__device__ __forceinline__ u64x2 lane_product(uint64_t lo, uint32_t hi)
{
    return u64x2{(uint32_t)lo, (uint32_t)(lo >> 32) + hi};
}

// The filter word of the canonical k-mer whose 2-bit words are c[0] (bases 0..15) and c[1] (bases 16..K-1, masked); tab:
// the shared address of the CTA's CodeTables<K>
template <int K>
__device__ __forceinline__ uint32_t code_filter_word(const ScanArgs &a, const uint32_t (&c)[2], uint32_t tab)
{
    using C = CodeShape<K>;
    using T = CodeTables<K>;
    constexpr int NP = MurmurShape<K>::NP;
    u64x2 p1[NP], p2[NP];
    p1[0] = lane_product(tab_u64<T::A>(tab, byte_of<0>(c[0])), tab_u32<T::B>(tab, byte_of<1>(c[0])));
    p2[0] = lane_product(tab_u64<T::C>(tab, byte_of<2>(c[0])), tab_u32<T::D>(tab, byte_of<3>(c[0])));
    if constexpr (C::TAIL_TABLE) {
        const uint64_t k1 = tab_u64<T::TAIL>(tab, c[1]);
        return murmur3_filter_mix<K, true>(p1, p2, a.seed, u64x2{(uint32_t)k1, (uint32_t)(k1 >> 32)});
    } else {
        // bases 16..23 (k1 of block 1 or of the tail): bases 16..19 are always whole for k >= 22
        const uint32_t b1 = byte_of<1>(c[1]);
        p1[NP - 1] = lane_product(tab_u64<T::A>(tab, byte_of<0>(c[1])), K >= 24 ? tab_u32<T::B>(tab, b1) : tab_u32<T::TAIL>(tab, 2 * b1));
        if constexpr (K >= 25) {   // bases 24..31 (k2 of block 1 or of the tail)
            const uint32_t b2 = byte_of<2>(c[1]), b3 = byte_of<3>(c[1]);
            const uint32_t hi = K == 32 ? tab_u32<T::D>(tab, b3) : K >= 29 ? tab_u32<T::TAIL>(tab, 2 * b3) : 0u;
            p2[NP - 1] = lane_product(K >= 28 ? tab_u64<T::C>(tab, b2) : tab_u64<T::TAIL>(tab, b2), hi);
        } else {
            p2[NP - 1] = u64x2{0u, 0u};
        }
        return murmur3_filter_mix<K>(p1, p2, a.seed);
    }
}

// reverse complement of the 16 codes of a word: code order reversed, every code complemented (xor 3)
__device__ __forceinline__ uint32_t revcomp16(uint32_t x)
{
    x = __brev(x);                          // code order reversed, the two bits of each code swapped
    return ~(((x >> 1) & 0x55555555u) | ((x << 1) & 0xAAAAAAAAu));
}

// 8 two-bit codes (16 bits) -> 8 nibbles
__device__ __forceinline__ uint32_t spread_codes8(uint32_t x)
{
    x = (x | (x << 8)) & 0x00FF00FFu;
    x = (x | (x << 4)) & 0x0F0F0F0Fu;
    x = (x | (x << 2)) & 0x33333333u;
    return x;
}

// Exact hash of the window at base `lp` of a warp tile, rebuilt from its code images (shared addresses c2 forward, rc2
// reverse complement) and its validity bitmap (inv).  Returns false when the window holds a base outside the alphabet.
template <int K, bool CANON>
__device__ __forceinline__ bool window_hash(const ScanArgs &a, uint32_t c2, uint32_t rc2, uint32_t inv, uint32_t lp, uint64_t &hash)
{
    using S = KmerShape<K>;
    using C = CodeShape<K>;
    uint32_t f[2], c[2];
    {
        const uint32_t w = c2 + 4 * (lp >> 4), sh = 2 * (lp & 15);      // word index <= 63 + 2
        const uint32_t x0 = lds_u32(w), x1 = lds_u32(w + 4), x2 = lds_u32(w + 8);
        f[0] = __funnelshift_r(x0, x1, sh);
        f[1] = __funnelshift_r(x1, x2, sh) & C::M1;
    }
    const uint32_t v = inv + 4 * (lp >> 5);
    const uint32_t bad = __funnelshift_r(lds_u32(v), lds_u32(v + 4), lp & 31) & (K == 32 ? 0xFFFFFFFFu : (1u << (K & 31)) - 1u);
    if (CANON) {
        const uint32_t q = 16 * SCAN_C2_IMAGE - lp - K;                 // the reverse complement's first base, word <= 66 + 2
        const uint32_t w = rc2 + 4 * (q >> 4), sh = 2 * (q & 15);
        const uint32_t y0 = lds_u32(w), y1 = lds_u32(w + 4), y2 = lds_u32(w + 8);
        const uint32_t r[2] = {__funnelshift_r(y0, y1, sh), __funnelshift_r(y1, y2, sh) & C::M1};
        canonical_words(f, r, c);
    } else {
        c[0] = f[0]; c[1] = f[1];
    }
    uint32_t n[S::NW];
#pragma unroll
    for (int i = 0; i < S::NW; i++) {
        n[i] = spread_codes8((c[i >> 1] >> (16 * (i & 1))) & 0xFFFFu);
        if (i == S::NW - 1) n[i] = (n[i] & S::LAST_MASK) | S::LAST_PAD;
    }
    uint32_t pool;
    asm("mov.u32 %0, 0x54474341;" : "=r"(pool));
    uint32_t asc[S::NA];
    expand_ascii<K>(n, asc, pool);
    const u64x2 h = murmur3_h1<K, S::NA>(asc, a.seed);
    hash = ((uint64_t)h.hi << 32) | h.lo;
    return bad == 0;
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
// tile, and queue the valid ones at or below the tile threshold for their table work.  Out of line: inlined into scan_kernel
// it measured slower (DESIGN.md §2.4).
template <int K, bool CANON>
static __device__ __noinline__ void scan_resolve(const ScanArgs &a, uint32_t pm, uint32_t c2, uint32_t rc2, uint32_t inv, uint64_t tile_base,
                                                uint64_t tmax)
{
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    while (__any_sync(0xFFFFFFFFu, pm != 0)) {
        if (pm) {
            const uint32_t bit = __ffs(pm) - 1;
            pm &= pm - 1;
            const uint32_t lp = 8 * (lane + 32 * (bit >> 3)) + (bit & 7);
            uint64_t hash;
            if (window_hash<K, CANON>(a, c2, rc2, inv, lp, hash) && hash <= tmax) {
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
        canonical_words(f, r, c);
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
// (tail_tab: the CTA's tail table in shared memory, used when KmerShape<K>::TAIL_TABLE)
template <int K, bool CANON, int J>
__device__ __forceinline__ bool scan_window(const ScanArgs &a, const uint32_t (&b)[KmerShape<K>::BW],
                                            const uint32_t (&rb)[KmerShape<K>::BW], uint64_t tmax, uint32_t pool, const uint64_t *tail_tab,
                                            u64x2 &h_out)
{
    using S = KmerShape<K>;
    u64x2 h;
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
        const uint64_t k1 = tail_tab[tail_index(c[S::NW - 1])];
        h = murmur3_h1<K, S::NA - 2, true>(asc, a.seed, u64x2{(uint32_t)k1, (uint32_t)(k1 >> 32)});
    } else {
        uint32_t asc[S::NA];
        window_ascii<K, CANON, J>(b, rb, pool, asc);
        h = murmur3_h1<K, S::NA>(asc, a.seed);
    }
    if (K <= 16) h.hi = 0;        // 32-bit hashes: |{A,C,G,T}|^k <= 2^32 (reference Sketch.cpp:1136, hash.cpp:31-35)
    // coarse filter on one 32-bit word; validity and the exact threshold are checked in the slow path
    h_out = h;
    return (K <= 16) ? (h.lo <= (uint32_t)tmax) : (h.hi <= (uint32_t)(tmax >> 32));
}

// Filter-word fast path (k > 16): only murmur3_h1_filter's word, to be tested against filter_threshold(tmax >> 32).  b, rb:
// the block's normalised code words (forward from the block's first base, reverse complement ending at its last), so window
// J's forward k-mer starts J bases into b and its reverse complement 16 NB - K - J bases into rb; both offsets are immediates.
template <int K, bool CANON, int J>
__device__ __forceinline__ uint32_t scan_window_filter(const ScanArgs &a, const uint32_t (&b)[CodeShape<K>::NB],
                                                       const uint32_t (&rb)[CodeShape<K>::NB], uint32_t tab)
{
    using C = CodeShape<K>;
    uint32_t f[2], c[2];
    f[0] = block_word<J, C::NB, 2>(b, 0);
    f[1] = block_word<J, C::NB, 2>(b, 1) & C::M1;
    if (CANON) {
        constexpr int RO = 16 * C::NB - K - J;
        const uint32_t r[2] = {block_word<RO, C::NB, 2>(rb, 0), block_word<RO, C::NB, 2>(rb, 1) & C::M1};
        canonical_words(f, r, c);
    } else {
        c[0] = f[0]; c[1] = f[1];
    }
    return scan_mb_extra(a, code_filter_word<K>(a, c, tab));
}

// The 8 windows of a block hashed back to back (independent multiply chains that ptxas can interleave), their pass flags
// at bits 24..31 of the result (bit 24 + j = window j).  No vote and no branch: the hot loop shifts the block's flags into
// the lane's pass mask, and the mask is resolved once per tile (scan_resolve).
template <int K, bool CANON, int... J>
__device__ __forceinline__ uint32_t scan_block_filter(const ScanArgs &a, const uint32_t (&b)[CodeShape<K>::NB], const uint32_t (&rb)[CodeShape<K>::NB],
                                                      uint32_t tf, uint32_t tab, std::integer_sequence<int, J...>)
{
    return (((scan_window_filter<K, CANON, J>(a, b, rb, tab) <= tf ? 1u : 0u) << (24 + J)) | ...);
}

// The lane's pass mask of a warp tile (filter-word kernels): block i = (g - lane) / 32 ends at bits 8 i .. 8 i + 7 after the
// tile's 4 trips.  Block g starts at base 8 g, bits 16 (g & 1) of code word g / 2, and a lane's g all have its parity, so
// one funnel shift per word by a per-lane amount normalises the block to start at bit 0 of b[0] (and its reverse
// complement, which ends at base 1087 - 8 g of the reverse-complement image, to end at the top of rb[NB - 1]).
template <int K, bool CANON>
__device__ __forceinline__ uint32_t scan_tile_filter(const ScanArgs &a, uint32_t c2, uint32_t rc2, uint32_t tab, uint32_t tf)
{
    using C = CodeShape<K>;
    const int lane = threadIdx.x & 31;
    const uint32_t par = 16u * (lane & 1);
    const uint32_t rc_lane = rc2 + 4u * (SCAN_C2_IMAGE - C::NB - (lane & 1));
    uint32_t pmask = 0;
#pragma unroll 1
    for (int g = lane; g < SCAN_WARP_TILE / 8; g += 32) {
        const uint32_t h = (uint32_t)g >> 1;
        uint32_t w[C::NB + 1], b[C::NB], rb[C::NB];
#pragma unroll
        for (int i = 0; i <= C::NB; i++) w[i] = lds_u32(c2 + 4u * (h + i));
#pragma unroll
        for (int i = 0; i < C::NB; i++) b[i] = __funnelshift_r(w[i], w[i + 1], par);
        if (CANON) {
#pragma unroll
            for (int i = 0; i <= C::NB; i++) w[i] = lds_u32(rc_lane - 4u * h + 4u * i);
#pragma unroll
            for (int i = 0; i < C::NB; i++) rb[i] = __funnelshift_r(w[i], w[i + 1], par);
        }
        pmask = (pmask >> 8) | scan_block_filter<K, CANON>(a, b, rb, tf, tab, std::make_integer_sequence<int, 8>());
    }
    return pmask;
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

// Full-hash variant: windows J0 and J0 + 1 hashed back to back, one warp vote, then the survivors of each window serialised by
// scan_emit_warp.  Two windows per vote beat four and eight on H100 (measured on the filter-word kernel before its pass masks,
// DESIGN.md §2.4).
template <int K, bool CANON, int J0>
__device__ __forceinline__ void scan_group(const ScanArgs &a, const uint32_t (&b)[KmerShape<K>::BW], const uint32_t (&rb)[KmerShape<K>::BW],
                                           uint64_t tile_base, uint32_t local0, uint64_t tmax, uint32_t pool, const uint32_t *sm_tile,
                                           const uint64_t *tail_tab)
{
    u64x2 h0, h1;
    const bool p0 = scan_window<K, CANON, J0>(a, b, rb, tmax, pool, tail_tab, h0);
    const bool p1 = scan_window<K, CANON, J0 + 1>(a, b, rb, tmax, pool, tail_tab, h1);
    if (__any_sync(0xFFFFFFFFu, p0 | p1)) {
        if (__any_sync(0xFFFFFFFFu, p0)) scan_emit_warp(a, p0, h0.lo, h0.hi, tile_base, local0 + J0, sm_tile, K, tmax);
        if (__any_sync(0xFFFFFFFFu, p1)) scan_emit_warp(a, p1, h1.lo, h1.hi, tile_base, local0 + J0 + 1, sm_tile, K, tmax);
    }
}

// 4 ASCII bytes -> 4 codes, one per byte: A=0 C=1 G=2 T=3 as ascii4_to_nibbles, anything else 8 | (bits 1-2 of the
// upper-cased byte's ((u >> 1) ^ (u >> 2)), which only the exact rebuild's validity test sees, and it looks at bit 3 alone)
__device__ __forceinline__ uint32_t ascii4_to_codes(uint32_t w, uint32_t fold)
{
    const uint32_t u = w & fold;
    const uint32_t t = (u >> 2) & ~(u >> 1) & 0x01010101u;                    // bit2 & ~bit1: 'T'
    const uint32_t expect = (0x41414141u | (u & 0x06060606u)) ^ (t * 0x11u);  // the ACGT byte with these bits 1,2
    const uint32_t bad = u ^ expect;
    const uint32_t nz = (((bad & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | bad) & 0x80808080u;  // bit7 set where byte != 0
    return (((u >> 1) ^ (u >> 2)) & 0x03030303u) | (nz >> 4);                  // A 0x41, C 0x43, G 0x47, T 0x54 -> 0 1 2 3
}

// 8 ASCII bytes -> one nibble word: the byte codes of both halves, even bytes and odd bytes gathered by two PRMT
__device__ __forceinline__ uint32_t ascii8_to_word(uint32_t lo, uint32_t hi, uint32_t fold)
{
    const uint32_t x0 = ascii4_to_codes(lo, fold), x1 = ascii4_to_codes(hi, fold);
    return __byte_perm(x0, x1, 0x6420) | (__byte_perm(x0, x1, 0x7531) << 4);
}

// 8 ASCII bytes -> one nibble word of the codes ((u >> 1) ^ (u >> 2)) & 3 alone (fold only touches bit 5, so the codes come
// from the raw bytes), and into `diff` the bits in which the upper-cased bytes differ from the ACGT bytes of their codes,
// rebuilt by PRMT from `pool`.  A byte is in the alphabet exactly when it equals the ACGT byte of its own code, so `diff`
// stays 0 exactly when all 8 bytes are, and then the word is what ascii8_to_word gives.
__device__ __forceinline__ uint32_t ascii8_to_code_word(uint32_t lo, uint32_t hi, uint32_t fold, uint32_t pool, uint32_t &diff)
{
    const uint32_t x0 = ((lo >> 1) ^ (lo >> 2)) & 0x03030303u, x1 = ((hi >> 1) ^ (hi >> 2)) & 0x03030303u;
    const uint32_t w = __byte_perm(x0, x1, 0x6420) | (__byte_perm(x0, x1, 0x7531) << 4);
    diff |= (prmt(pool, 0, w) ^ (lo & fold)) | (prmt(pool, 0, w >> 16) ^ (hi & fold));
    return w;
}

// the nibble word of the 8 bytes at stream offset `off`, with the bytes at or past stream_len made separators
__device__ __forceinline__ uint32_t clip_word(uint32_t w, uint64_t off, uint64_t stream_len)
{
    if (off >= stream_len) return 0x88888888u;
    if (off + 8 > stream_len) w |= 0x88888888u << (4 * (uint32_t)(stream_len - off));   // 1..7 bytes kept
    return w;
}

// 4 byte codes (bits 0-1 of each byte) -> one byte of 2-bit codes at bits 24..31: of the products of the multiply by
// 2^24 + 2^18 + 2^12 + 2^6, those that fall below bit 24 land in disjoint 2-bit fields, so nothing carries into bits 24..31
__device__ __forceinline__ uint32_t gather_codes4(uint32_t x) { return x * 0x01041040u; }

// 8 ASCII bytes -> 16 bits of 2-bit codes (the low half of the result; the high half is not zero), the codes of
// ascii8_to_code_word, which also tests the bytes into `diff`
__device__ __forceinline__ uint32_t ascii8_to_codes16(uint32_t lo, uint32_t hi, uint32_t fold, uint32_t pool, uint32_t &diff)
{
    ascii8_to_code_word(lo, hi, fold, pool, diff);
    const uint32_t x0 = ((lo >> 1) ^ (lo >> 2)) & 0x03030303u, x1 = ((hi >> 1) ^ (hi >> 2)) & 0x03030303u;
    return __byte_perm(gather_codes4(x0), gather_codes4(x1), 0x0073);
}

// nibble word (codes 0..3 in bits 0-1 of each nibble, bit 3 = outside the alphabet) -> 16 bits of 2-bit codes / 8 flag bits
__device__ __forceinline__ uint32_t nibbles_to_codes16(uint32_t w)
{
    w &= 0x33333333u;
    w = (w | (w >> 2)) & 0x0F0F0F0Fu;
    w = (w | (w >> 4)) & 0x00FF00FFu;
    return (w | (w >> 8)) & 0xFFFFu;
}
__device__ __forceinline__ uint32_t nibbles_to_flags8(uint32_t w)
{
    w = (w >> 3) & 0x11111111u;
    w = (w | (w >> 3)) & 0x03030303u;
    w = (w | (w >> 6)) & 0x000F000Fu;
    return (w | (w >> 12)) & 0xFFu;
}

__device__ __forceinline__ void sts_u16(uint32_t addr, uint32_t v) { asm volatile("st.shared.u16 [%0], %1;" :: "r"(addr), "h"((unsigned short)v) : "memory"); }
__device__ __forceinline__ void sts_u8(uint32_t addr, uint32_t v) { asm volatile("st.shared.u8 [%0], %1;" :: "r"(addr), "h"((unsigned short)v) : "memory"); }
__device__ __forceinline__ void sts_u32(uint32_t addr, uint32_t v) { asm volatile("st.shared.u32 [%0], %1;" :: "r"(addr), "r"(v) : "memory"); }

// Filter-word kernels, ASCII source: a lane's staged code words -- word lane (w0), word lane + 32 (w1) and halo half-word
// 128 + hw (h, bases 1024 + 8 hw ..) -- and their validity bits (v0, v1: 16 bits, vh: 8 bits) into the forward image, the
// validity bitmap and, canonical, the reverse-complement image (half-word H of the forward image is half-word 135 - H there)
template <bool CANON>
__device__ __forceinline__ void stage_codes(uint32_t c2, uint32_t rc2, uint32_t inv, int lane, int hw, uint32_t w0, uint32_t w1, uint32_t h,
                                            uint32_t v0, uint32_t v1, uint32_t vh)
{
    sts_u32(c2 + 4 * lane, w0);
    sts_u32(c2 + 4 * (lane + 32), w1);
    sts_u16(c2 + 2 * (128 + hw), h);
    sts_u16(inv + 2 * lane, v0);
    sts_u16(inv + 2 * (lane + 32), v1);
    sts_u8(inv + 128 + hw, vh);
    if (CANON) {
        sts_u32(rc2 + 4 * (SCAN_C2_IMAGE - 1 - lane), revcomp16(w0));
        sts_u32(rc2 + 4 * (SCAN_C2_IMAGE - 1 - 32 - lane), revcomp16(w1));
        sts_u16(rc2 + 2 * (2 * SCAN_C2_IMAGE - 1 - 128 - hw), revcomp16(h) >> 16);
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
// filter-word kernels into a per-warp shared landing buffer, which keeps those registers free through the hot loop.
#ifndef SCAN_MIN_BLOCKS
#define SCAN_MIN_BLOCKS 4      // filter-word kernels: resident CTAs per SM requested from ptxas (4 => 64 registers, no spills
                               // since the hot loop holds neither a survivor call nor prefetch registers; 3 => 80 registers, 1 %
                               // slower); tools/scan_microbench.cu compares the settings (-DSCAN_MIN_BLOCKS=n)
#endif
#ifndef SCAN_MIN_BLOCKS_FULL
#define SCAN_MIN_BLOCKS_FULL 3 // FULL kernels (=> 80 registers, no spills; 4 => 64 registers and spills)
#endif
__device__ __forceinline__ void sts_u64(uint32_t addr, uint32_t lo, uint32_t hi)
{
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" :: "r"(addr), "r"(lo), "r"(hi) : "memory");
}

// FULL: the fast path computes the whole 64-bit hash (k <= 16, where the filter is on the low word, and SCAN_SCREEN, where
// every lane probes the reference table with it) from nibble tiles; otherwise only murmur3_h1_filter's word, from 2-bit
// tiles, and the slow path recomputes.
template <int K, bool CANON, bool PACKED, bool FULL>
__global__ void __launch_bounds__(SCAN_THREADS, FULL ? ((K > 24 && SCAN_MIN_BLOCKS_FULL > 3) ? 3 : SCAN_MIN_BLOCKS_FULL) : SCAN_MIN_BLOCKS)
scan_kernel(const __grid_constant__ ScanArgs a)
{
    using S = KmerShape<K>;
    using C = CodeShape<(K > 16 ? K : 17)>;
    static_assert(FULL || K > 16, "the filter word is the high word of the hash");
    constexpr int NWARPS = FULL ? SCAN_WARPS : 1;    // nibble tiles (FULL kernels)
    constexpr int CWARPS = FULL ? 1 : SCAN_WARPS;    // code tiles and landing buffers (filter-word kernels)
    __shared__ __align__(16) uint32_t sm_all[NWARPS][SCAN_WARP_WORDS];
    // reverse-complement image of the tile (word i = nibble-reversed, complemented word NW-1-i), written once at staging so
    // that a block's reverse-complement words are 4 more LDS (the LSU is idle) instead of ~16 ALU instructions per block
    __shared__ __align__(16) uint32_t smr_all[CANON ? NWARPS : 1][SCAN_WARP_WORDS];
    __shared__ __align__(16) uint32_t c2_all[CWARPS][SCAN_C2_WORDS];
    __shared__ __align__(16) uint32_t rc2_all[CANON ? CWARPS : 1][SCAN_C2_WORDS];
    __shared__ __align__(16) uint32_t inv_all[CWARPS][SCAN_INV_WORDS];
    __shared__ __align__(16) uint4 land_all[CWARPS][FULL ? 1 : SCAN_WARP_VECS];   // next tile's raw bytes
    __shared__ __align__(16) uint8_t code_tab[FULL ? 16 : sizeof(CodeTables<(K > 16 ? K : 17)>)];
    __shared__ __align__(16) uint64_t tail_tab[FULL && S::TAIL_TABLE ? TAIL_TAB_SIZE : 1];
    if constexpr (!FULL) {
        fill_code_tables<K>(*reinterpret_cast<CodeTables<K> *>(code_tab));
        __syncthreads();
    } else if constexpr (S::TAIL_TABLE) {
        fill_tail_table<K>(tail_tab);
        __syncthreads();
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint32_t *sm = sm_all[FULL ? warp : 0];
    uint32_t *smr = smr_all[CANON && FULL ? warp : 0];
    // the hot loop and the slow path address the tiles as 32-bit shared-memory addresses, passed through a shuffle (they are
    // warp-uniform) so that ptxas keeps them in registers: it otherwise re-derives them (S2R SR_CgaCtaId, LEA, IMAD) on every
    // iteration of the hot loop to save a register
    const uint32_t sm_addr = __shfl_sync(0xFFFFFFFFu, (uint32_t)__cvta_generic_to_shared(FULL ? sm : c2_all[FULL ? 0 : warp]), 0);
    const uint32_t smr_addr = __shfl_sync(0xFFFFFFFFu, (uint32_t)__cvta_generic_to_shared(FULL ? smr : rc2_all[CANON && !FULL ? warp : 0]), 0);
    const uint32_t inv_addr = (uint32_t)__cvta_generic_to_shared(inv_all[FULL ? 0 : warp]);
    const uint32_t tab_addr = __shfl_sync(0xFFFFFFFFu, (uint32_t)__cvta_generic_to_shared(code_tab), 0);
    const uint32_t land = (uint32_t)__cvta_generic_to_shared(land_all[FULL ? 0 : warp]);
    const uint32_t fold = a.preserve_case ? 0xFFFFFFFFu : 0xDFDFDFDFu;
    // the bytes 'A','C','G','T' for PRMT.  Filter-word kernels: each lane reads the pool back from its own word of the warp's
    // tile (word lane, which only this lane stages later), so that ptxas keeps it in one register for the whole kernel.  A
    // constant, even through a shuffle or %laneid arithmetic, is rebuilt before every PRMT instead (an IMAD.U32 each).  The
    // FULL kernels keep the constant.
    uint32_t pool;
    if (FULL) {
        asm volatile("mov.u32 %0, 0x54474341;" : "=r"(pool));
    } else {
        const uint32_t at = sm_addr + 4u * lane;
        asm volatile("st.shared.u32 [%0], %1;" :: "r"(at), "r"(0x54474341u) : "memory");
        asm volatile("ld.volatile.shared.u32 %0, [%1];" : "=r"(pool) : "r"(at) : "memory");
    }

    const uint64_t wt_begin = a.tile_begin * (SCAN_TILE / SCAN_WARP_TILE);
    const uint64_t wt_end = a.tile_end * (SCAN_TILE / SCAN_WARP_TILE);
    const uint64_t wt_stride = (uint64_t)gridDim.x * SCAN_WARPS;
    uint64_t wt = wt_begin + (uint64_t)blockIdx.x * SCAN_WARPS + warp;
    if (wt >= wt_end) return;

    // FULL kernels: each lane stages vectors lane, lane+32 and one of the 4 halo vectors (64 + lane%4: eight lanes write the
    // same words with the same values -- no lane-dependent branch, the warp never splits): 16 bytes -> 2 words each.
    // Filter-word kernels: vectors lane and lane+32 (16 bytes -> one code word), and halo half-word 128 + lane%8 (8 bytes ->
    // 16 bits, four lanes alike).
    static_assert(SCAN_WARP_VECS - 64 == 4 && SCAN_HALO_WORDS == 8, "halo = 4 vectors = 8 words");
    const int v2 = 64 + (lane & 3);
    const int hw = lane & 7;
    uint4 q0, q1, q2;                      // ASCII source: three 16-byte vectors per lane
    uint64_t pc0 = 0, pc1 = 0;             // packed source: group (lane) and one of the 2 halo groups (32 + lane%2)
    uint32_t pm0 = 0, pm1 = 0;
    const int hg = 32 + (lane & 1);
    if constexpr (!FULL) {
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
        if (!FULL && !(SCAN_MB_STAGE_ONCE && wt != wt_first)) {   // this tile's bytes, copied in during the previous tile
            cp_async_wait_all();
            __syncwarp();
            if (PACKED) {
                pc0 = lds_u64(land + 8 * lane); pm0 = lds_u32(land + SCAN_LAND_INVAL + 4 * lane);
                pc1 = lds_u64(land + 8 * hg);   pm1 = lds_u32(land + SCAN_LAND_INVAL + 4 * hg);
            } else {
                q0 = lds_u128(land + 16 * lane);
                q1 = lds_u128(land + 16 * (lane + 32));
                const uint64_t h = lds_u64(land + 16 * 64 + 8 * hw);
                q2 = make_uint4((uint32_t)h, (uint32_t)(h >> 32), 0u, 0u);
            }
        }
        if (SCAN_MB_STAGE_ONCE && wt != wt_first) {
            // microbenchmark only: hash the first tile again
        } else if (PACKED && !FULL) {
            // the packed words are the code images' words as they stand: group g is code words 2g, 2g + 1 and validity word g
            sts_u64(sm_addr + 8 * lane, (uint32_t)pc0, (uint32_t)(pc0 >> 32));
            sts_u64(sm_addr + 8 * hg, (uint32_t)pc1, (uint32_t)(pc1 >> 32));
            sts_u32(inv_addr + 4 * lane, pm0);
            sts_u32(inv_addr + 4 * hg, pm1);
            if (CANON) {
                sts_u64(smr_addr + 4 * (SCAN_C2_IMAGE - 2 - 2 * lane), revcomp16((uint32_t)(pc0 >> 32)), revcomp16((uint32_t)pc0));
                sts_u64(smr_addr + 4 * (SCAN_C2_IMAGE - 2 - 2 * hg), revcomp16((uint32_t)(pc1 >> 32)), revcomp16((uint32_t)pc1));
            }
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
        } else if constexpr (!FULL) {
            // A tile of ACGT bytes alone (upper-cased unless preserve_case), halo included, is converted to codes only and
            // checked with one vote.  A tile with any other byte (N, IUPAC codes, a record separator, lower case under
            // preserve_case) is converted again with the validity test, as is the last tile of a launch, which reaches
            // past stream_len (warp-uniform); bit 3 of a nibble marks a base outside the alphabet as before.
            const bool ragged = base + 16ull * SCAN_WARP_VECS > a.stream_len;
            uint32_t w0, w1, h, v0 = 0, v1 = 0, vh = 0, diff = 0;
            if (!ragged) {
                w0 = __byte_perm(ascii8_to_codes16(q0.x, q0.y, fold, pool, diff), ascii8_to_codes16(q0.z, q0.w, fold, pool, diff), 0x5410);
                w1 = __byte_perm(ascii8_to_codes16(q1.x, q1.y, fold, pool, diff), ascii8_to_codes16(q1.z, q1.w, fold, pool, diff), 0x5410);
                h = ascii8_to_codes16(q2.x, q2.y, fold, pool, diff);
            }
            if (ragged || __any_sync(0xFFFFFFFFu, diff != 0)) {
                uint32_t n0 = ascii8_to_word(q0.x, q0.y, fold), n1 = ascii8_to_word(q0.z, q0.w, fold);
                uint32_t n2 = ascii8_to_word(q1.x, q1.y, fold), n3 = ascii8_to_word(q1.z, q1.w, fold);
                uint32_t n4 = ascii8_to_word(q2.x, q2.y, fold);
                if (ragged) {
                    const uint64_t o0 = base + 16ull * lane, o1 = o0 + 16ull * 32;
                    n0 = clip_word(n0, o0, a.stream_len);
                    n1 = clip_word(n1, o0 + 8, a.stream_len);
                    n2 = clip_word(n2, o1, a.stream_len);
                    n3 = clip_word(n3, o1 + 8, a.stream_len);
                    n4 = clip_word(n4, base + 16ull * 64 + 8ull * hw, a.stream_len);
                }
                w0 = nibbles_to_codes16(n0) | (nibbles_to_codes16(n1) << 16);
                w1 = nibbles_to_codes16(n2) | (nibbles_to_codes16(n3) << 16);
                h = nibbles_to_codes16(n4);
                v0 = nibbles_to_flags8(n0) | (nibbles_to_flags8(n1) << 8);
                v1 = nibbles_to_flags8(n2) | (nibbles_to_flags8(n3) << 8);
                vh = nibbles_to_flags8(n4);
            }
            stage_codes<CANON>(sm_addr, smr_addr, inv_addr, lane, hw, w0, w1, h, v0, v1, vh);
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
            if constexpr (!FULL) {
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
        if constexpr (!FULL) pmask = scan_tile_filter<K, CANON>(a, sm_addr, smr_addr, tab_addr, tf);
        else
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
            scan_group<K, CANON, 0>(a, b, rb, base, local0, tmax, pool, sm, tail_tab);
            scan_group<K, CANON, 2>(a, b, rb, base, local0, tmax, pool, sm, tail_tab);
            scan_group<K, CANON, 4>(a, b, rb, base, local0, tmax, pool, sm, tail_tab);
            scan_group<K, CANON, 6>(a, b, rb, base, local0, tmax, pool, sm, tail_tab);
        }
        if (SCAN_MB_CLOCK) mb_cycles += clock64() - c0;
        if constexpr (!FULL) {
            if (SCAN_MB_NO_SURVIVORS) mb_acc ^= pmask;
            else if (__any_sync(0xFFFFFFFFu, pmask != 0)) scan_resolve<K, CANON>(a, pmask, sm_addr, smr_addr, inv_addr, base, tmax);
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
