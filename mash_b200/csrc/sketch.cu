// sketch.cu -- hot path 1: batched bottom-s sketching on the GPU (C-ABI: mashgpu_sketch_*, mashgpu_hash_windows).
//
// Pipeline per batch (see DESIGN.md):
//   flat byte stream in HBM  ->  scan_kernel (scan.cuh): hash every valid canonical k-mer, keep hash <= T_unit
//   in the unit's open-addressing table (distinct keys + multiplicities)  ->  select_kernel: compact the table,
//   sort, emit the s smallest.  This replaces MinHashHeap::tryInsert / HashSet::toHashList
//   (reference MinHashHeap.cpp:68-146, HashSet.cpp:78-118): bottom-s of a set does not depend on insertion order.
//   T_unit is chosen so that ~SURVIVOR_FACTOR*s distinct hashes are expected; a unit that ends with fewer than s
//   distinct survivors (while k-mers were dropped) or overflows its table is re-run exactly with a larger T.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_segmented_radix_sort.cuh>

#include "common.cuh"
#include "scan.cuh"
#include "sketch_core.cuh"
#include "pack.h"
#include <chrono>
#include <condition_variable>
#include <future>
#include <mutex>
#include <thread>
#include <cstdlib>
#include <memory>

namespace mashgpu {

scan_launch_fn get_scan_launcher_part0(int, bool, bool);
scan_launch_fn get_scan_launcher_part1(int, bool, bool);
scan_launch_fn get_scan_launcher_part2(int, bool, bool);
scan_launch_fn get_scan_launcher_part3(int, bool, bool);

scan_launch_fn get_bytes_launcher_part0(int);
scan_launch_fn get_bytes_launcher_part1(int);
scan_launch_fn get_bytes_launcher_part2(int);
scan_launch_fn get_bytes_launcher_part3(int);

scan_launch_fn get_bytes_launcher(int k)
{
    if (auto f = get_bytes_launcher_part0(k)) return f;
    if (auto f = get_bytes_launcher_part1(k)) return f;
    if (auto f = get_bytes_launcher_part2(k)) return f;
    return get_bytes_launcher_part3(k);
}

scan_launch_fn get_scan_launcher(int k, bool canonical, bool packed)
{
    if (auto f = get_scan_launcher_part0(k, canonical, packed)) return f;
    if (auto f = get_scan_launcher_part1(k, canonical, packed)) return f;
    if (auto f = get_scan_launcher_part2(k, canonical, packed)) return f;
    return get_scan_launcher_part3(k, canonical, packed);
}

constexpr double SURVIVOR_FACTOR = 3.0;   // expected distinct survivors = 3 s
constexpr double TABLE_SLACK = 2.7;       // table slots per expected survivor
constexpr uint32_t SEL_MAX_LOG2 = 14;     // select_kernel sorts up to 2^14 keys in shared memory (128 KB)
constexpr int SEL_THREADS = 256;

// ---------------------------------------------------------------------------------------------------------
// per-tile coarse threshold: max T over the units a tile touches; and (tile_unit != NULL) the tile's first unit, from which
// the scan's slow path finds a survivor's unit with a short forward scan
// ---------------------------------------------------------------------------------------------------------
__global__ void tile_tmax_kernel(const uint64_t *unit_start, uint32_t n_units, const uint64_t *unit_t,
                                 uint64_t stream_len, int k, uint64_t tile_begin, uint64_t tile_end, uint64_t *tile_tmax,
                                 uint32_t *tile_unit)
{
    uint64_t tile = tile_begin + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (tile >= tile_end) return;
    uint64_t first = tile * (uint64_t)SCAN_TILE;
    uint64_t last = first + SCAN_TILE - 1;
    if (last >= stream_len) last = stream_len ? stream_len - 1 : 0;
    uint32_t lo = 0, hi = n_units;
    while (hi - lo > 1) { uint32_t mid = (lo + hi) >> 1; if (unit_start[mid] <= first) lo = mid; else hi = mid; }
    uint64_t t = 0;
    for (uint32_t u = lo; u < n_units && unit_start[u] <= last; u++) t = max(t, unit_t[u]);
    tile_tmax[tile] = t;
    if (tile_unit) tile_unit[tile] = lo;
}

// ---------------------------------------------------------------------------------------------------------
// select: table -> ascending bottom-s (+ counts)
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t table_count(const uint64_t *keys, const uint32_t *cnt, uint32_t log2cap, uint64_t key)
{
    const uint32_t mask = (1u << log2cap) - 1;
    uint32_t slot = slot_hash(key, log2cap);
    for (;;) {
        uint64_t k = keys[slot];
        if (k == key) return cnt[slot];
        if (k == EMPTY_KEY) return 0;
        slot = (slot + 1) & mask;
    }
}

// One CTA per unit; tables up to 2^SEL_MAX_LOG2 slots.  flags bit1 = fewer than s distinct survivors although
// k-mers were filtered (unit_t != max); units whose table is too large for shared memory are left to the batched
// segmented sort below (large sketch sizes: `-s 10000` needs ~2^17 candidate slots per unit).
__global__ void __launch_bounds__(SEL_THREADS) select_kernel(
    uint32_t unit_begin, uint32_t n_units, const uint64_t *unit_t, const uint64_t *tab_off, const uint32_t *tab_log2,
    const uint64_t *tab_keys, const uint32_t *tab_cnt, const uint32_t *unit_maxhash, uint32_t *unit_flags,
    uint32_t s, uint64_t capped_t, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint32_t min_copies)
{
    extern __shared__ uint64_t sk[];
    __shared__ uint32_t n_s;
    const uint32_t u = unit_begin + blockIdx.x;
    if (u >= unit_begin + n_units) return;
    const uint32_t log2cap = tab_log2[u];
    if (unit_flags[u] & 1u) return;                    // overflowed: will be re-run
    if (log2cap > SEL_MAX_LOG2) return;              // tables beyond the shared-memory sort: batched segmented sort (select_big_*)
    const uint32_t cap = 1u << log2cap;
    const uint64_t *keys = tab_keys + tab_off[u];
    const uint32_t *cnt = tab_cnt + tab_off[u];
    if (threadIdx.x == 0) n_s = 0;
    __syncthreads();
    for (uint32_t i = threadIdx.x; i < cap; i += SEL_THREADS) {
        uint64_t k = keys[i];
        if (k != EMPTY_KEY && cnt[i] >= min_copies) sk[atomicAdd(&n_s, 1u)] = k;      // `-m`: only hashes seen at least m times qualify
    }
    __syncthreads();
    const uint32_t n = n_s;
    uint32_t N = 2;
    while (N < n) N <<= 1;
    for (uint32_t i = n + threadIdx.x; i < N; i += SEL_THREADS) sk[i] = EMPTY_KEY;
    __syncthreads();
    for (uint32_t size = 2; size <= N; size <<= 1) {
        for (uint32_t stride = size >> 1; stride > 0; stride >>= 1) {
            for (uint32_t t = threadIdx.x; t < N / 2; t += SEL_THREADS) {
                uint32_t lo = 2 * t - (t & (stride - 1));
                uint32_t hi = lo + stride;
                bool up = (lo & size) == 0;
                uint64_t a = sk[lo], b = sk[hi];
                if ((a > b) == up) { sk[lo] = b; sk[hi] = a; }
            }
            __syncthreads();
        }
    }
    const uint32_t n_max = (unit_maxhash[u] && unit_maxhash[u] >= min_copies) ? 1u : 0u;          // the value 2^64-1 itself, largest possible
    const uint32_t total = n + n_max;
    const uint32_t m = total < s ? total : s;
    if (threadIdx.x == 0) {
        out_n[u] = m;
        // too few survivors although k-mers were dropped -- unless the threshold is the caller's cap (screen: the
        // running s-th smallest of the mixture; nothing above it can enter the bottom-s)
        if (total < s && unit_t[u] != EMPTY_KEY && unit_t[u] != capped_t) atomicOr(&unit_flags[u], 2u);
    }
    for (uint32_t i = threadIdx.x; i < m; i += SEL_THREADS) {
        uint64_t key = i < n ? sk[i] : EMPTY_KEY;
        out_hashes[(uint64_t)u * s + i] = key;
        if (out_counts) out_counts[(uint64_t)u * s + i] = i < n ? table_count(keys, cnt, log2cap, key) : unit_maxhash[u];
    }
}

// ---- big tables: compact the qualifying keys of every big unit into one buffer (segment b = unit big_units[b]), sort all
// segments with one segmented radix sort, emit the first s of each.  Same outputs and flags as select_kernel.
__global__ void select_big_compact_kernel(const uint32_t *big_units, uint32_t n_big, const uint64_t *seg_off, const uint64_t *tab_off, const uint32_t *tab_log2,
                                          const uint64_t *tab_keys, const uint32_t *tab_cnt, const uint32_t *unit_flags, uint32_t min_copies,
                                          uint64_t *comp, uint32_t *seg_n)
{
    const uint32_t b = blockIdx.y;
    if (b >= n_big) return;
    const uint32_t u = big_units[b];
    if (unit_flags[u] & 1u) return;                    // overflowed: will be re-run
    const uint64_t cap = 1ull << tab_log2[u];
    const uint64_t *keys = tab_keys + tab_off[u];
    const uint32_t *cnt = tab_cnt + tab_off[u];
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < cap; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t k = keys[i];
        if (k != EMPTY_KEY && cnt[i] >= min_copies) comp[seg_off[b] + atomicAdd(&seg_n[b], 1u)] = k;
    }
}

__global__ void select_big_bounds_kernel(const uint64_t *seg_off, const uint32_t *seg_n, uint32_t n_big, long long *seg_begin, long long *seg_end)
{
    const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= n_big) return;
    seg_begin[b] = (long long)seg_off[b];
    seg_end[b] = (long long)(seg_off[b] + seg_n[b]);
}

__global__ void __launch_bounds__(SEL_THREADS) select_big_emit_kernel(
    const uint32_t *big_units, uint32_t n_big, const uint64_t *seg_off, const uint32_t *seg_n, const uint64_t *sorted,
    const uint64_t *unit_t, const uint64_t *tab_off, const uint32_t *tab_log2, const uint64_t *tab_keys, const uint32_t *tab_cnt,
    const uint32_t *unit_maxhash, uint32_t *unit_flags, uint32_t s, uint64_t capped_t, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n,
    uint32_t min_copies)
{
    const uint32_t b = blockIdx.x;
    if (b >= n_big) return;
    const uint32_t u = big_units[b];
    if (unit_flags[u] & 1u) return;
    const uint32_t n = seg_n[b];
    const uint32_t n_max = (unit_maxhash[u] && unit_maxhash[u] >= min_copies) ? 1u : 0u;
    const uint64_t total = (uint64_t)n + n_max;
    const uint32_t m = (uint32_t)(total < s ? total : s);
    if (threadIdx.x == 0) {
        out_n[u] = m;
        if (total < s && unit_t[u] != EMPTY_KEY && unit_t[u] != capped_t) atomicOr(&unit_flags[u], 2u);
    }
    const uint64_t *keys = tab_keys + tab_off[u];
    const uint32_t *cnt = tab_cnt + tab_off[u];
    for (uint32_t i = threadIdx.x; i < m; i += SEL_THREADS) {
        const uint64_t key = i < n ? sorted[seg_off[b] + i] : EMPTY_KEY;
        out_hashes[(uint64_t)u * s + i] = key;
        if (out_counts) out_counts[(uint64_t)u * s + i] = i < n ? table_count(keys, cnt, tab_log2[u], key) : unit_maxhash[u];
    }
}

__device__ __forceinline__ int64_t table_find(const uint64_t *keys, uint32_t log2cap, uint64_t key)
{
    const uint32_t mask = (1u << log2cap) - 1;
    uint32_t slot = slot_hash(key, log2cap);
    for (;;) {
        uint64_t k = keys[slot];
        if (k == key) return slot;
        if (k == EMPTY_KEY) return -1;
        slot = (slot + 1) & mask;
    }
}

// Multiplicity counts, the reference's way.  MinHashHeap::tryInsert (MinHashHeap.cpp:68-74) only accepts a hash when
// the heap is not full or the hash is strictly below the current top, so once all s final hashes have been seen
// (stream position t* = the latest first occurrence among them) further occurrences of the largest final hash are
// neither inserted nor counted; every other count is the true multiplicity (SURVEY.md 8 a5).
// One CTA per full sketch: t* by max-reduction, then count[last] = occurrences of the largest hash at positions <= t*:
// equal to the table count if its last occurrence is <= t*, 1 if it was the last hash to arrive, otherwise the unit
// is flagged (bit 3) for a targeted recount over [unit start, t*].
__global__ void __launch_bounds__(SEL_THREADS) quirk_kernel(
    uint32_t unit_begin, uint32_t n_units, uint32_t s, const uint64_t *out_hashes, uint32_t *out_counts, const uint32_t *out_n,
    const uint64_t *tab_off, const uint32_t *tab_log2, const uint64_t *tab_keys, const uint32_t *tab_cnt,
    const uint64_t *tab_first, const uint64_t *tab_last, uint32_t *unit_flags, uint64_t *quirk_target, uint64_t *quirk_tstar, uint32_t m)
{
    // m = multiplicityMinimum: a hash is promoted into the heap at its m-th occurrence (tab_first level m-1) holding count m
    __shared__ unsigned long long tstar_s;
    const uint32_t u = unit_begin + blockIdx.x;
    if (u >= unit_begin + n_units) return;
    if (unit_flags[u] & 7u) return;                 // will be re-run
    if (out_n[u] < s) return;                       // heap never full: every count is exact
    const uint64_t *keys = tab_keys + tab_off[u];
    const uint32_t lg = tab_log2[u];
    if (threadIdx.x == 0) tstar_s = 0;
    __syncthreads();
    unsigned long long local = 0;
    for (uint32_t i = threadIdx.x; i < s; i += SEL_THREADS) {
        int64_t slot = table_find(keys, lg, out_hashes[(uint64_t)u * s + i]);
        if (slot >= 0) local = max(local, (unsigned long long)tab_first[(tab_off[u] + slot) * m + (m - 1)]);
    }
    atomicMax(&tstar_s, local);
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint64_t tstar = tstar_s;
        const uint64_t key = out_hashes[(uint64_t)u * s + s - 1];
        int64_t slot = table_find(keys, lg, key);
        if (slot >= 0) {
            const uint32_t c = tab_cnt[tab_off[u] + slot];
            const uint64_t f = tab_first[(tab_off[u] + slot) * m + (m - 1)], l = tab_last[tab_off[u] + slot];
            if (c > m && l > tstar) {
                if (f == tstar) out_counts[(uint64_t)u * s + s - 1] = m;
                else { quirk_target[u] = key; quirk_tstar[u] = tstar; atomicOr(&unit_flags[u], 8u); }
            }
        }
    }
}

// Large tables: compact non-empty keys to scratch (then cub radix sort on the host side of this file).
__global__ void compact_table_kernel(const uint64_t *keys, const uint32_t *cnt, uint32_t min_copies, uint64_t cap, uint64_t *out, unsigned long long *out_n)
{
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (i >= cap) return;
    uint64_t k = keys[i];
    if (k != EMPTY_KEY && cnt[i] >= min_copies) out[atomicAdd(out_n, 1ull)] = k;
}

// Packed source: expand the host's list of invalid runs into the 1-bit-per-position mask.  One warp per run; runs
// are disjoint, so interior words are plain stores and only the two edge words need atomics.
// record separators of the directly copied records of a wave (one launch instead of one 1-byte memset per record)
__global__ void write_separators_kernel(uint8_t *stream, const uint64_t *offsets, uint32_t n)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t < n) stream[offsets[t]] = 0;
}

__global__ void apply_runs_kernel(const PackRun *runs, uint64_t n_runs, uint32_t *mask)
{
    const uint64_t warp = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5, n_warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    const int lane = threadIdx.x & 31;
    for (uint64_t r = warp; r < n_runs; r += n_warps) {
        const uint64_t start = runs[r].start, end = start + runs[r].len;      // [start, end)
        if (end == start) continue;
        const uint64_t w0 = start >> 5, w1 = (end - 1) >> 5;
        const uint32_t first = 0xFFFFFFFFu << (start & 31), last = 0xFFFFFFFFu >> (31 - ((end - 1) & 31));
        if (w0 == w1) { if (lane == 0) atomicOr(&mask[w0], first & last); continue; }
        if (lane == 0) atomicOr(&mask[w0], first);
        if (lane == 1) atomicOr(&mask[w1], last);
        for (uint64_t w = w0 + 1 + lane; w < w1; w += 32) mask[w] = 0xFFFFFFFFu;
    }
}

// The bottom-m of a single-unit pass, ascending, each hash with its count and (first != NULL) its promoting occurrence (level mc-1)
// and its last occurrence, positions + base.  Entry n_sorted, when m > n_sorted, is the hash 2^64-1, which the table cannot hold: its
// side count, positions at the unit's start.
__global__ void unit_emit_kernel(const uint64_t *sorted, uint32_t n_sorted, uint32_t m, const uint64_t *keys, const uint32_t *cnt,
                                 const uint64_t *first, const uint64_t *last, uint32_t log2cap, uint32_t mc, uint32_t maxhash_cnt,
                                 uint64_t start, uint64_t base, uint64_t *c_key, uint32_t *c_cnt, uint64_t *c_first, uint64_t *c_last)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= m) return;
    if (i == n_sorted) {
        c_key[i] = EMPTY_KEY;
        c_cnt[i] = maxhash_cnt;
        if (first) c_first[i] = c_last[i] = base + start;
        return;
    }
    const uint64_t key = sorted[i];
    const int64_t slot = table_find(keys, log2cap, key);
    c_key[i] = key;
    c_cnt[i] = cnt[slot];
    if (first) {
        c_first[i] = base + first[slot * mc + mc - 1];
        c_last[i] = base + last[slot];
    }
}

// ---------------------------------------------------------------------------------------------------------
// host side
// ---------------------------------------------------------------------------------------------------------
int validate_sketch_params(mashgpu_ctx *ctx, const mashgpu_sketch_params *p, bool reads)
{
    if (!p) return fail(ctx, MASHGPU_ERR_INVALID, "params is NULL");
    if (p->kmer_size < 1 || p->kmer_size > 32) return fail(ctx, MASHGPU_ERR_INVALID, "kmer_size %d outside 1..32", p->kmer_size);
    if (p->sketch_size < 1) return fail(ctx, MASHGPU_ERR_INVALID, "sketch_size must be >= 1");
    int n = 0;
    for (int i = 0; i < 256; i++) n += p->alphabet[i] != 0;
    bool dna = n == 4 && p->alphabet['A'] && p->alphabet['C'] && p->alphabet['G'] && p->alphabet['T'];
    if (n == 0) return fail(ctx, MASHGPU_ERR_INVALID, "empty alphabet");
    if ((p->use64 != 0) != (std::pow((double)n, (double)p->kmer_size) > std::pow(2.0, 32.0)))
        return fail(ctx, MASHGPU_ERR_INVALID, "use64=%d contradicts the reference rule alphabetSize^k > 2^32 for k=%d, %d letters (Sketch.cpp:1136)", p->use64, p->kmer_size, n);
    if (p->alphabet[0]) return fail(ctx, MASHGPU_ERR_INVALID, "byte 0 cannot be an alphabet letter");
    if (p->min_copies > 255) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "min_copies (-m) above 255");
    if (p->bloom_bytes && !reads) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "bloom_bytes (-b) only applies to reads mode (mashgpu_reads_*, mashgpu_sketch_reads)");
    if (!dna && !p->noncanonical)
        return fail(ctx, MASHGPU_ERR_UNSUPPORTED,
                    "canonical k-mers are only defined for the alphabet {A,C,G,T}; other alphabets must be non-canonical "
                    "(the reference forces -n for -a / -z, sketchParameterSetup.cpp:79-95)");
    return MASHGPU_OK;
}

bool is_dna_alphabet(const mashgpu_sketch_params *p)
{
    int n = 0;
    for (int i = 0; i < 256; i++) n += p->alphabet[i] != 0;
    return n == 4 && p->alphabet['A'] && p->alphabet['C'] && p->alphabet['G'] && p->alphabet['T'];
}

static double kmer_space_of(const mashgpu_sketch_params *p)
{
    int n = 0;
    for (int i = 0; i < 256; i++) n += p->alphabet[i] != 0;
    return std::pow((double)n, (double)p->kmer_size);
}

// Threshold / table geometry of one unit. factor = expected-survivor multiple of s (<= 0: keep everything).
void plan_unit(const mashgpu_sketch_params *p, uint64_t span, double factor, uint64_t *t_out, uint32_t *log2_out)
{
    const double hash_space = p->use64 ? 18446744073709551616.0 : 4294967296.0;
    double kspace = kmer_space_of(p);
    double distinct_max = std::min((double)span, kspace);          // upper bound on distinct hashes
    double expect = factor * (double)p->sketch_size;
    if (factor <= 0 || expect >= (double)span * 0.5 || expect >= kspace * 0.25) {
        *t_out = EMPTY_KEY;                                            // keep all
        *log2_out = std::max(4u, ceil_log2((uint64_t)(2.0 * distinct_max) + 2));
        return;
    }
    double frac = expect / (double)span;
    double t = frac * hash_space;
    *t_out = t >= 18446744073709549568.0 ? (EMPTY_KEY - 1) : (uint64_t)t;
    *log2_out = std::max(4u, ceil_log2((uint64_t)(TABLE_SLACK * expect) + 2));
}

// The fields every pass over a stream shares: its source (ASCII, or packed codes and mask), its length and tiles, the hashing
// parameters; one unit, none skipped, no `-m`.
static ScanArgs scan_base(const mashgpu_sketch_params *p, const void *stream, uint64_t stream_len, const uint64_t *codes = nullptr,
                          const uint32_t *inval = nullptr)
{
    ScanArgs a;
    memset(&a, 0, sizeof a);
    a.stream = (const uint8_t *)stream;
    a.codes = codes;
    a.inval = inval;
    a.stream_len = stream_len;
    a.tile_end = (stream_len + SCAN_TILE - 1) / SCAN_TILE;
    a.seed = p->seed;
    a.use64 = p->use64;
    a.preserve_case = p->preserve_case;
    for (int b = 0; b < 256; b++) {
        int u = (!p->preserve_case && b > 96 && b < 123) ? b - 32 : b;     // reference Sketch.cpp:524-530
        a.byte_lut[b] = p->alphabet[u] ? (uint8_t)u : 0;
    }
    a.n_units = 1;
    a.only_unit = -1;
    a.min_copies = 1;
    return a;
}

// A job's device allocation: `bytes` follows what the job holds, `peak` its largest value.
template <typename T>
static bool tracked_alloc(DevBuf<T> &b, size_t n, uint64_t &bytes, uint64_t &peak)
{
    const size_t before = b.n * sizeof(T);
    if (b.alloc(n) != cudaSuccess) return false;
    bytes += n * sizeof(T);
    bytes -= before;
    peak = std::max(peak, bytes);
    return true;
}

static int launch_scan(mashgpu_ctx *ctx, const mashgpu_sketch_params *p, const ScanArgs &a, cudaStream_t st)
{
    const bool dna = is_dna_alphabet(p);
    if (!dna && !a.stream) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "the packed source only carries the alphabet {A,C,G,T}");
    scan_launch_fn fn = dna ? get_scan_launcher(p->kmer_size, !p->noncanonical, a.codes != nullptr) : get_bytes_launcher(p->kmer_size);
    if (!fn) return fail(ctx, MASHGPU_ERR_INVALID, "no scan kernel for k=%d", p->kmer_size);
    uint64_t ntiles = a.tile_end - a.tile_begin;
    if (ntiles == 0) return MASHGPU_OK;
    time_begin(ctx, ctx->scan_events, st);
    fn(a, 0, st);     // grid = resident CTAs (persistent warps striding over warp tiles)
    time_end(ctx, ctx->scan_events, st);
    ctx->kernel_launches++;
    ctx->scan_launches++;
    MG_CUDA(ctx, cudaGetLastError());
    return MASHGPU_OK;
}

// Occurrences of `target` at stream positions [lo, hi] -> d_count_slot (one uint32 in device memory)
static int recount_hash(mashgpu_ctx *ctx, const mashgpu_sketch_params *p, const ScanArgs &base, uint64_t lo, uint64_t hi, uint64_t target,
                        uint32_t *d_count_slot, cudaStream_t st)
{
    ScanArgs c = base;
    c.mode = SCAN_COUNT;
    c.tile_begin = lo / SCAN_TILE;
    c.tile_end = hi / SCAN_TILE + 1;
    c.tile_tmax = nullptr;
    c.tile_unit = nullptr;      // the first pass's per-tile buffers are not kept
    c.coarse_t = target;
    c.count_target = target; c.count_lo = lo; c.count_hi = hi; c.count_out = d_count_slot;
    MG_CUDA(ctx, cudaMemsetAsync(d_count_slot, 0, 4, st));
    return launch_scan(ctx, p, c, st);
}

// One unit sketched alone and exactly in a global-memory candidate table (DESIGN.md 2.3): the exact re-run of a flagged unit, and
// each stage of a unit job (2.7).  The owner sets the stream (`base`: its source and unit lookup), the unit (index u, stream
// positions [lo, hi)) and pos_base, which is added to every position the pass reports.  Buffers only grow; their bytes are counted
// in the owner's counters.
struct UnitPass {
    mashgpu_ctx *ctx = nullptr;
    const mashgpu_sketch_params *p = nullptr;
    cudaStream_t st = nullptr;
    uint64_t *bytes = nullptr, *peak = nullptr;
    bool positions = false;             // keep the first / last positions of every key (counts)
    uint32_t mc = 1;                    // `-m`: mc first positions per key; candidates need cnt >= mc
    ScanArgs base;
    uint32_t u = 0;
    uint64_t lo = 0, hi = 0, pos_base = 0;
    // the last scan: survivor factor, threshold (clamped to cap_t, above which nothing can enter), table size, scans of this unit
    double factor = 0;
    uint64_t t = 0, cap_t = EMPTY_KEY;
    uint32_t lg = 0, lg_cap = 0, scans = 0;
    DevBuf<uint64_t> keys, first, last, comp, sorted, c_key, c_first, c_last, meta;   // meta: [threshold, table offset 0]
    DevBuf<uint32_t> cnt, c_cnt, small;                                               // small: [log2, flags, maxhash, recount]
    DevBuf<unsigned long long> d_n;
    DevBuf<uint8_t> sort_tmp;
    size_t sort_tmp_bytes = 0;
    // the bottom-s of the last finish(): hash, count, promoting and last position
    std::vector<uint64_t> h_key, h_first, h_last;
    std::vector<uint32_t> h_cnt;

    template <typename T>
    bool alloc(DevBuf<T> &b, size_t n) { return tracked_alloc(b, n, *bytes, *peak); }

    int open(mashgpu_ctx *ctx_, const mashgpu_sketch_params *p_, cudaStream_t st_, bool positions_, uint64_t *bytes_, uint64_t *peak_)
    {
        ctx = ctx_; p = p_; st = st_; positions = positions_; bytes = bytes_; peak = peak_;
        mc = std::max(1u, p->min_copies);
        const uint32_t s = p->sketch_size;
        if (!alloc(meta, 2) || !alloc(small, 4) || !alloc(d_n, 1) || !alloc(c_key, s) || !alloc(c_cnt, s) ||
            (positions && (!alloc(c_first, s) || !alloc(c_last, s))))
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (single-unit pass)");
        return MASHGPU_OK;
    }

    // Table, compaction and sort buffers for 2^l slots.
    int reserve(uint32_t l)
    {
        if (l <= lg_cap) return MASHGPU_OK;
        const uint64_t cap = 1ull << l;
        size_t tmp = 0;
        cub::DeviceRadixSort::SortKeys(nullptr, tmp, (uint64_t *)nullptr, (uint64_t *)nullptr, (int)std::min<uint64_t>(cap, 0x7FFFFFFF), 0, 64, st);
        if (!alloc(keys, cap) || !alloc(cnt, cap) || (positions && (!alloc(first, cap * mc) || !alloc(last, cap))) || !alloc(comp, cap) ||
            !alloc(sorted, cap) || !alloc(sort_tmp, tmp))
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (single-unit table of %llu slots)", (unsigned long long)cap);
        sort_tmp_bytes = tmp;
        lg_cap = l;
        return MASHGPU_OK;
    }

    // Plan the threshold for f x s expected survivors, clamp it to `cap`, clear the table and enqueue the scan of the unit.
    int scan(double f, uint64_t cap)
    {
        factor = f;
        cap_t = cap;
        plan_unit(p, hi - lo, factor, &t, &lg);
        t = std::min(t, cap_t);
        MG_TRY(reserve(lg));
        const uint64_t n = 1ull << lg;
        MG_CUDA(ctx, cudaMemsetAsync(keys.p, 0xFF, n * 8, st));
        MG_CUDA(ctx, cudaMemsetAsync(cnt.p, 0, n * 4, st));
        if (positions) {
            MG_CUDA(ctx, cudaMemsetAsync(first.p, 0xFF, n * mc * 8, st));
            MG_CUDA(ctx, cudaMemsetAsync(last.p, 0, n * 8, st));
        }
        const uint64_t h_meta[2] = {t, 0};
        const uint32_t h_small[4] = {lg, 0, 0, 0};
        MG_CUDA(ctx, cudaMemcpyAsync(meta.p, h_meta, sizeof h_meta, cudaMemcpyHostToDevice, st));
        MG_CUDA(ctx, cudaMemcpyAsync(small.p, h_small, sizeof h_small, cudaMemcpyHostToDevice, st));
        ScanArgs a = base;
        a.mode = SCAN_SKETCH;           // a screen pass's reference hits were counted by its first scan
        a.tile_begin = lo / SCAN_TILE;
        a.tile_end = (hi + SCAN_TILE - 1) / SCAN_TILE;
        a.coarse_t = t;
        // the scan looks units up by index: views shifted so that index u lands on the pass's single entries
        a.only_unit = u;
        a.unit_t = meta.p - u;
        a.tab_off = meta.p + 1 - u;
        a.tab_log2 = small.p - u;
        a.unit_flags = small.p + 1 - u;
        a.unit_maxhash = small.p + 2 - u;
        a.tab_keys = keys.p;
        a.tab_cnt = cnt.p;
        a.tab_first = positions ? first.p : nullptr;
        a.tab_last = positions ? last.p : nullptr;
        a.min_copies = mc;
        return launch_scan(ctx, p, a, st);
    }

    // The exactness guard: while the table overflows, or fewer than s hashes survive a threshold that dropped k-mers and is not the
    // cap, scan again with 8x the survivor factor (ending at keep-all).  Then the bottom-s, ascending, into h_*.
    int finish()
    {
        const uint32_t s = p->sketch_size;
        uint32_t h_small[4];
        unsigned long long n = 0;
        uint64_t total = 0;
        for (scans = 1;; scans++) {
            MG_CUDA(ctx, cudaMemcpyAsync(h_small, small.p, sizeof h_small, cudaMemcpyDeviceToHost, st));
            MG_CUDA(ctx, cudaStreamSynchronize(st));
            bool again = (h_small[1] & 1u) != 0;
            if (!again) {
                const uint64_t cap = 1ull << lg;
                MG_CUDA(ctx, cudaMemsetAsync(d_n.p, 0, 8, st));
                compact_table_kernel<<<(unsigned)((cap + 255) / 256), 256, 0, st>>>(keys.p, cnt.p, mc, cap, comp.p, d_n.p);
                ctx->kernel_launches++;
                MG_CUDA(ctx, cudaGetLastError());
                MG_CUDA(ctx, cudaMemcpyAsync(&n, d_n.p, 8, cudaMemcpyDeviceToHost, st));
                MG_CUDA(ctx, cudaStreamSynchronize(st));
                total = n + (h_small[2] >= mc ? 1 : 0);
                again = total < s && t != EMPTY_KEY && t != cap_t;
            }
            if (!again) break;
            if (scans == 64) return fail(ctx, MASHGPU_ERR_CUDA, "exact sketch of one unit did not converge");
            MG_TRY(scan(factor * 8.0, cap_t));
        }
        const uint32_t m = (uint32_t)std::min<uint64_t>(total, s);
        if (n) {
            MG_CUDA(ctx, cub::DeviceRadixSort::SortKeys(sort_tmp.p, sort_tmp_bytes, comp.p, sorted.p, (int)n, 0, 64, st));
            ctx->kernel_launches += 8;
        }
        if (m) {
            unit_emit_kernel<<<(m + 255) / 256, 256, 0, st>>>(sorted.p, (uint32_t)std::min<uint64_t>(n, m), m, keys.p, cnt.p,
                                                              positions ? first.p : nullptr, last.p, lg, mc, h_small[2], lo, pos_base,
                                                              c_key.p, c_cnt.p, c_first.p, c_last.p);
            ctx->kernel_launches++;
            MG_CUDA(ctx, cudaGetLastError());
        }
        h_key.resize(m); h_cnt.resize(m); h_first.resize(m); h_last.resize(m);
        if (m) {
            MG_CUDA(ctx, cudaMemcpyAsync(h_key.data(), c_key.p, m * 8ull, cudaMemcpyDeviceToHost, st));
            MG_CUDA(ctx, cudaMemcpyAsync(h_cnt.data(), c_cnt.p, m * 4ull, cudaMemcpyDeviceToHost, st));
            if (positions) {
                MG_CUDA(ctx, cudaMemcpyAsync(h_first.data(), c_first.p, m * 8ull, cudaMemcpyDeviceToHost, st));
                MG_CUDA(ctx, cudaMemcpyAsync(h_last.data(), c_last.p, m * 8ull, cudaMemcpyDeviceToHost, st));
            }
            MG_CUDA(ctx, cudaStreamSynchronize(st));
        }
        return MASHGPU_OK;
    }

    // Occurrences of `key` at positions [unit start, tstar] (tstar as reported, pos_base included) -> *out.
    int recount(uint64_t key, uint64_t tstar, uint32_t *out)
    {
        MG_TRY(recount_hash(ctx, p, base, lo, tstar - pos_base, key, small.p + 3, st));
        MG_CUDA(ctx, cudaMemcpyAsync(out, small.p + 3, 4, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
        return MASHGPU_OK;
    }
};

// The bottom-s of a unit sketched in parts (DESIGN.md 2.7, tests/unit_stream_model.py): its hashes, their counts summed over the
// parts, and the current top's count at positions <= t*.
struct UnitSketch {
    std::vector<uint64_t> keys;
    std::vector<uint32_t> tot;
    uint32_t top_at_tstar = 0;
};

// Merge the bottom-s of a pass into R.  A part changes the set only when a hash first seen in it enters; t* is then the latest
// promoting position among those entrants.  The top's count at positions <= t* is its total before the part plus its occurrences in
// the part up to t*: all of them when its last position is <= t*, none when it was promoted after t*, mc when it was promoted at t*,
// otherwise a recount over [part start, t*].  For m = 1 this is MinHashHeap's top-of-heap quirk (MinHashHeap.cpp:70-74), and a
// merge into an empty state restates quirk_kernel for one unit.
static int unit_merge(UnitPass &P, UnitSketch &R)
{
    const uint32_t s = P.p->sketch_size;
    const std::vector<uint64_t> &ck = P.h_key, &cf = P.h_first, &cl = P.h_last, &rk = R.keys;
    const std::vector<uint32_t> &cc = P.h_cnt;
    const size_t nc = ck.size();
    std::vector<uint64_t> nk;
    std::vector<uint32_t> nt;
    nk.reserve(s); nt.reserve(s);
    size_t i = 0, j = 0;
    int64_t top_r = -1, top_c = -1;             // where the last emitted hash came from
    bool entered = false;
    uint64_t tstar = 0;
    while (nk.size() < s && (i < rk.size() || j < nc)) {
        if (j == nc || (i < rk.size() && rk[i] < ck[j])) { nk.push_back(rk[i]); nt.push_back(R.tot[i]); top_r = (int64_t)i++; top_c = -1; }
        else if (i == rk.size() || ck[j] < rk[i]) {
            nk.push_back(ck[j]); nt.push_back(cc[j]); top_r = -1; top_c = (int64_t)j;
            tstar = entered ? std::max(tstar, cf[j]) : cf[j];
            entered = true;
            j++;
        } else { nk.push_back(rk[i]); nt.push_back(R.tot[i] + cc[j]); top_r = (int64_t)i++; top_c = (int64_t)j++; }
    }
    if (entered && P.positions && nk.back() != EMPTY_KEY) {
        uint32_t part = 0;
        if (top_c >= 0) {
            const uint64_t f = cf[top_c], l = cl[top_c];
            if (l <= tstar) part = cc[top_c];
            else if (f > tstar) part = 0;
            else if (f == tstar) part = P.mc;
            else MG_TRY(P.recount(nk.back(), tstar, &part));
        }
        R.top_at_tstar = (top_r >= 0 ? R.tot[top_r] : 0) + part;
    }
    R.keys.swap(nk);
    R.tot.swap(nt);
    return MASHGPU_OK;
}

// The reference's counts: a full heap's top counts its occurrences up to t* only.
static void unit_counts(const UnitSketch &R, uint32_t s, uint32_t *out)
{
    std::copy(R.tot.begin(), R.tot.end(), out);
    if (R.keys.size() == s && R.keys.back() != EMPTY_KEY) out[s - 1] = R.top_at_tstar;
}

// Exact re-run of flagged unit u: the single-unit pass from 8x the survivor factor, uncapped, merged into an empty state.
static int rerun_unit(UnitPass &P, const SketchStream &S, uint32_t u, uint64_t *d_out_hashes, uint32_t *d_out_counts, uint32_t *d_out_n)
{
    const uint32_t s = P.p->sketch_size;
    P.ctx->exact_reruns++;
    P.u = u;
    P.lo = S.unit_start[u];
    P.hi = S.unit_start[u + 1];
    MG_TRY(P.scan(8.0 * SURVIVOR_FACTOR, EMPTY_KEY));
    MG_TRY(P.finish());
    UnitSketch R;
    MG_TRY(unit_merge(P, R));
    const uint32_t n = (uint32_t)R.keys.size();
    std::vector<uint32_t> counts(n);
    unit_counts(R, s, counts.data());
    MG_CUDA(P.ctx, cudaMemcpyAsync(d_out_hashes + (uint64_t)u * s, R.keys.data(), n * 8ull, cudaMemcpyHostToDevice, P.st));
    if (d_out_counts) MG_CUDA(P.ctx, cudaMemcpyAsync(d_out_counts + (uint64_t)u * s, counts.data(), n * 4ull, cudaMemcpyHostToDevice, P.st));
    MG_CUDA(P.ctx, cudaMemcpyAsync(d_out_n + u, &n, 4, cudaMemcpyHostToDevice, P.st));
    MG_CUDA(P.ctx, cudaStreamSynchronize(P.st));
    return MASHGPU_OK;
}

// Core: sketch every unit of a device-resident stream.
int sketch_stream_core(mashgpu_ctx *ctx, const mashgpu_sketch_params *p, const SketchStream &S,
                       uint64_t *d_out_hashes, uint32_t *d_out_counts, uint32_t *d_out_n, cudaStream_t st,
                       const ScreenProbe *probe)
{
    SketchTicket t;
    MG_TRY(sketch_stream_enqueue(ctx, p, S, d_out_hashes, d_out_counts, d_out_n, st, probe, t));
    return sketch_stream_finalize(ctx, t);
}

int sketch_stream_enqueue(mashgpu_ctx *ctx, const mashgpu_sketch_params *p, const SketchStream &S_in,
                          uint64_t *d_out_hashes, uint32_t *d_out_counts, uint32_t *d_out_n, cudaStream_t st,
                          const ScreenProbe *probe, SketchTicket &t)
{
    t.active = false;
    const uint32_t n_units = (uint32_t)S_in.n_units;
    if (n_units == 0) return MASHGPU_OK;
    t.params = *p;
    t.S = S_in;
    t.unit_start.assign(S_in.unit_start, S_in.unit_start + n_units + 1);
    t.S.unit_start = t.unit_start.data();
    t.d_out_hashes = d_out_hashes; t.d_out_counts = d_out_counts; t.d_out_n = d_out_n; t.st = st;
    const SketchStream &S = t.S;
    const uint32_t s = p->sketch_size;
    const uint64_t stream_len = S.unit_start[n_units];
    const uint64_t ntiles = (stream_len + SCAN_TILE - 1) / SCAN_TILE;

    // plan
    std::vector<uint64_t> h_t(n_units), h_off(n_units);
    std::vector<uint32_t> h_log2(n_units);
    uint64_t slots = 0;
    for (uint32_t u = 0; u < n_units; u++) {
        uint64_t span = S.unit_start[u + 1] - S.unit_start[u];
        plan_unit(p, span, S.force_keep_all ? 0.0 : SURVIVOR_FACTOR, &h_t[u], &h_log2[u]);
        // screen, mixture already holds s hashes: exactly the hashes <= its s-th smallest can still matter -- use that
        // value as the threshold whether the planned one is larger (fewer candidates) or smaller (it would miss some and
        // force an exact re-run when the chunk is full of repeats, e.g. reads at 5x coverage)
        if (S.t_cap) h_t[u] = S.t_cap_value;
        h_off[u] = slots;
        slots += 1ull << h_log2[u];
    }
    struct P64 { uint64_t *p; } d_start, d_t, d_off, d_keys, d_tmax;
    struct P32 { uint32_t *p; } d_log2, d_cnt, d_flags, d_maxhash;
    d_start.p = ctx->sc_start.get<uint64_t>(n_units + 1); d_t.p = ctx->sc_t.get<uint64_t>(n_units); d_off.p = ctx->sc_off.get<uint64_t>(n_units);
    d_log2.p = ctx->sc_log2.get<uint32_t>(n_units); d_flags.p = ctx->sc_flags.get<uint32_t>(n_units); d_maxhash.p = ctx->sc_maxhash.get<uint32_t>(n_units);
    d_keys.p = ctx->sc_keys.get<uint64_t>(slots); d_cnt.p = ctx->sc_cnt.get<uint32_t>(slots); d_tmax.p = ctx->sc_tmax.get<uint64_t>(ntiles);
    uint32_t *d_tunit = ctx->sc_tunit.get<uint32_t>(ntiles);
    if (!d_start.p || !d_t.p || !d_off.p || !d_log2.p || !d_flags.p || !d_maxhash.p || !d_keys.p || !d_cnt.p || !d_tmax.p || !d_tunit)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (%llu candidate slots for %u units)", (unsigned long long)slots, n_units);
    const bool want_counts = d_out_counts != nullptr;
    const uint32_t mc = probe ? 1u : std::max(1u, p->min_copies);      // the screen mixture is a plain MinHashHeap (CommandScreen.cpp:114-119)
    uint64_t *d_first = nullptr, *d_last = nullptr, *d_qtarget = nullptr, *d_qtstar = nullptr;
    if (want_counts) {
        d_first = ctx->sc_first.get<uint64_t>(slots * mc); d_last = ctx->sc_last.get<uint64_t>(slots);
        d_qtarget = ctx->sc_qtarget.get<uint64_t>(n_units); d_qtstar = ctx->sc_qtstar.get<uint64_t>(n_units);
        if (!d_first || !d_last || !d_qtarget || !d_qtstar) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (first/last occurrence tables)");
        MG_CUDA(ctx, cudaMemsetAsync(d_first, 0xFF, slots * mc * 8ull, st));
        MG_CUDA(ctx, cudaMemsetAsync(d_last, 0, slots * 8ull, st));
    }
    MG_CUDA(ctx, cudaMemcpyAsync(d_start.p, S.unit_start, (n_units + 1) * 8ull, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(d_t.p, h_t.data(), n_units * 8ull, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(d_off.p, h_off.data(), n_units * 8ull, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(d_log2.p, h_log2.data(), n_units * 4ull, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemsetAsync(d_flags.p, 0, n_units * 4ull, st));
    MG_CUDA(ctx, cudaMemsetAsync(d_maxhash.p, 0, n_units * 4ull, st));
    MG_CUDA(ctx, cudaMemsetAsync(d_keys.p, 0xFF, slots * 8ull, st));
    MG_CUDA(ctx, cudaMemsetAsync(d_cnt.p, 0, slots * 4ull, st));

    ScanArgs a = scan_base(p, S.d_stream, stream_len, S.d_codes, S.d_inval);
    a.mode = probe ? SCAN_SCREEN : SCAN_SKETCH;
    a.unit_start = d_start.p;
    a.n_units = n_units;
    a.unit_t = d_t.p;
    a.tab_off = d_off.p;
    a.tab_log2 = d_log2.p;
    a.tab_keys = d_keys.p;
    a.tab_cnt = d_cnt.p;
    a.unit_flags = d_flags.p;
    a.unit_maxhash = d_maxhash.p;
    a.tab_first = d_first;
    a.tab_last = d_last;
    a.min_copies = mc;
    if (probe) {
        a.ref_keys = probe->keys; a.ref_idx = probe->idx; a.ref_cnt = probe->cnt; a.ref_log2 = probe->log2cap; a.ref_hmax = probe->hmax;
        a.ref_bitmap = probe->bitmap; a.ref_bitmap_shift = probe->bitmap_shift;
    }
    if (ntiles) {
        tile_tmax_kernel<<<(unsigned)((ntiles + 255) / 256), 256, 0, st>>>(d_start.p, n_units, d_t.p, stream_len, p->kmer_size, 0, ntiles, d_tmax.p, d_tunit);
        ctx->kernel_launches++;
    }
    a.tile_tmax = d_tmax.p;
    a.tile_unit = d_tunit;
    if (probe) {
        // coarse filter must also let reference-hash candidates through
        a.tile_tmax = nullptr;
        uint64_t tm = 0;
        for (uint32_t u = 0; u < n_units; u++) tm = std::max(tm, h_t[u]);
        a.coarse_t = std::max(tm, probe->hmax);
        a.screen_mix_t = tm;
    }
    if (S.data_ready) MG_CUDA(ctx, cudaStreamWaitEvent(st, S.data_ready, 0));
    MG_TRY(launch_scan(ctx, p, a, st));

    const size_t sel_smem = (size_t)8 << SEL_MAX_LOG2;
    if (!ctx->attr_select) {   // per context: function attributes are per device
        MG_CUDA(ctx, cudaFuncSetAttribute(select_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sel_smem));
        ctx->attr_select = true;
    }
    uint32_t max_log2 = 4;
    for (uint32_t u = 0; u < n_units; u++) max_log2 = std::max(max_log2, std::min(h_log2[u], SEL_MAX_LOG2));
    select_kernel<<<n_units, SEL_THREADS, (size_t)8 << max_log2, st>>>(0, n_units, d_t.p, d_off.p, d_log2.p, d_keys.p, d_cnt.p,
                                                                     d_maxhash.p, d_flags.p, s, S.t_cap ? S.t_cap_value : EMPTY_KEY,
                                                                     d_out_hashes, d_out_counts, d_out_n, mc);
    ctx->kernel_launches++;
    MG_CUDA(ctx, cudaGetLastError());
    {   // units whose candidate table exceeds the shared-memory sort (large sketch sizes): one segmented sort for all of them
        std::vector<uint32_t> big;
        std::vector<uint64_t> seg_off;
        uint64_t comp_total = 0, max_cap = 0;
        for (uint32_t u = 0; u < n_units; u++)
            if (h_log2[u] > SEL_MAX_LOG2) { big.push_back(u); seg_off.push_back(comp_total); comp_total += 1ull << h_log2[u]; max_cap = std::max<uint64_t>(max_cap, 1ull << h_log2[u]); }
        if (!big.empty()) {
            if (comp_total >= 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "candidate tables of one wave exceed 2^31 slots (sketch_size %u x %zu units): feed fewer units per call", s, big.size());
            const uint32_t n_big = (uint32_t)big.size();
            uint32_t *d_big = ctx->sc_big_units.get<uint32_t>(n_big), *d_seg_n = ctx->sc_big_n.get<uint32_t>(n_big);
            uint64_t *d_seg_off = ctx->sc_big_off.get<uint64_t>(n_big);
            long long *d_bounds = ctx->sc_big_bounds.get<long long>(2ull * n_big);
            uint64_t *d_comp = ctx->sc_big_comp.get<uint64_t>(comp_total), *d_sorted = ctx->sc_big_sorted.get<uint64_t>(comp_total);
            if (!d_big || !d_seg_n || !d_seg_off || !d_bounds || !d_comp || !d_sorted) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sort buffers of %llu candidate slots)", (unsigned long long)comp_total);
            MG_CUDA(ctx, cudaMemcpyAsync(d_big, big.data(), n_big * 4ull, cudaMemcpyHostToDevice, st));
            MG_CUDA(ctx, cudaMemcpyAsync(d_seg_off, seg_off.data(), n_big * 8ull, cudaMemcpyHostToDevice, st));
            MG_CUDA(ctx, cudaMemsetAsync(d_seg_n, 0, n_big * 4ull, st));
            const unsigned bx = (unsigned)std::min<uint64_t>((max_cap + 255) / 256, 256);
            select_big_compact_kernel<<<dim3(bx, n_big), 256, 0, st>>>(d_big, n_big, d_seg_off, d_off.p, d_log2.p, d_keys.p, d_cnt.p, d_flags.p, mc, d_comp, d_seg_n);
            select_big_bounds_kernel<<<(n_big + 255) / 256, 256, 0, st>>>(d_seg_off, d_seg_n, n_big, d_bounds, d_bounds + n_big);
            size_t tmp_bytes = 0;
            cub::DeviceSegmentedRadixSort::SortKeys(nullptr, tmp_bytes, d_comp, d_sorted, (int)comp_total, (int)n_big, d_bounds, d_bounds + n_big, 0, 64, st);
            uint8_t *d_tmp = ctx->sc_big_tmp.get<uint8_t>(tmp_bytes);
            if (!d_tmp) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (segmented sort scratch)");
            MG_CUDA(ctx, cub::DeviceSegmentedRadixSort::SortKeys(d_tmp, tmp_bytes, d_comp, d_sorted, (int)comp_total, (int)n_big, d_bounds, d_bounds + n_big, 0, 64, st));
            select_big_emit_kernel<<<n_big, SEL_THREADS, 0, st>>>(d_big, n_big, d_seg_off, d_seg_n, d_sorted, d_t.p, d_off.p, d_log2.p, d_keys.p, d_cnt.p, d_maxhash.p, d_flags.p,
                                                                s, S.t_cap ? S.t_cap_value : EMPTY_KEY, d_out_hashes, d_out_counts, d_out_n, mc);
            ctx->kernel_launches += 4;
            MG_CUDA(ctx, cudaGetLastError());
        }
    }
    if (want_counts) {
        quirk_kernel<<<n_units, SEL_THREADS, 0, st>>>(0, n_units, s, d_out_hashes, d_out_counts, d_out_n, d_off.p, d_log2.p, d_keys.p, d_cnt.p,
                                                      d_first, d_last, d_flags.p, d_qtarget, d_qtstar, mc);
        ctx->kernel_launches++;
        MG_CUDA(ctx, cudaGetLastError());
    }

    // one ticket in flight per context: its flags land in the context's pinned buffer
    uint32_t *h_flags = ctx->flags_pinned.get<uint32_t>(n_units);
    if (!h_flags) return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory (unit flags)");
    MG_CUDA(ctx, cudaMemcpyAsync(h_flags, d_flags.p, n_units * 4ull, cudaMemcpyDeviceToHost, st));
    t.d_qtarget = d_qtarget; t.d_qtstar = d_qtstar;
    t.active = true;
    return MASHGPU_OK;
}

int sketch_stream_finalize(mashgpu_ctx *ctx, SketchTicket &t)
{
    if (!t.active) return MASHGPU_OK;
    t.active = false;
    const mashgpu_sketch_params *p = &t.params;
    const SketchStream &S = t.S;
    const uint32_t n_units = (uint32_t)S.n_units;
    const uint32_t s = p->sketch_size;
    cudaStream_t st = t.st;
    uint64_t *d_out_hashes = t.d_out_hashes; uint32_t *d_out_counts = t.d_out_counts, *d_out_n = t.d_out_n;
    uint64_t *d_qtarget = t.d_qtarget, *d_qtstar = t.d_qtstar;
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    const uint32_t *h_flags = static_cast<const uint32_t *>(ctx->flags_pinned.p);
    bool any_flag = false;
    for (uint32_t u = 0; u < n_units; u++) any_flag |= h_flags[u] != 0;
    if (!any_flag) return MASHGPU_OK;
    bool any_recount = false;
    for (uint32_t u = 0; u < n_units; u++) any_recount |= (h_flags[u] & 8u) && !(h_flags[u] & 7u);
    std::vector<uint64_t> h_qtarget, h_qtstar;
    if (any_recount) {
        h_qtarget.resize(n_units); h_qtstar.resize(n_units);
        MG_CUDA(ctx, cudaMemcpyAsync(h_qtarget.data(), d_qtarget, n_units * 8ull, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaMemcpyAsync(h_qtstar.data(), d_qtstar, n_units * 8ull, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
    }
    // re-runs and recounts scan the pass's stream again, finding units through its device copy of unit_start
    ScanArgs a = scan_base(p, S.d_stream, S.unit_start[n_units], S.d_codes, S.d_inval);
    a.unit_start = static_cast<const uint64_t *>(ctx->sc_start.p);
    a.n_units = n_units;
    UnitPass pass;
    uint64_t pass_bytes = 0, pass_peak = 0;
    for (uint32_t u = 0; u < n_units; u++) {
        if (h_flags[u] == 0) continue;
        if (h_flags[u] & 7u) {
            if (!pass.ctx) {
                MG_TRY(pass.open(ctx, p, st, d_out_counts != nullptr, &pass_bytes, &pass_peak));
                pass.base = a;
            }
            MG_TRY(rerun_unit(pass, S, u, d_out_hashes, d_out_counts, d_out_n));
        } else MG_TRY(recount_hash(ctx, p, a, S.unit_start[u], h_qtstar[u], h_qtarget[u], d_out_counts + (uint64_t)u * s + s - 1, st));
    }
    if (any_recount) MG_CUDA(ctx, cudaStreamSynchronize(st));
    return MASHGPU_OK;
}

}  // namespace mashgpu

using namespace mashgpu;

extern "C" uint32_t mashgpu_set_alphabet(mashgpu_sketch_params *p, const char *characters)
{
    // setAlphabetFromString, reference Sketch.cpp:1108-1137
    memset(p->alphabet, 0, 256);
    for (const char *c = characters; *c; c++) {
        unsigned char u = (unsigned char)*c;
        if (!p->preserve_case && u > 96 && u < 123) u -= 32;
        p->alphabet[u] = 1;
    }
    uint32_t n = 0;
    for (int i = 0; i < 256; i++) n += p->alphabet[i];
    p->use64 = std::pow((double)n, (double)p->kmer_size) > std::pow(2.0, 32.0);
    return n;
}

extern "C" int mashgpu_sketch_stream_dev(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                                         const void *d_stream, const uint64_t *unit_start, uint64_t n_units,
                                         uint64_t *d_out_hashes, uint32_t *d_out_counts, uint32_t *d_out_n, void *stream)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    MG_TRY(validate_sketch_params(ctx, params));
    if (n_units > 0xFFFFFFF0ull) return fail(ctx, MASHGPU_ERR_INVALID, "too many units");
    if (n_units && (!d_stream || !unit_start || !d_out_hashes || !d_out_n)) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    SketchStream S;
    S.d_stream = d_stream; S.unit_start = unit_start; S.n_units = n_units;
    return sketch_stream_core(ctx, params, S, d_out_hashes, d_out_counts, d_out_n, stream ? (cudaStream_t)stream : ctx->stream, nullptr);
}

namespace mashgpu {
static int unit_stream_limit(mashgpu_ctx *ctx, uint64_t *limit);
static int sketch_unit_streamed(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, uint64_t n_records, const char *const *seq,
                                const uint64_t *len, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_length,
                                uint64_t *out_records);
}  // namespace mashgpu

namespace {

constexpr uint64_t WAVE_BYTES = 1ull << 30;        // stream bytes per wave (the two feed paths share the waves of a batch: finer than 2 GiB balances better)
constexpr uint32_t SEP_LIST_MAX = 1u << 15;        // directly copied records per wave whose separators go through the list
constexpr uint64_t DIRECT_COPY_MIN = 1ull << 18;   // records at least this long are copied straight from the caller's buffer

// ---- the wave pieces of both batch calls (mashgpu_sketch_batch, mashgpu_sketch_batch_packed)

// Waves are cut by stream bytes and by unit count (outputs and candidate tables grow with the number of units, not with their
// length -- a multi-FASTA of millions of short records must not allocate units x s outputs at once).
struct WaveLimits { uint64_t bytes, units; };

WaveLimits wave_limits(uint32_t s)
{
    WaveLimits L{WAVE_BYTES, std::max<uint64_t>(64, (1ull << 28) / ((uint64_t)s * 8))};
    if (const char *env = getenv("MASHGPU_WAVE_BYTES")) L.bytes = std::max<uint64_t>(1024, strtoull(env, nullptr, 10));      // tests: many waves from little data
    if (const char *env = getenv("MASHGPU_WAVE_UNITS")) L.units = std::max<uint64_t>(1, strtoull(env, nullptr, 10));
    return L;
}

// The call's host outputs, indexed by unit (out_counts may be NULL), and the device outputs of one wave (the context's scratch).
struct WaveOut {
    uint64_t *out_hashes; uint32_t *out_counts, *out_n;
    uint64_t *d_hashes = nullptr; uint32_t *d_counts = nullptr, *d_n = nullptr;
};

int wave_outputs(mashgpu_ctx *ctx, uint32_t s, uint64_t max_units, WaveOut &o)
{
    o.d_hashes = ctx->sc_out_hashes.get<uint64_t>(max_units * s);
    o.d_n = ctx->sc_out_n.get<uint32_t>(max_units);
    o.d_counts = o.out_counts ? ctx->sc_out_counts.get<uint32_t>(max_units * s) : nullptr;
    if (!o.d_hashes || !o.d_n || (o.out_counts && !o.d_counts)) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (outputs)");
    return MASHGPU_OK;
}

// Sketches the wave S -- units [u0, u0 + S.n_units) of the call -- on the compute stream, copies its sketches back and waits for them.
int sketch_wave(mashgpu_ctx *ctx, const mashgpu_sketch_params *p, const SketchStream &S, uint64_t u0, const WaveOut &o)
{
    const uint64_t s = p->sketch_size, nu = S.n_units;
    MG_TRY(sketch_stream_core(ctx, p, S, o.d_hashes, o.d_counts, o.d_n, ctx->stream, nullptr));
    MG_CUDA(ctx, cudaMemcpyAsync(o.out_hashes + u0 * s, o.d_hashes, nu * s * 8, cudaMemcpyDeviceToHost, ctx->stream));
    MG_CUDA(ctx, cudaMemcpyAsync(o.out_n + u0, o.d_n, nu * 4, cudaMemcpyDeviceToHost, ctx->stream));
    if (o.out_counts) MG_CUDA(ctx, cudaMemcpyAsync(o.out_counts + u0 * s, o.d_counts, nu * s * 4, cudaMemcpyDeviceToHost, ctx->stream));
    MG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return MASHGPU_OK;
}

// Device slots for packed waves of up to max_len positions: 2-bit codes and the invalid-position mask, `groups` 32-position
// groups each (tile-padded + halo: the scan kernel reads whole tiles without looking at the stream length).  Uploads go on
// pack_stream and record pack_copied[b].
struct PackedSlots { uint64_t groups = 0; uint64_t *d_codes[2] = {}; uint32_t *d_inval[2] = {}; };

int packed_slots(mashgpu_ctx *ctx, int n_slots, uint64_t max_len, PackedSlots &P)
{
    P.groups = (max_len + SCAN_TILE - 1) / SCAN_TILE * (SCAN_TILE / 32) + 64;
    for (int b = 0; b < n_slots; b++) {
        P.d_codes[b] = ctx->sc_codes[b].get<uint64_t>(P.groups);
        P.d_inval[b] = ctx->sc_inval[b].get<uint32_t>(P.groups);
        if (!P.d_codes[b] || !P.d_inval[b]) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (packed stream of %llu groups)", (unsigned long long)P.groups);
        if (!ctx->pack_copied[b]) MG_CUDA(ctx, cudaEventCreateWithFlags(&ctx->pack_copied[b], cudaEventDisableTiming));
    }
    if (n_slots && !ctx->pack_stream) MG_CUDA(ctx, cudaStreamCreateWithFlags(&ctx->pack_stream, cudaStreamNonBlocking));
    return MASHGPU_OK;
}

// Enqueues the upload of a packed wave into slot b: `groups` code words, then the mask -- zeroed, and the invalid runs set (they
// must reach the end of the slot) by one apply_runs_kernel -- then records pack_copied[b].  The packer thread calls it too, so it
// returns a bare code: the launching thread reports the failure and counts the launch.
int upload_packed(mashgpu_ctx *ctx, const PackedSlots &P, int b, const uint64_t *h_codes, uint64_t groups, const std::vector<PackRun> &runs)
{
    cudaStream_t cs = ctx->pack_stream;
    if (groups && cudaMemcpyAsync(P.d_codes[b], h_codes, groups * 8, cudaMemcpyHostToDevice, cs) != cudaSuccess) return MASHGPU_ERR_CUDA;
    if (cudaMemsetAsync(P.d_inval[b], 0, P.groups * 4, cs) != cudaSuccess) return MASHGPU_ERR_CUDA;
    PackRun *d_runs = ctx->sc_runs[b].get<PackRun>(runs.size());
    if (!d_runs) return MASHGPU_ERR_NOMEM;
    if (cudaMemcpyAsync(d_runs, runs.data(), runs.size() * sizeof(PackRun), cudaMemcpyHostToDevice, cs) != cudaSuccess) return MASHGPU_ERR_CUDA;
    const uint64_t nr = runs.size();
    const unsigned blocks = (unsigned)std::min<uint64_t>((nr * 32 + 255) / 256, (uint64_t)ctx->sm_count * 16);
    apply_runs_kernel<<<std::max(1u, blocks), 256, 0, cs>>>(d_runs, nr, P.d_inval[b]);
    if (cudaGetLastError() != cudaSuccess) return MASHGPU_ERR_CUDA;
    if (cudaEventRecord(ctx->pack_copied[b], cs) != cudaSuccess) return MASHGPU_ERR_CUDA;
    return MASHGPU_OK;
}

// ---- mashgpu_sketch_batch

struct Wave { uint64_t unit_begin, unit_end, bytes; };     // its records: unit_rec_begin[unit_begin] .. unit_rec_begin[unit_end]

// Units [u0, u1) of a batch, none of them too large for the device, in waves.  Records, units and outputs are indexed as in the
// call: unit u holds the records unit_rec_begin[u] .. unit_rec_begin[u + 1], unit_bytes[u] stream bytes.
int sketch_units(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, const char *const *seq, const uint64_t *len,
                 const uint64_t *unit_rec_begin, const uint64_t *unit_bytes, uint64_t u0, uint64_t u1,
                 uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n)
{
    const uint32_t s = params->sketch_size;
    const uint64_t k = (uint64_t)params->kmer_size;
    const WaveLimits lim = wave_limits(s);
    std::vector<Wave> waves;
    {
        Wave w{u0, u0, 0};
        for (uint64_t u = u0; u < u1; u++) {
            if (w.unit_end > w.unit_begin && (w.bytes + unit_bytes[u] > lim.bytes || w.unit_end - w.unit_begin >= lim.units)) {
                waves.push_back(w);
                w = Wave{u, u, 0};
            }
            w.unit_end = u + 1;
            w.bytes += unit_bytes[u];
        }
        waves.push_back(w);
    }
    const size_t n_waves = waves.size();
    uint64_t max_bytes = 32, max_units = 1;
    for (auto &w : waves) { max_bytes = std::max(max_bytes, w.bytes); max_units = std::max(max_units, w.unit_end - w.unit_begin); }

    // ---- feed paths.  A wave reaches the GPU either as ASCII (DMA straight from the caller's buffers: no host CPU work, 1 byte
    // per base over PCIe) or 2-bit packed by host threads (pack.cpp: a quarter of the bytes, but ~6 GB/s per host core).  The two
    // producers run side by side and claim waves from one list, so the split follows their real speeds (bench.py's e2e object
    // reports the hybrid, ASCII-only and packed-only rates).  Packing is the only producer for waves with small records or pageable buffers (a
    // cudaMemcpyAsync from pageable memory is staged by the driver at a fraction of the PCIe rate and blocks this thread).
    // MASHGPU_HOST_PACK=0: ASCII only; =1: packed only; unset: both.  Non-DNA alphabets are ASCII only.
    enum { FEED_ASCII = 1, FEED_PACK = 2 };
    int feed = FEED_ASCII | FEED_PACK;
    if (const char *env = getenv("MASHGPU_HOST_PACK")) feed = env[0] == '0' ? FEED_ASCII : (env[0] == '1' ? FEED_PACK : feed);
    if (!is_dna_alphabet(params)) feed = FEED_ASCII;
    // ASCII-eligible waves: every kept record is long enough for a direct copy and lies in pinned (page-locked) memory
    std::vector<uint8_t> ascii_ok(n_waves, 1);
    if (feed == (FEED_ASCII | FEED_PACK)) {
        for (size_t wi = 0; wi < n_waves; wi++) {
            const Wave &w = waves[wi];
            bool ok = true;
            bool probed = false;
            for (uint64_t r = unit_rec_begin[w.unit_begin]; r < unit_rec_begin[w.unit_end] && ok; r++) {
                if (len[r] < k) continue;
                if (len[r] < DIRECT_COPY_MIN) ok = false;
                else if (!probed) {          // one probe per wave: callers allocate their records the same way
                    cudaPointerAttributes at;
                    if (cudaPointerGetAttributes(&at, seq[r]) != cudaSuccess) { cudaGetLastError(); ok = false; }
                    else if (at.type != cudaMemoryTypeHost && at.type != cudaMemoryTypeManaged) ok = false;
                    probed = true;
                }
            }
            ascii_ok[wi] = ok;
        }
    }
    // packer threads: as many as the process may actually run (pack.cpp: hardware threads, the container's CPU quota,
    // MASHGPU_PACK_THREADS) -- minus one for this thread when it also drives the ASCII copies
    int threads = host_pack_threads();
    if ((feed & FEED_ASCII) && !getenv("MASHGPU_PACK_THREADS")) threads = std::max(1, threads - 1);

    WaveOut out{out_hashes, out_counts, out_n};
    MG_TRY(wave_outputs(ctx, s, max_units, out));

    // ---- ASCII producer: two device wave buffers, copies on copy_stream
    struct AsciiSlot { int64_t wave = -1; uint8_t *d = nullptr; std::vector<uint64_t> unit_start; };
    AsciiSlot aslot[2];
    const uint64_t buf_bytes = ((max_bytes + 15) / 16) * 16 + 16;
    const int n_aslots = (feed & FEED_ASCII) ? (n_waves > 1 ? 2 : 1) : 0;
    cudaEvent_t *copied = ctx->wave_copied;
    for (int b = 0; b < n_aslots; b++) {
        aslot[b].d = ctx->sc_wave[b].get<uint8_t>(buf_bytes);
        if (!aslot[b].d) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (stream buffer %llu B)", (unsigned long long)buf_bytes);
        if (!copied[b]) MG_CUDA(ctx, cudaEventCreateWithFlags(&copied[b], cudaEventDisableTiming));
    }
    auto issue_copy = [&](size_t wi, int b) -> int {
        const Wave &w = waves[wi];
        uint8_t *dst = aslot[b].d;
        // staging size: all small records of the wave
        uint64_t small_bytes = 0;
        for (uint64_t r = unit_rec_begin[w.unit_begin]; r < unit_rec_begin[w.unit_end]; r++)
            if (len[r] >= k && len[r] < DIRECT_COPY_MIN) small_bytes += len[r] + 1;
        uint8_t *stage = ctx->pinned[b].get<uint8_t>(small_bytes);
        if (!stage) return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory (%llu B)", (unsigned long long)small_bytes);
        std::vector<uint64_t> &us = aslot[b].unit_start;
        us.assign(w.unit_end - w.unit_begin + 1, 0);
        // separator offsets of the directly copied records (pinned list -> device -> one kernel); list full: 1-byte memsets
        uint64_t *h_sep = ctx->pinned_sep[b].get<uint64_t>(SEP_LIST_MAX);
        if (!h_sep) return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory (separator list)");
        uint64_t *d_sep = ctx->sc_sep[b].get<uint64_t>(SEP_LIST_MAX);
        if (!d_sep) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (separator list)");
        uint32_t n_sep = 0;
        uint64_t off = 0, st_off = 0;
        uint64_t run_dst = 0, run_src = 0, run_len = 0;   // pending staged run
        auto flush_run = [&]() -> cudaError_t {
            if (!run_len) return cudaSuccess;
            cudaError_t e = cudaMemcpyAsync(dst + run_dst, stage + run_src, run_len, cudaMemcpyHostToDevice, ctx->copy_stream);
            run_len = 0;
            return e;
        };
        for (uint64_t u = w.unit_begin; u < w.unit_end; u++) {
            us[u - w.unit_begin] = off;
            for (uint64_t r = unit_rec_begin[u]; r < unit_rec_begin[u + 1]; r++) {
                if (len[r] < k) continue;
                if (len[r] >= DIRECT_COPY_MIN) {
                    MG_CUDA(ctx, flush_run());
                    MG_CUDA(ctx, cudaMemcpyAsync(dst + off, seq[r], len[r], cudaMemcpyHostToDevice, ctx->copy_stream));
                    if (n_sep < SEP_LIST_MAX) h_sep[n_sep++] = off + len[r];
                    else MG_CUDA(ctx, cudaMemsetAsync(dst + off + len[r], 0, 1, ctx->copy_stream));
                } else {
                    if (!run_len) { run_dst = off; run_src = st_off; }
                    memcpy(stage + st_off, seq[r], len[r]);
                    stage[st_off + len[r]] = 0;
                    st_off += len[r] + 1;
                    run_len += len[r] + 1;
                }
                off += len[r] + 1;
            }
        }
        MG_CUDA(ctx, flush_run());
        if (n_sep) {
            MG_CUDA(ctx, cudaMemcpyAsync(d_sep, h_sep, n_sep * 8ull, cudaMemcpyHostToDevice, ctx->copy_stream));
            write_separators_kernel<<<(n_sep + 255) / 256, 256, 0, ctx->copy_stream>>>(dst, d_sep, n_sep);
            MG_CUDA(ctx, cudaGetLastError());
            ctx->kernel_launches++;
        }
        us[w.unit_end - w.unit_begin] = off;
        MG_CUDA(ctx, cudaEventRecord(copied[b], ctx->copy_stream));
        aslot[b].wave = (int64_t)wi;
        return MASHGPU_OK;
    };

    // ---- packed producer: two pinned code buffers, one packing job at a time on `threads` host threads; the job itself enqueues
    // its upload (codes, invalid runs -> mask) on pack_stream, so a finished future means "event recorded"
    struct PackSlot {
        int64_t wave = -1;
        uint64_t *h_codes = nullptr;
        std::vector<uint64_t> unit_start; std::vector<PackRun> runs; uint64_t len = 0;
    };
    PackSlot pslot[2];
    const int n_pslots = (feed & FEED_PACK) ? (n_waves > 1 ? 2 : 1) : 0;
    PackedSlots slots;
    MG_TRY(packed_slots(ctx, n_pslots, max_bytes, slots));
    for (int b = 0; b < n_pslots; b++) {
        pslot[b].h_codes = ctx->pinned_codes[b].get<uint64_t>(slots.groups);
        if (!pslot[b].h_codes) return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory (%llu B)", (unsigned long long)(slots.groups * 8));
    }
    auto pack_job = [&](size_t wi, int b) -> int {
        cudaSetDevice(ctx->device);
        const Wave &w = waves[wi];
        PackSlot &P = pslot[b];
        std::vector<PackSegment> segs;
        segs.reserve(unit_rec_begin[w.unit_end] - unit_rec_begin[w.unit_begin]);
        P.unit_start.assign(w.unit_end - w.unit_begin + 1, 0);
        uint64_t off = 0;
        for (uint64_t u = w.unit_begin; u < w.unit_end; u++) {
            P.unit_start[u - w.unit_begin] = off;
            for (uint64_t r = unit_rec_begin[u]; r < unit_rec_begin[u + 1]; r++) {
                if (len[r] < k) continue;
                segs.push_back(PackSegment{(const uint8_t *)seq[r], off, len[r]});
                off += len[r] + 1;                     // one separator position after every record
            }
        }
        P.unit_start[w.unit_end - w.unit_begin] = off;
        P.len = off;
        pack_stream(segs.data(), segs.size(), off, params->preserve_case, threads, P.h_codes, P.runs);
        P.runs.push_back(PackRun{off, slots.groups * 32 - off});      // everything from the end of the stream to the end of the allocation is invalid
        // the upload is in flight when this returns: the slot is ready once the event has fired (its buffers are reused only after that)
        return upload_packed(ctx, slots, b, P.h_codes, (P.len + 31) / 32, P.runs);
    };

    // ---- scheduler: both producers claim the next unclaimed wave they may take; this thread runs the kernels of whichever
    // wave is ready first and hands its sketches back
    std::vector<uint8_t> claimed(n_waves, 0);
    size_t a_cursor = 0, p_cursor = 0, done = 0;
    std::mutex mu;                      // guards `claimed` and the packed slots' states (this thread and the packer thread)
    std::condition_variable cv;
    auto claim = [&](size_t &cursor, bool need_ascii) -> int64_t {
        std::lock_guard<std::mutex> lock(mu);
        for (size_t wi = cursor; wi < n_waves; wi++) {
            if (claimed[wi]) { if (wi == cursor) cursor++; continue; }
            if (need_ascii && !ascii_ok[wi] && (feed & FEED_PACK)) continue;      // left to the packer
            claimed[wi] = 1;
            return (int64_t)wi;
        }
        return -1;
    };
    int rc = MASHGPU_OK;
    enum { P_EMPTY, P_PACKING, P_UPLOADING };
    int pstate[2] = {P_EMPTY, P_EMPTY};         // under `mu`
    int pack_rc = MASHGPU_OK;                   // under `mu`: first failure of the packer thread
    bool stop = false, packer_done = n_pslots == 0;
    // the packer thread: claims a wave whenever one of its two slots is empty, packs it on `threads` host threads, enqueues the
    // upload and moves on -- it never waits for this thread's kernels
    std::thread packer;
    if (n_pslots)
        packer = std::thread([&]() {
            cudaSetDevice(ctx->device);
            for (;;) {
                int b = -1;
                {
                    std::unique_lock<std::mutex> lock(mu);
                    cv.wait(lock, [&] { return stop || pstate[0] == P_EMPTY || (n_pslots > 1 && pstate[1] == P_EMPTY); });
                    if (stop) break;
                    b = pstate[0] == P_EMPTY ? 0 : 1;
                }
                const int64_t wi = claim(p_cursor, false);
                if (wi < 0) break;
                { std::lock_guard<std::mutex> lock(mu); pslot[b].wave = wi; pstate[b] = P_PACKING; }
                const int r = pack_job((size_t)wi, b);
                std::lock_guard<std::mutex> lock(mu);
                if (r != MASHGPU_OK) { pack_rc = r; break; }
                pstate[b] = P_UPLOADING;
            }
            std::lock_guard<std::mutex> lock(mu);
            packer_done = true;
        });
    while (done < n_waves && rc == MASHGPU_OK) {
        // 1. keep the ASCII producer busy
        for (int b = 0; b < n_aslots && rc == MASHGPU_OK; b++)
            if (aslot[b].wave < 0) {
                const int64_t wi = claim(a_cursor, true);
                if (wi >= 0) rc = issue_copy((size_t)wi, b);
            }
        if (rc != MASHGPU_OK) break;
        // 2. a finished wave?  packed first, then ASCII copies in issue order
        int ready_p = -1, ready_a = -1, uploading = -1;
        bool packing = false, p_done = false;
        {
            std::lock_guard<std::mutex> lock(mu);
            if (pack_rc != MASHGPU_OK) { rc = fail(ctx, pack_rc, "host packing / packed upload failed"); break; }
            p_done = packer_done;
            for (int b = 0; b < n_pslots; b++) {
                if (pstate[b] == P_PACKING) packing = true;
                if (pstate[b] == P_UPLOADING) {
                    const cudaError_t q = cudaEventQuery(ctx->pack_copied[b]);
                    if (q == cudaSuccess) { if (ready_p < 0 || pslot[b].wave < pslot[ready_p].wave) ready_p = b; }
                    else if (q != cudaErrorNotReady) { rc = fail(ctx, MASHGPU_ERR_CUDA, "packed upload failed: %s", cudaGetErrorString(q)); break; }
                    else { cudaGetLastError(); uploading = b; }
                }
            }
        }
        if (rc != MASHGPU_OK) break;
        if (ready_p < 0) {
            int64_t best = -1;
            for (int b = 0; b < n_aslots; b++)
                if (aslot[b].wave >= 0 && (best < 0 || aslot[b].wave < best)) {
                    const cudaError_t q = cudaEventQuery(copied[b]);
                    if (q == cudaSuccess) { ready_a = b; best = aslot[b].wave; }
                    else if (q != cudaErrorNotReady) { rc = fail(ctx, MASHGPU_ERR_CUDA, "H2D copy failed: %s", cudaGetErrorString(q)); break; }
                    else cudaGetLastError();
                }
        }
        if (rc != MASHGPU_OK) break;
        if (ready_p >= 0) {
            PackSlot &P = pslot[ready_p];
            const Wave &w = waves[P.wave];
            ctx->kernel_launches++;             // apply_runs_kernel of the upload
            SketchStream S;
            S.d_codes = slots.d_codes[ready_p]; S.d_inval = slots.d_inval[ready_p]; S.unit_start = P.unit_start.data(); S.n_units = w.unit_end - w.unit_begin;
            rc = sketch_wave(ctx, params, S, w.unit_begin, out);
            { std::lock_guard<std::mutex> lock(mu); P.wave = -1; pstate[ready_p] = P_EMPTY; }
            cv.notify_all();
            done++;
        } else if (ready_a >= 0) {
            AsciiSlot &A = aslot[ready_a];
            const Wave &w = waves[A.wave];
            SketchStream S;
            S.d_stream = A.d; S.unit_start = A.unit_start.data(); S.n_units = w.unit_end - w.unit_begin;
            rc = sketch_wave(ctx, params, S, w.unit_begin, out);
            A.wave = -1;
            done++;
        } else {
            // nothing ready: wait for whichever producer is in flight
            int64_t best = -1; int bb = -1;
            for (int b = 0; b < n_aslots; b++)
                if (aslot[b].wave >= 0 && (best < 0 || aslot[b].wave < best)) { best = aslot[b].wave; bb = b; }
            if (uploading >= 0) cudaEventSynchronize(ctx->pack_copied[uploading]);
            else if (packing || (!p_done && bb < 0)) std::this_thread::sleep_for(std::chrono::microseconds(50));
            else if (bb >= 0) MG_CUDA(ctx, cudaEventSynchronize(copied[bb]));
            else { rc = fail(ctx, MASHGPU_ERR_INVALID, "feed scheduler stalled (%zu of %zu waves done)", done, n_waves); break; }
        }
    }
    if (packer.joinable()) {
        { std::lock_guard<std::mutex> lock(mu); stop = true; }
        cv.notify_all();
        packer.join();                           // never leave the packer thread behind (it references this frame)
    }
    cudaStreamSynchronize(ctx->copy_stream);
    if (ctx->pack_stream) cudaStreamSynchronize(ctx->pack_stream);
    return rc;
}

}  // namespace

extern "C" int mashgpu_sketch_batch(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                                    uint64_t n_records, const char *const *seq, const uint64_t *len,
                                    const uint32_t *unit_of_record, uint64_t n_units,
                                    uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_length)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    MG_TRY(validate_sketch_params(ctx, params));
    if (n_units == 0) return MASHGPU_OK;
    if (!out_hashes || !out_n) return fail(ctx, MASHGPU_ERR_INVALID, "out_hashes/out_n is NULL");
    if (n_records && (!seq || !len)) return fail(ctx, MASHGPU_ERR_INVALID, "seq/len is NULL");
    if (n_units > 0xFFFFFFF0ull) return fail(ctx, MASHGPU_ERR_INVALID, "too many units");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint32_t s = params->sketch_size;
    const uint64_t k = (uint64_t)params->kmer_size;

    // unit spans in the flat stream: kept records back to back, one separator byte after each
    std::vector<uint64_t> unit_bytes(n_units, 0), unit_rec_begin(n_units + 1, 0);
    {
        uint64_t r = 0;
        for (uint64_t u = 0; u < n_units; u++) {
            unit_rec_begin[u] = r;
            while (r < n_records && (unit_of_record ? unit_of_record[r] : r) == u) {
                if (len[r] >= k) unit_bytes[u] += len[r] + 1;
                r++;
            }
            if (r < n_records && unit_of_record && unit_of_record[r] < u)
                return fail(ctx, MASHGPU_ERR_INVALID, "unit_of_record must be non-decreasing");
        }
        unit_rec_begin[n_units] = r;
        if (r != n_records) return fail(ctx, MASHGPU_ERR_INVALID, "unit_of_record refers to units >= n_units or is not sorted");
    }
    if (out_length)
        for (uint64_t u = 0; u < n_units; u++) {
            uint64_t L = 0;
            for (uint64_t r = unit_rec_begin[u]; r < unit_rec_begin[u + 1]; r++)
                if (len[r] >= k) L += len[r];
            out_length[u] = L;
        }

    // a unit whose stream does not fit on the device at once (the whole-set rule of mashgpu_sketch_reads) streams through a unit job
    // fed from the caller's buffers; each run of units between such units takes the waves of sketch_units (DESIGN.md 2.7)
    uint64_t limit = UINT64_MAX;
    if (params->min_copies <= 1) MG_TRY(unit_stream_limit(ctx, &limit));
    mashgpu_sketch_params q = *params;
    q.target_cov = 0;                    // not a reads-mode setting: ignored here as in the waves
    for (uint64_t u0 = 0; u0 < n_units;) {
        if (unit_bytes[u0] > limit) {
            const uint64_t rb = unit_rec_begin[u0];
            MG_TRY(sketch_unit_streamed(ctx, &q, unit_rec_begin[u0 + 1] - rb, seq + rb, len + rb, out_hashes + u0 * s,
                                        out_counts ? out_counts + u0 * s : nullptr, out_n + u0, out_length ? out_length + u0 : nullptr, nullptr));
            u0++;
            continue;
        }
        uint64_t u1 = u0 + 1;
        while (u1 < n_units && unit_bytes[u1] <= limit) u1++;
        MG_TRY(sketch_units(ctx, params, seq, len, unit_rec_begin.data(), unit_bytes.data(), u0, u1, out_hashes, out_counts, out_n));
        u0 = u1;
    }
    return MASHGPU_OK;
}

extern "C" int mashgpu_sketch_batch_packed(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                                           const uint64_t *codes, uint64_t stream_len, const uint64_t *runs, uint64_t n_runs,
                                           const uint64_t *unit_start, uint64_t n_units,
                                           uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    MG_TRY(validate_sketch_params(ctx, params));
    if (n_units == 0) return MASHGPU_OK;
    if (!is_dna_alphabet(params)) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "the packed source only carries the alphabet {A,C,G,T}");
    if (!codes || !unit_start || !out_hashes || !out_n || (n_runs && !runs)) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    if (n_units > 0xFFFFFFF0ull) return fail(ctx, MASHGPU_ERR_INVALID, "too many units");
    for (uint64_t u = 0; u < n_units; u++)
        if (unit_start[u + 1] < unit_start[u]) return fail(ctx, MASHGPU_ERR_INVALID, "unit_start must be ascending");
    if (unit_start[n_units] > stream_len) return fail(ctx, MASHGPU_ERR_INVALID, "unit_start exceeds stream_len");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint32_t s = params->sketch_size;
    // waves of whole units, each starting at the 32-position group that holds its first unit's first position
    struct PWave { uint64_t u0, u1, g0, g1; };      // units [u0, u1), groups [g0, g1)
    const WaveLimits lim = wave_limits(s);
    std::vector<PWave> waves;
    for (uint64_t u = 0; u < n_units;) {
        uint64_t v = u + 1;
        while (v < n_units && v - u < lim.units && unit_start[v + 1] - unit_start[u] <= lim.bytes) v++;
        waves.push_back(PWave{u, v, unit_start[u] / 32, (unit_start[v] + 31) / 32});
        u = v;
    }
    uint64_t max_groups = 1, max_units = 1;
    for (auto &w : waves) { max_groups = std::max(max_groups, w.g1 - w.g0); max_units = std::max(max_units, w.u1 - w.u0); }
    const int nbuf = waves.size() > 1 ? 2 : 1;
    PackedSlots slots;
    MG_TRY(packed_slots(ctx, nbuf, max_groups * 32, slots));
    WaveOut out{out_hashes, out_counts, out_n};
    MG_TRY(wave_outputs(ctx, s, max_units, out));

    std::vector<PackRun> wruns[2];
    std::vector<uint64_t> wstart[2];
    uint64_t run_cursor = 0;        // first run that may still reach into the current wave (runs ascending)
    auto upload = [&](size_t wi) -> int {
        const PWave &w = waves[wi];
        const int b = (int)(wi % nbuf);
        const uint64_t p0 = w.g0 * 32, p1 = unit_start[w.u1];           // wave-local position = position - p0
        std::vector<PackRun> &R = wruns[b];
        R.clear();
        if (unit_start[w.u0] > p0) R.push_back(PackRun{0, unit_start[w.u0] - p0});       // the tail of the previous unit in the first group
        while (run_cursor < n_runs && runs[2 * run_cursor] + runs[2 * run_cursor + 1] <= unit_start[w.u0]) run_cursor++;
        for (uint64_t r = run_cursor; r < n_runs && runs[2 * r] < p1; r++) {
            const uint64_t a = std::max(runs[2 * r], unit_start[w.u0]), e = std::min(runs[2 * r] + runs[2 * r + 1], p1);
            if (e > a) R.push_back(PackRun{a - p0, e - a});
        }
        R.push_back(PackRun{p1 - p0, slots.groups * 32 - (p1 - p0)});                  // everything past the wave's last unit
        const int rc = upload_packed(ctx, slots, b, codes + w.g0, w.g1 - w.g0, R);
        if (rc != MASHGPU_OK) return fail(ctx, rc, "packed upload failed");
        ctx->kernel_launches++;             // apply_runs_kernel
        wstart[b].resize(w.u1 - w.u0 + 1);
        for (uint64_t u = w.u0; u <= w.u1; u++) wstart[b][u - w.u0] = unit_start[u] - p0;
        return MASHGPU_OK;
    };
    MG_TRY(upload(0));
    int rc = MASHGPU_OK;
    for (size_t wi = 0; wi < waves.size() && rc == MASHGPU_OK; wi++) {
        const PWave &w = waves[wi];
        const int b = (int)(wi % nbuf);
        if (wi + 1 < waves.size()) {
            // buffer (wi+1)%2 was last read by the kernels of wave wi-1 (synchronised below); its run list by upload(wi-1)
            if (wi >= 1) MG_CUDA(ctx, cudaEventSynchronize(ctx->pack_copied[(wi + 1) % nbuf]));
            rc = upload(wi + 1);
            if (rc != MASHGPU_OK) break;
        }
        MG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, ctx->pack_copied[b], 0));
        SketchStream S;
        S.d_codes = slots.d_codes[b]; S.d_inval = slots.d_inval[b]; S.unit_start = wstart[b].data(); S.n_units = w.u1 - w.u0;
        rc = sketch_wave(ctx, params, S, w.u0, out);
    }
    cudaStreamSynchronize(ctx->pack_stream);
    return rc;
}

// ---------------------------------------------------------------------------------------------------------
// `mash sketch -r [-m] [-c] [-b]`: a streaming reads job, replayed exactly through the reference's heap (DESIGN.md 2.6).
//
// MinHashHeap::tryInsert only looks at a k-mer when the heap is not full or its hash is below the heap's top (MinHashHeap.cpp:70-74),
// and once the heap is full the top never rises.  So the top at the start of any stretch of the stream (no limit while the heap is
// not full) bounds every k-mer of the stretch that can change the heap.  Each stretch of a staged buffer is scanned once with that
// threshold (SCAN_EVENTS); the events {position, hash} are sorted by position and replayed by reads_replay_kernel -- a faithful,
// sequential restatement of MinHashHeap::tryInsert (MinHashHeap.cpp:68-146, the Bloom branch :78-95 included) with the stop test of
// Sketch.cpp:1258-1262 -- through a replay state that stays in device memory for the whole job.  Device memory is fixed by the
// parameters (staging, event buffers, O(s + pending) replay tables, the Bloom bits), never by the size of the read set.
// ---------------------------------------------------------------------------------------------------------
namespace mashgpu {

struct ReplayMap { uint64_t *key; uint32_t *cnt; uint64_t mask; };     // open addressing, cnt == 0 marks a free slot

__device__ __forceinline__ uint64_t rm_slot(const ReplayMap &m, uint64_t key) { return ((key * 0x9E3779B97F4A7C15ULL) >> 11) & m.mask; }
__device__ uint32_t *rm_find(const ReplayMap &m, uint64_t key)
{
    uint64_t i = rm_slot(m, key);
    while (m.cnt[i]) {
        if (m.key[i] == key) return &m.cnt[i];
        i = (i + 1) & m.mask;
    }
    return nullptr;
}
__device__ void rm_insert_new(const ReplayMap &m, uint64_t key, uint32_t cnt)
{
    uint64_t i = rm_slot(m, key);
    while (m.cnt[i]) i = (i + 1) & m.mask;
    m.key[i] = key; m.cnt[i] = cnt;
}
__device__ void rm_erase(const ReplayMap &m, uint64_t key)      // backward-shift deletion
{
    uint64_t i = rm_slot(m, key);
    while (m.cnt[i] && m.key[i] != key) i = (i + 1) & m.mask;
    if (!m.cnt[i]) return;
    uint64_t j = i;
    for (;;) {
        j = (j + 1) & m.mask;
        if (!m.cnt[j]) break;
        const uint64_t k = rm_slot(m, m.key[j]);
        const bool between = (i <= j) ? (i < k && k <= j) : (i < k || k <= j);
        if (!between) { m.key[i] = m.key[j]; m.cnt[i] = m.cnt[j]; i = j; }
    }
    m.cnt[i] = 0;
}
__device__ void rh_push(uint64_t *heap, uint64_t &n, uint64_t v)     // binary max-heap
{
    uint64_t i = n++;
    while (i > 0) {
        const uint64_t p = (i - 1) / 2;
        if (heap[p] >= v) break;
        heap[i] = heap[p]; i = p;
    }
    heap[i] = v;
}
__device__ void rh_pop(uint64_t *heap, uint64_t &n)
{
    const uint64_t v = heap[--n];
    uint64_t i = 0;
    for (;;) {
        uint64_t c = 2 * i + 1;
        if (c >= n) break;
        if (c + 1 < n && heap[c + 1] > heap[c]) c++;
        if (heap[c] <= v) break;
        heap[i] = heap[c]; i = c;
    }
    if (n) heap[i] = v;
}

constexpr uint64_t NO_RECORD = ~0ull;

// The heap between launches.  acc = hashes + hashesQueue, pend = hashesPending + hashesQueuePending of MinHashHeap.
struct ReplayState {
    uint64_t size, heap_n, pend_n, msum;
    uint64_t cur;                   // record of the last event that passed the gate and has not had its stop test yet
    uint64_t used;                  // records used, once stopped
    uint64_t gate_t;                // EMPTY_KEY while the heap is not full, else its top: the scan threshold of the next stretch
    unsigned long long ev_count;    // events of the last scan (may exceed the buffer: the stretch is then split)
    uint32_t stopped;
};

// Bloom filter of MinHashHeap(use64, s, 1, b) (bloom_filter.hpp with false_positive_probability 0): one hash function, 8 b bits,
// salt = predef_salt[0]^2 + (uint32)(random_seed * 0xA5A5A5A5 + 1) with the default random_seed, bit = hash_ap(key) mod 8 b
// (the 32-bit hash_ap reaches only the first 2^32 bits).  The key is the hash's 8 little-endian bytes, or 4 with 32-bit hashes.
constexpr uint32_t BLOOM_SALT = 0x9A0876E7u;
constexpr uint64_t BLOOM_MAX_BYTES = 1ull << 29;

__host__ __device__ inline uint32_t bloom_hash_ap(uint64_t key, bool use64)
{
    uint32_t h = BLOOM_SALT;
    const uint32_t i1 = (uint32_t)key, i2 = (uint32_t)(key >> 32);
    if (use64) h ^= (h << 7) ^ i1 * (h >> 3) ^ (~((h << 11) + (i2 ^ (h >> 5))));    // one 8-byte block
    else h ^= ~((h << 11) + (i1 ^ (h >> 5)));                                        // the 4-byte tail, loop == 0
    return h;
}

// After the sort: the record of every event (first record whose separator lies after the position) and its Bloom bit.
__global__ void reads_event_meta_kernel(uint64_t *ev_pos_to_rec, const uint64_t *ev_hash, uint64_t n_ev, const uint64_t *rec_end,
                                        uint64_t n_rec, uint64_t rec_base, uint64_t bloom_bits, int use64, uint32_t *ev_bit)
{
    const uint64_t e = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (e >= n_ev) return;
    const uint64_t pos = ev_pos_to_rec[e];
    uint64_t lo = 0, hi = n_rec;
    while (lo < hi) { const uint64_t mid = (lo + hi) >> 1; if (rec_end[mid] <= pos) lo = mid + 1; else hi = mid; }
    ev_pos_to_rec[e] = rec_base + lo;
    if (bloom_bits) ev_bit[e] = (uint32_t)(bloom_hash_ap(ev_hash[e], use64) % bloom_bits);
}

__global__ void reads_fill_tmax_kernel(uint64_t *tile_tmax, uint64_t t0, uint64_t t1, const ReplayState *st)
{
    const uint64_t t = t0 + blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t < t1) tile_tmax[t] = st->gate_t;
}

__device__ __forceinline__ bool reads_stop_test(ReplayState &S, double target_cov)
{
    if (S.cur == NO_RECORD) return false;
    const bool stop = target_cov > 0 && S.size && (double)S.msum / (double)S.size >= target_cov;      // Sketch.cpp:1258-1262
    if (stop) { S.used = S.cur + 1; S.stopped = 1; }
    S.cur = NO_RECORD;
    return stop;
}

// One warp replays the events in order.  The heap's state only changes at events that pass its gate, so the stop test of record r
// (after its last k-mer) is due when the next passing event lies in a later record, or at the end of a feed.  Lanes load 32 events
// at a time and vote on the gate with the current top; lane 0 applies the passing ones one by one (the top only falls, so an
// event that fails the vote fails the gate at its turn too).
__global__ void reads_replay_kernel(ReplayState *state, const uint64_t *ev_rec, const uint64_t *ev_hash, const uint32_t *ev_bit, uint64_t n_ev,
                                    uint32_t s, uint32_t m, double target_cov, ReplayMap acc, uint64_t *acc_heap, ReplayMap pend, uint64_t *pend_heap,
                                    uint32_t *bloom)
{
    if (blockIdx.x) return;
    const uint32_t lane = threadIdx.x;
    ReplayState S = *state;
    if (S.stopped) return;
    bool stopped = false;
    for (uint64_t base = 0; base < n_ev && !stopped; base += 32) {
        const uint64_t e = base + lane;
        const bool valid = e < n_ev;
        const uint64_t h = valid ? ev_hash[e] : 0, r = valid ? ev_rec[e] : 0;
        const uint32_t bit = (valid && bloom) ? ev_bit[e] : 0;
        uint32_t todo = __ballot_sync(0xFFFFFFFFu, valid);
        for (;;) {
            const uint64_t size = __shfl_sync(0xFFFFFFFFu, S.size, 0), top = __shfl_sync(0xFFFFFFFFu, S.gate_t, 0);
            const uint32_t pass = __ballot_sync(0xFFFFFFFFu, valid && (size < s || h < top)) & todo;     // MinHashHeap.cpp:70-74
            if (!pass) break;
            const int src = __ffs(pass) - 1;
            todo &= ~((2u << src) - 1u);
            const uint64_t hash = __shfl_sync(0xFFFFFFFFu, h, src), rec = __shfl_sync(0xFFFFFFFFu, r, src);
            const uint32_t b = __shfl_sync(0xFFFFFFFFu, bit, src);
            int stop = 0;
            if (lane == 0) {
                if (S.cur != rec && reads_stop_test(S, target_cov)) stop = 1;
                else {
                    S.cur = rec;
                    uint32_t *c = rm_find(acc, hash);
                    if (!c) {
                        if (bloom) {                                        // :78-95
                            const uint32_t w = b >> 5, mask = 1u << (b & 31);
                            if (bloom[w] & mask) {
                                rm_insert_new(acc, hash, 2);
                                rh_push(acc_heap, S.heap_n, hash);
                                S.size++; S.msum += 2;
                            } else bloom[w] |= mask;
                        } else {
                            uint32_t *pc = m > 1 ? rm_find(pend, hash) : nullptr;
                            const uint64_t pending = pc ? *pc : 0;
                            if (m == 1 || pending == m - 1) {               // :96-108
                                rm_insert_new(acc, hash, m);
                                rh_push(acc_heap, S.heap_n, hash);
                                S.size++; S.msum += m;
                                if (m > 1 && pc) rm_erase(pend, hash);
                            } else if (!pc) {                               // :110-118
                                rh_push(pend_heap, S.pend_n, hash);
                                rm_insert_new(pend, hash, 1);
                            } else (*pc)++;
                        }
                    } else { (*c)++; S.msum++; }                            // :120-124
                    if (S.size > s) {                                       // :126-144
                        const uint64_t t = acc_heap[0];
                        uint32_t *tc = rm_find(acc, t);
                        S.msum -= tc ? *tc : 0;
                        rm_erase(acc, t);
                        while (S.pend_n > 0 && t < pend_heap[0]) {
                            if (rm_find(pend, pend_heap[0])) rm_erase(pend, pend_heap[0]);
                            rh_pop(pend_heap, S.pend_n);
                        }
                        rh_pop(acc_heap, S.heap_n);
                        S.size--;
                    }
                    S.gate_t = S.size >= s ? acc_heap[0] : EMPTY_KEY;
                }
            }
            if (__shfl_sync(0xFFFFFFFFu, stop, 0)) { stopped = true; break; }
        }
    }
    if (lane == 0) *state = S;
}

// The stop test of the last record of a feed (a feed always ends with a whole record).
__global__ void reads_feed_end_kernel(ReplayState *state, double target_cov)
{
    ReplayState S = *state;
    if (!S.stopped) reads_stop_test(S, target_cov);
    *state = S;
}

// Pending map growth: re-insert every entry of the old table into the new one (keys are distinct).
__global__ void reads_rehash_kernel(ReplayMap from, ReplayMap to)
{
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i <= from.mask; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t c = from.cnt[i];
        if (!c) continue;
        const uint64_t key = from.key[i];
        uint64_t j = ((key * 0x9E3779B97F4A7C15ULL) >> 11) & to.mask;
        while (atomicCAS(&to.cnt[j], 0u, c) != 0u) j = (j + 1) & to.mask;
        to.key[j] = key;
    }
}

// toHashList: ascending hashes + counts (HashSet.cpp:78-118); popping a copy of the max-heap yields them in descending order (the
// job's own heap stays intact, so finish may be called again)
__global__ void reads_emit_kernel(const ReplayState *state, ReplayMap acc, const uint64_t *acc_heap, uint64_t *heap_copy,
                                  uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n)
{
    if (blockIdx.x || threadIdx.x) return;
    uint64_t n = state->heap_n;
    for (uint64_t i = 0; i < n; i++) heap_copy[i] = acc_heap[i];
    const uint64_t size = state->size;
    *out_n = (uint32_t)size;
    for (uint64_t i = size; i-- > 0;) {
        const uint64_t v = heap_copy[0];
        out_hashes[i] = v;
        const uint32_t *c = rm_find(acc, v);
        out_counts[i] = c ? *c : 0;
        rh_pop(heap_copy, n);
    }
}

// Pinned staging of whole records for the streaming jobs (reads and unit jobs): kept records back to back, one separator byte after
// each, and the offsets of those separators.  A record longer than the space left is split; the buffer after the split starts with
// its last k-1 bases (the carry), so each window of the record lies whole in exactly one stage.  With two buffers the caller fills
// one while the other is still being copied to the device.
struct RecordStage {
    PinnedBuf<uint8_t> buf[2];
    int nbuf = 1, cur = 0;
    uint64_t cap = 0, k = 0, fill = 0;
    uint64_t records = 0, bases = 0;    // kept records staged so far and the sum of their lengths
    std::vector<uint64_t> rec_end;      // separator offsets of the records that end in the current buffer
    std::vector<uint8_t> carry;         // the last k-1 bases of a record split across stages
    uint8_t *h() { return buf[cur].p; }
    cudaError_t open(uint64_t cap_, uint64_t k_, int nbuf_)
    {
        cap = cap_; k = k_; nbuf = nbuf_;
        for (int b = 0; b < nbuf; b++)
            if (const cudaError_t e = buf[b].alloc(cap)) return e;
        return cudaSuccess;
    }
};

// Hand the current buffer (fill bytes, rec_end) to `process`; keep the last k-1 bases when a record continues into the next stage.
template <typename F>
static int stage_flush(RecordStage &S, bool record_continues, F &&process)
{
    if (record_continues) {
        const uint64_t keep = std::min<uint64_t>(S.k - 1, S.fill);
        S.carry.assign(S.h() + S.fill - keep, S.h() + S.fill);
    } else S.carry.clear();
    MG_TRY(process());
    S.rec_end.clear();
    S.fill = 0;
    S.cur = (S.cur + 1) % S.nbuf;
    if (!S.carry.empty()) { memcpy(S.h(), S.carry.data(), S.carry.size()); S.fill = S.carry.size(); }
    return MASHGPU_OK;
}

// Stage the next records in order (those shorter than k are skipped, Sketch.cpp:1222-1226); flush(record_continues) runs whenever
// the buffer is full, and staging ends early once stopped() holds.
template <typename Flush, typename Stopped>
static int stage_records(RecordStage &S, uint64_t n_records, const char *const *seq, const uint64_t *len, Flush &&flush, Stopped &&stopped)
{
    for (uint64_t r = 0; r < n_records && !stopped(); r++) {
        if (len[r] < S.k) continue;
        if (S.fill + len[r] + 1 > S.cap && S.fill) MG_TRY(flush(false));
        if (stopped()) break;
        uint64_t done = 0;
        while (len[r] - done + 1 > S.cap - S.fill) {           // longer than the stage: split with a (k-1)-base overlap
            const uint64_t take = S.cap - S.fill;
            memcpy(S.h() + S.fill, seq[r] + done, take);
            S.fill += take; done += take;
            MG_TRY(flush(true));
            if (stopped()) break;
        }
        if (stopped()) break;
        memcpy(S.h() + S.fill, seq[r] + done, len[r] - done);
        S.fill += len[r] - done;
        S.rec_end.push_back(S.fill);
        S.h()[S.fill++] = 0;                                    // separator
        S.records++;
        S.bases += len[r];
    }
    return MASHGPU_OK;
}

}  // namespace mashgpu

struct mashgpu_reads_job {
    mashgpu_ctx *ctx = nullptr;
    mashgpu_sketch_params params{};
    uint32_t s = 0, m = 1;
    uint64_t k = 0;
    uint64_t ev_cap = 0, bloom_bits = 0;
    // staging: one pinned buffer (records: kept records fed, the ones before the stop once stopped), its device copy
    mashgpu::RecordStage stage;
    mashgpu::DevBuf<uint8_t> d_stage;
    mashgpu::DevBuf<uint64_t> d_rec_end, d_tmax;
    uint64_t rec_base = 0;          // kept records that ended in earlier stages
    // events
    mashgpu::DevBuf<uint64_t> ev_pos, ev_hash, ev_pos2, ev_hash2;
    mashgpu::DevBuf<uint32_t> ev_bit;
    mashgpu::DevBuf<uint8_t> sort_tmp;
    size_t sort_tmp_bytes = 0;
    // replay state
    mashgpu::DevBuf<mashgpu::ReplayState> d_state;
    mashgpu::PinnedBuf<mashgpu::ReplayState> h_state;
    mashgpu::DevBuf<uint64_t> a_key, a_heap, p_key, p_heap;
    mashgpu::DevBuf<uint32_t> a_cnt, p_cnt, bloom;
    uint64_t cap_a = 0, cap_p = 0, cap_ph = 0;
    uint64_t gate_t = mashgpu::EMPTY_KEY;   // host copy of the threshold as of the last read-back (an older top is a valid bound)
    bool stopped = false;
    cudaEvent_t replay_ev[2] = {nullptr, nullptr};
    uint64_t dev_bytes = 0;
};

namespace mashgpu {

static uint64_t env_u64(const char *name, uint64_t dflt, uint64_t lo)
{
    const char *env = getenv(name);
    return env ? std::max<uint64_t>(lo, strtoull(env, nullptr, 10)) : dflt;
}

// Pending tables for `extra` more entries at load <= 1/2 (grown on the device, before the replay launch that needs them).
static int reads_reserve_pending(mashgpu_reads_job *job, uint64_t pend_n, uint64_t extra)
{
    mashgpu_ctx *ctx = job->ctx;
    cudaStream_t st = ctx->stream;
    const uint64_t need = pend_n + extra;
    if (need + 2 > job->cap_ph) {
        uint64_t cap = std::max<uint64_t>(2 * job->cap_ph, need + 2);
        DevBuf<uint64_t> nh;
        if (!tracked_alloc(nh, cap, job->dev_bytes, ctx->reads_peak_bytes)) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (pending heap of %llu)", (unsigned long long)cap);
        if (pend_n) MG_CUDA(ctx, cudaMemcpyAsync(nh.p, job->p_heap.p, pend_n * 8, cudaMemcpyDeviceToDevice, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
        job->dev_bytes -= job->p_heap.n * 8;
        std::swap(job->p_heap.p, nh.p); std::swap(job->p_heap.n, nh.n);
        job->cap_ph = cap;
    }
    if (2 * need + 16 > job->cap_p) {
        uint64_t cap = std::max<uint64_t>(16, job->cap_p);
        while (cap < 2 * need + 16) cap <<= 1;
        DevBuf<uint64_t> nk; DevBuf<uint32_t> nc;
        if (!tracked_alloc(nk, cap, job->dev_bytes, ctx->reads_peak_bytes) || !tracked_alloc(nc, cap, job->dev_bytes, ctx->reads_peak_bytes)) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (pending map of %llu)", (unsigned long long)cap);
        MG_CUDA(ctx, cudaMemsetAsync(nc.p, 0, cap * 4, st));
        if (job->cap_p) {
            ReplayMap from{job->p_key.p, job->p_cnt.p, job->cap_p - 1}, to{nk.p, nc.p, cap - 1};
            reads_rehash_kernel<<<(unsigned)std::min<uint64_t>((job->cap_p + 255) / 256, (uint64_t)ctx->sm_count * 8), 256, 0, st>>>(from, to);
            ctx->kernel_launches++;
            MG_CUDA(ctx, cudaGetLastError());
        }
        MG_CUDA(ctx, cudaStreamSynchronize(st));
        job->dev_bytes -= job->p_key.n * 8 + job->p_cnt.n * 4;
        std::swap(job->p_key.p, nk.p); std::swap(job->p_key.n, nk.n);
        std::swap(job->p_cnt.p, nc.p); std::swap(job->p_cnt.n, nc.n);
        job->cap_p = cap;
    }
    return MASHGPU_OK;
}

// Scan, sort and replay the staged buffer, stretch by stretch.
static int reads_process_stage(mashgpu_reads_job *job)
{
    mashgpu_ctx *ctx = job->ctx;
    const mashgpu_sketch_params *p = &job->params;
    cudaStream_t st = ctx->stream;
    const uint64_t len = job->stage.fill;
    const uint64_t n_rec = job->stage.rec_end.size();
    if (len == 0 || job->stopped) return MASHGPU_OK;
    MG_CUDA(ctx, cudaMemcpyAsync(job->d_stage.p, job->stage.h(), len, cudaMemcpyHostToDevice, st));
    if (n_rec) MG_CUDA(ctx, cudaMemcpyAsync(job->d_rec_end.p, job->stage.rec_end.data(), n_rec * 8, cudaMemcpyHostToDevice, st));
    ScanArgs a = scan_base(p, job->d_stage.p, len);
    a.tile_tmax = job->d_tmax.p;
    a.mode = SCAN_EVENTS;
    a.unit_t = &job->d_state.p->gate_t;
    a.ev_pos = job->ev_pos.p; a.ev_hash = job->ev_hash.p; a.ev_count = &job->d_state.p->ev_count; a.ev_capacity = job->ev_cap;
    const uint64_t ntiles = (len + SCAN_TILE - 1) / SCAN_TILE;
    const double space = p->use64 ? 18446744073709551616.0 : 4294967296.0;
    const uint64_t budget = std::max<uint64_t>(SCAN_TILE, job->ev_cap / 4);     // expected events per stretch
    const uint32_t sort_bits = std::max(1u, ceil_log2(len + 1));
    uint64_t t0 = 0, span = 0;
    while (t0 < ntiles) {
        if (span == 0) {                     // stretch size from the threshold as of the last read-back
            const double f = job->gate_t == EMPTY_KEY ? 1.0 : std::max(1.0, (double)job->gate_t) / space;
            const double windows = std::max((double)(1 << 16), (double)budget / f);
            span = (uint64_t)std::min<double>((double)ntiles, std::ceil(windows / SCAN_TILE));
        }
        const uint64_t t1 = std::min(ntiles, t0 + std::max<uint64_t>(1, span));
        reads_fill_tmax_kernel<<<(unsigned)((t1 - t0 + 255) / 256), 256, 0, st>>>(job->d_tmax.p, t0, t1, job->d_state.p);
        ctx->kernel_launches++;
        MG_CUDA(ctx, cudaMemsetAsync(&job->d_state.p->ev_count, 0, sizeof(unsigned long long), st));
        a.tile_begin = t0; a.tile_end = t1;
        MG_TRY(launch_scan(ctx, p, a, st));
        MG_CUDA(ctx, cudaMemcpyAsync(job->h_state.p, job->d_state.p, sizeof(ReplayState), cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
        const ReplayState H = *job->h_state.p;
        if (H.stopped) break;                // the previous stretch's replay reached the target coverage
        job->gate_t = H.gate_t;
        const uint64_t n_ev = H.ev_count;
        if (n_ev > job->ev_cap) {            // more events than the buffer holds: split the stretch, its bytes are still resident
            span = std::max<uint64_t>(1, (t1 - t0) / 2);
            if (t1 - t0 == 1) return fail(ctx, MASHGPU_ERR_INVALID, "event buffer below one tile");
            continue;
        }
        if (n_ev) {
            MG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(job->sort_tmp.p, job->sort_tmp_bytes, job->ev_pos.p, job->ev_pos2.p, job->ev_hash.p,
                                                         job->ev_hash2.p, (int)n_ev, 0, (int)sort_bits, st));
            ctx->kernel_launches += 4;
            reads_event_meta_kernel<<<(unsigned)((n_ev + 255) / 256), 256, 0, st>>>(job->ev_pos2.p, job->ev_hash2.p, n_ev, job->d_rec_end.p, n_rec,
                                                                                    job->rec_base, job->bloom_bits, p->use64, job->ev_bit.p);
            ctx->kernel_launches++;
            if (job->m > 1 && !job->bloom_bits) MG_TRY(reads_reserve_pending(job, H.pend_n, n_ev));
            ReplayMap acc{job->a_key.p, job->a_cnt.p, job->cap_a - 1}, pend{job->p_key.p, job->p_cnt.p, job->cap_p ? job->cap_p - 1 : 0};
            if (ctx->timing) MG_CUDA(ctx, cudaEventRecord(job->replay_ev[0], st));
            reads_replay_kernel<<<1, 32, 0, st>>>(job->d_state.p, job->ev_pos2.p, job->ev_hash2.p, job->ev_bit.p, n_ev, job->s, job->m,
                                                  p->target_cov, acc, job->a_heap.p, pend, job->p_heap.p, job->bloom_bits ? job->bloom.p : nullptr);
            ctx->kernel_launches++;
            MG_CUDA(ctx, cudaGetLastError());
            if (ctx->timing) {
                MG_CUDA(ctx, cudaEventRecord(job->replay_ev[1], st));
                MG_CUDA(ctx, cudaEventSynchronize(job->replay_ev[1]));
                float ms = 0;
                cudaEventElapsedTime(&ms, job->replay_ev[0], job->replay_ev[1]);
                ctx->reads_replay_ms += ms;
            }
            ctx->reads_events += n_ev;
        }
        t0 = t1;
        span = 0;
    }
    return MASHGPU_OK;
}

// Hand the staged buffer to the device; keep the last k-1 bases when a record continues into the next stage.
static int reads_flush(mashgpu_reads_job *job, bool record_continues)
{
    return stage_flush(job->stage, record_continues, [&]() -> int {
        MG_TRY(reads_process_stage(job));
        MG_CUDA(job->ctx, cudaMemcpyAsync(job->h_state.p, job->d_state.p, sizeof(ReplayState), cudaMemcpyDeviceToHost, job->ctx->stream));
        MG_CUDA(job->ctx, cudaStreamSynchronize(job->ctx->stream));
        if (job->h_state.p->stopped) job->stopped = true;
        job->rec_base += job->stage.rec_end.size();
        return MASHGPU_OK;
    });
}

}  // namespace mashgpu

extern "C" int mashgpu_reads_open(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, mashgpu_reads_job **out)
{
    using namespace mashgpu;
    if (!ctx || !out) return MASHGPU_ERR_INVALID;
    *out = nullptr;
    MG_TRY(validate_sketch_params(ctx, params, true));
    if (!is_dna_alphabet(params)) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "reads mode is only provided for the alphabet {A,C,G,T}");
    if (params->bloom_bytes && params->min_copies > 1)
        return fail(ctx, MASHGPU_ERR_INVALID, "bloom_bytes (-b) and min_copies (-m) > 1 exclude each other (as in the reference CLI)");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    auto *job = new mashgpu_reads_job();
    std::unique_ptr<mashgpu_reads_job> guard(job);
    job->ctx = ctx;
    job->params = *params;
    job->s = params->sketch_size;
    job->m = std::max(1u, params->min_copies);
    job->k = (uint64_t)params->kmer_size;
    const uint64_t stage_cap = env_u64("MASHGPU_READS_STAGE_BYTES", 128ull << 20, 4 * job->k + 64);
    job->ev_cap = std::min<uint64_t>(env_u64("MASHGPU_READS_EVENT_CAP", 1ull << 21, SCAN_TILE), 1ull << 30);    // cub takes int counts
    job->bloom_bits = params->bloom_bytes * 8;
    ctx->reads_peak_bytes = 0;
    cudaStream_t st = ctx->stream;
    const uint64_t max_rec = stage_cap / (job->k + 1) + 2;
    const uint64_t max_tiles = (stage_cap + SCAN_TILE - 1) / SCAN_TILE;
    job->cap_a = 16;
    while (job->cap_a < 4ull * (job->s + 2)) job->cap_a <<= 1;
    cub::DeviceRadixSort::SortPairs(nullptr, job->sort_tmp_bytes, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint64_t *)nullptr, (uint64_t *)nullptr,
                                    (int)job->ev_cap, 0, 64, st);
    if (job->stage.open(stage_cap, job->k, 1) != cudaSuccess || job->h_state.alloc(1) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory");
    auto alloc = [&](auto &b, size_t n) { return tracked_alloc(b, n, job->dev_bytes, ctx->reads_peak_bytes); };
    if (!alloc(job->d_stage, ((stage_cap + 15) / 16) * 16 + 64) || !alloc(job->d_rec_end, max_rec) ||
        !alloc(job->d_tmax, max_tiles) || !alloc(job->ev_pos, job->ev_cap) || !alloc(job->ev_hash, job->ev_cap) ||
        !alloc(job->ev_pos2, job->ev_cap) || !alloc(job->ev_hash2, job->ev_cap) || (job->bloom_bits && !alloc(job->ev_bit, job->ev_cap)) ||
        !alloc(job->sort_tmp, job->sort_tmp_bytes) || !alloc(job->d_state, 1) || !alloc(job->a_key, job->cap_a) ||
        !alloc(job->a_cnt, job->cap_a) || !alloc(job->a_heap, job->s + 2) ||
        (job->bloom_bits && !alloc(job->bloom, (std::min(params->bloom_bytes, BLOOM_MAX_BYTES) + 3) / 4)))
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (reads job)");
    MG_CUDA(ctx, cudaMemsetAsync(job->a_cnt.p, 0, job->cap_a * 4, st));
    if (job->bloom_bits) MG_CUDA(ctx, cudaMemsetAsync(job->bloom.p, 0, job->bloom.n * 4, st));
    ReplayState init;
    memset(&init, 0, sizeof init);
    init.cur = NO_RECORD; init.gate_t = EMPTY_KEY;
    *job->h_state.p = init;
    MG_CUDA(ctx, cudaMemcpyAsync(job->d_state.p, job->h_state.p, sizeof init, cudaMemcpyHostToDevice, st));
    if (job->m > 1 && !job->bloom_bits) MG_TRY(reads_reserve_pending(job, 0, 1024));
    MG_CUDA(ctx, cudaEventCreate(&job->replay_ev[0]));
    MG_CUDA(ctx, cudaEventCreate(&job->replay_ev[1]));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    *out = guard.release();
    return MASHGPU_OK;
}

extern "C" int mashgpu_reads_feed(mashgpu_reads_job *job, uint64_t n_records, const char *const *seq, const uint64_t *len, int *stopped)
{
    using namespace mashgpu;
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (n_records && (!seq || !len)) return fail(ctx, MASHGPU_ERR_INVALID, "seq/len is NULL");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_TRY(stage_records(job->stage, n_records, seq, len, [&](bool cont) { return reads_flush(job, cont); }, [&] { return job->stopped; }));
    if (!job->stopped && job->stage.fill) MG_TRY(reads_flush(job, false));
    if (!job->stopped) {
        reads_feed_end_kernel<<<1, 1, 0, ctx->stream>>>(job->d_state.p, job->params.target_cov);
        ctx->kernel_launches++;
        MG_CUDA(ctx, cudaGetLastError());
        MG_CUDA(ctx, cudaMemcpyAsync(job->h_state.p, job->d_state.p, sizeof(ReplayState), cudaMemcpyDeviceToHost, ctx->stream));
        MG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
        if (job->h_state.p->stopped) job->stopped = true;
    }
    if (stopped) *stopped = job->stopped ? 1 : 0;
    return MASHGPU_OK;
}

extern "C" int mashgpu_reads_finish(mashgpu_reads_job *job, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_records_used)
{
    using namespace mashgpu;
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (!out_hashes || !out_n || !out_records_used) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    DevBuf<uint64_t> d_hashes, d_heap; DevBuf<uint32_t> d_counts, d_n;
    if (d_hashes.alloc(job->s) != cudaSuccess || d_heap.alloc(job->s + 2) != cudaSuccess || d_counts.alloc(job->s) != cudaSuccess || d_n.alloc(1) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (outputs)");
    ReplayMap acc{job->a_key.p, job->a_cnt.p, job->cap_a - 1};
    reads_emit_kernel<<<1, 1, 0, st>>>(job->d_state.p, acc, job->a_heap.p, d_heap.p, d_hashes.p, d_counts.p, d_n.p);
    ctx->kernel_launches++;
    MG_CUDA(ctx, cudaGetLastError());
    uint32_t n = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&n, d_n.p, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(job->h_state.p, job->d_state.p, sizeof(ReplayState), cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    if (n) MG_CUDA(ctx, cudaMemcpyAsync(out_hashes, d_hashes.p, n * 8ull, cudaMemcpyDeviceToHost, st));
    if (n && out_counts) MG_CUDA(ctx, cudaMemcpyAsync(out_counts, d_counts.p, n * 4ull, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    *out_n = n;
    *out_records_used = job->h_state.p->stopped ? job->h_state.p->used : job->stage.records;
    return MASHGPU_OK;
}

extern "C" int mashgpu_reads_close(mashgpu_reads_job *job)
{
    if (!job) return MASHGPU_OK;
    cudaSetDevice(job->ctx->device);
    cudaStreamSynchronize(job->ctx->stream);
    for (cudaEvent_t &e : job->replay_ev) if (e) cudaEventDestroy(e);
    delete job;
    return MASHGPU_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Streaming unit job (mashgpu_unit_*, DESIGN.md 2.7): one sketchFile unit with minCov 1 and no Bloom filter, of any size, in device
// memory fixed by the parameters.  The bottom-s of a set does not depend on order, so each stage of the stream is sketched on its
// own by the single-unit pass, with the running s-th smallest hash as the cap of its threshold once s hashes are held, and its
// bottom-s (count, first and last position of each hash) is merged into the running state (unit_merge).
// ---------------------------------------------------------------------------------------------------------

struct mashgpu_unit_job {
    mashgpu_ctx *ctx = nullptr;
    mashgpu_sketch_params params{};
    uint32_t s = 0;
    mashgpu::RecordStage stage;                 // two pinned buffers: one fills while the other is copied
    mashgpu::DevBuf<uint8_t> d_stage[2];
    cudaEvent_t copied[2] = {nullptr, nullptr};
    int pending = -1;                           // buffer of the stage in flight (scanned or being scanned, not merged), -1 = none
    uint64_t next_base = 0;                     // global stream position of the next stage's first byte
    mashgpu::UnitPass pass;                     // the stage in flight: unit 0 of its buffer, positions + its global start
    mashgpu::UnitSketch sketch;                 // running state
    bool finished = false;
    uint64_t dev_bytes = 0;
};

namespace mashgpu {

// Finish the pending stage: exactness guard (re-scans while its bytes are resident), its bottom-s, and the merge.
static int unit_complete(mashgpu_unit_job *job)
{
    if (job->pending < 0) return MASHGPU_OK;
    MG_TRY(job->pass.finish());
    job->ctx->exact_reruns += job->pass.scans - 1;
    MG_TRY(unit_merge(job->pass, job->sketch));
    job->pending = -1;
    job->ctx->unit_stages++;
    return MASHGPU_OK;
}

// The current buffer is full (or the unit ends): copy it to the device, merge the stage before it (whose running top caps this
// stage's threshold), then enqueue this stage's scan.  The host fills the other buffer while the scan runs.
static int unit_process(mashgpu_unit_job *job)
{
    mashgpu_ctx *ctx = job->ctx;
    const int b = job->stage.cur;
    const uint64_t len = job->stage.fill;
    if (len == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaMemcpyAsync(job->d_stage[b].p, job->stage.h(), len, cudaMemcpyHostToDevice, ctx->copy_stream));
    MG_CUDA(ctx, cudaEventRecord(job->copied[b], ctx->copy_stream));
    MG_TRY(unit_complete(job));
    job->pending = b;
    UnitPass &P = job->pass;
    P.base = scan_base(&job->params, job->d_stage[b].p, len);
    P.hi = len;
    P.pos_base = job->next_base;
    job->next_base += len - job->stage.carry.size();      // the next stage starts with the carried k-1 bases
    const std::vector<uint64_t> &keys = job->sketch.keys;
    MG_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, job->copied[b], 0));
    return P.scan(SURVIVOR_FACTOR, keys.size() == job->s ? keys.back() : EMPTY_KEY);
}

static int unit_flush(mashgpu_unit_job *job, bool record_continues)
{
    return stage_flush(job->stage, record_continues, [&]() { return unit_process(job); });
}

// Device bytes of a one-unit stream above which the unit streams through a unit job (half of the free device memory, as
// sketch_reads_whole_set uses; MASHGPU_UNIT_STREAM_BYTES lowers it, for tests).
static int unit_stream_limit(mashgpu_ctx *ctx, uint64_t *limit)
{
    size_t free_b = 0, total_b = 0;
    MG_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    *limit = free_b / 2;
    if (const char *env = getenv("MASHGPU_UNIT_STREAM_BYTES")) *limit = std::min<uint64_t>(*limit, strtoull(env, nullptr, 10));
    return MASHGPU_OK;
}

// One unit through a unit job, fed from the caller's buffers.
static int sketch_unit_streamed(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, uint64_t n_records, const char *const *seq,
                                const uint64_t *len, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_length,
                                uint64_t *out_records)
{
    mashgpu_unit_job *job = nullptr;
    MG_TRY(mashgpu_unit_open(ctx, params, &job));
    uint64_t length = 0, records = 0;
    int rc = mashgpu_unit_feed(job, n_records, seq, len);
    if (rc == MASHGPU_OK) rc = mashgpu_unit_finish(job, out_hashes, out_counts, out_n, &length, &records);
    mashgpu_unit_close(job);
    if (out_length) *out_length = length;
    if (out_records) *out_records = records;
    return rc;
}

}  // namespace mashgpu

extern "C" int mashgpu_unit_open(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, mashgpu_unit_job **out)
{
    using namespace mashgpu;
    if (!ctx || !out) return MASHGPU_ERR_INVALID;
    *out = nullptr;
    MG_TRY(validate_sketch_params(ctx, params));
    if (params->min_copies > 1 || params->target_cov > 0)
        return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "the unit job takes neither min_copies (-m) > 1 nor target_cov (-c): use mashgpu_reads_*");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    auto *job = new mashgpu_unit_job();
    std::unique_ptr<mashgpu_unit_job> guard(job);
    job->ctx = ctx;
    job->params = *params;
    job->s = params->sketch_size;
    const uint64_t k = (uint64_t)params->kmer_size;
    const uint64_t stage_cap = env_u64("MASHGPU_UNIT_STAGE_BYTES", 128ull << 20, 4 * k + 64);
    ctx->unit_peak_bytes = 0;
    if (job->stage.open(stage_cap, k, 2) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory (unit job staging)");
    const uint64_t d_stage_bytes = ((stage_cap + 15) / 16) * 16 + 64;
    if (!tracked_alloc(job->d_stage[0], d_stage_bytes, job->dev_bytes, ctx->unit_peak_bytes) ||
        !tracked_alloc(job->d_stage[1], d_stage_bytes, job->dev_bytes, ctx->unit_peak_bytes))
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (unit job)");
    MG_TRY(job->pass.open(ctx, &job->params, ctx->stream, true, &job->dev_bytes, &ctx->unit_peak_bytes));
    // the table of any stage's first pass: a full stage, or a short one that plan_unit keeps whole (span <= 6 s)
    uint64_t t; uint32_t lg_full, lg_short;
    plan_unit(params, stage_cap, SURVIVOR_FACTOR, &t, &lg_full);
    plan_unit(params, std::min<uint64_t>(stage_cap, 2 * (uint64_t)(SURVIVOR_FACTOR * job->s) + 2), SURVIVOR_FACTOR, &t, &lg_short);
    MG_TRY(job->pass.reserve(std::max(lg_full, lg_short)));
    MG_CUDA(ctx, cudaEventCreateWithFlags(&job->copied[0], cudaEventDisableTiming));
    MG_CUDA(ctx, cudaEventCreateWithFlags(&job->copied[1], cudaEventDisableTiming));
    *out = guard.release();
    return MASHGPU_OK;
}

extern "C" int mashgpu_unit_feed(mashgpu_unit_job *job, uint64_t n_records, const char *const *seq, const uint64_t *len)
{
    using namespace mashgpu;
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (job->finished) return fail(ctx, MASHGPU_ERR_INVALID, "mashgpu_unit_feed after mashgpu_unit_finish");
    if (n_records && (!seq || !len)) return fail(ctx, MASHGPU_ERR_INVALID, "seq/len is NULL");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    return stage_records(job->stage, n_records, seq, len, [&](bool cont) { return unit_flush(job, cont); }, [] { return false; });
}

extern "C" int mashgpu_unit_finish(mashgpu_unit_job *job, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_length,
                                   uint64_t *out_records)
{
    using namespace mashgpu;
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (!out_hashes || !out_n || !out_length || !out_records) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (!job->finished) {
        if (job->stage.fill) MG_TRY(unit_flush(job, false));
        MG_TRY(unit_complete(job));
        job->finished = true;
    }
    const std::vector<uint64_t> &keys = job->sketch.keys;
    const size_t n = keys.size();
    std::copy(keys.begin(), keys.end(), out_hashes);
    if (out_counts) unit_counts(job->sketch, job->s, out_counts);
    *out_n = (uint32_t)n;
    *out_length = job->stage.bases;
    *out_records = job->stage.records;
    return MASHGPU_OK;
}

extern "C" int mashgpu_unit_close(mashgpu_unit_job *job)
{
    if (!job) return MASHGPU_OK;
    cudaSetDevice(job->ctx->device);
    cudaStreamSynchronize(job->ctx->stream);
    cudaStreamSynchronize(job->ctx->copy_stream);
    for (cudaEvent_t &e : job->copied) if (e) cudaEventDestroy(e);
    delete job;
    return MASHGPU_OK;
}

namespace mashgpu {

// Without -c and -b the heap's result does not depend on the order of the reads: the s smallest hashes seen at least m times, with
// the heap's multiplicities (DESIGN.md 2.6), which sketch_stream_core computes in one parallel pass.  A read set that fits in half
// of the free device memory is sketched that way in one resident stream (0.2 s against 1.2 s for the replay at -m 2 on 0.5 Gbp,
// DESIGN.md 2.6); MASHGPU_ERR_NOMEM sends a larger one to the streaming job.
static int sketch_reads_whole_set(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, uint64_t n_records, const char *const *seq,
                                  const uint64_t *len, uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_used)
{
    MG_TRY(validate_sketch_params(ctx, params, true));
    if (!is_dna_alphabet(params)) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "reads mode is only provided for the alphabet {A,C,G,T}");
    if (n_records && (!seq || !len)) return fail(ctx, MASHGPU_ERR_INVALID, "seq/len is NULL");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const uint32_t s = params->sketch_size;
    const uint64_t k = (uint64_t)params->kmer_size;
    uint64_t total = 0, n_rec = 0;
    for (uint64_t r = 0; r < n_records; r++)
        if (len[r] >= k) { total += len[r] + 1; n_rec++; }
    if (n_rec == 0) return MASHGPU_OK;
    uint64_t limit = 0;
    MG_TRY(unit_stream_limit(ctx, &limit));
    if (total > limit) return MASHGPU_ERR_NOMEM;
    DevBuf<uint8_t> d_stream; DevBuf<uint64_t> d_hashes; DevBuf<uint32_t> d_n, d_counts;
    if (d_stream.alloc(((total + 15) / 16) * 16 + 64) != cudaSuccess || d_hashes.alloc(s) != cudaSuccess || d_n.alloc(1) != cudaSuccess ||
        d_counts.alloc(s) != cudaSuccess)
        return MASHGPU_ERR_NOMEM;
    {
        const size_t chunk = 64ull << 20;
        PinnedBuf<uint8_t> stage[2];
        if (stage[0].alloc(chunk) != cudaSuccess || stage[1].alloc(chunk) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory");
        cudaEvent_t done[2];
        MG_CUDA(ctx, cudaEventCreateWithFlags(&done[0], cudaEventDisableTiming));
        MG_CUDA(ctx, cudaEventCreateWithFlags(&done[1], cudaEventDisableTiming));
        uint64_t fill = 0, base = 0;
        int b = 0;
        bool used_ev[2] = {false, false};
        auto flush = [&]() -> cudaError_t {           // double-buffered: the copy of one chunk overlaps the packing of the next
            if (!fill) return cudaSuccess;
            cudaError_t e = cudaMemcpyAsync(d_stream.p + base, stage[b].p, fill, cudaMemcpyHostToDevice, st);
            if (e != cudaSuccess) return e;
            e = cudaEventRecord(done[b], st);
            used_ev[b] = true;
            b ^= 1;
            if (used_ev[b]) cudaEventSynchronize(done[b]);
            base += fill; fill = 0;
            return e;
        };
        cudaError_t e = cudaSuccess;
        for (uint64_t r = 0; r < n_records && e == cudaSuccess; r++) {
            if (len[r] < k) continue;
            uint64_t done_r = 0;
            while (done_r < len[r] + 1 && e == cudaSuccess) {            // the record's bytes, then its separator
                const uint64_t take = std::min<uint64_t>(chunk - fill, len[r] + 1 - done_r);
                const uint64_t from_seq = done_r < len[r] ? std::min(take, len[r] - done_r) : 0;
                if (from_seq) memcpy(stage[b].p + fill, seq[r] + done_r, from_seq);
                if (take > from_seq) stage[b].p[fill + from_seq] = 0;
                fill += take; done_r += take;
                if (fill == chunk) e = flush();
            }
        }
        if (e == cudaSuccess) e = flush();
        cudaStreamSynchronize(st);
        cudaEventDestroy(done[0]); cudaEventDestroy(done[1]);
        if (e != cudaSuccess) return fail(ctx, MASHGPU_ERR_CUDA, "upload of the read set failed: %s", cudaGetErrorString(e));
    }
    uint64_t us[2] = {0, total};
    SketchStream S;
    S.d_stream = d_stream.p; S.unit_start = us; S.n_units = 1;
    MG_TRY(sketch_stream_core(ctx, params, S, d_hashes.p, out_counts ? d_counts.p : nullptr, d_n.p, st, nullptr));
    uint32_t n = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&n, d_n.p, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    if (n) MG_CUDA(ctx, cudaMemcpyAsync(out_hashes, d_hashes.p, n * 8ull, cudaMemcpyDeviceToHost, st));
    if (n && out_counts) MG_CUDA(ctx, cudaMemcpyAsync(out_counts, d_counts.p, n * 4ull, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    *out_n = n; *out_used = n_rec;
    return MASHGPU_OK;
}

}  // namespace mashgpu

extern "C" int mashgpu_sketch_reads(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                                    uint64_t n_records, const char *const *seq, const uint64_t *len,
                                    uint64_t *out_hashes, uint32_t *out_counts, uint32_t *out_n, uint64_t *out_records_used)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!out_hashes || !out_n || !out_records_used) return mashgpu::fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    *out_n = 0; *out_records_used = 0;
    if (params && params->bloom_bytes == 0 && !(params->target_cov > 0)) {
        const int rc = mashgpu::sketch_reads_whole_set(ctx, params, n_records, seq, len, out_hashes, out_counts, out_n, out_records_used);
        if (rc != MASHGPU_ERR_NOMEM) return rc;                     // too large for one resident stream: stream it through a job
        if (params->min_copies <= 1)                                // order-independent: the parallel unit job, not the replay
            return mashgpu::sketch_unit_streamed(ctx, params, n_records, seq, len, out_hashes, out_counts, out_n, nullptr, out_records_used);
    }
    mashgpu_reads_job *job = nullptr;
    MG_TRY(mashgpu_reads_open(ctx, params, &job));
    int rc = mashgpu_reads_feed(job, n_records, seq, len, nullptr);
    if (rc == MASHGPU_OK) rc = mashgpu_reads_finish(job, out_hashes, out_counts, out_n, out_records_used);
    mashgpu_reads_close(job);
    return rc;
}

extern "C" int mashgpu_host_pack(const mashgpu_sketch_params *params, uint64_t n_records, const char *const *seq, const uint64_t *len,
                                 int threads, uint64_t *codes, uint64_t *runs, uint64_t runs_capacity, uint64_t *n_runs)
{
    if (!params || !codes || !n_runs || (n_records && (!seq || !len))) return MASHGPU_ERR_INVALID;
    std::vector<PackSegment> segs;
    uint64_t off = 0;
    for (uint64_t r = 0; r < n_records; r++) {
        segs.push_back(PackSegment{(const uint8_t *)seq[r], off, len[r]});
        off += len[r] + 1;
    }
    std::vector<PackRun> found;
    pack_stream(segs.data(), segs.size(), off, params->preserve_case, threads, codes, found);
    *n_runs = found.size();
    for (uint64_t i = 0; i < found.size() && i < runs_capacity; i++) { runs[2 * i] = found[i].start; runs[2 * i + 1] = found[i].len; }
    return MASHGPU_OK;
}

extern "C" int mashgpu_hash_windows(mashgpu_ctx *ctx, const mashgpu_sketch_params *params,
                                    const char *seq, uint64_t len, uint64_t *out_hash, uint8_t *out_valid)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    MG_TRY(validate_sketch_params(ctx, params));
    const uint64_t k = (uint64_t)params->kmer_size;
    if (len < k) return MASHGPU_OK;
    if (!seq || !out_hash || !out_valid) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint64_t nwin = len - k + 1;
    DevBuf<uint8_t> d_seq, d_valid; DevBuf<uint64_t> d_hash;
    const uint64_t padded = ((len + 15) / 16) * 16;
    if (d_seq.alloc(padded) != cudaSuccess || d_valid.alloc(len) != cudaSuccess || d_hash.alloc(len) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory");
    cudaStream_t st = ctx->stream;
    MG_CUDA(ctx, cudaMemcpyAsync(d_seq.p, seq, len, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemsetAsync(d_valid.p, 0, len, st));
    MG_CUDA(ctx, cudaMemsetAsync(d_hash.p, 0, len * 8, st));
    ScanArgs a = scan_base(params, d_seq.p, len);
    a.coarse_t = EMPTY_KEY;
    a.mode = SCAN_DUMP;
    a.out_hash = d_hash.p; a.out_valid = d_valid.p;
    MG_TRY(launch_scan(ctx, params, a, st));
    MG_CUDA(ctx, cudaMemcpyAsync(out_hash, d_hash.p, nwin * 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(out_valid, d_valid.p, nwin, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    return MASHGPU_OK;
}
