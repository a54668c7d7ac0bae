// dist.cu -- hot path 2: all-pairs sketch comparison (C-ABI: mashgpu_dist_*).
//
// Replaces compare / compareSketches / pValue (reference CommandDistance.cpp:306-448).
//
// Data layout (DESIGN.md): at open time every hash of every sketch is replaced by its rank in the sorted set of
// all distinct hashes (an order- and equality-preserving 32-bit dictionary, built with one radix sort), and each
// sketch becomes a row of P = sketch_size+1 uint32 ranks padded with the sentinel 0xFFFFFFFF.  The merge kernel
// keeps a tile of 32 reference rows in shared memory, element-interleaved so that lane r only ever touches bank r,
// and streams query rows through per-warp shared buffers; each lane runs the reference's sequential merge for its
// (query, reference) pair for exactly sketch_size steps (every step adds one element to the union):
//      a <= b -> advance ref;  b <= a -> advance query;   common = i + j - steps.
// Steps that consume sentinels on both sides are the "list ran out" case of CommandDistance.cpp:367-385 and are
// subtracted afterwards.
//
// A run is three kernels (DESIGN.md 3.2-3.2c):
//   dist_probe_kernel  tile prefilter: a cuckoo filter over each 32-reference tile decides which (query, tile) combinations
//                      share a hash at all; the others get the closed form of an empty intersection for all 32 pairs
//   dist_kernel        the merge, on the tiles' work lists (or on every pair when the prefilter is off)
//   dist_fix_kernel    p-value / pass flag / pass-list entry of the pairs with shared hashes, evaluated densely
// Results are identical with and without the prefilter (tests/test_gpu_dist_prefilter.py).
// A best run (mashgpu_dist_run_best, DESIGN.md 3.7) runs the same kernels with no dense output: the two places that know a pair's
// final pass flag, dist_emit and dist_fix_kernel, capture the hits, and dist_best.cuh selects the N nearest of every query.
// A component run (mashgpu_dist_components, DESIGN.md 3.8) is the same again: at those two places dist_cc.cuh unions the two sketches
// of every hit of the lower triangle into a forest, whose roots become the components' labels.
// A spanning-forest run (mashgpu_dist_spanning_forest, DESIGN.md 3.9) repeats such runs in Boruvka rounds: at the same places
// dist_msf.cuh offers every hit to the cheapest-edge slots of its two components.
// Greedy dereplication (mashgpu_dist_representatives, DESIGN.md 3.12) runs the query rows in blocks, strictly in order: at the same
// places dist_greedy.cuh marks rows covered by earlier representatives and records each block's own edges in a bit matrix, which
// greedy_resolve_kernel decides in rounds; one more run offers each member its nearest representative.
// Neighbor joining (mashgpu_dist_neighbor_joining, DESIGN.md 3.10) and average / complete linkage (mashgpu_dist_linkage, 3.11)
// fill an n x n matrix with plain lower-triangle runs (distance output only) and hand it to nj.cu or linkage.cu.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cstdlib>
#include <chrono>
#include <memory>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

#include "common.cuh"
#include "binom.cuh"
#include "dict.cuh"
#include "dist_filter.cuh"
#include "dist_best.cuh"
#include "dist_cc.cuh"
#include "dist_msf.cuh"
#include "dist_greedy.cuh"
#include "linkage_cta.cuh"

namespace mashgpu {

struct FixEntry;
struct DistArgs {
    const uint32_t *ranks;      // rows of P ranks: references first, then queries (or shared when self)
    uint32_t P;                 // row pitch = sketch_size + 1
    uint32_t S;                 // sketch_size (merge steps)
    const uint32_t *ref_n;      // min(n_hashes, P) per reference row
    const uint32_t *qry_n;
    const uint64_t *ref_len;
    const uint64_t *qry_len;
    uint64_t ref_row0, qry_row0;   // first row of each set in `ranks`
    uint32_t n_ref;
    uint32_t q_begin, q_count;
    uint32_t q_per_cta;         // queries handled by one CTA (grid.y slices the query range)
    int kmer_size;
    double kmer_space, max_distance, max_pvalue;
    const double *dist_lut;     // distance for (common, denom == S), S+1 entries
    BinomTable binom;           // C(S, x) for the p-value of pairs with denom == S
    uint32_t *numer; uint32_t *denom; double *distance; double *pvalue; uint8_t *pass;   // outputs, (q - q_begin) * n_ref + r
    // compacted pass-list (filtered runs): passing pairs are appended in arbitrary order, then sorted by pair index
    uint64_t *list_idx; uint32_t *list_numer; uint32_t *list_denom; double *list_distance; double *list_pvalue;
    unsigned long long *list_count; uint64_t list_capacity;
    // prefilter work lists (dist_probe_kernel -> dist_kernel): per reference tile the queries that share a hash with it
    uint32_t *qlist; uint32_t *qcount; uint64_t qlist_stride; unsigned long long *flag_total;
    int triangle;               // lower triangle only: pairs with tri_r0 + r >= q are neither computed nor written
    uint32_t tri_r0;            // row of reference 0 in the query numbering (0 for a self comparison; the shard offset of an encoded job)
    int use_qlist;              // dist_kernel: take the queries of a tile from qlist instead of the dense range
    // sparse related pairs (dist_probe_kernel -> dist_pair_kernel): when a query may share hashes with at most pair_max references
    // of a tile, only those (query, reference) pairs are merged, one warp per pair, instead of all 32 in lockstep.  A warp reserves its
    // slots with one atomicAdd on pair_count; pair_full holds ~(start of the first reservation that did not fit), 0 while all fit
    // (complemented so that zeroed memory means "none" and atomicMax keeps the smallest start).  Slots from that start on may be
    // unwritten -- a reservation that straddles the capacity writes nothing -- and are not merged.
    uint2 *pair_list; unsigned long long *pair_count, *pair_full; uint64_t pair_capacity; unsigned long long *pair_total;
    int pair_max;               // 0: every flagged (query, tile) combination goes to the tile's work list
    int pair_dense;             // dist_pair_kernel enumerates every pair of the run itself (sketch sizes beyond the tiled merge)
    // deferred p-values (dist_fix_kernel): pairs with shared hashes whose binomial tail is evaluated in a dense second pass
    struct FixEntry *fix_list; unsigned long long *fix_count; uint64_t fix_capacity;
    BestCapture best;           // best runs: hits (pass, common > 0) are captured here; every dense output and the pass list are NULL then
    GraphCapture graph;         // component runs and spanning-forest rounds: hits are unioned or offered here (the sketches q and tri_r0 + r);
                                // NULL outputs and pass list, as for best
};

struct FixEntry { uint64_t o; uint32_t common, denom; };

__device__ __forceinline__ void dist_list_append(const DistArgs &a, uint64_t o, uint32_t common, uint32_t denom, double dist, double p)
{
    const unsigned long long at = atomicAdd(a.list_count, 1ull);
    if (at < a.list_capacity) {
        a.list_idx[at] = o; a.list_numer[at] = common; a.list_denom[at] = denom; a.list_distance[at] = dist; a.list_pvalue[at] = p;
    }
}

// distance of compareSketches (CommandDistance.cpp:387-407)
__device__ __forceinline__ double mash_distance(uint32_t common, uint32_t denom, int k)
{
    if (common == denom) return 0.0;
    if (common == 0) return 1.0;
    const double j = (double)common / (double)denom;
    double d = -log(2 * j / (1. + j)) / k;
    return d > 1 ? 1.0 : d;
}

// Epilogue of compareSketches for one pair (CommandDistance.cpp:387-424) given the merge result.
// The binomial tail of a pair with shared hashes costs more than its merge (up to `common` multiply-divide steps), and such
// pairs are a small, scattered minority of a large grid: evaluated in place they leave 31 lanes of the warp waiting (measured
// on configs[2] in shuffled order: 94 of 275 ms).  They are queued instead and dist_fix_kernel evaluates them densely; when
// the queue is full (data sets where most pairs share hashes -- then the lanes of a warp are busy together anyway) the tail
// is evaluated here.
__device__ __forceinline__ void dist_emit(const DistArgs &a, uint32_t q, uint32_t r, uint32_t common, uint32_t denom, uint64_t lenA)
{
    double dist = (denom == a.S) ? a.dist_lut[common] : mash_distance(common, denom, a.kmer_size);
    const uint64_t o = (uint64_t)(q - a.q_begin) * a.n_ref + r;
    bool pass = true, deferred = false;
    double p = 0.0;
    if (a.max_distance >= 0 && dist > a.max_distance) pass = false;     // CommandDistance.cpp:409-412
    else if (common == 0) {                                             // pValue: x == 0 -> 1 (:429-432)
        p = 1.0;
        if (a.max_pvalue >= 0 && p > a.max_pvalue) pass = false;
    } else {
        if (a.fix_list) {
            const unsigned long long at = atomicAdd(a.fix_count, 1ull);
            if (at < a.fix_capacity) {
                a.fix_list[at] = FixEntry{o, common, denom};
                deferred = true;
            }
        }
        if (!deferred) {
            p = mash_pvalue(common, lenA, a.qry_len[q], a.kmer_space, denom, &a.binom);
            if (a.max_pvalue >= 0 && p > a.max_pvalue) pass = false;    // :419-422
        }
    }
    if (a.numer) a.numer[o] = common;
    if (a.denom) a.denom[o] = denom;
    if (a.distance) a.distance[o] = dist;
    if (deferred) return;
    if (a.list_idx && pass) dist_list_append(a, o, common, denom, dist, p);
    if (a.best.cand && pass && common) dist_best_append(a.best, q - a.q_begin, r, common, denom, dist, p);
    if (a.graph.forest && pass && common) dist_graph_hit(a.graph, q, a.tri_r0 + r, dist);
    if (a.pvalue) a.pvalue[o] = p;
    if (a.pass) a.pass[o] = pass ? 1 : 0;
}

// second pass over the queued pairs: p-value, pass flag, pass-list entry
__global__ void __launch_bounds__(256) dist_fix_kernel(const DistArgs a)
{
    const unsigned long long queued = *a.fix_count;
    const uint64_t n = queued < a.fix_capacity ? queued : a.fix_capacity;
    for (uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; t < n; t += (uint64_t)gridDim.x * blockDim.x) {
        const FixEntry e = a.fix_list[t];
        const uint32_t q = a.q_begin + (uint32_t)(e.o / a.n_ref), r = (uint32_t)(e.o % a.n_ref);
        const double p = mash_pvalue(e.common, a.ref_len[r], a.qry_len[q], a.kmer_space, e.denom, &a.binom);
        const bool pass = !(a.max_pvalue >= 0 && p > a.max_pvalue);
        if ((a.list_idx || a.best.cand || a.graph.forest) && pass) {        // queued pairs share a hash
            const double dist = (e.denom == a.S) ? a.dist_lut[e.common] : mash_distance(e.common, e.denom, a.kmer_size);
            if (a.list_idx) dist_list_append(a, e.o, e.common, e.denom, dist, p);
            else if (a.best.cand) dist_best_append(a.best, q - a.q_begin, r, e.common, e.denom, dist, p);
            else dist_graph_hit(a.graph, q, a.tri_r0 + r, dist);
        }
        if (a.pvalue) a.pvalue[e.o] = p;
        if (a.pass) a.pass[e.o] = pass ? 1 : 0;
    }
}

// (reference tile and query rows: stage_ref_tile / bulk_span / bulk_copy_wait, layout: dist_qpitch / dist_smem_bytes, all in dict.cuh)
__global__ void __launch_bounds__(DIST_THREADS, 1) dist_kernel(const DistArgs a)
{
    extern __shared__ __align__(16) uint32_t smem[];
    const uint32_t qpitch = dist_qpitch(a.P);
    uint32_t *s_ref = smem;                                  // [P][32]
    uint32_t *s_qry = smem + (((size_t)a.P * DIST_TILE_R + 3) & ~(size_t)3);      // [DIST_WARPS][DIST_ILP][qpitch]
    uint64_t *s_bar = reinterpret_cast<uint64_t *>(s_qry + (size_t)DIST_WARPS * DIST_ILP * qpitch);     // one mbarrier per warp
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t r0 = blockIdx.x * DIST_TILE_R;
    const uint32_t r = r0 + lane;
    const bool r_ok = r < a.n_ref;

    // The CTA's items: the dense query range [q_begin, q_begin + q_count), or (prefiltered runs) the tile's work list.
    // Item index -> query: q_begin + item, or qlist[tile][item].  A CTA takes q_per_cta items at a time, gridDim.y apart.
    const uint32_t n_items = a.use_qlist ? a.qcount[blockIdx.x] : a.q_count;
    const uint32_t *my_list = a.use_qlist ? a.qlist + (uint64_t)blockIdx.x * a.qlist_stride : nullptr;
    if ((uint64_t)blockIdx.y * a.q_per_cta >= n_items) return;          // nothing to do: do not even stage the tile

    stage_ref_tile(s_ref, a.ranks, a.ref_row0, a.P, r0, a.n_ref);
    __syncthreads();
    const uint32_t nA = r_ok ? a.ref_n[r] : 0;
    const uint64_t lenA = r_ok ? a.ref_len[r] : 1;
    const uint32_t sref_base = (uint32_t)__cvta_generic_to_shared(s_ref) + lane * 4;
    uint32_t *my_q = s_qry + (size_t)warp * DIST_ILP * qpitch;
    const uint32_t bar = warp_bar_init(s_bar + warp);
    uint32_t phase = 0;

    for (uint64_t it_lo = (uint64_t)blockIdx.y * a.q_per_cta; it_lo < n_items; it_lo += (uint64_t)gridDim.y * a.q_per_cta) {
    const uint32_t it_hi = (uint32_t)min((uint64_t)n_items, it_lo + a.q_per_cta);
    for (uint32_t ib = (uint32_t)it_lo + warp * DIST_ILP; ib < it_hi; ib += DIST_WARPS * DIST_ILP) {
        uint32_t qs[DIST_ILP];
        bool all_skipped = true;
#pragma unroll
        for (int c = 0; c < DIST_ILP; c++) {
            const uint32_t item = ib + c;
            qs[c] = item < it_hi ? (my_list ? my_list[item] : a.q_begin + item) : 0xFFFFFFFFu;
            if (a.triangle && qs[c] <= a.tri_r0 + r0) qs[c] = 0xFFFFFFFFu;        // the whole tile lies on or above the diagonal
            all_skipped &= qs[c] == 0xFFFFFFFFu;
        }
        if (all_skipped) continue;                      // warp-uniform
        // load DIST_ILP query rows into this warp's buffers; a skipped one is padding (the merge still takes its S steps)
        uint32_t skew[DIST_ILP], bytes[DIST_ILP], total = 0;
        const uint32_t *src[DIST_ILP];
#pragma unroll
        for (int c = 0; c < DIST_ILP; c++) {
            skew[c] = 0; bytes[c] = 0; src[c] = nullptr;
            if (qs[c] != 0xFFFFFFFFu) {
                bytes[c] = bulk_span(a.ranks + (a.qry_row0 + qs[c]) * (uint64_t)a.P, a.P, src[c], skew[c]);
                total += bytes[c];
            } else {
                uint32_t *dst = my_q + (size_t)c * qpitch;
                for (uint32_t i = lane; i < a.P; i += 32) dst[i] = RANK_PAD;
            }
        }
        bulk_copy_wait(src, bytes, total, my_q, qpitch, bar, phase);
        uint32_t pa[DIST_ILP], pb[DIST_ILP], va[DIST_ILP], vb[DIST_ILP], pb0[DIST_ILP];
#pragma unroll
        for (int c = 0; c < DIST_ILP; c++) {
            pa[c] = sref_base;
            pb0[c] = pb[c] = (uint32_t)__cvta_generic_to_shared(my_q + (size_t)c * qpitch) + skew[c];
            va[c] = lds32(pa[c]);
            vb[c] = lds32(pb[c]);
        }
        // One merge step per chain = 6 instructions: 2 compares, 2 predicated pointer bumps, 2 predicated loads, written
        // as one PTX block so that the pointer update stays in place (the C++ form compiled to 9 instructions).
        // 9 -> 6 instructions and a 2-deep register lookahead that takes the LDS latency out of the dependent chain both
        // left the rate unchanged (tools/dist_probe.py) -- the kernel is bound by the shared-memory pipe: two
        // half-populated LDS wavefronts per warp-step, see DESIGN.md 3.3.
#pragma unroll 4
        for (uint32_t t = 0; t < a.S; t++) {
#pragma unroll
            for (int c = 0; c < DIST_ILP; c++) {
                asm volatile("{\n\t.reg .pred pa, pb;\n\t"
                             "setp.le.u32 pa, %0, %1;\n\t"
                             "setp.le.u32 pb, %1, %0;\n\t"
                             "@pa add.u32 %2, %2, 128;\n\t"
                             "@pb add.u32 %3, %3, 4;\n\t"
                             "@pa ld.shared.u32 %0, [%2];\n\t"
                             "@pb ld.shared.u32 %1, [%3];\n\t}"
                             : "+r"(va[c]), "+r"(vb[c]), "+r"(pa[c]), "+r"(pb[c]));
            }
        }
        // epilogue
#pragma unroll
        for (int c = 0; c < DIST_ILP; c++) {
            const uint32_t q = qs[c];
            if (q == 0xFFFFFFFFu || !r_ok || (a.triangle && a.tri_r0 + r >= q)) continue;
            const uint32_t i_end = (pa[c] - sref_base) / (DIST_TILE_R * 4);
            const uint32_t j_end = (pb[c] - pb0[c]) / 4;
            const uint32_t bogus = i_end > nA ? i_end - nA : 0;   // steps that consumed padding on both sides
            const uint32_t denom = a.S - bogus;
            const uint32_t common = (i_end - bogus) + (j_end - bogus) - denom;
            dist_emit(a, q, r, common, denom, lenA);
        }
        __syncwarp();
    }
    }
}

// ---------------------------------------------------------------------------------------------------------
// Prefilter: which (query, reference tile) combinations share a hash at all?
//
// For most pairs of a large all-vs-all run the answer of the merge is "no shared hash": common = 0, denom =
// min(s', |A| + |B|), distance 1, p-value 1 (CommandDistance.cpp:347-407 with an empty intersection).  One CTA builds a
// cuckoo filter (dist_filter.cuh) over the <= 32 x s' ranks of its reference tile, then streams the queries through it:
// a warp looks 32 ranks of a query up per step (two shared-memory loads each, no loop) instead of running 32 x s' merge
// steps.  A filter hit is confirmed exactly (each lane binary-searches the rank in its reference's row); the first
// confirmed hit puts the query on the tile's work list for dist_kernel and ends the query early.  Queries without a
// confirmed hit get the closed-form result for all 32 pairs written here.  Only ranks at index < s' take part: the merge
// cannot reach a match at a later index (it would need more than s' union steps).
// ---------------------------------------------------------------------------------------------------------
constexpr int PROBE_WARPS = 32;
constexpr int PROBE_THREADS = PROBE_WARPS * 32;
constexpr int PROBE_DEPTH = 4;          // 32-rank batches in flight per warp
constexpr int PROBE_MAX_CONFIRMS = 3;   // exact confirmations of shared-slot hits per (query, tile) before the combination is merged as a whole
constexpr size_t PROBE_SMEM = CF_BUCKETS * sizeof(uint32_t) + 2 * CF_BUCKETS;      // the filter + one owner byte per slot

// A filter hit somewhere in the group b[] (ranks base + 32 c + lane): which references of the tile may share it?  The id side
// table (dist_filter.cuh) names the reference when the fingerprint's slot belongs to one; slots shared by several references
// (the rule in a tile of related sketches) and, when the pair path is off, every hit are confirmed exactly: each lane
// binary-searches the rank in its own reference's row (global memory) and the ballot is the set of references that hold it.
// Returns the updated candidate mask; stops confirming once more than pair_max references are in it (the combination is merged
// as a whole then).
template <bool FULL>
__device__ __noinline__ uint2 probe_resolve(uint32_t b0, uint32_t b1, uint32_t b2, uint32_t b3, uint32_t base, uint32_t nB, const uint32_t *rowA,
                                            uint32_t nA_lim, uint32_t mask, int pair_max, int confirms)
{
    // (the filter's address, the lane and the running state travel in as few registers as possible: what is live across this call
    // is live across the caller's hot loop, and at 1024 threads per CTA the loop has 64 registers)
    extern __shared__ uint32_t s_tab[];
    const uint8_t *s_ids = reinterpret_cast<const uint8_t *>(s_tab + CF_BUCKETS);
    const int lane = threadIdx.x & 31;
    const uint32_t b[PROBE_DEPTH] = {b0, b1, b2, b3};      // by value: an array reference would pin the caller's ranks in local memory
#pragma unroll
    for (int c = 0; c < PROBE_DEPTH; c++) {
        bool multi = false;
        uint32_t bits = 0;
        if (FULL || base + 32 * c + lane < nB) {
            if (pair_max > 0) bits = cf_owner_bits(s_tab, s_ids, b[c], &multi);
            else multi = cf_lookup(s_tab, b[c]);             // pair path off (no owner bytes): a hit only counts once confirmed
        }
        mask |= __reduce_or_sync(0xFFFFFFFFu, bits);
        unsigned m = __ballot_sync(0xFFFFFFFFu, multi);
        while (m && __popc(mask) <= pair_max) {
            // A confirmation costs ~10 dependent global loads.  A query that keeps hitting shared slots is related to several
            // references of the tile (same family): after a few confirmations merge the whole combination instead.
            if (pair_max > 0 && ++confirms > PROBE_MAX_CONFIRMS) return make_uint2(0xFFFFFFFFu, (uint32_t)confirms);
            const int src = __ffs(m) - 1;
            m &= m - 1;
            const uint32_t bb = __shfl_sync(0xFFFFFFFFu, b[c], src);
            uint32_t lo = 0, hi = nA_lim;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (rowA[mid] < bb) lo = mid + 1; else hi = mid;
            }
            mask |= __ballot_sync(0xFFFFFFFFu, lo < nA_lim && rowA[lo] == bb);
        }
    }
    return make_uint2(mask, (uint32_t)confirms);
}

// One group of PROBE_DEPTH x 32 ranks of a query against the filter.  FULL: the whole group lies inside the query's list.
// Returns true when some lane has a fingerprint match.
template <bool FULL>
__device__ __forceinline__ bool probe_group(uint32_t tab_s, const uint32_t (&b)[PROBE_DEPTH], uint32_t base, uint32_t nB, int lane)
{
    // b[c] = rank base + 32 c + lane of the query (RANK_PAD past the end of its list)
    static_assert(PROBE_DEPTH == 4, "cf_group_any takes four probes");
    CfProbe pr[PROBE_DEPTH];
#pragma unroll
    for (int c = 0; c < PROBE_DEPTH; c++) {
        pr[c] = cf_fetch_s(tab_s, b[c]);
        if (!FULL && base + 32 * c + lane >= nB) pr[c].f2 = 0x7E007E00u;       // past the end of the list: never matches
    }
    return cf_group_any(pr[0], pr[1], pr[2], pr[3]);
}

__global__ void __launch_bounds__(PROBE_THREADS, 1) dist_probe_kernel(const DistArgs a)
{
    extern __shared__ uint32_t s_tab[];                      // CF_BUCKETS words, then 2 * CF_BUCKETS id bytes
    uint8_t *s_ids = reinterpret_cast<uint8_t *>(s_tab + CF_BUCKETS);
    __shared__ int s_fail;
    __shared__ uint32_t s_mx[32];                            // s_mx[l] = max over the tile's references of their rank at index 32 l (probe cut-off, below)
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t r0 = blockIdx.x * DIST_TILE_R;
    const uint32_t q_lo = a.q_begin + blockIdx.y * a.q_per_cta;
    const uint32_t q_hi = min(q_lo + a.q_per_cta, a.q_begin + a.q_count);
    if (q_lo >= q_hi) return;

    for (uint32_t i = threadIdx.x; i < CF_BUCKETS; i += PROBE_THREADS) s_tab[i] = 0;
    if (a.pair_max > 0)       // the owner bytes exist only when the pair path is on (the launch then asks for 64 KB more shared memory)
        for (uint32_t i = threadIdx.x; i < CF_BUCKETS / 2; i += PROBE_THREADS) reinterpret_cast<uint32_t *>(s_ids)[i] = 0xFFFFFFFFu;     // CF_ID_NONE
    if (threadIdx.x == 0) s_fail = 0;
    if (threadIdx.x < 32) s_mx[threadIdx.x] = 0;
    __syncthreads();
    for (uint32_t rr = warp; rr < DIST_TILE_R; rr += PROBE_WARPS) {
        const uint32_t rb = r0 + rr;
        if (rb >= a.n_ref) break;
        const uint32_t n = min(a.ref_n[rb], a.S);
        const uint32_t *row = a.ranks + (a.ref_row0 + rb) * (uint64_t)a.P;
        for (uint32_t i = lane; i < n; i += 32)
            if (!cf_insert(s_tab, row[i], threadIdx.x * 2654435761u + i)) s_fail = 1;
        atomicMax(&s_mx[lane], 32u * lane < n ? row[32 * lane] : RANK_PAD);       // a list that ends before index 32 l bounds nothing there
    }
    __syncthreads();
    // id side table: one reference per phase, so that only ranks of the same reference ever write a slot concurrently
    if (a.pair_max > 0)
        for (uint32_t rr = 0; rr < DIST_TILE_R; rr++) {
            const uint32_t rb = r0 + rr;
            if (rb < a.n_ref) {
                const uint32_t n = min(a.ref_n[rb], a.S);
                const uint32_t *row = a.ranks + (a.ref_row0 + rb) * (uint64_t)a.P;
                for (uint32_t i = threadIdx.x; i < n; i += PROBE_THREADS) cf_mark_ids(s_tab, s_ids, row[i], rr);
            }
            __syncthreads();
        }
    const uint32_t tab_s = (uint32_t)__cvta_generic_to_shared(s_tab);
    const bool tile_failed = s_fail != 0;       // filter overflow (cannot happen at <= 32 x 1035 ranks): merge everything

    const uint32_t r = r0 + lane;
    const bool r_ok = r < a.n_ref;
    const uint32_t nA = r_ok ? a.ref_n[r] : 0;
    const uint32_t nA_lim = min(nA, a.S);
    const uint64_t lenA = r_ok ? a.ref_len[r] : 1;
    const uint32_t *rowA = a.ranks + (a.ref_row0 + (r_ok ? r : r0)) * (uint64_t)a.P;
    // closed form of a pair without shared hashes whose union still reaches s' elements (the usual case): constants
    const double lut0 = a.dist_lut[0];
    const bool far = a.max_distance >= 0 && lut0 > a.max_distance;           // dist_emit: filtered by -d, p-value left 0
    const double p_const = far ? 0.0 : 1.0;
    const uint8_t pass_const = (far || (a.max_pvalue >= 0 && 1.0 > a.max_pvalue)) ? 0 : 1;
    const int pair_max = a.pair_max;
    // Cut-off.  In the merge of a reference A with the query B (both sorted, ties kept apart) only the first s' elements matter: if none
    // of them is shared they are the first s' elements of the union, common = 0 and denom = s' whatever lies behind.  A query element
    // B[j] is among them iff j + |{a in A: a < B[j]}| < s', so once j + (a lower bound of that count for every reference of the tile)
    // reaches s' the rest of the query need not be looked up: unrelated sketches of similar size are done after about half their
    // ranks.  Lower bound: lane l holds mx = max over the tile of A[32 l]; mx < x means every reference has more than 32 l ranks
    // below x, and mx grows with l, so with L lanes below x the count is at least 32 L - 31.
    const uint32_t mx = s_mx[lane];
    const uint32_t cut_at = a.S + 31;

    for (uint32_t q = q_lo + warp; q < q_hi; q += PROBE_WARPS) {
        if (a.triangle && q <= a.tri_r0 + r0) continue;            // the whole tile lies on or above the diagonal
        const uint32_t nB_all = a.qry_n[q];
        const uint32_t nB = min(nB_all, a.S);
        const uint32_t *rowB = a.ranks + (a.qry_row0 + q) * (uint64_t)a.P;
        uint32_t mask = tile_failed ? 0xFFFFFFFFu : 0u;     // references of the tile the query may share a hash with
        bool dense = tile_failed;                           // more than pair_max of them: the combination is merged as a whole
        int confirms = 0;
        uint32_t base = 0;
        const uint32_t *pB = rowB + lane;
        constexpr uint32_t GROUP = 32 * PROBE_DEPTH;
        // full groups; the lines of the group after next are requested into L1 first (one prefetch instruction, lanes 0-3
        // name the four 128-byte lines): 8 warps per sub-partition do not cover the L2 latency on their own.  ptxas sinks
        // register prefetches to the end of the body.
        uint32_t cur[PROBE_DEPTH];
        // (two groups per iteration -- 8 lookups in flight per lane, one vote per 256 ranks -- was slower: the loop is bound by
        // ALU-pipe and shared-memory throughput, not by latency)
        if (2 * GROUP <= nB) asm volatile("prefetch.global.L1 [%0];" :: "l"(rowB + GROUP + 32 * (lane & 3)));
        while (base + GROUP <= nB && !dense) {
            if (base + 3 * GROUP <= nB) asm volatile("prefetch.global.L1 [%0];" :: "l"(rowB + base + 2 * GROUP + 32 * (lane & 3)));
#pragma unroll
            for (int c = 0; c < PROBE_DEPTH; c++) cur[c] = __ldg(pB + 32 * c);
            if (probe_group<true>(tab_s, cur, base, nB, lane)) {
                const uint2 st = probe_resolve<true>(cur[0], cur[1], cur[2], cur[3], base, nB, rowA, nA_lim, mask, a.pair_max, confirms);
                mask = st.x; confirms = (int)st.y;
                if (__popc(mask) > a.pair_max) { dense = true; break; }
            }
            base += GROUP; pB += GROUP;
            // cut-off test for the next group with the last rank of this one (already in a register; B[base] > B[base - 1], so the
            // bound is merely a little weaker than with B[base], which would have to be waited for)
            if (base + 32 * __popc(__ballot_sync(0xFFFFFFFFu, mx < __shfl_sync(0xFFFFFFFFu, cur[PROBE_DEPTH - 1], 31))) >= cut_at) { base = nB; break; }
        }
        if (base < nB && !dense) {      // ragged last group
#pragma unroll
            for (int c = 0; c < PROBE_DEPTH; c++) cur[c] = (base + 32 * c + lane < nB) ? __ldg(pB + 32 * c) : RANK_PAD;
            if (probe_group<false>(tab_s, cur, base, nB, lane)) {
                const uint2 st = probe_resolve<false>(cur[0], cur[1], cur[2], cur[3], base, nB, rowA, nA_lim, mask, pair_max, confirms);
                mask = st.x;
                dense = __popc(mask) > pair_max;
            }
        }
        const bool mine = r_ok && !(a.triangle && a.tri_r0 + r >= q);       // this lane's pair exists
        if (!dense && mask) {
            // a few candidate references: their pairs go to the pair list (one warp merges one pair, dist_pair_kernel), the other
            // lanes get the closed form below.  List full: merge the whole combination instead.
            const unsigned want = __ballot_sync(0xFFFFFFFFu, mine && ((mask >> lane) & 1u));
            if (want) {
                unsigned long long at = 0;
                if (lane == 0) at = atomicAdd(a.pair_count, (unsigned long long)__popc(want));
                at = __shfl_sync(0xFFFFFFFFu, at, 0);
                if (at + __popc(want) <= a.pair_capacity) {
                    if ((want >> lane) & 1u) a.pair_list[at + __popc(want & ((1u << lane) - 1u))] = make_uint2(q, r);
                } else {
                    // the counter has moved past slots this warp leaves unwritten: the consumer stops at the first such start
                    if (lane == 0) atomicMax(a.pair_full, ~at);
                    dense = true;
                }
            }
        }
        if (dense) {
            if (lane == 0) {
                const uint32_t at = atomicAdd(&a.qcount[blockIdx.x], 1u);
                a.qlist[(uint64_t)blockIdx.x * a.qlist_stride + at] = q;
                atomicAdd(a.flag_total, 1ull);
            }
        } else if (mine && !((mask >> lane) & 1u)) {
            // empty intersection: the merge would take min(s', |A| + |B|) union steps and count nothing
            const uint32_t denom = min(a.S, nA + nB_all);
            if (a.best.cand || a.graph.forest) {
                // best, component or spanning-forest run: a pair without a shared hash is not a hit, whatever its denominator
            } else if (denom == a.S && a.list_idx && pass_const == 0) {
                // filtered run (-d / -v) and distance 1 / p-value 1 does not pass: nothing to write for this pair
            } else if (denom == a.S && !a.list_idx) {
                const uint64_t o = (uint64_t)(q - a.q_begin) * a.n_ref + r;
                if (a.numer) a.numer[o] = 0;
                if (a.denom) a.denom[o] = denom;
                if (a.distance) a.distance[o] = lut0;
                if (a.pvalue) a.pvalue[o] = p_const;
                if (a.pass) a.pass[o] = pass_const;
            } else {
                dist_emit(a, q, r, 0u, denom, lenA);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------------------
// One warp per (query, reference) pair: the sorted merge of compareSketches (CommandDistance.cpp:347-385) as a union count.
//   common = ties among the first min(s', |A u B|) elements of the sorted union, denom = min(s', |A u B|)
// (lists cut to their first s' elements: an element beyond index s' can never be among the first s' of the union).
// Both rows are staged in the warp's shared memory; the query row is cut into 32 runs, lane l takes run l and the reference
// elements that fall into its value range (one binary search per lane), merges them sequentially counting union elements and
// ties; a warp scan finds the lane in which the s'-th union element falls, and the search zooms into that lane's run with all 32
// lanes again (runs of one query element end in a closed form).  ~2 log_32(s') rounds of ~2 s'/32 steps instead of s' lockstep
// steps for 32 pairs: the path for the few related pairs of a (query, tile) combination (dist_probe_kernel's pair list), where the
// lockstep kernel would run 32 lanes for one or two useful ones, and for sketch sizes whose 32-reference tile does not fit shared
// memory (pair_dense).
// ---------------------------------------------------------------------------------------------------------
constexpr int PAIR_WARPS_MAX = 8;

__device__ __forceinline__ uint32_t warp_incl_scan(uint32_t v, int lane)
{
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        const uint32_t t = __shfl_up_sync(0xFFFFFFFFu, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

// Shared-memory layout: both rows linear, each preceded by up to 3 words of skew (the TMA bulk copy that stages a row needs
// 16-byte aligned ends, a row starts on a 4-byte boundary) and followed by the sentinel 0xFFFFFFFF.  Bank conflicts are avoided by
// the run length instead of padding: lane l's run starts at element l * run, and with an ODD run the 32 starts fall into 32
// different banks, so lanes that step through their runs at similar speeds do not collide (an even run of 32 put every start
// into bank 0: 32-way conflicts on every load, 2e7 pairs/s; the padded variant of the same idea measured 1.5e8).
// The sequential part reads past a lane's ranges on purpose: the element after a lane's query run is the first of the next
// lane's run, larger than every reference element of this lane, and the element after its reference range is not below that one
// -- so an exhausted side never wins a comparison and the loop needs no bounds selects, only the two end tests.
__global__ void __launch_bounds__(PAIR_WARPS_MAX * 32) dist_pair_kernel(const DistArgs a, uint32_t row_pitch, uint32_t run0)
{
    extern __shared__ __align__(16) uint32_t smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, warps = blockDim.x >> 5;
    uint32_t *bufA = smem + (size_t)warp * 2 * row_pitch, *bufB = bufA + row_pitch;
    uint64_t *s_bar = reinterpret_cast<uint64_t *>(smem + (size_t)warps * 2 * row_pitch);
    const uint32_t bar = warp_bar_init(s_bar + warp);
    uint32_t phase = 0;
    uint64_t total;
    if (a.pair_dense) total = (uint64_t)a.q_count * a.n_ref;
    else {
        // every slot below both bounds was written by this run (a reservation below the first failed one fit); without a failed
        // reservation pair_count <= pair_capacity
        const unsigned long long listed = *a.pair_count, written = ~*a.pair_full;
        total = listed < written ? listed : written;
        if (blockIdx.x == 0 && threadIdx.x == 0 && a.pair_total) atomicAdd(a.pair_total, (unsigned long long)total);
    }
    for (uint64_t idx = (uint64_t)blockIdx.x * warps + warp; idx < total; idx += (uint64_t)gridDim.x * warps) {
        uint32_t q, r;
        if (a.pair_dense) {
            q = a.q_begin + (uint32_t)(idx / a.n_ref); r = (uint32_t)(idx % a.n_ref);
            if (a.triangle && a.tri_r0 + r >= q) continue;
        } else {
            const uint2 e = a.pair_list[idx];
            q = e.x; r = e.y;
        }
        const uint32_t nA = min(a.ref_n[r], a.S), nB = min(a.qry_n[q], a.S);
        // stage both rows cut to their first n elements (bufB = bufA + row_pitch), then the sentinels
        const uint32_t *src[2];
        uint32_t skew[2];
        const uint32_t spanA = bulk_span(a.ranks + (a.ref_row0 + r) * (uint64_t)a.P, nA, src[0], skew[0]);
        const uint32_t spanB = bulk_span(a.ranks + (a.qry_row0 + q) * (uint64_t)a.P, nB, src[1], skew[1]);
        const uint32_t bytes[2] = {nA ? spanA : 0u, nB ? spanB : 0u};
        bulk_copy_wait(src, bytes, bytes[0] + bytes[1], bufA, row_pitch, bar, phase);
        uint32_t *sA = bufA + skew[0] / 4, *sB = bufB + skew[1] / 4;
        if (lane == 0) { sA[nA] = RANK_PAD; sB[nB] = RANK_PAD; }
        __syncwarp();
        uint32_t i0 = 0, i1 = nA, j0 = 0, j1 = nB;          // the segment still to be resolved
        uint32_t need = a.S;                                 // union elements still to be taken
        uint32_t common = 0, taken = 0;
        bool first = true;
        for (;;) {
            const uint32_t lenB = j1 - j0;
            // query elements per lane: odd (bank-conflict-free run starts); 0 when only reference elements are left
            uint32_t run = first ? run0 : (lenB + 31) / 32;
            if (run > 1) run |= 1u;
            first = false;
            const uint32_t jb = min(j0 + (uint32_t)lane * run, j1), je = min(jb + run, j1);
            uint32_t ib;
            if (lane == 0) ib = i0;                          // reference elements below the first query element belong to lane 0
            else if (jb >= j1) ib = i1;
            else {
                const uint32_t v = sB[jb];
                uint32_t lo = i0, hi = i1;
                while (lo < hi) {
                    const uint32_t mid = (lo + hi) >> 1;
                    if (sA[mid] < v) lo = mid + 1; else hi = mid;
                }
                ib = lo;
            }
            uint32_t ie = __shfl_down_sync(0xFFFFFFFFu, ib, 1);
            if (lane == 31) ie = i1;
            uint32_t u = 0, t = 0;
            if (ib < ie || jb < je) {
                // pointers in the shared window; an exhausted side holds an element that cannot win (see above)
                uint32_t pa = (uint32_t)__cvta_generic_to_shared(sA + ib), pb = (uint32_t)__cvta_generic_to_shared(sB + jb);
                const uint32_t ea = (uint32_t)__cvta_generic_to_shared(sA + ie), eb = (uint32_t)__cvta_generic_to_shared(sB + je);
                uint32_t av = lds32(pa), bv = lds32(pb);
                // the element after the segment's last query element must exceed every reference element of the segment; at the top
                // level that is the sentinel, below it the next lane's first query element -- except for the LAST lane with query
                // elements of a zoomed segment, whose successor belongs to the parent's next lane: also larger.  A reference range
                // that ends at i1 reads sA[i1]: the sentinel or the parent's next element, not below the query run's successor.
                asm volatile("{\n\t.reg .pred pa, pb, pt, pc;\n\t"
                             "PAIR_MERGE_LOOP:\n\t"
                             "setp.le.u32 pa, %0, %1;\n\t"
                             "setp.le.u32 pb, %1, %0;\n\t"
                             "and.pred pt, pa, pb;\n\t"
                             "@pa add.u32 %2, %2, 4;\n\t"
                             "@pb add.u32 %3, %3, 4;\n\t"
                             "@pt add.u32 %5, %5, 1;\n\t"
                             "@pa ld.shared.u32 %0, [%2];\n\t"
                             "@pb ld.shared.u32 %1, [%3];\n\t"
                             "add.u32 %4, %4, 1;\n\t"
                             "setp.lt.u32 pc, %2, %6;\n\t"
                             "setp.lt.or.u32 pc, %3, %7, pc;\n\t"
                             "@pc bra PAIR_MERGE_LOOP;\n\t}"
                             : "+r"(av), "+r"(bv), "+r"(pa), "+r"(pb), "+r"(u), "+r"(t) : "r"(ea), "r"(eb) : "memory");
            }
            const uint32_t U = warp_incl_scan(u, lane), T = warp_incl_scan(t, lane);
            const uint32_t totalU = __shfl_sync(0xFFFFFFFFu, U, 31), totalT = __shfl_sync(0xFFFFFFFFu, T, 31);
            if (totalU <= need) { common += totalT; taken += totalU; break; }      // the segment ends before the s'-th union element
            const int L = __ffs(__ballot_sync(0xFFFFFFFFu, U >= need)) - 1;       // the lane in which it falls
            const uint32_t Uprev = __shfl_sync(0xFFFFFFFFu, U - u, L), Tprev = __shfl_sync(0xFFFFFFFFu, T - t, L);
            common += Tprev; taken += Uprev; need -= Uprev;
            i0 = __shfl_sync(0xFFFFFFFFu, ib, L); i1 = __shfl_sync(0xFFFFFFFFu, ie, L);
            j0 = __shfl_sync(0xFFFFFFFFu, jb, L); j1 = __shfl_sync(0xFFFFFFFFu, je, L);
            if (j1 - j0 <= 1) {
                // at most one query element b left: the union runs (reference elements below b), b -- a tie when the next
                // reference element equals it --, (the rest); `need` (>= 1, fewer than the segment holds) of them are taken
                if (j1 > j0) {
                    const uint32_t b = sB[j0];
                    uint32_t k = 0;
                    for (uint32_t i = i0 + lane; i < i1; i += 32) k += sA[i] < b;
#pragma unroll
                    for (int d = 16; d > 0; d >>= 1) k += __shfl_xor_sync(0xFFFFFFFFu, k, d);
                    const bool tie = i0 + k < i1 && sA[i0 + k] == b;
                    if (tie && need >= k + 1) common++;
                }
                taken += need;
                break;
            }
        }
        if (lane == 0) dist_emit(a, q, r, common, taken, a.ref_len[r]);
    }
}

// The sequential merge of one pair (query q, reference r) straight from global memory: (common, denom).
__device__ __forceinline__ uint2 dist_merge_pair(const DistArgs &a, uint32_t q, uint32_t r)
{
    const uint32_t *A = a.ranks + (a.ref_row0 + r) * (uint64_t)a.P;
    const uint32_t *B = a.ranks + (a.qry_row0 + q) * (uint64_t)a.P;
    uint32_t i = 0, j = 0;
    uint32_t va = A[0], vb = B[0];
    for (uint32_t step = 0; step < a.S; step++) {
        const bool adv_a = va <= vb, adv_b = vb <= va;
        if (adv_a) va = A[++i];
        if (adv_b) vb = B[++j];
    }
    const uint32_t nA = a.ref_n[r];
    const uint32_t bogus = i > nA ? i - nA : 0;
    const uint32_t denom = a.S - bogus;
    return make_uint2((i - bogus) + (j - bogus) - denom, denom);
}

// General fallback for sketch sizes whose tiles do not fit in shared memory (s > ~1035): one thread per pair, rows read
// straight from global memory (L1/L2).  Same arithmetic, an order of magnitude slower; large -s is the rare case.
__global__ void __launch_bounds__(256) dist_kernel_general(const DistArgs a)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    const uint64_t total = (uint64_t)a.q_count * a.n_ref;
    if (t >= total) return;
    const uint32_t q = a.q_begin + (uint32_t)(t / a.n_ref), r = (uint32_t)(t % a.n_ref);
    if (a.triangle && a.tri_r0 + r >= q) return;
    const uint2 cd = dist_merge_pair(a, q, r);
    dist_emit(a, q, r, cd.x, cd.y, a.ref_len[r]);
}

// dist_emit's distance of a pair from its merge result
__device__ __forceinline__ double dist_value(const DistArgs &a, uint32_t common, uint32_t denom)
{
    return (denom == a.S) ? a.dist_lut[common] : mash_distance(common, denom, a.kmer_size);
}

// The values of a graph edge (q, r) recomputed on its own: the sequential merge of dist_kernel_general and the arithmetic of dist_emit /
// dist_fix_kernel, so every value is the one a dense run returns for (q, r).  Every edge shares a hash, so its p-value is the binomial
// tail.
__device__ __forceinline__ void dist_edge_values(const DistArgs &a, uint32_t q, uint32_t r, uint32_t *numer, uint32_t *denom, double *distance,
                                                 double *pvalue)
{
    const uint2 cd = dist_merge_pair(a, q, r);
    *numer = cd.x; *denom = cd.y;
    *distance = dist_value(a, cd.x, cd.y);
    *pvalue = mash_pvalue(cd.x, a.ref_len[r], a.qry_len[q], a.kmer_space, cd.y, &a.binom);
}

// Values of the spanning forest's edges, once after its last round, for (q = i, r = j - tri_r0).  `lo` holds the edges (j << 32 | i)
// in forest order.
__global__ void __launch_bounds__(256) msf_values_kernel(const DistArgs a, const unsigned long long *lo, uint64_t m, uint32_t *row,
                                                         uint32_t *col, uint32_t *numer, uint32_t *denom, double *distance, double *pvalue)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= m) return;
    const uint32_t q = (uint32_t)lo[t], j = (uint32_t)(lo[t] >> 32);
    row[t] = q; col[t] = j;
    dist_edge_values(a, q, j - a.tri_r0, numer + t, denom + t, distance + t, pvalue + t);
}

// The outputs of greedy dereplication, one thread per sketch of a self job: a representative is its own with zero values; a member's
// representative is the other end of the key in its slot, and its values are those of that edge.  counters[1] counts the
// representatives; counters[2] |= 2 for a member without a slot (cannot happen: an earlier representative is always adjacent).
__global__ void __launch_bounds__(256) greedy_values_kernel(const DistArgs a, const uint32_t *status, const MsfKey *slot, uint64_t n, uint32_t *rep,
                                                           uint32_t *numer, uint32_t *denom, double *distance, double *pvalue,
                                                           unsigned long long *counters)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    const MsfKey k = slot[t];
    const bool is_rep = status[t] & GREEDY_REP;
    if (is_rep || k.hi == MSF_NONE) {
        rep[t] = (uint32_t)t; numer[t] = 0; denom[t] = 0; distance[t] = 0.0; pvalue[t] = 0.0;
        if (is_rep) atomicAdd(counters + 1, 1ull);
        else atomicOr(counters + 2, 2ull);
        return;
    }
    const uint32_t q = (uint32_t)k.lo, r = (uint32_t)(k.lo >> 32);
    rep[t] = q == (uint32_t)t ? r : q;
    dist_edge_values(a, q, r, numer + t, denom + t, distance + t, pvalue + t);
}

// ---------------------------------------------------------------------------------------------------------
// dictionary encoding
// ---------------------------------------------------------------------------------------------------------
// n_eff[row0 + row] = number of hashes of the row that take part: min(n_hashes, P, stride)
__global__ void dict_neff_kernel(const uint32_t *n_hashes, uint64_t n_rows, uint32_t P, uint64_t stride, uint64_t row0, uint32_t *n_eff)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_rows) return;
    n_eff[row0 + t] = (uint32_t)min((uint64_t)min(n_hashes[t], P), stride);
}

// valid hashes only, compacted: entry off[row] + i = hash i of the row, with its slot (row0 + row) * P + i
__global__ void dict_gather_kernel(const uint64_t *hashes, uint64_t stride, uint64_t n_rows, uint32_t P, uint64_t row0,
                                   const uint32_t *n_eff, const uint32_t *off, uint64_t out0, uint64_t *keys, uint32_t *slots)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_rows * P) return;
    const uint64_t row = t / P;
    const uint32_t i = (uint32_t)(t % P);
    if (i >= n_eff[row0 + row]) return;
    const uint64_t o = out0 + off[row] + i;
    keys[o] = hashes[row * stride + i];
    slots[o] = (uint32_t)((row0 + row) * P + i);
}

__global__ void dict_flag_kernel(const uint64_t *sorted_keys, uint64_t n, uint32_t *flags)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    flags[t] = (t == 0 || sorted_keys[t] != sorted_keys[t - 1]) ? 1u : 0u;
}

// out[value of sorted entry t] = rank of its key among the distinct keys
__global__ void dict_scatter_kernel(const uint32_t *sorted_vals, const uint32_t *scan, uint64_t n, uint32_t *out)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    out[sorted_vals[t]] = scan[t] - 1u;
}

// sharded build: rows[slots[t]] = codes[t] + base of the segment (hash range) entry t was sent to
__global__ void dict_scatter_seg_kernel(const uint32_t *codes, const uint32_t *slots, uint64_t n, const uint64_t *seg_end, const uint64_t *seg_base,
                                        uint32_t n_segs, uint32_t *rows, uint32_t *err)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint32_t g = 0;
    while (g + 1 < n_segs && t >= seg_end[g]) g++;
    const uint64_t c = (uint64_t)codes[t] + seg_base[g];
    if (c >= 0xFFFFFFFFull) { atomicOr(err, 1u); return; }
    rows[slots[t]] = (uint32_t)c;
}

// lower bounds of the splitters in an ascending key list
__global__ void dict_split_kernel(const uint64_t *keys, uint64_t n, const uint64_t *splitters, uint32_t n_split, uint64_t *pos)
{
    const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= n_split) return;
    const uint64_t v = splitters[t];
    uint64_t lo = 0, hi = n;
    while (lo < hi) {
        const uint64_t mid = (lo + hi) >> 1;
        if (keys[mid] < v) lo = mid + 1; else hi = mid;
    }
    pos[t] = lo;
}

__global__ void list_gather_kernel(const uint32_t *order, uint64_t n, const uint32_t *numer, const uint32_t *denom, const double *distance,
                                   const double *pvalue, uint32_t *o_numer, uint32_t *o_denom, double *o_distance, double *o_pvalue)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    const uint32_t src = order[t];
    o_numer[t] = numer[src]; o_denom[t] = denom[src]; o_distance[t] = distance[src]; o_pvalue[t] = pvalue[src];
}

__global__ void iota_kernel(uint32_t *v, uint64_t n)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t < n) v[t] = (uint32_t)t;
}

// ---------------------------------------------------------------------------------------------------------
// Linkage cut (mashgpu_dist_linkage_cut, DESIGN.md 3.13): the CTA tier and the large tier's row gather
// ---------------------------------------------------------------------------------------------------------
struct CutComp { uint32_t first, m, merge0; };      // a component: members[first .. first + m), merges rec[merge0 .. merge0 + m - 2]

// One CTA per component of a size class (m <= the class's bound, THREADS for it): the component's lower triangle of run()'s
// distances into shared memory -- D(i, j), j < i, of the pair (q = members[i], r = members[j]) by the sequential merge and
// dist_emit's arithmetic, as dist_edge_values computes it -- then its whole linkage there (linkage_cta.cuh).
template <unsigned THREADS, bool AVERAGE>
__global__ void __launch_bounds__(THREADS) cut_cta_kernel(const DistArgs a, const uint32_t *__restrict__ members, const CutComp *__restrict__ comps,
                                                          LkMerge *rec, int *no_pair)
{
    extern __shared__ __align__(16) double cut_smem[];
    const CutComp c = comps[blockIdx.x];
    const uint32_t *mem = members + c.first;
    const CtaLinkage L = cta_layout(cut_smem, c.m);
    const uint32_t pairs = cta_tri(c.m);
    for (uint32_t p = threadIdx.x; p < pairs; p += THREADS) {
        uint32_t i = (uint32_t)((1.0f + sqrtf(1.0f + 8.0f * (float)p)) * 0.5f);     // the row: cta_tri(i) <= p < cta_tri(i + 1)
        while (i > 1 && cta_tri(i) > p) i--;
        while (cta_tri(i + 1) <= p) i++;
        const uint2 cd = dist_merge_pair(a, mem[i], mem[p - cta_tri(i)]);
        L.tri[p] = dist_value(a, cd.x, cd.y);
    }
    __syncthreads();
    cta_linkage<THREADS, AVERAGE>(L, c.m, rec + c.merge0, no_pair);
}

// Empty sketches share no hash, yet are at distance 0 from one another (common = denom = 0): at any T they are one component, whose
// label is the first of them.  (Every other pair without a shared hash is at distance 1.)
__global__ void cut_empty_first_kernel(const uint32_t *n_eff, uint64_t n, uint32_t *first)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t < n && n_eff[t] == 0) atomicMin(first, (uint32_t)t);
}

__global__ void cut_empty_join_kernel(const uint32_t *n_eff, uint64_t n, const uint32_t *first, uint32_t *label)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t < n && n_eff[t] == 0) label[t] = *first;
}

// The components' first positions in the sorted keys: flag[t] = 1 where a run of equal keys starts, then (with scan = the inclusive sum of
// the flags) first[scan[t] - 1] = t there
__global__ void cut_start_kernel(const uint32_t *key, uint64_t n, uint32_t *flag)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t < n) flag[t] = (t == 0 || key[t] != key[t - 1]) ? 1u : 0u;
}

__global__ void cut_first_kernel(const uint32_t *key, const uint32_t *scan, uint64_t n, uint32_t *first)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t < n && (t == 0 || key[t] != key[t - 1])) first[scan[t] - 1] = (uint32_t)t;
}

// The large tier's rows: row t := the self job's row members[t], with its hash count and length
__global__ void cut_gather_kernel(const uint32_t *ranks, uint32_t P, const uint32_t *n_eff, const uint64_t *len, const uint32_t *members, uint64_t m,
                                  uint32_t *o_ranks, uint32_t *o_n_eff, uint64_t *o_len)
{
    for (uint64_t x = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; x < m * P; x += (uint64_t)gridDim.x * blockDim.x) {
        const uint64_t t = x / P;
        const uint32_t i = (uint32_t)(x % P), src = members[t];
        o_ranks[x] = ranks[(uint64_t)src * P + i];
        if (i == 0) { o_n_eff[t] = n_eff[src]; o_len[t] = len[src]; }
    }
}

}  // namespace mashgpu

using namespace mashgpu;

struct mashgpu_dist_job {
    mashgpu_ctx *ctx = nullptr;
    mashgpu_dist_params params{};
    uint64_t n_ref = 0, n_qry = 0;
    bool self = false;
    bool encoded = false;               // mashgpu_dist_open_encoded: queries are all rows, references a contiguous range of them
    uint32_t P = 0;
    // rank rows: views used by the kernels (into the buffers below, or the caller's arrays for mashgpu_dist_open_encoded)
    const uint32_t *d_ranks = nullptr, *d_n_eff = nullptr;
    const uint64_t *d_lens = nullptr;
    uint64_t ref_row0 = 0, qry_row0 = 0;     // first row of each set
    DevBuf<uint32_t> ranks, n_eff;
    DevBuf<uint64_t> lens;          // ref lengths then query lengths
    DevBuf<double> lut, binom_m;
    DevBuf<int> binom_e;
    bool tiled = true;
    // grow-only buffers of mashgpu_dist_run_list (no cudaMalloc per call after the first)
    DevBuf<uint64_t> l_idx, s_idx; DevBuf<uint32_t> l_n, l_d, l_order, s_order, o_n, o_d; DevBuf<double> l_D, l_P, o_D, o_P;
    DevBuf<unsigned long long> l_cnt; DevBuf<uint8_t> l_tmp;
    // best hits (mashgpu_dist_run_best_dev): grow-only buffers, counters since the job was opened
    uint64_t best_capacity = 0;         // mashgpu_dist_set_best_capacity; 0 = default
    DevBuf<BestCand> b_cand, b_grouped;
    DevBuf<uint32_t> b_q;               // per query of a block: hits, segment offset, scatter cursor
    DevBuf<unsigned long long> b_cnt;
    DevBuf<uint8_t> b_tmp;
    uint64_t best_blocks = 0, best_splits = 0, best_candidates = 0;
    double best_select_ms = 0;
    std::vector<EventPair> best_events;
    DevBuf<unsigned long long> cc_edges;        // edge counter of mashgpu_dist_components_dev
    uint64_t greedy_block = 0;          // mashgpu_dist_set_representative_block; 0 = default
    uint64_t cut_cta_max = 0;           // mashgpu_dist_set_linkage_cut_cta_max; 0 = default
    double cut_ms[4] = {0, 0, 0, 0};    // device time of the last linkage cut's phases: components, grouping, CTA tier, large tier
    // prefilter (dist_probe_kernel): -1 = auto (on; switched off when most combinations turn out to share hashes), 0 = off, 1 = on
    int prefilter_mode = -1;
    bool triangle = false;
    bool auto_off = false;
    DevBuf<uint32_t> qlist, qcount;
    DevBuf<uint2> pair_list;            // sparse related pairs of the run in flight (dist_probe_kernel -> dist_pair_kernel)
    DevBuf<unsigned long long> pair_count;      // [0] slots reserved by the run in flight, [1] its DistArgs::pair_full, [2] pairs merged from
                                                // lists since the job was opened
    int pair_max = 4;                   // a (query, tile) combination with at most this many candidate references goes to the pair list;
                                        // 0 = pair path off (MASHGPU_DIST_PAIR_MAX)
    DevBuf<FixEntry> fix_list;
    DevBuf<unsigned long long> fix_count;
    DevBuf<unsigned long long> flag_total;
    PinnedBuf<unsigned long long> h_flag_total;
    cudaEvent_t flag_event = nullptr;
    bool flag_pending = false;          // a snapshot of the device counter is on its way to h_flag_total
    uint64_t snap_combos = 0;           // combinations probed up to the run the snapshot was taken after
    uint64_t combos_probed = 0;         // (query, tile) combinations probed so far; flag_total (device) counts the flagged ones
    ~mashgpu_dist_job() { if (flag_event) cudaEventDestroy(flag_event); }
};

namespace mashgpu {

int stage_set(mashgpu_ctx *ctx, const mashgpu_sketch_set *s, SetOnDevice &d, cudaStream_t st, bool want_length)
{
    if (s->on_device) { d.hashes = s->hashes; d.n_hashes = s->n_hashes; d.length = s->length; return MASHGPU_OK; }
    if (d.h.alloc(s->n * s->stride) != cudaSuccess || d.n.alloc(s->n) != cudaSuccess || (want_length && d.l.alloc(s->n) != cudaSuccess))
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sketch set of %llu x %llu)", (unsigned long long)s->n, (unsigned long long)s->stride);
    MG_CUDA(ctx, cudaMemcpyAsync(d.h.p, s->hashes, s->n * s->stride * 8, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(d.n.p, s->n_hashes, s->n * 4, cudaMemcpyHostToDevice, st));
    if (want_length) MG_CUDA(ctx, cudaMemcpyAsync(d.l.p, s->length, s->n * 8, cudaMemcpyHostToDevice, st));
    d.hashes = d.h.p; d.n_hashes = d.n.p; d.length = d.l.p;
    return MASHGPU_OK;
}

int check_set(mashgpu_ctx *ctx, const mashgpu_sketch_set *s, const char *what, bool want_length)
{
    if (!s) return fail(ctx, MASHGPU_ERR_INVALID, "%s set is NULL", what);
    if (s->n && (!s->hashes || !s->n_hashes || (want_length && !s->length))) return fail(ctx, MASHGPU_ERR_INVALID, "%s set has NULL arrays", what);
    return MASHGPU_OK;
}

int dict_gather(mashgpu_ctx *ctx, const SetOnDevice &d, uint64_t n_rows, uint64_t stride, uint32_t P, uint64_t row0, uint32_t *n_eff,
                uint64_t out0, uint64_t *keys, uint32_t *slots, uint64_t *n_out, cudaStream_t st)
{
    *n_out = 0;
    if (n_rows == 0) return MASHGPU_OK;
    if (n_rows * P >= 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^31 dictionary slots (%llu rows x %u)", (unsigned long long)n_rows, P);
    DevBuf<uint32_t> off; DevBuf<uint8_t> tmp;
    if (off.alloc(n_rows + 1) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (row offsets)");
    dict_neff_kernel<<<blocks_for(n_rows), 256, 0, st>>>(d.n_hashes, n_rows, P, stride, row0, n_eff);
    size_t tb = 0;
    cub::DeviceScan::ExclusiveSum(nullptr, tb, n_eff + row0, off.p, (int)n_rows, st);
    if (tmp.alloc(tb) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (scan scratch)");
    MG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tb, n_eff + row0, off.p, (int)n_rows, st));
    uint32_t last_off = 0, last_n = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&last_off, off.p + (n_rows - 1), 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(&last_n, n_eff + row0 + (n_rows - 1), 4, cudaMemcpyDeviceToHost, st));
    dict_gather_kernel<<<blocks_for(n_rows * P), 256, 0, st>>>(d.hashes, stride, n_rows, P, row0, n_eff, off.p, out0, keys, slots);
    MG_CUDA(ctx, cudaGetLastError());
    MG_CUDA(ctx, cudaStreamSynchronize(st));      // off / tmp go out of scope
    ctx->kernel_launches += 4;
    *n_out = (uint64_t)last_off + last_n;
    return MASHGPU_OK;
}

int dict_rank(mashgpu_ctx *ctx, uint64_t *keys, uint32_t *vals, uint64_t n, uint32_t *out, uint64_t *n_distinct, cudaStream_t st)
{
    *n_distinct = 0;
    if (n == 0) return MASHGPU_OK;
    if (n >= 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^31 hashes in one dictionary sort");
    DevBuf<uint64_t> keys2; DevBuf<uint32_t> vals2; DevBuf<uint8_t> tmp;
    if (keys2.alloc(n) != cudaSuccess || vals2.alloc(n) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (dictionary scratch for %llu hashes)", (unsigned long long)n);
    size_t tmp_sort = 0, tmp_scan = 0;
    uint32_t *flags = reinterpret_cast<uint32_t *>(keys), *scan = flags + n;        // the unsorted keys are dead after the sort
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_sort, keys, keys2.p, vals, vals2.p, (int)n, 0, 64, st);
    cub::DeviceScan::InclusiveSum(nullptr, tmp_scan, flags, scan, (int)n, st);
    if (tmp.alloc(std::max(tmp_sort, tmp_scan)) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sort scratch)");
    cudaError_t e = cub::DeviceRadixSort::SortPairs(tmp.p, tmp_sort, keys, keys2.p, vals, vals2.p, (int)n, 0, 64, st);
    if (e != cudaSuccess) return fail(ctx, MASHGPU_ERR_CUDA, "radix sort failed: %s", cudaGetErrorString(e));
    dict_flag_kernel<<<blocks_for(n), 256, 0, st>>>(keys2.p, n, flags);
    e = cub::DeviceScan::InclusiveSum(tmp.p, tmp_scan, flags, scan, (int)n, st);
    if (e != cudaSuccess) return fail(ctx, MASHGPU_ERR_CUDA, "scan failed: %s", cudaGetErrorString(e));
    dict_scatter_kernel<<<blocks_for(n), 256, 0, st>>>(vals2.p, scan, n, out);
    MG_CUDA(ctx, cudaGetLastError());
    uint32_t nd = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&nd, scan + (n - 1), 4, cudaMemcpyDeviceToHost, st));
    e = cudaStreamSynchronize(st);
    if (e != cudaSuccess) return fail(ctx, MASHGPU_ERR_CUDA, "dictionary build failed: %s", cudaGetErrorString(e));
    ctx->kernel_launches += 12;
    *n_distinct = nd;
    return MASHGPU_OK;
}

int encode_rows(mashgpu_ctx *ctx, const SetOnDevice &ref, uint64_t n_ref, uint64_t ref_stride, const SetOnDevice *qry, uint64_t n_qry,
                uint64_t qry_stride, uint32_t P, uint32_t *ranks, uint32_t *n_eff, cudaStream_t st)
{
    const uint64_t rows = n_ref + (qry ? n_qry : 0), total = rows * P;
    if (rows == 0) return MASHGPU_OK;
    DevBuf<uint64_t> keys; DevBuf<uint32_t> slots;
    if (keys.alloc(total) != cudaSuccess || slots.alloc(total) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (dictionary scratch for %llu hashes)", (unsigned long long)total);
    uint64_t n_r = 0, n_q = 0, n_distinct = 0;
    MG_TRY(dict_gather(ctx, ref, n_ref, ref_stride, P, 0, n_eff, 0, keys.p, slots.p, &n_r, st));
    if (qry) MG_TRY(dict_gather(ctx, *qry, n_qry, qry_stride, P, n_ref, n_eff, n_r, keys.p, slots.p, &n_q, st));
    MG_CUDA(ctx, cudaMemsetAsync(ranks, 0xFF, total * 4, st));                  // padding code everywhere, then the real ranks
    MG_TRY(dict_rank(ctx, keys.p, slots.p, n_r + n_q, ranks, &n_distinct, st));
    if (n_distinct >= 0xFFFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^32 - 1 distinct hashes");
    return MASHGPU_OK;
}

}  // namespace mashgpu

namespace {

// distance LUT, binomial table, kernel attributes and the environment switches: everything of a job but the rank rows
int dist_job_tables(mashgpu_ctx *ctx, mashgpu_dist_job *job, cudaStream_t st)
{
    const mashgpu_dist_params *params = &job->params;
    const uint64_t S = params->sketch_size;
    if (job->lut.alloc(S + 1) != cudaSuccess || job->binom_m.alloc(S + 1) != cudaSuccess || job->binom_e.alloc(S + 1) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (distance / binomial tables)");
    // distance LUT for denom == sketch_size, computed with the host libm exactly as the reference does
    std::vector<double> lut(S + 1);
    for (uint64_t c = 0; c <= S; c++) {
        double d;
        double j = (double)c / (double)S;
        if (c == S) d = 0; else if (c == 0) d = 1.; else { d = -log(2 * j / (1. + j)) / params->kmer_size; if (d > 1) d = 1; }
        lut[c] = d;
    }
    MG_CUDA(ctx, cudaMemcpyAsync(job->lut.p, lut.data(), (S + 1) * 8, cudaMemcpyHostToDevice, st));
    // C(S, x) as mant * 2^expo for the device binomial tail (binom.cuh), running product in long double
    std::vector<double> bm(S + 1);
    std::vector<int> be(S + 1);
    {
        long double m = 1.0L;
        int e = 0;
        bm[0] = 1.0; be[0] = 0;
        for (uint64_t x = 1; x <= S; x++) {
            m *= (long double)(S - x + 1) / (long double)x;
            int k;
            m = frexpl(m, &k);
            e += k;
            bm[x] = (double)m; be[x] = e;
        }
    }
    MG_CUDA(ctx, cudaMemcpyAsync(job->binom_m.p, bm.data(), (S + 1) * 8, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(job->binom_e.p, be.data(), (S + 1) * 4, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));      // the host vectors go out of scope
    if (!ctx->attr_dist) {   // per context: function attributes are per device
        cudaError_t e = cudaFuncSetAttribute(dist_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(dist_probe_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)PROBE_SMEM);
        if (e == cudaSuccess) e = cudaFuncSetAttribute(dist_pair_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024);
        if (e != cudaSuccess) return fail(ctx, MASHGPU_ERR_CUDA, "cudaFuncSetAttribute: %s", cudaGetErrorString(e));
        ctx->attr_dist = true;
    }
    if (const char *env = getenv("MASHGPU_DIST_PAIR_MAX")) job->pair_max = std::max(0, std::min(31, atoi(env)));
    if (const char *env = getenv("MASHGPU_DIST_PREFILTER")) job->prefilter_mode = atoi(env) > 0 ? 1 : (atoi(env) == 0 ? 0 : -1);
    // s <= 1034: the tiled merge (dist_kernel); larger sketches run the warp-per-pair merge or dist_kernel_general
    job->tiled = dist_smem_bytes(job->P) <= 227 * 1024;
    return MASHGPU_OK;
}

int check_dist_params(mashgpu_ctx *ctx, const mashgpu_dist_params *params)
{
    if (params->sketch_size < 1 || params->sketch_size > 0x7FFFFFF0ull) return fail(ctx, MASHGPU_ERR_INVALID, "sketch_size out of range");
    if (params->kmer_size < 1) return fail(ctx, MASHGPU_ERR_INVALID, "kmer_size out of range");
    return MASHGPU_OK;
}

}  // namespace

extern "C" int mashgpu_dist_open(mashgpu_ctx *ctx, const mashgpu_sketch_set *ref, const mashgpu_sketch_set *qry,
                                 const mashgpu_dist_params *params, mashgpu_dist_job **job_out)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!params || !job_out) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    MG_TRY(check_set(ctx, ref, "reference"));
    const bool self = (qry == nullptr || qry == ref);
    if (!self) MG_TRY(check_set(ctx, qry, "query"));
    MG_TRY(check_dist_params(ctx, params));
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;

    std::unique_ptr<mashgpu_dist_job> job(new mashgpu_dist_job());      // every early return below frees the job and its buffers
    job->ctx = ctx; job->params = *params; job->self = self;
    job->n_ref = ref->n; job->n_qry = self ? ref->n : qry->n;
    const uint32_t P = (uint32_t)params->sketch_size + 1;
    job->P = P;
    const uint64_t rows = job->n_ref + (self ? 0 : job->n_qry);
    const uint64_t total = rows * P;
    if (total >= 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^31 dictionary slots (%llu rows x %u)", (unsigned long long)rows, P);

    const bool trace = getenv("MASHGPU_TRACE") != nullptr;
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t_open = now();
    SetOnDevice dr, dq;
    MG_TRY(stage_set(ctx, ref, dr, st));
    if (!self) MG_TRY(stage_set(ctx, qry, dq, st));

    if (job->ranks.alloc(total) != cudaSuccess || job->n_eff.alloc(rows) != cudaSuccess || job->lens.alloc(rows) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (rank rows)");
    job->d_ranks = job->ranks.p; job->d_n_eff = job->n_eff.p; job->d_lens = job->lens.p;
    job->ref_row0 = 0; job->qry_row0 = self ? 0 : job->n_ref;
    if (rows) {
        if (trace) fprintf(stderr, "[mashgpu] dist_open: staging + rank rows (%.0f MB) %.2f ms\n", total * 4e-6, now() - t_open);
        MG_TRY(encode_rows(ctx, dr, job->n_ref, ref->stride, self ? nullptr : &dq, job->n_qry, self ? 0 : qry->stride, P, job->ranks.p,
                           job->n_eff.p, st));
        MG_CUDA(ctx, cudaMemcpyAsync(job->lens.p, dr.length, job->n_ref * 8, cudaMemcpyDeviceToDevice, st));
        if (!self && job->n_qry)
            MG_CUDA(ctx, cudaMemcpyAsync(job->lens.p + job->n_ref, dq.length, job->n_qry * 8, cudaMemcpyDeviceToDevice, st));
        if (trace) fprintf(stderr, "[mashgpu] dist_open: dictionary built at %.2f ms\n", now() - t_open);
    }
    if (trace) fprintf(stderr, "[mashgpu] dist_open: scratch freed at %.2f ms\n", now() - t_open);
    MG_TRY(dist_job_tables(ctx, job.get(), st));
    if (trace) fprintf(stderr, "[mashgpu] dist_open: tables at %.2f ms\n", now() - t_open);
    *job_out = job.release();
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_open_encoded(mashgpu_ctx *ctx, const uint32_t *d_rows, const uint32_t *d_n_eff, const uint64_t *d_length,
                                         uint64_t n_rows, uint64_t ref_begin, uint64_t ref_count, const mashgpu_dist_params *params,
                                         mashgpu_dist_job **job_out)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!params || !job_out) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    if (n_rows && (!d_rows || !d_n_eff || !d_length)) return fail(ctx, MASHGPU_ERR_INVALID, "NULL row arrays");
    if (ref_begin + ref_count > n_rows) return fail(ctx, MASHGPU_ERR_INVALID, "reference rows [%llu, %llu) exceed %llu rows", (unsigned long long)ref_begin,
                                                    (unsigned long long)(ref_begin + ref_count), (unsigned long long)n_rows);
    if (n_rows >= 0xFFFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^32 - 1 rows");
    MG_TRY(check_dist_params(ctx, params));
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    std::unique_ptr<mashgpu_dist_job> job(new mashgpu_dist_job());
    job->ctx = ctx; job->params = *params; job->self = false; job->encoded = true;
    job->n_ref = ref_count; job->n_qry = n_rows;
    job->P = (uint32_t)params->sketch_size + 1;
    job->d_ranks = d_rows; job->d_n_eff = d_n_eff; job->d_lens = d_length;
    job->ref_row0 = ref_begin; job->qry_row0 = 0;
    MG_TRY(dist_job_tables(ctx, job.get(), ctx->stream));
    *job_out = job.release();
    return MASHGPU_OK;
}

// ---- sharded dictionary build (see include/mashgpu.h) ----------------------------------------------------------------
extern "C" int mashgpu_dict_local_sort(mashgpu_ctx *ctx, const mashgpu_sketch_set *set, uint64_t sketch_size,
                                       uint64_t *d_keys, uint32_t *d_slots, uint64_t *n_valid, void *stream)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!n_valid) return fail(ctx, MASHGPU_ERR_INVALID, "n_valid is NULL");
    *n_valid = 0;
    MG_TRY(check_set(ctx, set, "sketch", false));
    if (sketch_size < 1 || sketch_size > 0x7FFFFFF0ull) return fail(ctx, MASHGPU_ERR_INVALID, "sketch_size out of range");
    if (set->n == 0) return MASHGPU_OK;
    if (!d_keys || !d_slots) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    const uint32_t P = (uint32_t)sketch_size + 1;
    SetOnDevice d;
    MG_TRY(stage_set(ctx, set, d, st, false));
    DevBuf<uint32_t> n_eff, slots0; DevBuf<uint64_t> keys0; DevBuf<uint8_t> tmp;
    const uint64_t cap = set->n * std::min<uint64_t>(set->stride, P);
    if (n_eff.alloc(set->n) != cudaSuccess || keys0.alloc(cap) != cudaSuccess || slots0.alloc(cap) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (dictionary scratch for %llu hashes)", (unsigned long long)cap);
    uint64_t n = 0;
    MG_TRY(dict_gather(ctx, d, set->n, set->stride, P, 0, n_eff.p, 0, keys0.p, slots0.p, &n, st));
    if (n) {
        size_t tb = 0;
        cub::DeviceRadixSort::SortPairs(nullptr, tb, keys0.p, d_keys, slots0.p, d_slots, (int)n, 0, 64, st);
        if (tmp.alloc(tb) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sort scratch)");
        MG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp.p, tb, keys0.p, d_keys, slots0.p, d_slots, (int)n, 0, 64, st));
        ctx->kernel_launches += 8;
    }
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    *n_valid = n;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dict_split(mashgpu_ctx *ctx, const uint64_t *d_keys, uint64_t n, const uint64_t *splitters, uint32_t n_parts,
                                  uint64_t *counts, void *stream)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (n_parts == 0 || !counts || (n_parts > 1 && !splitters) || (n && !d_keys)) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    if (n_parts == 1) { counts[0] = n; return MASHGPU_OK; }
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    const uint32_t ns = n_parts - 1;
    for (uint32_t i = 1; i < ns; i++)
        if (splitters[i] < splitters[i - 1]) return fail(ctx, MASHGPU_ERR_INVALID, "splitters must be ascending");
    DevBuf<uint64_t> d_spl, d_pos;
    if (d_spl.alloc(ns) != cudaSuccess || d_pos.alloc(ns) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory");
    std::vector<uint64_t> pos(ns);
    MG_CUDA(ctx, cudaMemcpyAsync(d_spl.p, splitters, ns * 8ull, cudaMemcpyHostToDevice, st));
    dict_split_kernel<<<blocks_for(ns, 64), 64, 0, st>>>(d_keys, n, d_spl.p, ns, d_pos.p);
    MG_CUDA(ctx, cudaGetLastError());
    MG_CUDA(ctx, cudaMemcpyAsync(pos.data(), d_pos.p, ns * 8ull, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->kernel_launches++;
    uint64_t prev = 0;
    for (uint32_t p = 0; p < ns; p++) { counts[p] = pos[p] - prev; prev = pos[p]; }
    counts[ns] = n - prev;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dict_rank(mashgpu_ctx *ctx, const uint64_t *d_keys, uint64_t n, uint32_t *d_codes, uint64_t *n_distinct, void *stream)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!n_distinct) return fail(ctx, MASHGPU_ERR_INVALID, "n_distinct is NULL");
    *n_distinct = 0;
    if (n == 0) return MASHGPU_OK;
    if (!d_keys || !d_codes) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    if (n >= 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^31 hashes in one dictionary sort");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    DevBuf<uint64_t> keys; DevBuf<uint32_t> pos;
    if (keys.alloc(n) != cudaSuccess || pos.alloc(n) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (dictionary scratch for %llu hashes)", (unsigned long long)n);
    MG_CUDA(ctx, cudaMemcpyAsync(keys.p, d_keys, n * 8, cudaMemcpyDeviceToDevice, st));
    iota_kernel<<<blocks_for(n), 256, 0, st>>>(pos.p, n);
    ctx->kernel_launches++;
    return dict_rank(ctx, keys.p, pos.p, n, d_codes, n_distinct, st);
}

extern "C" int mashgpu_dict_scatter(mashgpu_ctx *ctx, const uint32_t *d_codes, const uint32_t *d_slots, const uint64_t *seg_counts,
                                    const uint64_t *seg_base, uint32_t n_segs, const mashgpu_sketch_set *set, uint64_t sketch_size,
                                    uint32_t *d_rows, uint32_t *d_n_eff, void *stream)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    MG_TRY(check_set(ctx, set, "sketch", false));
    if (sketch_size < 1 || sketch_size > 0x7FFFFFF0ull) return fail(ctx, MASHGPU_ERR_INVALID, "sketch_size out of range");
    if (set->n == 0) return MASHGPU_OK;
    if (!d_rows || !d_n_eff || !seg_counts || !seg_base || n_segs == 0) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    const uint32_t P = (uint32_t)sketch_size + 1;
    uint64_t n = 0;
    std::vector<uint64_t> seg_end(n_segs);
    for (uint32_t g = 0; g < n_segs; g++) { n += seg_counts[g]; seg_end[g] = n; }
    if (n && (!d_codes || !d_slots)) return fail(ctx, MASHGPU_ERR_INVALID, "NULL codes");
    DevBuf<uint64_t> d_seg; DevBuf<uint32_t> d_err, d_nh;
    if (d_seg.alloc(2ull * n_segs) != cudaSuccess || d_err.alloc(1) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory");
    MG_CUDA(ctx, cudaMemcpyAsync(d_seg.p, seg_end.data(), n_segs * 8ull, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(d_seg.p + n_segs, seg_base, n_segs * 8ull, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemsetAsync(d_err.p, 0, 4, st));
    MG_CUDA(ctx, cudaMemsetAsync(d_rows, 0xFF, set->n * (uint64_t)P * 4, st));
    const uint32_t *n_hashes = set->n_hashes;
    if (!set->on_device) {
        if (d_nh.alloc(set->n) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory");
        MG_CUDA(ctx, cudaMemcpyAsync(d_nh.p, set->n_hashes, set->n * 4, cudaMemcpyHostToDevice, st));
        n_hashes = d_nh.p;
    }
    dict_neff_kernel<<<blocks_for(set->n), 256, 0, st>>>(n_hashes, set->n, P, set->stride, 0, d_n_eff);
    if (n) dict_scatter_seg_kernel<<<blocks_for(n), 256, 0, st>>>(d_codes, d_slots, n, d_seg.p, d_seg.p + n_segs, n_segs, d_rows, d_err.p);
    MG_CUDA(ctx, cudaGetLastError());
    uint32_t err = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&err, d_err.p, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->kernel_launches += 2;
    if (err) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^32 - 1 distinct hashes in the collection");
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_set_prefilter(mashgpu_dist_job *job, int mode)
{
    if (!job) return MASHGPU_ERR_INVALID;
    job->prefilter_mode = mode > 0 ? 1 : (mode == 0 ? 0 : -1);
    job->auto_off = false;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_set_triangle(mashgpu_dist_job *job, int on)
{
    if (!job) return MASHGPU_ERR_INVALID;
    if (on && !job->self && job->d_ranks == job->ranks.p)
        return fail(job->ctx, MASHGPU_ERR_INVALID, "triangle enumeration needs a self comparison (qry == NULL) or an encoded job");
    job->triangle = on != 0;
    return MASHGPU_OK;
}

// auto mode: looks at the last snapshot of the flagged-combination counter, if it has arrived.  When most (query, tile)
// combinations share hashes the probe is pure overhead -- merge everything from then on.
static void dist_collect_flags(mashgpu_dist_job *job)
{
    if (!job->flag_pending) return;
    if (cudaEventQuery(job->flag_event) != cudaSuccess) { cudaGetLastError(); return; }
    job->flag_pending = false;
    const uint64_t flagged = *job->h_flag_total.p;
    if (job->prefilter_mode < 0 && job->snap_combos >= 64 && flagged * 2 > job->snap_combos) job->auto_off = true;
}

extern "C" int mashgpu_dist_prefilter_stats(mashgpu_dist_job *job, uint64_t *combos_probed, uint64_t *combos_flagged, int *active)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    unsigned long long flagged = 0;
    if (job->flag_total.p) {
        MG_CUDA(ctx, cudaDeviceSynchronize());
        MG_CUDA(ctx, cudaMemcpy(&flagged, job->flag_total.p, 8, cudaMemcpyDeviceToHost));
    }
    dist_collect_flags(job);
    if (combos_probed) *combos_probed = job->combos_probed;
    if (combos_flagged) *combos_flagged = flagged;
    if (active) *active = job->tiled && (job->prefilter_mode > 0 || (job->prefilter_mode < 0 && !job->auto_off));
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_pair_stats(mashgpu_dist_job *job, uint64_t *pairs_merged_from_lists)
{
    if (!job || !pairs_merged_from_lists) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    *pairs_merged_from_lists = 0;
    if (!job->pair_count.p) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_CUDA(ctx, cudaDeviceSynchronize());
    unsigned long long v = 0;
    MG_CUDA(ctx, cudaMemcpy(&v, job->pair_count.p + 2, 8, cudaMemcpyDeviceToHost));
    *pairs_merged_from_lists = v;
    return MASHGPU_OK;
}

namespace {

// The arguments of a run of queries [q_begin, q_begin + q_count): the job's tables and rows, the range and the triangle.  Every
// output field is NULL; the caller sets the run's target (dense outputs, pass list or best-hit capture) before dist_enqueue.
DistArgs dist_args(const mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count)
{
    DistArgs a{};
    a.ranks = job->d_ranks; a.P = job->P; a.S = (uint32_t)job->params.sketch_size;
    a.ref_n = job->d_n_eff + job->ref_row0; a.ref_len = job->d_lens + job->ref_row0; a.ref_row0 = job->ref_row0;
    a.qry_n = job->d_n_eff + job->qry_row0; a.qry_len = job->d_lens + job->qry_row0; a.qry_row0 = job->qry_row0;
    a.n_ref = (uint32_t)job->n_ref; a.q_begin = (uint32_t)q_begin; a.q_count = (uint32_t)q_count;
    a.kmer_size = job->params.kmer_size; a.kmer_space = job->params.kmer_space;
    a.max_distance = job->params.max_distance; a.max_pvalue = job->params.max_pvalue;
    a.dist_lut = job->lut.p;
    a.binom.mant = job->binom_m.p; a.binom.expo = job->binom_e.p; a.binom.n0 = job->params.sketch_size;
    a.triangle = job->triangle ? 1 : 0;
    a.tri_r0 = job->self ? 0u : (uint32_t)job->ref_row0;
    return a;
}

// Enqueues a run on `st` (a.q_count >= 1, n_ref >= 1, the device current): the merge path for the job (prefilter and pair list,
// dense tiles, warp per pair or one thread per pair), the p-value pass, the launch counters and the prefilter's flag snapshot.
int dist_enqueue(mashgpu_dist_job *job, DistArgs a, cudaStream_t st)
{
    mashgpu_ctx *ctx = job->ctx;
    const uint64_t q_count = a.q_count;
    {   // queue for the deferred p-values: 1/16 of the pairs (at least 2^20); beyond that dist_emit evaluates in place
        const uint64_t pairs = q_count * job->n_ref;
        const uint64_t cap = std::min<uint64_t>(pairs, std::max<uint64_t>(1ull << 20, pairs / 16));
        if (job->fix_list.n < cap && job->fix_list.alloc(cap) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (p-value queue)");
        if (!job->fix_count.p && job->fix_count.alloc(1) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (p-value queue)");
        MG_CUDA(ctx, cudaMemsetAsync(job->fix_count.p, 0, 8, st));
        a.fix_list = job->fix_list.p; a.fix_count = job->fix_count.p; a.fix_capacity = cap;
    }
    auto launch_fix = [&]() {
        dist_fix_kernel<<<ctx->sm_count * 8, 256, 0, st>>>(a);
        ctx->kernel_launches++;
        return cudaGetLastError();
    };
    // warp-per-pair merge: shared memory for two rows of S ranks per warp
    const uint32_t run0 = ((a.S + 31u) / 32u) | 1u;          // first-round run: odd, 32 runs cover the row
    const uint32_t row_pitch = (a.S + 1u + 8u + 3u) & ~3u;    // S elements + sentinel + skew and 16-byte rounding of the bulk copy
    const int pair_warps = (int)std::min<size_t>(PAIR_WARPS_MAX, (220 * 1024) / ((size_t)row_pitch * 8));
    auto launch_pairs = [&]() {
        const size_t smem_p = (size_t)pair_warps * 2 * row_pitch * 4 + (size_t)pair_warps * 8;
        const int ctas_per_sm = (int)std::max<size_t>(1, std::min<size_t>(4, (220 * 1024) / std::max<size_t>(smem_p, 1)));
        dist_pair_kernel<<<ctx->sm_count * ctas_per_sm, pair_warps * 32, smem_p, st>>>(a, row_pitch, run0);
        ctx->kernel_launches++;
        return cudaGetLastError();
    };
    if (!job->tiled && pair_warps >= 1) {
        // sketch sizes whose 32-reference tile does not fit shared memory (s >= 1035, e.g. `-s 10000`): every pair by the warp-per-pair merge
        a.pair_dense = 1;
        time_begin(ctx, ctx->dist_events, st);
        MG_CUDA(ctx, launch_pairs());
        MG_CUDA(ctx, launch_fix());
        time_end(ctx, ctx->dist_events, st);
        ctx->dist_launches++;
        return MASHGPU_OK;
    }
    if (!job->tiled) {
        const uint64_t total = q_count * job->n_ref;
        time_begin(ctx, ctx->dist_events, st);
        dist_kernel_general<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(a);
        MG_CUDA(ctx, cudaGetLastError());
        MG_CUDA(ctx, launch_fix());
        time_end(ctx, ctx->dist_events, st);
        ctx->kernel_launches++;
        ctx->dist_launches++;
        return MASHGPU_OK;
    }
    const uint32_t r_tiles = (uint32_t)((job->n_ref + DIST_TILE_R - 1) / DIST_TILE_R);
    const uint32_t round = DIST_WARPS * DIST_ILP;
    const size_t smem = dist_smem_bytes(a.P);
    dist_collect_flags(job);
    const bool prefilter = job->prefilter_mode > 0 || (job->prefilter_mode < 0 && !job->auto_off);
    if (prefilter) {
        // pass 1: dist_probe_kernel writes the closed form for (query, tile) combinations without a shared hash and
        // lists the others per tile; pass 2: dist_kernel merges the listed ones.
        const uint64_t need = (uint64_t)r_tiles * q_count;
        if (job->qlist.n < need && job->qlist.alloc(need + need / 4) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (prefilter work lists)");
        if (job->qcount.n < r_tiles && job->qcount.alloc(r_tiles) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (prefilter counters)");
        if (!job->flag_total.p) {
            if (job->flag_total.alloc(1) != cudaSuccess || job->h_flag_total.alloc(1) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of memory (prefilter counter)");
            MG_CUDA(ctx, cudaEventCreateWithFlags(&job->flag_event, cudaEventDisableTiming));
            MG_CUDA(ctx, cudaMemsetAsync(job->flag_total.p, 0, 8, st));
        }
        MG_CUDA(ctx, cudaMemsetAsync(job->qcount.p, 0, (size_t)r_tiles * 4, st));
        a.qlist = job->qlist.p; a.qcount = job->qcount.p; a.qlist_stride = q_count; a.flag_total = job->flag_total.p;
        if (job->pair_max > 0 && pair_warps >= 1) {
            const uint64_t pairs = q_count * job->n_ref;
            const uint64_t cap = std::max<uint64_t>(1ull << 20, pairs / 16);
            if (job->pair_list.n < cap && job->pair_list.alloc(cap) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (pair list)");
            if (!job->pair_count.p) {
                if (job->pair_count.alloc(3) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (pair counter)");
                MG_CUDA(ctx, cudaMemsetAsync(job->pair_count.p, 0, 24, st));
            }
            MG_CUDA(ctx, cudaMemsetAsync(job->pair_count.p, 0, 16, st));
            a.pair_list = job->pair_list.p; a.pair_count = job->pair_count.p; a.pair_full = job->pair_count.p + 1; a.pair_total = job->pair_count.p + 2;
            a.pair_capacity = job->pair_list.n; a.pair_max = job->pair_max;
        }
        // probe: one CTA keeps its filter for a long run of queries (the build costs about as much as probing ~100 queries)
        uint32_t p_slices = std::max(1u, (uint32_t)(2 * ctx->sm_count + r_tiles - 1) / r_tiles);
        uint32_t p_per_cta = (uint32_t)((q_count + p_slices - 1) / p_slices);
        p_per_cta = std::max<uint32_t>(p_per_cta, PROBE_WARPS);
        p_slices = (uint32_t)((q_count + p_per_cta - 1) / p_per_cta);
        a.q_per_cta = p_per_cta;
        time_begin(ctx, ctx->dist_events, st);
        // without the pair path the kernel keeps 128 KB of shared memory and twice the L1 (query rows stream through L1)
        const size_t probe_smem = a.pair_max > 0 ? PROBE_SMEM : CF_BUCKETS * sizeof(uint32_t);
        dist_probe_kernel<<<dim3(r_tiles, p_slices), PROBE_THREADS, probe_smem, st>>>(a);
        time_end(ctx, ctx->dist_events, st);
        MG_CUDA(ctx, cudaGetLastError());
        // merge the listed combinations: a few CTAs per tile walk its list (CTAs of tiles with short lists exit at once)
        a.use_qlist = 1;
        a.q_per_cta = 2 * round;
        const uint32_t m_slices = (uint32_t)std::min<uint64_t>(8, (q_count + a.q_per_cta - 1) / a.q_per_cta);
        time_begin(ctx, ctx->dist_events, st);
        dist_kernel<<<dim3(r_tiles, m_slices), DIST_THREADS, smem, st>>>(a);
        MG_CUDA(ctx, cudaGetLastError());
        if (a.pair_list) MG_CUDA(ctx, launch_pairs());
        MG_CUDA(ctx, launch_fix());
        time_end(ctx, ctx->dist_events, st);
        job->combos_probed += need;
        if (!job->flag_pending) {           // snapshot of the running flagged count for the auto switch (never waited for)
            MG_CUDA(ctx, cudaMemcpyAsync(job->h_flag_total.p, job->flag_total.p, 8, cudaMemcpyDeviceToHost, st));
            MG_CUDA(ctx, cudaEventRecord(job->flag_event, st));
            job->flag_pending = true;
            job->snap_combos = job->combos_probed;
        }
        ctx->kernel_launches += 2;
        ctx->dist_launches += 2;
        return MASHGPU_OK;
    }
    const dim3 grid = dense_grid(r_tiles, q_count, ctx->sm_count, a.q_per_cta);
    time_begin(ctx, ctx->dist_events, st);
    dist_kernel<<<grid, DIST_THREADS, smem, st>>>(a);
    MG_CUDA(ctx, cudaGetLastError());
    MG_CUDA(ctx, launch_fix());
    time_end(ctx, ctx->dist_events, st);
    ctx->kernel_launches++;
    ctx->dist_launches++;
    return MASHGPU_OK;
}

}  // namespace

extern "C" int mashgpu_dist_run_dev(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count,
                                    uint32_t *d_numer, uint32_t *d_denom, double *d_distance, double *d_pvalue, uint8_t *d_pass,
                                    void *stream)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (q_begin + q_count > job->n_qry) return fail(ctx, MASHGPU_ERR_INVALID, "query range [%llu, %llu) exceeds %llu", (unsigned long long)q_begin, (unsigned long long)(q_begin + q_count), (unsigned long long)job->n_qry);
    if (q_count == 0 || job->n_ref == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    DistArgs a = dist_args(job, q_begin, q_count);
    a.numer = d_numer; a.denom = d_denom; a.distance = d_distance; a.pvalue = d_pvalue; a.pass = d_pass;
    return dist_enqueue(job, a, stream ? (cudaStream_t)stream : ctx->stream);
}

extern "C" int mashgpu_dist_run(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count,
                                uint32_t *numer, uint32_t *denom, double *distance, double *pvalue, uint8_t *pass)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (q_begin + q_count > job->n_qry) return fail(ctx, MASHGPU_ERR_INVALID, "query range exceeds query count");
    if (q_count == 0 || job->n_ref == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    // bound the device outputs: chunks of queries, 128 Mi pairs (~3.2 GB of outputs) per launch
    const uint64_t n_ref = job->n_ref;
    const uint64_t q_chunk = std::min(q_count, std::max<uint64_t>(1, (1ull << 27) / n_ref));
    const HostOut out[] = {{numer, 4 * n_ref}, {denom, 4 * n_ref}, {distance, 8 * n_ref}, {pvalue, 8 * n_ref}, {pass, n_ref}};
    // pairs on or above the diagonal of a triangle run are not written by the kernels: hand zeros back for them
    return run_host_chunks(ctx, out, q_count, q_chunk, job->triangle, "pair outputs", [&](uint64_t q, uint64_t qc, void *const *d) {
        return mashgpu_dist_run_dev(job, q_begin + q, qc, (uint32_t *)d[0], (uint32_t *)d[1], (double *)d[2], (double *)d[3], (uint8_t *)d[4], ctx->stream);
    });
}

extern "C" int mashgpu_dist_run_list(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count, uint64_t capacity,
                                     uint64_t *pair_index, uint32_t *numer, uint32_t *denom, double *distance, double *pvalue, uint64_t *n_pass)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (!n_pass) return fail(ctx, MASHGPU_ERR_INVALID, "n_pass is NULL");
    *n_pass = 0;
    if (q_begin + q_count > job->n_qry) return fail(ctx, MASHGPU_ERR_INVALID, "query range exceeds query count");
    if (q_count == 0 || job->n_ref == 0) return MASHGPU_OK;
    if (capacity >= 0xFFFFFFFFull) return fail(ctx, MASHGPU_ERR_INVALID, "capacity must be below 2^32");
    if (capacity && (!pair_index || !numer || !denom || !distance || !pvalue)) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    const uint64_t cap = std::max<uint64_t>(capacity, 1);
    mashgpu_dist_job &J = *job;       // grow-only list buffers: no cudaMalloc per call once they are large enough
    if (J.l_idx.reserve(cap) != cudaSuccess || J.s_idx.reserve(cap) != cudaSuccess || J.l_n.reserve(cap) != cudaSuccess || J.l_d.reserve(cap) != cudaSuccess ||
        J.l_D.reserve(cap) != cudaSuccess || J.l_P.reserve(cap) != cudaSuccess || J.l_order.reserve(cap) != cudaSuccess || J.s_order.reserve(cap) != cudaSuccess ||
        J.o_n.reserve(cap) != cudaSuccess || J.o_d.reserve(cap) != cudaSuccess || J.o_D.reserve(cap) != cudaSuccess || J.o_P.reserve(cap) != cudaSuccess ||
        J.l_cnt.reserve(1) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (pass list of %llu entries)", (unsigned long long)cap);
    MG_CUDA(ctx, cudaMemsetAsync(J.l_cnt.p, 0, 8, st));
    DistArgs a = dist_args(job, q_begin, q_count);
    a.list_idx = J.l_idx.p; a.list_numer = J.l_n.p; a.list_denom = J.l_d.p; a.list_distance = J.l_D.p; a.list_pvalue = J.l_P.p;
    a.list_count = J.l_cnt.p; a.list_capacity = capacity;
    MG_TRY(dist_enqueue(job, a, st));
    unsigned long long n = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&n, J.l_cnt.p, 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    *n_pass = n;
    if (n == 0 || n > capacity) return MASHGPU_OK;      // overflow: the caller retries with a larger capacity (or the dense call)
    // restore the reference's output order (query-major pair index): sort the list by pair index on the device
    const unsigned tb = 256, nb = (unsigned)((n + tb - 1) / tb);
    iota_kernel<<<nb, tb, 0, st>>>(J.l_order.p, n);
    // the pair index is below q_count * n_ref: sort only the bits that can be set
    int end_bit = 1;
    while (end_bit < 64 && ((q_count * job->n_ref) >> end_bit)) end_bit++;
    size_t tmp_bytes = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, J.l_idx.p, J.s_idx.p, J.l_order.p, J.s_order.p, (int)n, 0, end_bit, st);
    if (J.l_tmp.reserve(tmp_bytes) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sort scratch)");
    MG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(J.l_tmp.p, tmp_bytes, J.l_idx.p, J.s_idx.p, J.l_order.p, J.s_order.p, (int)n, 0, end_bit, st));
    list_gather_kernel<<<nb, tb, 0, st>>>(J.s_order.p, n, J.l_n.p, J.l_d.p, J.l_D.p, J.l_P.p, J.o_n.p, J.o_d.p, J.o_D.p, J.o_P.p);
    ctx->kernel_launches += 10;
    MG_CUDA(ctx, cudaMemcpyAsync(pair_index, J.s_idx.p, n * 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(numer, J.o_n.p, n * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(denom, J.o_d.p, n * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(distance, J.o_D.p, n * 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(pvalue, J.o_P.p, n * 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    return MASHGPU_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Best hits (DESIGN.md 3.7)
// ---------------------------------------------------------------------------------------------------------
constexpr uint64_t BEST_DEFAULT_CAPACITY = 1ull << 25;      // candidates: 1 GiB of capture buffer and 1 GiB of grouped copy
constexpr uint64_t BEST_BLOCK_PAIRS = 1ull << 31;           // pairs of a starting block: bounds the work lists and queues of one run
constexpr uint64_t BEST_HOST_ENTRIES = 1ull << 24;          // q x n_best entries per device output chunk of the host call

extern "C" int mashgpu_dist_set_best_capacity(mashgpu_dist_job *job, uint64_t entries)
{
    if (!job) return MASHGPU_ERR_INVALID;
    job->best_capacity = std::min<uint64_t>(entries, 0xFFFFFFFFull);       // segment offsets are 32-bit
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_best_stats(mashgpu_dist_job *job, uint64_t *blocks_run, uint64_t *blocks_split, uint64_t *candidates, double *select_ms)
{
    if (!job) return MASHGPU_ERR_INVALID;
    cudaSetDevice(job->ctx->device);
    for (auto &ev : job->best_events) {
        cudaEventSynchronize(ev.b);
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ev.a, ev.b) == cudaSuccess) job->best_select_ms += ms;
        cudaEventDestroy(ev.a);
        cudaEventDestroy(ev.b);
    }
    job->best_events.clear();
    if (blocks_run) *blocks_run = job->best_blocks;
    if (blocks_split) *blocks_split = job->best_splits;
    if (candidates) *candidates = job->best_candidates;
    if (select_ms) *select_ms = job->best_select_ms;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_run_best_dev(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count, uint32_t n_best,
                                         uint32_t *d_n_hits, uint32_t *d_n_total, uint32_t *d_ref, uint32_t *d_numer, uint32_t *d_denom,
                                         double *d_distance, double *d_pvalue, void *stream)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (n_best == 0) return fail(ctx, MASHGPU_ERR_INVALID, "n_best must be at least 1");
    if (n_best > BEST_MAX_N) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "n_best %u exceeds %u", n_best, BEST_MAX_N);
    if (q_begin + q_count > job->n_qry) return fail(ctx, MASHGPU_ERR_INVALID, "query range [%llu, %llu) exceeds %llu", (unsigned long long)q_begin, (unsigned long long)(q_begin + q_count), (unsigned long long)job->n_qry);
    if (q_count == 0) return MASHGPU_OK;
    if (!d_n_hits || !d_ref || !d_numer || !d_denom || !d_distance || !d_pvalue) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    const uint64_t n_ref = job->n_ref;
    if (n_ref == 0) {       // no reference, no hit
        const uint64_t e = q_count * n_best;
        MG_CUDA(ctx, cudaMemsetAsync(d_n_hits, 0, q_count * 4, st));
        if (d_n_total) MG_CUDA(ctx, cudaMemsetAsync(d_n_total, 0, q_count * 4, st));
        MG_CUDA(ctx, cudaMemsetAsync(d_ref, 0, e * 4, st)); MG_CUDA(ctx, cudaMemsetAsync(d_numer, 0, e * 4, st)); MG_CUDA(ctx, cudaMemsetAsync(d_denom, 0, e * 4, st));
        MG_CUDA(ctx, cudaMemsetAsync(d_distance, 0, e * 8, st)); MG_CUDA(ctx, cudaMemsetAsync(d_pvalue, 0, e * 8, st));
        return MASHGPU_OK;
    }
    // never below n_ref: a block of one query always fits, which is where the halving below ends
    const uint64_t capacity = std::max<uint64_t>(n_ref, job->best_capacity ? job->best_capacity : BEST_DEFAULT_CAPACITY);
    const uint64_t block0 = std::max<uint64_t>(1, BEST_BLOCK_PAIRS / n_ref);
    uint32_t kw = 1;
    while (kw < n_best) kw <<= 1;
    mashgpu_dist_job &J = *job;
    // blocks still to run, next one last; a block whose candidates overflow the buffer is replaced by its two halves
    std::vector<std::pair<uint64_t, uint64_t>> todo;
    for (uint64_t q = (q_count + block0 - 1) / block0; q-- > 0;) todo.push_back({q * block0, std::min(block0, q_count - q * block0)});
    while (!todo.empty()) {
        const uint64_t b0 = todo.back().first, bn = todo.back().second;
        todo.pop_back();
        const uint64_t cap = std::min(capacity, bn * n_ref);        // a block has at most bn * n_ref hits
        if (J.b_cand.reserve(cap) != cudaSuccess || J.b_grouped.reserve(cap) != cudaSuccess || J.b_q.reserve(3 * bn) != cudaSuccess || J.b_cnt.reserve(1) != cudaSuccess)
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (best-hit candidates: %llu entries)", (unsigned long long)cap);
        uint32_t *qcnt = J.b_q.p, *qoff = qcnt + bn, *cursor = qoff + bn;
        MG_CUDA(ctx, cudaMemsetAsync(J.b_cnt.p, 0, 8, st));
        MG_CUDA(ctx, cudaMemsetAsync(qcnt, 0, 3 * bn * 4, st));
        DistArgs a = dist_args(job, q_begin + b0, bn);
        a.best = BestCapture{J.b_cand.p, J.b_cnt.p, cap, qcnt};
        MG_TRY(dist_enqueue(job, a, st));
        unsigned long long n = 0;
        MG_CUDA(ctx, cudaMemcpyAsync(&n, J.b_cnt.p, 8, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
        job->best_blocks++;
        if (n > cap) {      // bn >= 2 here: one query has at most n_ref <= cap hits
            job->best_splits++;
            todo.push_back({b0 + bn / 2, bn - bn / 2});
            todo.push_back({b0, bn / 2});
            continue;
        }
        job->best_candidates += n;
        time_begin(ctx, job->best_events, st);
        size_t tb = 0;
        cub::DeviceScan::ExclusiveSum(nullptr, tb, qcnt, qoff, (int)bn, st);
        if (J.b_tmp.reserve(tb) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (scan scratch)");
        MG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(J.b_tmp.p, tb, qcnt, qoff, (int)bn, st));
        if (n) best_scatter_kernel<<<blocks_for(n), 256, 0, st>>>(J.b_cand.p, n, qoff, cursor, J.b_grouped.p);
        const BestOut o{d_n_hits + b0, d_n_total ? d_n_total + b0 : nullptr, d_ref + b0 * n_best, d_numer + b0 * n_best, d_denom + b0 * n_best,
                        d_distance + b0 * n_best, d_pvalue + b0 * n_best};
        dist_best_kernel<<<blocks_for(bn, BEST_WARPS), BEST_THREADS, 0, st>>>(J.b_grouped.p, qoff, qcnt, (uint32_t)bn, n_best, kw, o);
        MG_CUDA(ctx, cudaGetLastError());
        time_end(ctx, job->best_events, st);
        ctx->kernel_launches += 4;
    }
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_run_best(mashgpu_dist_job *job, uint64_t q_begin, uint64_t q_count, uint32_t n_best,
                                     uint32_t *n_hits, uint32_t *n_total, uint32_t *ref, uint32_t *numer, uint32_t *denom, double *distance, double *pvalue)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (n_best == 0) return fail(ctx, MASHGPU_ERR_INVALID, "n_best must be at least 1");
    if (n_best > BEST_MAX_N) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "n_best %u exceeds %u", n_best, BEST_MAX_N);
    if (q_begin + q_count > job->n_qry) return fail(ctx, MASHGPU_ERR_INVALID, "query range exceeds query count");
    if (q_count == 0) return MASHGPU_OK;
    if (!n_hits || !ref || !numer || !denom || !distance || !pvalue) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    // bound the device outputs: chunks of queries (each is cut into blocks by the device call)
    const uint64_t q_chunk = std::min<uint64_t>(q_count, std::max<uint64_t>(1, BEST_HOST_ENTRIES / n_best));
    const uint64_t e4 = 4ull * n_best, e8 = 8ull * n_best;
    const HostOut out[] = {{n_hits, 4}, {n_total, 4}, {ref, e4}, {numer, e4}, {denom, e4}, {distance, e8}, {pvalue, e8}};
    return run_host_chunks(ctx, out, q_count, q_chunk, false, "best-hit outputs", [&](uint64_t q, uint64_t qc, void *const *d) {
        return mashgpu_dist_run_best_dev(job, q_begin + q, qc, n_best, (uint32_t *)d[0], (uint32_t *)d[1], (uint32_t *)d[2], (uint32_t *)d[3],
                                         (uint32_t *)d[4], (double *)d[5], (double *)d[6], ctx->stream);
    });
}

// ---------------------------------------------------------------------------------------------------------
// Connected components (DESIGN.md 3.8)
// ---------------------------------------------------------------------------------------------------------
constexpr uint64_t TRIANGLE_RUN_PAIRS = 1ull << 31;     // pairs of one lower-triangle run: bounds its work lists, pair list and p-value queue

// components and spanning forests read the lower triangle of a self or encoded job; `what` starts the refusal
static int need_self_or_encoded(mashgpu_dist_job *job, const char *what)
{
    return job->self || job->encoded ? MASHGPU_OK : fail(job->ctx, MASHGPU_ERR_INVALID, "%s a self comparison (qry == NULL) or an encoded job", what);
}

// Queries of one lower-triangle run by default
static uint64_t triangle_block(const mashgpu_dist_job *job)
{
    return std::max<uint64_t>(1, TRIANGLE_RUN_PAIRS / std::max<uint64_t>(job->n_ref, 1));
}

// Runs every pair of the lower triangle of a self or encoded job once, in blocks of `block` queries (0: triangle_block), with the capture
// that set_target puts into each run's arguments; after_run(a) enqueues what follows each block's run (greedy dereplication resolves the
// block there).  Lower triangle whatever the job's own setting: query q meets the rows below it only, so the queries up to the first
// reference row have no pair at all.  Nothing can overflow, so no block is ever run twice.
template <class SetTarget, class AfterRun>
static int enqueue_lower_triangle(mashgpu_dist_job *job, cudaStream_t st, SetTarget set_target, uint64_t block, AfterRun after_run)
{
    const uint64_t n = job->n_qry, n_ref = job->n_ref;
    const uint64_t q_first = job->self ? 1 : job->ref_row0 + 1;
    if (block == 0) block = triangle_block(job);
    for (uint64_t q0 = q_first; n_ref && q0 < n; q0 += block) {
        DistArgs a = dist_args(job, q0, std::min(block, n - q0));
        a.triangle = 1;
        set_target(a);
        MG_TRY(dist_enqueue(job, a, st));
        MG_TRY(after_run(a));
    }
    return MASHGPU_OK;
}

template <class SetTarget>
static int enqueue_lower_triangle(mashgpu_dist_job *job, cudaStream_t st, SetTarget set_target)
{
    return enqueue_lower_triangle(job, st, set_target, 0, [](const DistArgs &) { return (int)MASHGPU_OK; });
}

extern "C" int mashgpu_dist_components_dev(mashgpu_dist_job *job, uint32_t *d_labels, uint64_t *n_edges, void *stream)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    MG_TRY(need_self_or_encoded(job, "components need"));
    if (!d_labels || !n_edges) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    *n_edges = 0;
    const uint64_t n = job->n_qry;
    if (n == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    if (job->cc_edges.reserve(1) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (edge counter)");
    MG_CUDA(ctx, cudaMemsetAsync(job->cc_edges.p, 0, 8, st));
    cc_init_kernel<<<blocks_for(n), 256, 0, st>>>(d_labels, n);
    MG_CUDA(ctx, cudaGetLastError());
    // the labels are the forest
    MG_TRY(enqueue_lower_triangle(job, st, [&](DistArgs &a) { a.graph = GraphCapture{d_labels, job->cc_edges.p, nullptr}; }));
    cc_flatten_kernel<<<blocks_for(n), 256, 0, st>>>(d_labels, n);
    MG_CUDA(ctx, cudaGetLastError());
    ctx->kernel_launches += 2;
    unsigned long long e = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&e, job->cc_edges.p, 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    *n_edges = e;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_components(mashgpu_dist_job *job, uint32_t *labels, uint64_t *n_edges)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    MG_TRY(need_self_or_encoded(job, "components need"));
    if (!labels || !n_edges) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    *n_edges = 0;
    const uint64_t n = job->n_qry;
    if (n == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    DevBuf<uint32_t> d;
    if (d.alloc(n) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (%llu labels)", (unsigned long long)n);
    MG_TRY(mashgpu_dist_components_dev(job, d.p, n_edges, ctx->stream));
    MG_CUDA(ctx, cudaMemcpyAsync(labels, d.p, n * 4, cudaMemcpyDeviceToHost, ctx->stream));
    MG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    return MASHGPU_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Minimum spanning forest (DESIGN.md 3.9)
// ---------------------------------------------------------------------------------------------------------
extern "C" int mashgpu_dist_spanning_forest_dev(mashgpu_dist_job *job, uint32_t *d_row, uint32_t *d_col, uint32_t *d_numer, uint32_t *d_denom,
                                                double *d_distance, double *d_pvalue, uint64_t *n_edges, uint64_t *n_rounds, void *stream)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    MG_TRY(need_self_or_encoded(job, "a spanning forest needs"));
    if (!d_row || !d_col || !d_numer || !d_denom || !d_distance || !d_pvalue || !n_edges || !n_rounds) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    *n_edges = 0; *n_rounds = 0;
    const uint64_t n = job->n_qry;
    if (n < 2 || job->n_ref == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    const uint64_t cap = n - 1;
    // O(n) state: labels, the union-find of the forest, one slot per component, the forest's keys and their sorted copy
    DevBuf<uint32_t> label, parent; DevBuf<MsfKey> best; DevBuf<unsigned long long> lo, hi, lo2, hi2, count; DevBuf<uint8_t> tmp;
    if (label.alloc(n) != cudaSuccess || parent.alloc(n) != cudaSuccess || best.alloc(n) != cudaSuccess || lo.alloc(cap) != cudaSuccess ||
        hi.alloc(cap) != cudaSuccess || lo2.alloc(cap) != cudaSuccess || hi2.alloc(cap) != cudaSuccess || count.alloc(1) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (spanning forest of %llu sketches)", (unsigned long long)n);
    cc_init_kernel<<<blocks_for(n), 256, 0, st>>>(label.p, n);
    cc_init_kernel<<<blocks_for(n), 256, 0, st>>>(parent.p, n);
    MG_CUDA(ctx, cudaMemsetAsync(count.p, 0, 8, st));
    MG_CUDA(ctx, cudaGetLastError());
    ctx->kernel_launches += 2;
    // A productive round joins every component that has an edge to another one, so it at least halves their number: more than
    // ceil(log2 n) + 1 rounds (the last one finds no edge) cannot happen.
    uint64_t max_rounds = 1;
    while ((1ull << (max_rounds - 1)) < n) max_rounds++;
    unsigned long long edges = 0;
    uint64_t rounds = 0;
    while (edges < cap) {
        if (rounds == max_rounds) return fail(ctx, MASHGPU_ERR_CUDA, "internal error: spanning forest not done after %llu rounds", (unsigned long long)rounds);
        MG_CUDA(ctx, cudaMemsetAsync(best.p, 0xFF, n * sizeof(MsfKey), st));
        MG_TRY(enqueue_lower_triangle(job, st, [&](DistArgs &a) { a.graph = GraphCapture{label.p, nullptr, best.p}; }));
        msf_hook_kernel<<<blocks_for(n), 256, 0, st>>>(label.p, best.p, parent.p, count.p, lo.p, hi.p, cap, n);
        cc_flatten_kernel<<<blocks_for(n), 256, 0, st>>>(parent.p, n);
        MG_CUDA(ctx, cudaGetLastError());
        MG_CUDA(ctx, cudaMemcpyAsync(label.p, parent.p, n * 4, cudaMemcpyDeviceToDevice, st));
        ctx->kernel_launches += 2;
        unsigned long long now = 0;
        MG_CUDA(ctx, cudaMemcpyAsync(&now, count.p, 8, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
        rounds++;
        if (now > cap) return fail(ctx, MASHGPU_ERR_CUDA, "internal error: %llu spanning forest edges over %llu sketches", now, (unsigned long long)n);
        if (now == edges) break;
        edges = now;
    }
    *n_rounds = rounds;
    if (edges == 0) return MASHGPU_OK;
    // forest order: (j, i) first, then a stable pass on the distance bits
    size_t tb = 0;
    cub::DeviceRadixSort::SortPairs(nullptr, tb, lo.p, lo2.p, hi.p, hi2.p, (int)edges, 0, 64, st);
    if (tmp.alloc(tb) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sort scratch)");
    MG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp.p, tb, lo.p, lo2.p, hi.p, hi2.p, (int)edges, 0, 64, st));
    MG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp.p, tb, hi2.p, hi.p, lo2.p, lo.p, (int)edges, 0, 64, st));
    DistArgs a = dist_args(job, 0, n);
    msf_values_kernel<<<blocks_for(edges), 256, 0, st>>>(a, lo.p, edges, d_row, d_col, d_numer, d_denom, d_distance, d_pvalue);
    MG_CUDA(ctx, cudaGetLastError());
    MG_CUDA(ctx, cudaStreamSynchronize(st));        // the scratch goes out of scope
    ctx->kernel_launches += 9;         // two radix sorts and the values
    *n_edges = edges;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_spanning_forest(mashgpu_dist_job *job, uint32_t *row, uint32_t *col, uint32_t *numer, uint32_t *denom,
                                            double *distance, double *pvalue, uint64_t *n_edges, uint64_t *n_rounds)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    MG_TRY(need_self_or_encoded(job, "a spanning forest needs"));
    if (!row || !col || !numer || !denom || !distance || !pvalue || !n_edges || !n_rounds) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    *n_edges = 0; *n_rounds = 0;
    const uint64_t n = job->n_qry;
    if (n < 2) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    const uint64_t cap = n - 1;
    DevBuf<uint32_t> d32; DevBuf<double> d64;
    if (d32.alloc(4 * cap) != cudaSuccess || d64.alloc(2 * cap) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (%llu forest edges)", (unsigned long long)cap);
    MG_TRY(mashgpu_dist_spanning_forest_dev(job, d32.p, d32.p + cap, d32.p + 2 * cap, d32.p + 3 * cap, d64.p, d64.p + cap, n_edges, n_rounds, ctx->stream));
    const uint64_t m = *n_edges;
    cudaStream_t st = ctx->stream;
    MG_CUDA(ctx, cudaMemcpyAsync(row, d32.p, m * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(col, d32.p + cap, m * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(numer, d32.p + 2 * cap, m * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(denom, d32.p + 3 * cap, m * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(distance, d64.p, m * 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(pvalue, d64.p + cap, m * 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    return MASHGPU_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Greedy dereplication (DESIGN.md 3.12)
// ---------------------------------------------------------------------------------------------------------
extern "C" int mashgpu_dist_set_representative_block(mashgpu_dist_job *job, uint64_t rows)
{
    if (!job) return MASHGPU_ERR_INVALID;
    job->greedy_block = std::min<uint64_t>(rows, GREEDY_MAX_BLOCK);
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_representatives_dev(mashgpu_dist_job *job, uint32_t *d_rep, uint32_t *d_numer, uint32_t *d_denom, double *d_distance,
                                                double *d_pvalue, uint64_t *n_reps, uint64_t *n_rounds, void *stream)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (job->encoded) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "representatives of an encoded (sharded) job");
    if (!job->self) return fail(ctx, MASHGPU_ERR_INVALID, "representatives need a self comparison (qry == NULL)");
    if (!d_rep || !d_numer || !d_denom || !d_distance || !d_pvalue || !n_reps || !n_rounds) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    *n_reps = 0; *n_rounds = 0;
    const uint64_t n = job->n_qry;
    if (n == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    // pass-1 blocks of `block` rows from row 1 (sketch 0 is a representative from the start), each with its GreedyRun header; one
    // header more for pass 2
    const uint64_t block = std::min<uint64_t>({job->greedy_block ? job->greedy_block : triangle_block(job), GREEDY_MAX_BLOCK, std::max<uint64_t>(n - 1, 1)});
    const uint64_t pitch = (block + 31) / 32, n_blocks = (n - 1 + block - 1) / block;
    // O(n) state plus one block's bit matrix, its two pairs of row sets and the rows' extents
    DevBuf<uint32_t> status, bits, masks, extent; DevBuf<MsfKey> slot; DevBuf<GreedyRun> runs; DevBuf<int> ctl; DevBuf<unsigned long long> counters;
    if (status.alloc(n) != cudaSuccess || slot.alloc(n) != cudaSuccess || runs.alloc(n_blocks + 1) != cudaSuccess || counters.alloc(3) != cudaSuccess ||
        (n_blocks && (bits.alloc(block * pitch) != cudaSuccess || masks.alloc(4 * pitch) != cudaSuccess || extent.alloc(2 * block) != cudaSuccess ||
                      ctl.alloc(6) != cudaSuccess)))
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (representatives of %llu sketches in blocks of %llu)", (unsigned long long)n,
                    (unsigned long long)block);
    std::vector<GreedyRun> h_runs(n_blocks + 1);
    for (uint64_t b = 0; b < n_blocks; b++) h_runs[b] = GreedyRun{status.p, bits.p, nullptr, (uint32_t)(1 + b * block), (uint32_t)pitch};
    h_runs[n_blocks] = GreedyRun{status.p, nullptr, slot.p, 0, 0};
    MG_CUDA(ctx, cudaMemcpyAsync(runs.p, h_runs.data(), h_runs.size() * sizeof(GreedyRun), cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemsetAsync(counters.p, 0, 3 * 8, st));
    MG_CUDA(ctx, cudaMemsetAsync(slot.p, 0xFF, n * sizeof(MsfKey), st));
    if (n_blocks) MG_CUDA(ctx, cudaMemsetAsync(bits.p, 0, block * pitch * 4, st));
    greedy_init_kernel<<<blocks_for(n), 256, 0, st>>>(status.p, n);
    MG_CUDA(ctx, cudaGetLastError());
    ctx->kernel_launches++;
    int per_sm = 0;
    MG_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, greedy_resolve_kernel, GREEDY_THREADS, 0));
    // pass 1: each block's run, then its resolve (one cooperative launch), then the matrix cleared for the next block
    auto resolve = [&](const DistArgs &a) -> int {
        GreedyResolve p{bits.p, (uint32_t)pitch, a.q_count, a.q_begin, status.p, masks.p, masks.p + 2 * pitch, extent.p, extent.p + block, ctl.p,
                        counters.p};
        MG_CUDA(ctx, cudaMemsetAsync(ctl.p, 0, 3 * 4, st));
        MG_CUDA(ctx, cudaMemsetAsync(ctl.p + 3, 0xFF, 3 * 4, st));
        const uint64_t warps_needed = (a.q_count + 31) / 32;
        const unsigned grid = (unsigned)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)per_sm * ctx->sm_count,
                                                                                 (warps_needed * 32 + GREEDY_THREADS - 1) / GREEDY_THREADS));
        void *args[] = {&p};
        MG_CUDA(ctx, cudaLaunchCooperativeKernel((const void *)greedy_resolve_kernel, grid, GREEDY_THREADS, args, 0, st));
        MG_CUDA(ctx, cudaMemsetAsync(bits.p, 0, (uint64_t)a.q_count * pitch * 4, st));
        ctx->kernel_launches++;
        return MASHGPU_OK;
    };
    MG_TRY(enqueue_lower_triangle(job, st, [&](DistArgs &a) {
        a.graph = GraphCapture{reinterpret_cast<uint32_t *>(runs.p + (a.q_begin - 1) / block), nullptr, nullptr};
    }, block, resolve));
    // pass 2: every member's nearest representative, at the default run size
    MG_TRY(enqueue_lower_triangle(job, st, [&](DistArgs &a) { a.graph = GraphCapture{reinterpret_cast<uint32_t *>(runs.p + n_blocks), nullptr, nullptr}; }));
    greedy_values_kernel<<<blocks_for(n), 256, 0, st>>>(dist_args(job, 0, n), status.p, slot.p, n, d_rep, d_numer, d_denom, d_distance, d_pvalue,
                                                         counters.p);
    MG_CUDA(ctx, cudaGetLastError());
    ctx->kernel_launches++;
    unsigned long long c[3] = {0, 0, 0};
    MG_CUDA(ctx, cudaMemcpyAsync(c, counters.p, sizeof c, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));        // the state and the headers go out of scope
    if (c[2] & 1) return fail(ctx, MASHGPU_ERR_CUDA, "internal error: a block of representatives not resolved in as many rounds as rows");
    if (c[2] & 2) return fail(ctx, MASHGPU_ERR_CUDA, "internal error: a sketch with neither a representative status nor a representative");
    *n_reps = c[1]; *n_rounds = c[0];
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_representatives(mashgpu_dist_job *job, uint32_t *rep, uint32_t *numer, uint32_t *denom, double *distance, double *pvalue,
                                            uint64_t *n_reps, uint64_t *n_rounds)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (job->encoded) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "representatives of an encoded (sharded) job");
    if (!job->self) return fail(ctx, MASHGPU_ERR_INVALID, "representatives need a self comparison (qry == NULL)");
    if (!rep || !numer || !denom || !distance || !pvalue || !n_reps || !n_rounds) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    *n_reps = 0; *n_rounds = 0;
    const uint64_t n = job->n_qry;
    if (n == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    DevBuf<uint32_t> d32; DevBuf<double> d64;
    if (d32.alloc(3 * n) != cudaSuccess || d64.alloc(2 * n) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (representatives of %llu sketches)", (unsigned long long)n);
    MG_TRY(mashgpu_dist_representatives_dev(job, d32.p, d32.p + n, d32.p + 2 * n, d64.p, d64.p + n, n_reps, n_rounds, ctx->stream));
    cudaStream_t st = ctx->stream;
    MG_CUDA(ctx, cudaMemcpyAsync(rep, d32.p, n * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(numer, d32.p + n, n * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(denom, d32.p + 2 * n, n * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(distance, d64.p, n * 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(pvalue, d64.p + n, n * 8, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    return MASHGPU_OK;
}

// ---------------------------------------------------------------------------------------------------------
// Trees over every pair's distance of a self job: neighbor joining (DESIGN.md 3.10; the joins are in nj.cu) and average /
// complete linkage (DESIGN.md 3.11; the merges are in linkage.cu)
// ---------------------------------------------------------------------------------------------------------
// The n x n matrix of a self job's distances, lower triangle filled (row q at matrix + q * n), for `what` of at least min_n
// sketches.  outputs = the caller's outputs are all non-NULL.  8 n^2 bytes beyond the free device memory are refused before
// anything is allocated.
static int fill_distance_matrix(mashgpu_dist_job *job, const char *what, uint64_t min_n, bool outputs, DevBuf<double> &matrix)
{
    mashgpu_ctx *ctx = job->ctx;
    if (job->encoded) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "%s of an encoded (sharded) job", what);
    if (!job->self) return fail(ctx, MASHGPU_ERR_INVALID, "%s needs a self comparison (qry == NULL)", what);
    if (!outputs) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    const uint64_t n = job->n_qry;
    if (n < min_n) return fail(ctx, MASHGPU_ERR_INVALID, "%s needs at least %llu sketches (got %llu)", what, (unsigned long long)min_n, (unsigned long long)n);
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    size_t free_b = 0, total_b = 0;
    MG_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    if ((double)n * (double)n * 8.0 > (double)free_b)
        return fail(ctx, MASHGPU_ERR_NOMEM, "a %llu x %llu distance matrix needs %.3g GB, the device has %.3g GB free", (unsigned long long)n,
                    (unsigned long long)n, (double)n * (double)n * 8e-9, (double)free_b * 1e-9);
    if (matrix.alloc(n * n) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (%llu x %llu distance matrix)", (unsigned long long)n, (unsigned long long)n);
    // distance output only; the lower triangle is all the trees read
    return enqueue_lower_triangle(job, ctx->stream, [&](DistArgs &a) { a.distance = matrix.p + (uint64_t)a.q_begin * n; });
}

extern "C" int mashgpu_dist_neighbor_joining(mashgpu_dist_job *job, uint32_t *parent, double *length)
{
    if (!job) return MASHGPU_ERR_INVALID;
    DevBuf<double> matrix;
    MG_TRY(fill_distance_matrix(job, "neighbor joining", 3, parent && length, matrix));
    const uint64_t n = job->n_qry;
    return mashgpu_neighbor_joining_matrix(job->ctx, matrix.p, n, n, parent, length, job->ctx->stream);
}

extern "C" int mashgpu_dist_linkage(mashgpu_dist_job *job, int method, uint32_t *id_lo, uint32_t *id_hi, double *height, uint32_t *size,
                                    uint64_t *rows_rescanned)
{
    if (!job) return MASHGPU_ERR_INVALID;
    if (method != MASHGPU_LINKAGE_AVERAGE && method != MASHGPU_LINKAGE_COMPLETE)
        return fail(job->ctx, MASHGPU_ERR_INVALID, "unknown linkage method %d", method);
    DevBuf<double> matrix;
    MG_TRY(fill_distance_matrix(job, "linkage", 2, id_lo && id_hi && height && size, matrix));
    const uint64_t n = job->n_qry;
    return mashgpu_linkage_matrix(job->ctx, matrix.p, n, n, method, id_lo, id_hi, height, size, rows_rescanned, job->ctx->stream);
}

// ---------------------------------------------------------------------------------------------------------
// Flat clusters of average / complete linkage at a height, linked per component (DESIGN.md 3.13)
// ---------------------------------------------------------------------------------------------------------
// Upper member counts of the CTA tier's size classes below its largest one: a small component is not charged the shared memory of
// the largest, so many of them are resident per SM.
static const uint32_t CUT_CLASSES[] = {2, 4, 8, 16, 32, 64, 96, 128, 160};

// The largest component whose triangle and linkage state fit one CTA's shared memory next to the static block minimum (238)
static uint32_t cut_cta_limit()
{
    const size_t avail = 227 * 1024 - 256;
    uint32_t m = 2;
    while (cta_linkage_smem(m + 1) <= avail) m++;
    return m;
}

// T = t (1 + 8 n 2^-53), rounded up.  A merge at a height <= t never joins two components of the graph whose edges are the pairs within
// T that share a hash: between components every leaf pair is above T, and n nested averages lose less than a factor 1 - 3 n 2^-53.
static double cut_threshold(double t, uint64_t n)
{
    return std::nextafter(t * (1.0 + 8.0 * (double)n * 0x1p-53), INFINITY);
}

template <unsigned THREADS>
static cudaError_t cut_cta_launch(bool average, uint32_t n_comps, size_t smem, cudaStream_t st, const DistArgs &a, const uint32_t *members,
                                  const CutComp *comps, LkMerge *rec, int *no_pair)
{
    void (*k)(const DistArgs, const uint32_t *, const CutComp *, LkMerge *, int *) =
        average ? cut_cta_kernel<THREADS, true> : cut_cta_kernel<THREADS, false>;
    cudaError_t e = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    k<<<n_comps, THREADS, smem, st>>>(a, members, comps, rec, no_pair);
    return cudaGetLastError();
}

// The m x m matrix of the lower triangle of run()'s distances among `members` (device, ascending) of a self job, through the tiled merge
// kernels: the job itself when the component is the whole set, else an encoded job over a gathered copy of the members' rows.
static int cut_fill_matrix(mashgpu_dist_job *job, const uint32_t *d_members, uint64_t m, double *matrix, cudaStream_t st)
{
    mashgpu_ctx *ctx = job->ctx;
    auto target = [&](DistArgs &a) { a.distance = matrix + (uint64_t)a.q_begin * m; };
    if (m == job->n_qry) return enqueue_lower_triangle(job, st, target);
    DevBuf<uint32_t> rows, n_eff; DevBuf<uint64_t> len;
    if (rows.alloc(m * job->P) != cudaSuccess || n_eff.alloc(m) != cudaSuccess || len.alloc(m) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (rows of a %llu-sketch component)", (unsigned long long)m);
    cut_gather_kernel<<<ctx->sm_count * 8, 256, 0, st>>>(job->d_ranks, job->P, job->d_n_eff, job->d_lens, d_members, m, rows.p, n_eff.p, len.p);
    MG_CUDA(ctx, cudaGetLastError());
    ctx->kernel_launches++;
    mashgpu_dist_job *sub = nullptr;
    MG_TRY(mashgpu_dist_open_encoded(ctx, rows.p, n_eff.p, len.p, m, 0, m, &job->params, &sub));
    const int rc = enqueue_lower_triangle(sub, st, target);
    mashgpu_dist_close(sub);            // synchronises the stream before the rows are freed
    return rc;
}

extern "C" int mashgpu_dist_set_linkage_cut_cta_max(mashgpu_dist_job *job, uint64_t members)
{
    if (!job) return MASHGPU_ERR_INVALID;
    job->cut_cta_max = members;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_linkage_cut_stats(mashgpu_dist_job *job, double *phase_ms)
{
    if (!job) return MASHGPU_ERR_INVALID;
    if (!phase_ms) return fail(job->ctx, MASHGPU_ERR_INVALID, "NULL output");
    for (int i = 0; i < 4; i++) phase_ms[i] = job->cut_ms[i];
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_linkage_cut(mashgpu_dist_job *job, int method, double t, uint32_t *labels, uint32_t *id_lo, uint32_t *id_hi,
                                        double *height, uint32_t *size, uint64_t *n_clusters, uint64_t *n_components, uint64_t *largest_component)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (job->encoded) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "linkage cut of an encoded (sharded) job");
    if (!job->self) return fail(ctx, MASHGPU_ERR_INVALID, "linkage cut needs a self comparison (qry == NULL)");
    if (method != MASHGPU_LINKAGE_AVERAGE && method != MASHGPU_LINKAGE_COMPLETE)
        return fail(ctx, MASHGPU_ERR_INVALID, "unknown linkage method %d", method);
    if (!(t >= 0)) return fail(ctx, MASHGPU_ERR_INVALID, "cut height %g is NaN or negative", t);
    if (!labels || !n_clusters || !n_components || !largest_component) return fail(ctx, MASHGPU_ERR_INVALID, "NULL output");
    const int forest = (id_lo != nullptr) + (id_hi != nullptr) + (height != nullptr) + (size != nullptr);
    if (forest != 0 && forest != 4) return fail(ctx, MASHGPU_ERR_INVALID, "the merge forest needs all four outputs or none");
    const uint64_t n = job->n_qry;
    *n_clusters = *n_components = *largest_component = n;        // 0 or 1 sketch: the identity
    for (double &ms : job->cut_ms) ms = 0;
    if (n == 1) labels[0] = 0;
    if (n < 2) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    struct Events {
        EventPair e[4] = {};
        ~Events() { for (EventPair &p : e) { if (p.a) cudaEventDestroy(p.a); if (p.b) cudaEventDestroy(p.b); } }
    } events;
    EventPair *ev = events.e;
    for (int i = 0; i < 4; i++) {
        MG_CUDA(ctx, cudaEventCreate(&ev[i].a));
        MG_CUDA(ctx, cudaEventCreate(&ev[i].b));
    }

    // 1. components of the pairs within T: those that share a hash (no p-value test: every p-value is <= 1), and the empty sketches
    // joined; one component when T >= 1
    const double T = cut_threshold(t, n);
    DevBuf<uint32_t> d_label, d_key, d_idx, d_member, d_first;
    if (d_label.alloc(n) != cudaSuccess || d_key.alloc(n) != cudaSuccess || d_idx.alloc(n) != cudaSuccess || d_member.alloc(n) != cudaSuccess ||
        d_first.alloc(n) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (components of %llu sketches)", (unsigned long long)n);
    MG_CUDA(ctx, cudaEventRecord(ev[0].a, st));
    if (T < 1) {
        const double md = job->params.max_distance, mp = job->params.max_pvalue;
        job->params.max_distance = T;
        job->params.max_pvalue = -1;
        uint64_t edges = 0;
        const int rc = mashgpu_dist_components_dev(job, d_label.p, &edges, st);
        job->params.max_distance = md;
        job->params.max_pvalue = mp;
        MG_TRY(rc);
        uint32_t *first_empty = d_key.p;                    // scratch until the sort
        MG_CUDA(ctx, cudaMemsetAsync(first_empty, 0xFF, 4, st));
        cut_empty_first_kernel<<<blocks_for(n), 256, 0, st>>>(job->d_n_eff, n, first_empty);
        cut_empty_join_kernel<<<blocks_for(n), 256, 0, st>>>(job->d_n_eff, n, first_empty, d_label.p);
        MG_CUDA(ctx, cudaGetLastError());
        ctx->kernel_launches += 2;
    } else {
        MG_CUDA(ctx, cudaMemsetAsync(d_label.p, 0, n * 4, st));
    }
    MG_CUDA(ctx, cudaEventRecord(ev[0].b, st));

    // 2. grouping: (label, index) sorted by label -- stable, so each component's members are ascending and the components come in the
    // order of their smallest member, the label -- and where each component starts
    MG_CUDA(ctx, cudaEventRecord(ev[1].a, st));
    iota_kernel<<<blocks_for(n), 256, 0, st>>>(d_idx.p, n);
    MG_CUDA(ctx, cudaGetLastError());
    int bits = 1;
    while (bits < 32 && (1ull << bits) < n) bits++;
    size_t tb_sort = 0, tb_scan = 0;
    DevBuf<uint8_t> tmp;
    uint32_t *flag = d_idx.p, *scan = d_label.p;            // the sort's inputs are dead after it
    MG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(nullptr, tb_sort, d_label.p, d_key.p, d_idx.p, d_member.p, (int)n, 0, bits, st));
    MG_CUDA(ctx, cub::DeviceScan::InclusiveSum(nullptr, tb_scan, flag, scan, (int)n, st));
    if (tmp.alloc(std::max(tb_sort, tb_scan)) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sort scratch)");
    MG_CUDA(ctx, cub::DeviceRadixSort::SortPairs(tmp.p, tb_sort, d_label.p, d_key.p, d_idx.p, d_member.p, (int)n, 0, bits, st));
    cut_start_kernel<<<blocks_for(n), 256, 0, st>>>(d_key.p, n, flag);
    MG_CUDA(ctx, cub::DeviceScan::InclusiveSum(tmp.p, tb_scan, flag, scan, (int)n, st));
    cut_first_kernel<<<blocks_for(n), 256, 0, st>>>(d_key.p, scan, n, d_first.p);
    MG_CUDA(ctx, cudaGetLastError());
    uint32_t runs = 0;
    std::vector<uint32_t> first, member(n);
    MG_CUDA(ctx, cudaMemcpyAsync(&runs, scan + (n - 1), 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(member.data(), d_member.p, n * 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->kernel_launches += 8;
    first.resize(runs + 1);
    MG_CUDA(ctx, cudaMemcpy(first.data(), d_first.p, (size_t)runs * 4, cudaMemcpyDeviceToHost));
    first[runs] = (uint32_t)n;
    MG_CUDA(ctx, cudaEventRecord(ev[1].b, st));
    // the components in order, each with its members' offset and its merges' offset; the CTA tier's components by size class, the
    // large tier's in a list
    const uint32_t limit = cut_cta_limit();
    const uint32_t M = job->cut_cta_max ? (uint32_t)std::min<uint64_t>(job->cut_cta_max, limit) : limit;
    std::vector<uint32_t> bound;
    for (uint32_t b : CUT_CLASSES) if (b < M) bound.push_back(b);
    if (M >= 2) bound.push_back(M);
    std::vector<CutComp> comp(runs);
    std::vector<std::vector<CutComp>> cls(bound.size());
    std::vector<CutComp> large;
    uint64_t merges = 0, largest = 0, largest_large = 0;
    for (uint32_t c = 0; c < runs; c++) {
        const uint32_t m = first[c + 1] - first[c];
        comp[c] = CutComp{first[c], m, (uint32_t)merges};
        merges += m - 1;
        largest = std::max<uint64_t>(largest, m);
        if (m < 2) continue;
        if (m > M) { large.push_back(comp[c]); largest_large = std::max<uint64_t>(largest_large, m); continue; }
        size_t k = 0;
        while (bound[k] < m) k++;
        cls[k].push_back(comp[c]);
    }
    size_t free_b = 0, total_b = 0;
    MG_CUDA(ctx, cudaMemGetInfo(&free_b, &total_b));
    if ((double)largest_large * (double)largest_large * 8.0 > (double)free_b)
        return fail(ctx, MASHGPU_ERR_NOMEM, "at t = %g the largest component has %llu sketches: its %llu x %llu distance matrix needs %.3g GB, the device has %.3g GB free",
                    t, (unsigned long long)largest_large, (unsigned long long)largest_large, (unsigned long long)largest_large,
                    (double)largest_large * (double)largest_large * 8e-9, (double)free_b * 1e-9);

    // 3. the CTA tier: one launch per size class
    std::vector<LkMerge> rec(merges);
    DevBuf<LkMerge> d_rec; DevBuf<CutComp> d_comp; DevBuf<int> d_no_pair;
    uint64_t in_cta = 0;
    for (auto &v : cls) in_cta += v.size();
    MG_CUDA(ctx, cudaEventRecord(ev[2].a, st));
    if (in_cta) {
        if (d_rec.alloc(merges) != cudaSuccess || d_comp.alloc(in_cta) != cudaSuccess || d_no_pair.alloc(1) != cudaSuccess)
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (merges of %llu components)", (unsigned long long)in_cta);
        std::vector<CutComp> flat;
        flat.reserve(in_cta);
        for (auto &v : cls) flat.insert(flat.end(), v.begin(), v.end());
        MG_CUDA(ctx, cudaMemcpyAsync(d_comp.p, flat.data(), in_cta * sizeof(CutComp), cudaMemcpyHostToDevice, st));
        MG_CUDA(ctx, cudaMemsetAsync(d_no_pair.p, 0, sizeof(int), st));
        const DistArgs a = dist_args(job, 0, n);
        const bool average = method == MASHGPU_LINKAGE_AVERAGE;
        uint64_t off = 0;
        for (size_t k = 0; k < cls.size(); k++) {
            const uint32_t nc = (uint32_t)cls[k].size();
            if (!nc) continue;
            const size_t smem = cta_linkage_smem(bound[k]);
            const CutComp *dc = d_comp.p + off;
            cudaError_t e;
            if (bound[k] <= 32) e = cut_cta_launch<32>(average, nc, smem, st, a, d_member.p, dc, d_rec.p, d_no_pair.p);
            else if (bound[k] <= 64) e = cut_cta_launch<64>(average, nc, smem, st, a, d_member.p, dc, d_rec.p, d_no_pair.p);
            else if (bound[k] <= 128) e = cut_cta_launch<128>(average, nc, smem, st, a, d_member.p, dc, d_rec.p, d_no_pair.p);
            else e = cut_cta_launch<256>(average, nc, smem, st, a, d_member.p, dc, d_rec.p, d_no_pair.p);
            MG_CUDA(ctx, e);
            ctx->kernel_launches++;
            off += nc;
        }
        int no_pair = 0;
        MG_CUDA(ctx, cudaMemcpyAsync(rec.data(), d_rec.p, merges * sizeof(LkMerge), cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaMemcpyAsync(&no_pair, d_no_pair.p, sizeof(int), cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
        if (no_pair) return fail(ctx, MASHGPU_ERR_INVALID, "linkage found no pair with a comparable distance (an update overflowed)");
    }
    MG_CUDA(ctx, cudaEventRecord(ev[2].b, st));

    // 4. the large tier: per component an m x m matrix through the tiled merge kernels, then mashgpu_linkage_matrix
    MG_CUDA(ctx, cudaEventRecord(ev[3].a, st));
    for (const CutComp &c : large) {
        const uint64_t m = c.m;
        DevBuf<double> matrix;
        if (matrix.alloc(m * m) != cudaSuccess)
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (%llu x %llu distance matrix of a component at t = %g)", (unsigned long long)m,
                        (unsigned long long)m, t);
        MG_TRY(cut_fill_matrix(job, d_member.p + c.first, m, matrix.p, st));
        std::vector<uint32_t> lo(m - 1), hi(m - 1), sz(m - 1);
        std::vector<double> h(m - 1);
        MG_TRY(mashgpu_linkage_matrix(ctx, matrix.p, m, m, method, lo.data(), hi.data(), h.data(), sz.data(), nullptr, st));
        for (uint64_t s = 0; s + 1 < m; s++) rec[c.merge0 + s] = LkMerge{h[s], lo[s], hi[s], sz[s]};
    }
    MG_CUDA(ctx, cudaEventRecord(ev[3].b, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    for (int i = 0; i < 4; i++) {
        float ms = 0;
        MG_CUDA(ctx, cudaEventElapsedTime(&ms, ev[i].a, ev[i].b));
        job->cut_ms[i] = ms;
    }

    // 5. per component the cut (writeLinkage's: a maximal subtree whose largest merge height is <= t), labelled by its smallest member,
    // and the merges with the set's ids: leaf j -> members[first + j], node m + s -> n + merge0 + s
    std::vector<double> worst;
    std::vector<uint32_t> top, low;
    for (const CutComp &c : comp) {
        const uint32_t m = c.m, *mem = member.data() + c.first;
        if (m == 1) { labels[mem[0]] = mem[0]; continue; }
        const LkMerge *r = rec.data() + c.merge0;
        const uint32_t nodes = 2 * m - 1;
        worst.assign(nodes, 0.0);
        low.resize(nodes);
        top.resize(nodes);
        for (uint32_t j = 0; j < m; j++) low[j] = j;
        for (uint32_t s = 0; s + 1 < m; s++) {
            worst[m + s] = std::max(r[s].height, std::max(worst[r[s].lo], worst[r[s].hi]));
            low[m + s] = std::min(low[r[s].lo], low[r[s].hi]);
        }
        top[nodes - 1] = nodes - 1;
        for (uint32_t s = m - 1; s-- > 0;) {
            const uint32_t u = m + s;
            top[r[s].lo] = worst[u] <= t ? top[u] : r[s].lo;
            top[r[s].hi] = worst[u] <= t ? top[u] : r[s].hi;
        }
        for (uint32_t j = 0; j < m; j++) labels[mem[j]] = mem[low[top[j]]];
        if (forest) {
            auto global = [&](uint32_t x) { return x < m ? mem[x] : (uint32_t)(n + c.merge0 + (x - m)); };
            for (uint32_t s = 0; s + 1 < m; s++) {
                id_lo[c.merge0 + s] = global(r[s].lo);
                id_hi[c.merge0 + s] = global(r[s].hi);
                height[c.merge0 + s] = r[s].height;
                size[c.merge0 + s] = r[s].size;
            }
        }
    }
    uint64_t clusters = 0;
    for (uint64_t i = 0; i < n; i++) clusters += labels[i] == i;
    *n_clusters = clusters;
    *n_components = runs;
    *largest_component = largest;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist_close(mashgpu_dist_job *job)
{
    if (!job) return MASHGPU_ERR_INVALID;
    cudaSetDevice(job->ctx->device);
    cudaStreamSynchronize(job->ctx->stream);
    for (auto &ev : job->best_events) { cudaEventDestroy(ev.a); cudaEventDestroy(ev.b); }
    delete job;
    return MASHGPU_OK;
}

extern "C" int mashgpu_dist(mashgpu_ctx *ctx, const mashgpu_sketch_set *ref, const mashgpu_sketch_set *qry,
                            const mashgpu_dist_params *params,
                            uint32_t *numer, uint32_t *denom, double *distance, double *pvalue, uint8_t *pass)
{
    mashgpu_dist_job *job = nullptr;
    MG_TRY(mashgpu_dist_open(ctx, ref, qry, params, &job));
    int rc = mashgpu_dist_run(job, 0, job->n_qry, numer, denom, distance, pvalue, pass);
    mashgpu_dist_close(job);
    return rc;
}
