// dist_best.cuh -- best hits of a dist run (mashgpu_dist_run_best, DESIGN.md 3.7): the device side.
//
// A best run keeps, per query, the N nearest references among its hits (pairs that pass and share a hash) instead of the dense
// grid.  Three steps:
//   capture   dist_emit / dist_fix_kernel append one BestCand per hit to a bounded buffer and count it per query
//   grouping  exclusive scan of the per-query counts, then best_scatter_kernel moves every candidate into its query's segment
//   selection dist_best_kernel picks the N smallest (distance bits, reference) of every segment and writes them in rank order
// The reference has no counterpart (its users pipe `mash dist` into sort); the result is defined as the first N rows of a stable
// sort of the query's row of the dense grid, which is what the tests compare it with.
#pragma once
#include <cstdint>

namespace mashgpu {

// One hit.  A distance is a non-negative double, so its bit pattern orders as the value does: the key is integer compares only.
struct __align__(16) BestCand {
    uint64_t dbits;         // __double_as_longlong(distance)
    double pvalue;
    uint32_t q;             // query, relative to the first query of the block in flight
    uint32_t ref;
    uint32_t numer, denom;
};
static_assert(sizeof(BestCand) == 32, "a candidate is two 16-byte stores");

// Capture target inside DistArgs; cand == nullptr outside best runs.
struct BestCapture {
    BestCand *cand;
    unsigned long long *count;      // candidates reserved; above `capacity` the block is run again in halves
    uint64_t capacity;
    uint32_t *qcount;               // hits per query of the block
};

// Appends a hit.  A reservation beyond the capacity writes nothing (the host sees count > capacity and discards the block).  The
// lanes of a warp mostly report the same query (the tiled merge holds one query against 32 references): one counter update per
// distinct query of the warp.  Not inlined: the merge kernels' epilogues keep their register allocation.
__device__ __noinline__ void dist_best_append(const BestCapture b, uint32_t q_rel, uint32_t r, uint32_t common, uint32_t denom, double dist, double p)
{
    const unsigned peers = __match_any_sync(__activemask(), q_rel);
    if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(&b.qcount[q_rel], (uint32_t)__popc(peers));
    const unsigned long long at = atomicAdd(b.count, 1ull);
    if (at < b.capacity) b.cand[at] = BestCand{(uint64_t)__double_as_longlong(dist), p, q_rel, r, common, denom};
}

// grouped[off[q] + (arrival order)] = candidate; the order inside a segment is arbitrary, the selection key is a total order
__global__ void __launch_bounds__(256) best_scatter_kernel(const BestCand *cand, uint64_t n, const uint32_t *off, uint32_t *cursor, BestCand *grouped)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    const BestCand c = cand[t];
    grouped[off[c.q] + atomicAdd(&cursor[c.q], 1u)] = c;
}

constexpr int BEST_WARPS = 8;
constexpr int BEST_THREADS = BEST_WARPS * 32;
constexpr uint32_t BEST_TILE = 1024;            // candidates sorted at a time; also the largest N
constexpr uint32_t BEST_MAX_N = BEST_TILE;

struct BestKey { uint64_t d; uint32_t ref, idx; };     // idx: position in the query's segment
__device__ __forceinline__ bool best_less(const BestKey &a, const BestKey &b) { return a.d < b.d || (a.d == b.d && a.ref < b.ref); }
__device__ __forceinline__ BestKey best_inf() { return BestKey{~0ull, 0xFFFFFFFFu, 0xFFFFFFFFu}; }

struct BestOut {
    uint32_t *n_hits, *n_total;                 // [q]; n_total may be NULL
    uint32_t *ref, *numer, *denom; double *distance, *pvalue;      // [q * n_best + rank]
};

__device__ __forceinline__ void best_write(const BestOut &o, uint64_t at, const BestCand &c)
{
    o.ref[at] = c.ref; o.numer[at] = c.numer; o.denom[at] = c.denom;
    o.distance[at] = __longlong_as_double((long long)c.dbits); o.pvalue[at] = c.pvalue;
}
__device__ __forceinline__ void best_write_zero(const BestOut &o, uint64_t at)
{
    o.ref[at] = 0; o.numer[at] = 0; o.denom[at] = 0; o.distance[at] = 0.0; o.pvalue[at] = 0.0;
}

// compare-exchange of s[i], s[p] (i < p): afterwards s[i] <= s[p] when `asc`, s[i] >= s[p] otherwise
__device__ __forceinline__ void best_cmpx(BestKey *s, uint32_t i, uint32_t p, bool asc)
{
    const BestKey a = s[i], b = s[p];
    if (best_less(b, a) == asc) { s[i] = b; s[p] = a; }
}

// The N best of every query of a block, in rank order, with n_hits = min(N, hits) and n_total = hits; ranks past n_hits are zero.
// A CTA takes BEST_WARPS consecutive queries.
//   up to 32 hits (the usual case against a diverse database): one warp per query, one candidate per lane, its rank is the number
//     of smaller keys among the 32 (keys of a query are distinct: they differ in the reference)
//   more: the CTA streams the segment through shared memory, BEST_THREADS candidates a step.  It keeps the best `kw` (N rounded up
//     to a power of two) sorted in s_key[0, kw); candidates below the current N-th best collect in s_key[BEST_TILE, ...) and, when
//     that tile fills up or the segment ends, are sorted (bitonic, descending) and merged in: kept ascending next to tile
//     descending is a bitonic sequence, so the element-wise minimum holds the kw smallest of both and log2(kw) merge steps sort
//     it again.  After the first tiles of a long segment nearly every candidate fails the N-th-best test and costs one compare.
__global__ void __launch_bounds__(BEST_THREADS) dist_best_kernel(const BestCand *grouped, const uint32_t *off, const uint32_t *qcnt, uint32_t q_count,
                                                                 uint32_t n_best, uint32_t kw, const BestOut o)
{
    __shared__ BestKey s_key[2 * BEST_TILE];
    __shared__ uint32_t s_fill;
    const uint32_t tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t q0 = blockIdx.x * BEST_WARPS;
    {
        const uint32_t q = q0 + warp;
        const uint32_t cnt = q < q_count ? qcnt[q] : 0xFFFFFFFFu;
        if (cnt <= 32) {
            const bool have = lane < cnt;
            BestCand c{};
            if (have) c = grouped[off[q] + lane];
            const uint64_t d = have ? c.dbits : ~0ull;
            const uint32_t ref = have ? c.ref : 0xFFFFFFFFu;
            uint32_t rank = 0;
#pragma unroll
            for (int j = 0; j < 32; j++) {
                const uint64_t dj = __shfl_sync(0xFFFFFFFFu, d, j);
                const uint32_t rj = __shfl_sync(0xFFFFFFFFu, ref, j);
                rank += (dj < d || (dj == d && rj < ref)) ? 1u : 0u;
            }
            const uint32_t hits = min(cnt, n_best);
            const uint64_t row = (uint64_t)q * n_best;
            if (have && rank < n_best) best_write(o, row + rank, c);
            for (uint32_t i = hits + lane; i < n_best; i += 32) best_write_zero(o, row + i);
            if (lane == 0) { o.n_hits[q] = hits; if (o.n_total) o.n_total[q] = cnt; }
        }
    }
    BestKey *kept = s_key, *tile = s_key + BEST_TILE;
    for (uint32_t w = 0; w < BEST_WARPS; w++) {
        const uint32_t q = q0 + w;
        if (q >= q_count) break;
        const uint32_t cnt = qcnt[q];
        if (cnt <= 32) continue;                    // CTA-uniform
        const BestCand *seg = grouped + off[q];
        __syncthreads();                            // the previous long query's output has been read from s_key
        for (uint32_t i = tid; i < kw; i += BEST_THREADS) kept[i] = best_inf();
        if (tid == 0) s_fill = 0;
        __syncthreads();
        BestKey thresh = best_inf();                // the N-th best so far
        for (uint32_t base = 0; base < cnt; base += BEST_THREADS) {
            const uint32_t i = base + tid;
            if (i < cnt) {
                const BestCand c = seg[i];
                const BestKey key{c.dbits, c.ref, i};
                if (best_less(key, thresh)) tile[atomicAdd(&s_fill, 1u)] = key;
            }
            __syncthreads();
            const uint32_t fill = s_fill;
            __syncthreads();                        // everyone has read s_fill before the next step adds to it
            if (fill == 0 || (fill + BEST_THREADS <= BEST_TILE && base + BEST_THREADS < cnt)) continue;
            // sort the tile's first n2 >= fill entries descending
            uint32_t n2 = 2;
            while (n2 < fill) n2 <<= 1;
            for (uint32_t t = fill + tid; t < n2; t += BEST_THREADS) tile[t] = best_inf();
            __syncthreads();
            for (uint32_t k = 2; k <= n2; k <<= 1)
                for (uint32_t j = k >> 1; j > 0; j >>= 1) {
                    for (uint32_t t = tid; t < n2 / 2; t += BEST_THREADS) {
                        const uint32_t lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                        best_cmpx(tile, lo, lo | j, (lo & k) != 0);
                    }
                    __syncthreads();
                }
            // the kw smallest of kept (ascending) and tile (descending; its kw smallest are its last kw entries)
            for (uint32_t t = tid; t < kw; t += BEST_THREADS) {
                const int src = (int)t + (int)n2 - (int)kw;
                if (src >= 0 && best_less(tile[src], kept[t])) kept[t] = tile[src];
            }
            __syncthreads();
            for (uint32_t j = kw >> 1; j > 0; j >>= 1) {
                for (uint32_t t = tid; t < kw / 2; t += BEST_THREADS) {
                    const uint32_t lo = ((t & ~(j - 1)) << 1) | (t & (j - 1));
                    best_cmpx(kept, lo, lo | j, true);
                }
                __syncthreads();
            }
            thresh = kept[n_best - 1];
            if (tid == 0) s_fill = 0;
            __syncthreads();
        }
        const uint32_t hits = min(cnt, n_best);
        const uint64_t row = (uint64_t)q * n_best;
        for (uint32_t i = tid; i < n_best; i += BEST_THREADS) {
            if (i < hits) best_write(o, row + i, seg[kept[i].idx]);
            else best_write_zero(o, row + i);
        }
        if (tid == 0) { o.n_hits[q] = hits; if (o.n_total) o.n_total[q] = cnt; }
    }
}

}  // namespace mashgpu
