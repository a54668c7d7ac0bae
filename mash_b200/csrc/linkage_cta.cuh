// linkage_cta.cuh -- average / complete linkage of one small matrix inside one CTA: the CTA tier of the linkage cut
// (mashgpu_dist_linkage_cut, DESIGN.md 3.13).  dist.cu fills the component's lower triangle into shared memory and calls
// cta_linkage, so each component costs one CTA instead of three launches per merge.
//
// The algorithm is linkage.cu's (DESIGN.md 3.11) with __syncthreads in place of its launches: per-row nearest-neighbour caches, the
// least (cache value, row) as the pair, the update of row a with lk_value and the cache rule lk_offer (dense.cuh), and rescans of
// the listed rows.  The merges are therefore mashgpu_linkage_matrix's bit for bit, ties included.  Only the storage differs: the
// lower triangle alone, packed (entry (i, j), j < i, at i (i - 1) / 2 + j), so D(a, k) and D(k, a) are one entry, and dead slots are
// a flag instead of a NaN column (a rescan skips them the same way).
#pragma once
#include <cstdint>

#include "dense.cuh"

namespace mashgpu {
namespace {

__host__ __device__ __forceinline__ uint32_t cta_tri(uint32_t m) { return m * (m - 1) / 2; }      // entries of the packed triangle

// shared memory of an m-member component: the triangle and the caches (double), cj, sizes, ids and the rescan list (uint32), liveness
__host__ __device__ __forceinline__ size_t cta_linkage_smem(uint32_t m)
{
    return ((8 * ((size_t)cta_tri(m) + m) + 16 * (size_t)m + m) + 15) & ~(size_t)15;
}

struct CtaLinkage {
    double *tri, *cv;
    uint32_t *cj, *size, *id, *list;
    uint8_t *alive;
};

__device__ __forceinline__ CtaLinkage cta_layout(void *smem, uint32_t m)
{
    CtaLinkage L;
    L.tri = reinterpret_cast<double *>(smem);
    L.cv = L.tri + cta_tri(m);
    L.cj = reinterpret_cast<uint32_t *>(L.cv + m);
    L.size = L.cj + m; L.id = L.size + m; L.list = L.id + m;
    L.alive = reinterpret_cast<uint8_t *>(L.list + m);
    return L;
}

// D(i, j), i != j
__device__ __forceinline__ double &cta_at(const CtaLinkage &L, uint32_t i, uint32_t j)
{
    return i > j ? L.tri[cta_tri(i) + j] : L.tri[cta_tri(j) + i];
}

// One warp: row i's cache := the least (D(i, j), j) over live j < i; (+inf, none) when there is none.
__device__ __forceinline__ void cta_rescan(const CtaLinkage &L, uint32_t i)
{
    const uint32_t lane = threadIdx.x & 31;
    const double *row = L.tri + cta_tri(i);
    double bq = __longlong_as_double(0x7FF0000000000000ll);
    unsigned long long bk = DENSE_NO_KEY;
    for (uint32_t j = lane; j < i; j += 32)
        if (L.alive[j] && dense_before(row[j], j, bq, bk)) { bq = row[j]; bk = j; }
    dense_warp_min(bq, bk);
    if (lane == 0) {
        L.cv[i] = bk == DENSE_NO_KEY ? __longlong_as_double(0x7FF0000000000000ll) : bq;
        L.cj[i] = bk == DENSE_NO_KEY ? DENSE_NONE : (uint32_t)bk;
    }
}

// The m - 1 merges of the filled triangle (m >= 2), into rec[0 .. m - 2] with the component's own node ids: leaves 0..m-1, merge s
// makes node m + s.  The triangle is scratch.  *no_pair := 1 when a step finds no pair (a non-comparable distance; not reachable
// with Mash distances, which are finite).
template <unsigned THREADS, bool AVERAGE>
__device__ void cta_linkage(const CtaLinkage &L, uint32_t m, LkMerge *rec, int *no_pair)
{
    constexpr uint32_t WARPS = THREADS / 32;
    __shared__ uint32_t count;
    const uint32_t warp = threadIdx.x >> 5;
    for (uint32_t k = threadIdx.x; k < m; k += THREADS) { L.alive[k] = 1; L.size[k] = 1; L.id[k] = k; }
    __syncthreads();
    for (uint32_t i = warp; i < m; i += WARPS) cta_rescan(L, i);
    __syncthreads();
    for (uint32_t s = 0; s + 1 < m; s++) {
        // the pair: the least (cache value, row << 32 | neighbour)
        double bq = __longlong_as_double(0x7FF0000000000000ll);
        unsigned long long bk = DENSE_NO_KEY;
        for (uint32_t i = threadIdx.x; i < m; i += THREADS) {
            const uint32_t j = L.cj[i];
            const unsigned long long key = (unsigned long long)i << 32 | j;
            if (j != DENSE_NONE && dense_before(L.cv[i], key, bq, bk)) { bq = L.cv[i]; bk = key; }
        }
        if (threadIdx.x == 0) count = 0;
        const DenseMin best = dense_block_min<THREADS>(bq, bk);
        if (best.key == DENSE_NO_KEY) {
            if (threadIdx.x == 0) *no_pair = 1;
            return;
        }
        const uint32_t b = (uint32_t)(best.key >> 32), a = (uint32_t)best.key;
        const uint32_t na = L.size[a], nb = L.size[b];
        // the update: slot k is thread k's alone (D(a, k) is one entry of the packed triangle)
        for (uint32_t k = threadIdx.x; k < m; k += THREADS) {
            if (k == b) {
                L.cv[b] = __longlong_as_double(0x7FF0000000000000ll);
                L.cj[b] = DENSE_NONE;
                L.alive[b] = 0;
                continue;
            }
            if (!L.alive[k]) continue;
            if (k == a) {
                const uint32_t ia = L.id[a], ib = L.id[b];
                rec[s] = LkMerge{best.q, min(ia, ib), max(ia, ib), na + nb};
                L.list[atomicAdd(&count, 1u)] = a;
                continue;
            }
            double &dak = cta_at(L, a, k);
            const double v = lk_value<AVERAGE>(na, nb, dak, cta_at(L, b, k));
            dak = v;
            if (k < a) continue;
            const int o = lk_offer(v, a, b, L.cv[k], L.cj[k]);
            if (o == LK_TAKE) { L.cv[k] = v; L.cj[k] = a; }
            else if (o == LK_RESCAN) L.list[atomicAdd(&count, 1u)] = k;
        }
        __syncthreads();
        if (threadIdx.x == 0) { L.size[a] = na + nb; L.id[a] = m + s; }
        const uint32_t listed = count;
        for (uint32_t r = warp; r < listed; r += WARPS) cta_rescan(L, L.list[r]);
        __syncthreads();
    }
}

}  // namespace
}  // namespace mashgpu
