// dense.cuh -- pieces shared by the passes over a dense float64 distance matrix in device memory: neighbor joining (nj.cu,
// DESIGN.md 3.10) and average / complete linkage (linkage.cu, DESIGN.md 3.11).  A strict total order on (value, key), its warp and
// block minimum, and the mirror of the lower triangle with its finiteness test.
#pragma once
#include <cstdint>

namespace mashgpu {
namespace {

constexpr unsigned NJ_THREADS = 256;
constexpr unsigned long long NJ_NO_KEY = ~0ull;

struct NjBest { double q; unsigned long long key; };

// strict total order on (value, key); a NaN value is never before anything
__device__ __forceinline__ bool nj_before(double q1, unsigned long long k1, double q2, unsigned long long k2)
{
    return q1 < q2 || (q1 == q2 && k1 < k2);
}

__device__ __forceinline__ void nj_warp_min(double &q, unsigned long long &k)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const double q2 = __shfl_xor_sync(0xFFFFFFFFu, q, o);
        const unsigned long long k2 = __shfl_xor_sync(0xFFFFFFFFu, k, o);
        if (nj_before(q2, k2, q, k)) { q = q2; k = k2; }
    }
}

// the minimum over the block of THREADS threads, returned to every thread
template <unsigned THREADS = NJ_THREADS>
__device__ NjBest nj_block_min(double q, unsigned long long k)
{
    __shared__ double sq[THREADS / 32];
    __shared__ unsigned long long sk[THREADS / 32];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    nj_warp_min(q, k);
    if (lane == 0) { sq[warp] = q; sk[warp] = k; }
    __syncthreads();
    if (warp == 0) {
        q = lane < THREADS / 32 ? sq[lane] : __longlong_as_double(0x7FF0000000000000ll);
        k = lane < THREADS / 32 ? sk[lane] : NJ_NO_KEY;
        nj_warp_min(q, k);
        if (lane == 0) { sq[0] = q; sk[0] = k; }
    }
    __syncthreads();
    return NjBest{sq[0], sk[0]};
}

// Lower triangle -> upper triangle through 32 x 32 tiles in shared memory, diagonal := 0, and the finiteness test of every
// lower-triangle entry.  Grid (tiles, tiles); tiles above the diagonal exit.  Upper entries are only written and lower ones only
// read, so tiles need no ordering.
__global__ void __launch_bounds__(256) nj_mirror_kernel(double *D, uint64_t ld, uint32_t n, int *nonfinite)
{
    __shared__ double t[32][33];
    const uint32_t bi = blockIdx.y, bj = blockIdx.x;
    if (bj > bi) return;
    const uint32_t i0 = bi * 32, j0 = bj * 32, x = threadIdx.x;
    bool bad = false;
    for (uint32_t y = threadIdx.y; y < 32; y += 8) {
        const uint32_t i = i0 + y, j = j0 + x;
        if (i < n && j < i) {
            const double v = D[(uint64_t)i * ld + j];
            t[y][x] = v;
            bad |= !isfinite(v);
        }
    }
    if (__syncthreads_or(bad) && x == 0 && threadIdx.y == 0) *nonfinite = 1;
    for (uint32_t y = threadIdx.y; y < 32; y += 8) {         // upper entry (r, c), r < c, is D(c, r) = t[x][y]
        const uint32_t r = j0 + y, c = i0 + x;
        if (c < n && r < c) D[(uint64_t)r * ld + c] = t[x][y];
        else if (c < n && r == c) D[(uint64_t)r * ld + c] = 0.0;
    }
}

}  // namespace
}  // namespace mashgpu
