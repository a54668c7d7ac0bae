// dense.cuh -- pieces shared by the passes over a dense float64 distance matrix in device memory: neighbor joining (nj.cu,
// DESIGN.md 3.10) and average / complete linkage (linkage.cu, DESIGN.md 3.11, and its CTA tier linkage_cta.cuh, 3.13).  A strict
// total order on (value, key) with its block minimum, the linkage update, the mirror of the lower triangle with its finiteness
// test, and what every pass does before its first step.
#pragma once
#include <algorithm>
#include <cstdint>

#include "common.cuh"

namespace mashgpu {
namespace {

constexpr unsigned DENSE_THREADS = 256;
constexpr unsigned long long DENSE_NO_KEY = ~0ull;
constexpr uint32_t DENSE_NONE = 0xFFFFFFFFu;          // no node, no neighbour

struct DenseMin { double q; unsigned long long key; };

unsigned dense_blocks(uint64_t n, unsigned tb = DENSE_THREADS) { return (unsigned)std::max<uint64_t>(1, (n + tb - 1) / tb); }

// strict total order on (value, key); a NaN value is never before anything
__device__ __forceinline__ bool dense_before(double q1, unsigned long long k1, double q2, unsigned long long k2)
{
    return q1 < q2 || (q1 == q2 && k1 < k2);
}

__device__ __forceinline__ void dense_warp_min(double &q, unsigned long long &k)
{
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const double q2 = __shfl_xor_sync(0xFFFFFFFFu, q, o);
        const unsigned long long k2 = __shfl_xor_sync(0xFFFFFFFFu, k, o);
        if (dense_before(q2, k2, q, k)) { q = q2; k = k2; }
    }
}

// the minimum over the block of THREADS threads, returned to every thread
template <unsigned THREADS = DENSE_THREADS>
__device__ DenseMin dense_block_min(double q, unsigned long long k)
{
    __shared__ double sq[THREADS / 32];
    __shared__ unsigned long long sk[THREADS / 32];
    const unsigned lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    dense_warp_min(q, k);
    if (lane == 0) { sq[warp] = q; sk[warp] = k; }
    __syncthreads();
    if (warp == 0) {
        q = lane < THREADS / 32 ? sq[lane] : __longlong_as_double(0x7FF0000000000000ll);
        k = lane < THREADS / 32 ? sk[lane] : DENSE_NO_KEY;
        dense_warp_min(q, k);
        if (lane == 0) { sq[0] = q; sk[0] = k; }
    }
    __syncthreads();
    return DenseMin{sq[0], sk[0]};
}

// Average / complete linkage (linkage.cu, and the CTA tier of the linkage cut, linkage_cta.cuh): merge s in scipy's Z layout, and the
// two steps of a merge of (a, b) that every slot k does for itself.
struct LkMerge { double height; uint32_t lo, hi, size; };   // node ids (smaller first), height, leaves

// D(u, k) from D(a, k) and D(b, k): one IEEE double operation at a time, never fused
template <bool AVERAGE>
__device__ __forceinline__ double lk_value(uint32_t na, uint32_t nb, double dak, double dbk)
{
    if (AVERAGE) return __ddiv_rn(__dadd_rn(__dmul_rn((double)na, dak), __dmul_rn((double)nb, dbk)), (double)(na + nb));
    return dbk > dak ? dbk : dak;
}

// What a merge of (a, b) does to the cache (c, j) of a row k > a, given v = D(u, k): a neighbour a or b becomes (v, a) when v <= c,
// else the row is rescanned; any other neighbour is lowered to (v, a) when that is before it, else kept.
enum { LK_KEEP, LK_TAKE, LK_RESCAN };
__device__ __forceinline__ int lk_offer(double v, uint32_t a, uint32_t b, double c, uint32_t j)
{
    if (j == a || j == b) return v <= c ? LK_TAKE : LK_RESCAN;
    return dense_before(v, a, c, j) ? LK_TAKE : LK_KEEP;
}

// the minimum of an argmin's n_partial per-CTA partials, reduced by a block of DENSE_THREADS threads and returned to every thread
__device__ __forceinline__ DenseMin dense_partials_min(const DenseMin *__restrict__ partial, uint32_t n_partial)
{
    double bq = __longlong_as_double(0x7FF0000000000000ll);
    unsigned long long bk = DENSE_NO_KEY;
    for (uint32_t t = threadIdx.x; t < n_partial; t += DENSE_THREADS) {
        const DenseMin c = partial[t];
        if (dense_before(c.q, c.key, bq, bk)) { bq = c.q; bk = c.key; }
    }
    return dense_block_min(bq, bk);
}

// Lower triangle -> upper triangle through 32 x 32 tiles in shared memory, diagonal := 0, and the finiteness test of every
// lower-triangle entry.  Grid (tiles, tiles); tiles above the diagonal exit.  Upper entries are only written and lower ones only
// read, so tiles need no ordering.
__global__ void __launch_bounds__(256) dense_mirror_kernel(double *D, uint64_t ld, uint32_t n, int *nonfinite)
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

// Before the first step of a pass over the caller's n x ld matrix: the checks of n (at least min_n leaves for `what`) and ld, the
// device, the stream (the caller's, else the context's), and the mirror; a NaN or infinite lower-triangle entry is refused.
int dense_begin(mashgpu_ctx *ctx, double *D, uint64_t n, uint64_t ld, uint64_t min_n, const char *what, void *stream, cudaStream_t &st)
{
    if (n < min_n) return fail(ctx, MASHGPU_ERR_INVALID, "%s needs at least %llu leaves (got %llu)", what, (unsigned long long)min_n, (unsigned long long)n);
    if (ld < n) return fail(ctx, MASHGPU_ERR_INVALID, "leading dimension %llu below n = %llu", (unsigned long long)ld, (unsigned long long)n);
    if (n >= 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^31 - 1 leaves");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    st = stream ? (cudaStream_t)stream : ctx->stream;
    DevBuf<int> flag;
    if (flag.alloc(1) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (%s state of %llu leaves)", what, (unsigned long long)n);
    MG_CUDA(ctx, cudaMemsetAsync(flag.p, 0, sizeof(int), st));
    const uint32_t tiles = ((uint32_t)n + 31) / 32;
    dense_mirror_kernel<<<dim3(tiles, tiles), dim3(32, 8), 0, st>>>(D, ld, (uint32_t)n, flag.p);
    MG_CUDA(ctx, cudaGetLastError());
    int nonfinite = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&nonfinite, flag.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->kernel_launches++;
    return nonfinite ? fail(ctx, MASHGPU_ERR_INVALID, "the distance matrix has a NaN or infinite entry in its lower triangle") : MASHGPU_OK;
}

}  // namespace
}  // namespace mashgpu
