// linkage.cu -- average (UPGMA) and complete linkage over a dense float64 distance matrix in device memory (C-ABI:
// mashgpu_linkage_matrix, DESIGN.md 3.11).  No counterpart in the reference: its users feed the `mash triangle` matrix to scipy.
//
// The definition (mashgpu.h) merges, at every step, the least (D(a, b), b, a) over live slots a < b.  Both methods are reducible,
// so a per-row nearest-neighbour cache finds that pair without scanning the matrix: cache[i] is the least (D(i, j), j) over live
// j < i, and the least (cache[i].value, i) over the rows is the pair.  After a merge of (a, b) into slot a only rows whose cached
// neighbour was a or b and whose new distance to a is larger than the cached value need a rescan (plus row a itself); every other
// row's cache is lowered to (D(i, a), a) or kept (lk_update_kernel).  The same rule is restated in tests/linkage_model.py, which
// checks it against the naive global minimum.
//
// Matrix: the caller's n x ld array, mirrored by dense_mirror_kernel (dense.cuh) so that rows a and b hold every column.  A merge
// writes row a and column a; rows after b get NaN in column b, so a rescan of row i reads its i entries and skips dead ones (a
// NaN is never before anything, and a live entry may be +inf: an average that overflowed is still a distance).  Row b is never
// written.  Per merge the host enqueues three kernels and never synchronises; the merge records are copied back at the end.
// Every device arithmetic step is one IEEE double operation (__dmul_rn, __dadd_rn, __ddiv_rn); __ddiv_rn is the correctly rounded
// quotient, so the DFMAs of its Newton steps are the only ones in linkage.o.
#include <vector>

#include "dense.cuh"

namespace mashgpu {
namespace {

constexpr unsigned LK_RESCAN_THREADS = 1024;    // one CTA per rescanned row: a row of n doubles in a few round trips

struct LkStep { uint32_t a, b; };                           // the slots of the merge in flight

// slot i: a leaf of size 1, no cached neighbour, and on the rescan list (which therefore holds every row)
__global__ void lk_init_kernel(double *cv, uint32_t *cj, uint8_t *alive, uint32_t *size, uint32_t *id, uint32_t *list, uint32_t *count,
                               uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i == 0) *count = n;
    if (i >= n) return;
    cv[i] = __longlong_as_double(0x7FF0000000000000ll);
    cj[i] = DENSE_NONE;
    alive[i] = 1;
    size[i] = 1;
    id[i] = list[i] = i;
}

// The least (cache value, row) over the rows with a cached neighbour, one partial per CTA; key = row << 32 | neighbour.  Block 0
// also empties the rescan list for this step's lk_update_kernel.
__global__ void __launch_bounds__(DENSE_THREADS) lk_argmin_kernel(const double *__restrict__ cv, const uint32_t *__restrict__ cj, uint32_t n,
                                                                  DenseMin *partial, uint32_t *count)
{
    if (blockIdx.x == 0 && threadIdx.x == 0) *count = 0;
    double bq = __longlong_as_double(0x7FF0000000000000ll);
    unsigned long long bk = DENSE_NO_KEY;
    for (uint32_t i = blockIdx.x * DENSE_THREADS + threadIdx.x; i < n; i += gridDim.x * DENSE_THREADS) {
        const uint32_t j = cj[i];
        const unsigned long long key = (unsigned long long)i << 32 | j;
        if (j != DENSE_NONE && dense_before(cv[i], key, bq, bk)) { bq = cv[i]; bk = key; }
    }
    const DenseMin b = dense_block_min(bq, bk);
    if (threadIdx.x == 0) partial[blockIdx.x] = b;
}

// Merge s of the pair lk_argmin_kernel found (every CTA reduces the partials itself): b = the row, a = its cached neighbour, a < b.
// Thread k owns slot k: it reads D(a, k) and D(b, k) (rows a and b), writes D(u, k) to row a and column a, NaN to column b of a row
// after b, and its own cache:
//   average:  D(u, k) = ((double)n_a * D(a, k) + (double)n_b * D(b, k)) / (double)(n_a + n_b)
//   complete: D(u, k) = max(D(a, k), D(b, k)), D(a, k) when they are equal
//   k > a, cached neighbour a or b: (D(u, k), a) if D(u, k) <= the cached value, else k goes on the rescan list
//   k > a, any other neighbour:     lowered to (D(u, k), a) when that is before the cached pair
// Thread a writes the merge record and puts row a on the list; thread b retires slot b.  Sizes and ids are only read here (the
// rescan kernel updates slot a's), and no entry is touched by two threads.
template <bool AVERAGE>
__global__ void __launch_bounds__(DENSE_THREADS) lk_update_kernel(double *D, uint64_t ld, const DenseMin *__restrict__ partial, uint32_t n_partial,
                                                                  uint32_t n, double *cv, uint32_t *cj, uint8_t *alive,
                                                                  const uint32_t *__restrict__ size, const uint32_t *__restrict__ id,
                                                                  uint32_t *list, uint32_t *count, LkMerge *rec, LkStep *step, int *no_pair)
{
    const DenseMin best = dense_partials_min(partial, n_partial);
    if (best.key == DENSE_NO_KEY) {         // no row has a live neighbour with a comparable distance: the result is refused
        if (blockIdx.x == 0 && threadIdx.x == 0) *no_pair = 1;
        return;
    }
    const uint32_t b = (uint32_t)(best.key >> 32), a = (uint32_t)best.key;
    const uint32_t k = blockIdx.x * DENSE_THREADS + threadIdx.x;
    if (k >= n) return;
    if (k == b) {
        cv[b] = __longlong_as_double(0x7FF0000000000000ll);
        cj[b] = DENSE_NONE;
        alive[b] = 0;
        return;
    }
    if (!alive[k]) return;
    if (k > b) D[(uint64_t)k * ld + b] = __longlong_as_double(0x7FF8000000000000ll);
    const uint32_t na = size[a], nb = size[b];
    if (k == a) {
        const uint32_t ia = id[a], ib = id[b];
        *rec = LkMerge{best.q, min(ia, ib), max(ia, ib), na + nb};
        *step = LkStep{a, b};
        list[atomicAdd(count, 1u)] = a;
        return;
    }
    double *row_a = D + (uint64_t)a * ld;
    const double dak = row_a[k], dbk = D[(uint64_t)b * ld + k];
    const double v = lk_value<AVERAGE>(na, nb, dak, dbk);
    row_a[k] = v;
    D[(uint64_t)k * ld + a] = v;
    if (k < a) return;
    const int o = lk_offer(v, a, b, cv[k], cj[k]);
    if (o == LK_TAKE) { cv[k] = v; cj[k] = a; }
    else if (o == LK_RESCAN) list[atomicAdd(count, 1u)] = k;
}

// Grid-stride CTAs over the rescan list (its length read here): row i's cache := the least (D(i, j), j) over j < i, NaN (dead)
// entries skipped; (+inf, none) when there is no such j.  With a step, block 0 first makes slot a the merged node u (size and id)
// and adds the list's length to the count of rows rescanned; the initial pass over every row has none.
__global__ void __launch_bounds__(LK_RESCAN_THREADS) lk_rescan_kernel(const double *__restrict__ D, uint64_t ld, const uint32_t *__restrict__ list,
                                                                      const uint32_t *count, double *cv, uint32_t *cj, const LkStep *step,
                                                                      uint32_t u, uint32_t *size, uint32_t *id, unsigned long long *rescanned)
{
    const uint32_t m = *count;
    if (step && blockIdx.x == 0 && threadIdx.x == 0) {
        const LkStep s = *step;
        size[s.a] += size[s.b];
        id[s.a] = u;
        *rescanned += m;
    }
    constexpr uint32_t T = LK_RESCAN_THREADS;
    for (uint32_t r = blockIdx.x; r < m; r += gridDim.x) {
        const uint32_t i = list[r];
        const double *row = D + (uint64_t)i * ld;
        double bq = __longlong_as_double(0x7FF0000000000000ll);
        unsigned long long bk = DENSE_NO_KEY;
        uint32_t j = threadIdx.x;
        for (; j + 3 * T < i; j += 4 * T) {         // four independent loads in flight per thread
            double d[4];
#pragma unroll
            for (int x = 0; x < 4; x++) d[x] = row[j + x * T];
#pragma unroll
            for (int x = 0; x < 4; x++)
                if (dense_before(d[x], j + x * T, bq, bk)) { bq = d[x]; bk = j + x * T; }
        }
        for (; j < i; j += T)
            if (dense_before(row[j], j, bq, bk)) { bq = row[j]; bk = j; }
        const DenseMin b = dense_block_min<T>(bq, bk);
        if (threadIdx.x == 0) {
            cv[i] = b.key == DENSE_NO_KEY ? __longlong_as_double(0x7FF0000000000000ll) : b.q;
            cj[i] = b.key == DENSE_NO_KEY ? DENSE_NONE : (uint32_t)b.key;
        }
        __syncthreads();                            // the block minimum's shared slots are reused by the next row
    }
}

}  // namespace
}  // namespace mashgpu

using namespace mashgpu;

extern "C" int mashgpu_linkage_matrix(mashgpu_ctx *ctx, double *d_matrix, uint64_t n, uint64_t ld, int method, uint32_t *id_lo, uint32_t *id_hi,
                                      double *height, uint32_t *size, uint64_t *rows_rescanned, void *stream)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!d_matrix || !id_lo || !id_hi || !height || !size) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    if (method != MASHGPU_LINKAGE_AVERAGE && method != MASHGPU_LINKAGE_COMPLETE)
        return fail(ctx, MASHGPU_ERR_INVALID, "unknown linkage method %d", method);
    cudaStream_t st;
    MG_TRY(dense_begin(ctx, d_matrix, n, ld, 2, "linkage", stream, st));
    const uint32_t N = (uint32_t)n;
    const uint32_t g = std::min<uint32_t>((uint32_t)ctx->sm_count * 8, dense_blocks(n));
    const uint32_t rescan_grid = (uint32_t)ctx->sm_count * 2;
    // O(n) state: the caches (value, neighbour), liveness, sizes, ids, the rescan list, the argmin's partials, the merge records
    DevBuf<double> cv; DevBuf<uint32_t> words; DevBuf<uint8_t> alive; DevBuf<DenseMin> partial; DevBuf<LkMerge> d_rec; DevBuf<LkStep> d_step;
    DevBuf<unsigned long long> d_rescanned; DevBuf<int> d_no_pair;
    if (cv.alloc(n) != cudaSuccess || words.alloc(4 * n + 1) != cudaSuccess || alive.alloc(n) != cudaSuccess || partial.alloc(g) != cudaSuccess ||
        d_rec.alloc(n - 1) != cudaSuccess || d_step.alloc(1) != cudaSuccess || d_rescanned.alloc(1) != cudaSuccess || d_no_pair.alloc(1) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (linkage state of %llu leaves)", (unsigned long long)n);
    uint32_t *cj = words.p, *sz = words.p + n, *id = words.p + 2 * n, *list = words.p + 3 * n, *count = words.p + 4 * n;
    MG_CUDA(ctx, cudaMemsetAsync(d_no_pair.p, 0, sizeof(int), st));
    MG_CUDA(ctx, cudaMemsetAsync(d_rescanned.p, 0, sizeof(unsigned long long), st));
    lk_init_kernel<<<dense_blocks(n), DENSE_THREADS, 0, st>>>(cv.p, cj, alive.p, sz, id, list, count, N);
    lk_rescan_kernel<<<std::min<uint32_t>(N, ctx->sm_count * 16u), LK_RESCAN_THREADS, 0, st>>>(d_matrix, ld, list, count, cv.p, cj, nullptr, 0, sz,
                                                                                               id, d_rescanned.p);
    MG_CUDA(ctx, cudaGetLastError());
    ctx->kernel_launches += 2;
    const bool average = method == MASHGPU_LINKAGE_AVERAGE;
    for (uint32_t s = 0; s + 1 < N; s++) {
        lk_argmin_kernel<<<g, DENSE_THREADS, 0, st>>>(cv.p, cj, N, partial.p, count);
        if (average)
            lk_update_kernel<true><<<dense_blocks(n), DENSE_THREADS, 0, st>>>(d_matrix, ld, partial.p, g, N, cv.p, cj, alive.p, sz, id, list, count,
                                                                          d_rec.p + s, d_step.p, d_no_pair.p);
        else
            lk_update_kernel<false><<<dense_blocks(n), DENSE_THREADS, 0, st>>>(d_matrix, ld, partial.p, g, N, cv.p, cj, alive.p, sz, id, list, count,
                                                                           d_rec.p + s, d_step.p, d_no_pair.p);
        lk_rescan_kernel<<<rescan_grid, LK_RESCAN_THREADS, 0, st>>>(d_matrix, ld, list, count, cv.p, cj, d_step.p, N + s, sz, id, d_rescanned.p);
        MG_CUDA(ctx, cudaGetLastError());
        ctx->kernel_launches += 3;
    }
    std::vector<LkMerge> rec(n - 1);
    unsigned long long rescanned = 0;
    int no_pair = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(rec.data(), d_rec.p, (n - 1) * sizeof(LkMerge), cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(&rescanned, d_rescanned.p, sizeof(rescanned), cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(&no_pair, d_no_pair.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    if (no_pair) return fail(ctx, MASHGPU_ERR_INVALID, "linkage found no pair with a comparable distance (an update overflowed)");
    for (uint64_t s = 0; s + 1 < n; s++) {
        id_lo[s] = rec[s].lo;
        id_hi[s] = rec[s].hi;
        height[s] = rec[s].height;
        size[s] = rec[s].size;
    }
    if (rows_rescanned) *rows_rescanned = rescanned;
    return MASHGPU_OK;
}
