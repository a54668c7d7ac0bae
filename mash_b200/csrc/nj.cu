// nj.cu -- neighbor joining over a dense float64 distance matrix in device memory (C-ABI: mashgpu_neighbor_joining_matrix,
// DESIGN.md 3.10).  No counterpart in the reference: its users feed the `mash triangle` matrix to an NJ program on the CPU.
//
// Canonical Saitou-Nei / Studier-Keppler NJ with a fixed floating-point operation order, so that tests/nj_model.py (numpy)
// reproduces every output bit.  Every device arithmetic step is one IEEE double operation written as a __d*_rn intrinsic, which
// nvcc never contracts into an FMA; the one division per join (of the branch lengths) is done on the host from the join records.
// Per step the host only enqueues two kernels; nothing is read back until the end.
//
// Matrix: the caller's n x ld array.  dense_mirror_kernel (dense.cuh) copies the lower triangle to the upper one and zeroes the
// diagonal, so that every live row holds all live columns and the join writes a row and a column.  Rows never move: row slot a stays the row
// of the node at that position (a join puts u into the slot of a, the smaller position).  The live positions are kept as lists of
// row slot, column index, node id and row sum, in position order (double-buffered, rewritten by each join).  Columns are
// compacted in place, row by row, whenever the live count falls to 3/4 of the column span, so a scan reads at most 4/3 of the
// live lower triangle's bytes (plus sector rounding) and never the full n x n.  Dead rows are skipped outright.
#include <vector>

#include "dense.cuh"

namespace mashgpu {
namespace {

struct NjJoin { uint32_t a, b; double dab, diff; };     // join s: node ids of a and b, D(a, b) and r_a - r_b
struct NjLast { uint32_t id[3]; double len[3]; };       // the last three nodes and their branches

// r_i = sum over ascending k of D(i, k), the diagonal's 0 included; thread i walks column i, so a warp reads 32 adjacent doubles
__global__ void __launch_bounds__(64) nj_rowsum_kernel(const double *__restrict__ D, uint64_t ld, uint32_t n, double *r)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    double s = D[i];
#pragma unroll 8
    for (uint32_t k = 1; k < n; k++) s = __dadd_rn(s, D[(uint64_t)k * ld + i]);
    r[i] = s;
}

// both buffers of the position lists: slot = column = node id = position (the second buffer only ever holds valid indices)
__global__ void nj_init_kernel(uint32_t *rs, uint32_t *cs, uint32_t *id, uint32_t n)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    rs[i] = rs[n + i] = cs[i] = cs[n + i] = id[i] = id[n + i] = i;
}

// Moves the live columns of every live row to their positions: row rs[k], column cs[p] -> column p.  cs is ascending, so
// cs[p] >= p: a chunk of positions reads only columns at or after its own start, and later chunks only columns after its end.
// One barrier between a chunk's reads and its writes is all the ordering needed.  Rows are independent.
__global__ void __launch_bounds__(DENSE_THREADS) nj_compact_kernel(double *D, uint64_t ld, const uint32_t *__restrict__ rs,
                                                                   const uint32_t *__restrict__ cs, uint32_t m)
{
    for (uint32_t k = blockIdx.x; k < m; k += gridDim.x) {
        double *row = D + (uint64_t)rs[k] * ld;
        for (uint32_t c0 = 0; c0 < m; c0 += DENSE_THREADS) {
            const uint32_t p = c0 + threadIdx.x;
            const double v = p < m ? row[cs[p]] : 0.0;
            __syncthreads();
            if (p < m) row[p] = v;
        }
    }
}

__global__ void nj_iota_kernel(uint32_t *v, uint32_t m)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < m) v[i] = i;
}

// One warp per item of two rows (q = 1 + it and q = m - 1 - it: m positions per item), grid-stride.  Q is never stored: each lane
// keeps its least (Q, q, p) and the block writes one partial.
//   Q(p, q) = ((m - 2) * D(a, b) - r_a) - r_b,  a = L[p], b = L[q], p < q
__global__ void __launch_bounds__(DENSE_THREADS) nj_scan_kernel(const double *__restrict__ D, uint64_t ld, const uint32_t *__restrict__ rs,
                                                                const uint32_t *__restrict__ cs, const double *__restrict__ r, uint32_t m,
                                                                DenseMin *partial)
{
    const double mm2 = (double)(m - 2);
    double bq = __longlong_as_double(0x7FF0000000000000ll);
    unsigned long long bk = DENSE_NO_KEY;
    const uint32_t lane = threadIdx.x & 31, items = m / 2;
    const uint32_t warps = (gridDim.x * DENSE_THREADS) >> 5;
    for (uint32_t it = (blockIdx.x * DENSE_THREADS + threadIdx.x) >> 5; it < items; it += warps) {
        for (int h = 0; h < 2; h++) {
            const uint32_t q = h ? m - 1 - it : it + 1;
            if (h && q == it + 1) break;
            const double *row = D + (uint64_t)rs[q] * ld;
            const double rq = r[q];
            const unsigned long long kq = (unsigned long long)q << 32;
            uint32_t p = lane;
            for (; p + 96 < q; p += 128) {          // four independent loads in flight per lane
                double d[4], rp[4];
#pragma unroll
                for (int u = 0; u < 4; u++) { d[u] = row[cs[p + 32 * u]]; rp[u] = r[p + 32 * u]; }
#pragma unroll
                for (int u = 0; u < 4; u++) {
                    const double Q = __dsub_rn(__dsub_rn(__dmul_rn(mm2, d[u]), rp[u]), rq);
                    if (dense_before(Q, kq | (p + 32 * u), bq, bk)) { bq = Q; bk = kq | (p + 32 * u); }
                }
            }
            for (; p < q; p += 32) {
                const double Q = __dsub_rn(__dsub_rn(__dmul_rn(mm2, row[cs[p]]), r[p]), rq);
                if (dense_before(Q, kq | p, bq, bk)) { bq = Q; bk = kq | p; }
            }
        }
    }
    const DenseMin b = dense_block_min(bq, bk);
    if (threadIdx.x == 0) partial[blockIdx.x] = b;
}

// Join s (u = n + s) of the pair the scan found; every block reduces the partials itself.  Thread k handles position k:
//   D(u, k) = ((D(a, k) + D(b, k)) - D(a, b)) * 0.5, written to row a and column a
//   r_k     = ((r_k - D(a, k)) - D(b, k)) + D(u, k)
//   r_u     = ((r_a + r_b) - m * D(a, b)) * 0.5
// u takes position p, q is removed.  The record keeps D(a, b) and r_a - r_b: the branch lengths need one division, which the host
// does when it reads the records back (nj_tree), so no device arithmetic of the joins is a DFMA.  Thread k reads row a and row b
// at column cs[k] and writes row a at cs[k] and row rs[k] at cs[p]; no other thread touches those entries, and D(a, b) (row b) is
// not written.
__global__ void __launch_bounds__(DENSE_THREADS) nj_join_kernel(double *D, uint64_t ld, const DenseMin *__restrict__ partial, uint32_t n_partial,
                                                                uint32_t m, uint32_t u, const uint32_t *__restrict__ rs, const uint32_t *__restrict__ cs,
                                                                const uint32_t *__restrict__ id, const double *__restrict__ r, uint32_t *rs2,
                                                                uint32_t *cs2, uint32_t *id2, double *r2, NjJoin *rec, int *no_pair)
{
    const DenseMin best = dense_partials_min(partial, n_partial);
    if (best.key == DENSE_NO_KEY) {         // every Q was NaN (sums that overflowed): the result is refused
        if (blockIdx.x == 0 && threadIdx.x == 0) *no_pair = 1;
        return;
    }
    const uint32_t p = (uint32_t)best.key, q = (uint32_t)(best.key >> 32);
    const uint32_t k = blockIdx.x * DENSE_THREADS + threadIdx.x;
    if (k >= m || k == q) return;
    const uint32_t a = rs[p], ca = cs[p];
    double *row_a = D + (uint64_t)a * ld;
    const double *row_b = D + (uint64_t)rs[q] * ld;
    const double dab = row_b[ca], ra = r[p], rb = r[q];
    const uint32_t k2 = k < q ? k : k - 1;
    if (k == p) {
        *rec = NjJoin{id[p], id[q], dab, __dsub_rn(ra, rb)};
        r2[p] = __dmul_rn(__dsub_rn(__dadd_rn(ra, rb), __dmul_rn((double)m, dab)), 0.5);
        rs2[p] = a; cs2[p] = ca; id2[p] = u;
        return;
    }
    const uint32_t ck = cs[k], sk = rs[k];
    const double dak = row_a[ck], dbk = row_b[ck];
    const double duk = __dmul_rn(__dsub_rn(__dadd_rn(dak, dbk), dab), 0.5);
    row_a[ck] = duk;
    D[(uint64_t)sk * ld + ca] = duk;
    r2[k2] = __dadd_rn(__dsub_rn(__dsub_rn(r[k], dak), dbk), duk);
    rs2[k2] = sk; cs2[k2] = ck; id2[k2] = id[k];
}

// the last three positions x, y, z: lx = ((D(x, y) + D(x, z)) - D(y, z)) * 0.5 and so on
__global__ void nj_final_kernel(const double *D, uint64_t ld, const uint32_t *rs, const uint32_t *cs, const uint32_t *id, NjLast *last)
{
    const double dxy = D[(uint64_t)rs[1] * ld + cs[0]], dxz = D[(uint64_t)rs[2] * ld + cs[0]], dyz = D[(uint64_t)rs[2] * ld + cs[1]];
    *last = NjLast{{id[0], id[1], id[2]},
                   {__dmul_rn(__dsub_rn(__dadd_rn(dxy, dxz), dyz), 0.5), __dmul_rn(__dsub_rn(__dadd_rn(dxy, dyz), dxz), 0.5),
                    __dmul_rn(__dsub_rn(__dadd_rn(dxz, dyz), dxy), 0.5)}};
}

}  // namespace
}  // namespace mashgpu

using namespace mashgpu;

extern "C" int mashgpu_neighbor_joining_matrix(mashgpu_ctx *ctx, double *d_matrix, uint64_t n, uint64_t ld, uint32_t *parent, double *length,
                                               void *stream)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!d_matrix || !parent || !length) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    cudaStream_t st;
    MG_TRY(dense_begin(ctx, d_matrix, n, ld, 3, "neighbor joining", stream, st));
    const uint32_t N = (uint32_t)n, nodes = 2 * N - 2;
    const uint32_t max_partials = (uint32_t)ctx->sm_count * 8;
    // O(n) state: two buffers of the position lists (slot, column, node id; row sums), the join records, the scan's partials, a flag
    DevBuf<uint32_t> lists; DevBuf<double> sums; DevBuf<NjJoin> d_rec; DevBuf<NjLast> d_last; DevBuf<DenseMin> partial; DevBuf<int> d_no_pair;
    if (lists.alloc(6ull * n) != cudaSuccess || sums.alloc(2ull * n) != cudaSuccess || d_rec.alloc(n - 3) != cudaSuccess ||
        d_last.alloc(1) != cudaSuccess || partial.alloc(max_partials) != cudaSuccess || d_no_pair.alloc(1) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (neighbor joining state of %llu leaves)", (unsigned long long)n);
    uint32_t *rs[2] = {lists.p, lists.p + n}, *cs[2] = {lists.p + 2 * n, lists.p + 3 * n}, *id[2] = {lists.p + 4 * n, lists.p + 5 * n};
    double *r[2] = {sums.p, sums.p + n};
    MG_CUDA(ctx, cudaMemsetAsync(d_no_pair.p, 0, sizeof(int), st));
    nj_rowsum_kernel<<<dense_blocks(n, 64), 64, 0, st>>>(d_matrix, ld, N, r[0]);
    nj_init_kernel<<<dense_blocks(n), DENSE_THREADS, 0, st>>>(rs[0], cs[0], id[0], N);
    MG_CUDA(ctx, cudaGetLastError());
    ctx->kernel_launches += 2;
    uint32_t span = N;          // columns in use: [0, span)
    for (uint32_t s = 0; s + 3 < N; s++) {
        const uint32_t m = N - s, c = s & 1;
        if (4ull * m <= 3ull * span) {
            nj_compact_kernel<<<std::min<uint32_t>(m, ctx->sm_count * 16u), DENSE_THREADS, 0, st>>>(d_matrix, ld, rs[c], cs[c], m);
            nj_iota_kernel<<<dense_blocks(m), DENSE_THREADS, 0, st>>>(cs[c], m);
            ctx->kernel_launches += 2;
            span = m;
        }
        const uint32_t g = std::min<uint32_t>(max_partials, dense_blocks(m / 2, DENSE_THREADS / 32));
        nj_scan_kernel<<<g, DENSE_THREADS, 0, st>>>(d_matrix, ld, rs[c], cs[c], r[c], m, partial.p);
        nj_join_kernel<<<dense_blocks(m), DENSE_THREADS, 0, st>>>(d_matrix, ld, partial.p, g, m, N + s, rs[c], cs[c], id[c], r[c], rs[c ^ 1], cs[c ^ 1],
                                                               id[c ^ 1], r[c ^ 1], d_rec.p + s, d_no_pair.p);
        MG_CUDA(ctx, cudaGetLastError());
        ctx->kernel_launches += 2;
    }
    const uint32_t c = (N - 3) & 1;
    nj_final_kernel<<<1, 1, 0, st>>>(d_matrix, ld, rs[c], cs[c], id[c], d_last.p);
    MG_CUDA(ctx, cudaGetLastError());
    ctx->kernel_launches++;
    std::vector<NjJoin> rec(n - 3);
    NjLast last;
    int no_pair = 0;
    if (n > 3) MG_CUDA(ctx, cudaMemcpyAsync(rec.data(), d_rec.p, (n - 3) * sizeof(NjJoin), cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(&last, d_last.p, sizeof(NjLast), cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(&no_pair, d_no_pair.p, sizeof(int), cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    if (no_pair) return fail(ctx, MASHGPU_ERR_INVALID, "neighbor joining found no pair with a comparable Q (row sums overflowed)");
    // la = D(a, b) * 0.5 + (r_a - r_b) / (2 * (m - 2)), lb = D(a, b) - la: IEEE double operations in this order (x86-64 without FMA
    // code generation, so nothing is contracted)
    for (uint32_t s = 0; s + 3 < N; s++) {
        const NjJoin &j = rec[s];
        const double half = j.dab * 0.5, den = 2.0 * (double)(N - s - 2), share = j.diff / den, la = half + share;
        parent[j.a] = parent[j.b] = N + s;
        length[j.a] = la;
        length[j.b] = j.dab - la;
    }
    for (int i = 0; i < 3; i++) { parent[last.id[i]] = nodes - 1; length[last.id[i]] = last.len[i]; }
    parent[nodes - 1] = DENSE_NONE;
    length[nodes - 1] = 0.0;
    return MASHGPU_OK;
}
