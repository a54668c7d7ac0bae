// within.cu -- containment of query sketches in reference sketches, every pair on the GPU (C-ABI: mashgpu_within_*).
//
// Replaces contain / containSketches (reference CommandContain.cpp:205-265).  containSketches(R, Q) walks the two sorted lists
// with denom = min(|R|, |Q|):
//      while (steps < denom && i < |R|):  R[i] < Q[j] -> i++ (not a step);  Q[j] < R[i] -> j++;  tie -> i++, j++, common++
// and returns score = common / j, error = 1 / sqrt(j): j, the number of query hashes examined, ends at
//      j_end = min(denom, #{t : Q[t] <= R[|R|-1]})      (0 for an empty R),    common = |Q[0 .. j_end) n R|
// (DESIGN.md 3.6; tests/within_model.py pins this to the reference's object code).
//
// Rows are the dictionary ranks of dist.cu (dict.cuh), with one difference: the reference side of the walk is NOT cut to the
// sketch size -- a row of R takes part in full, so the row pitch is P = max |R| + 1 and a query row keeps its first P ranks
// (only min(|Q|, max |R|) of them can be examined).  Two kernels, selected by P as dist selects them:
//   within_kernel       P <= 1035: dist_kernel's layout (32 references element-interleaved in shared memory, query rows staged
//                       by TMA into per-warp buffers), one lane per (query, reference) pair running the reference's loop in lockstep
//   within_pair_kernel  larger P (`-s 10000`): one warp per pair; the examined query prefix Q[0 .. j_end) is cut into 32 runs and
//                       each lane counts the ties of its run with one binary search into R and a sequential walk
#include <algorithm>
#include <cmath>
#include <cstring>
#include <memory>
#include <vector>

#include "common.cuh"
#include "dict.cuh"

namespace mashgpu {

struct WithinArgs {
    const uint32_t *ranks;      // rows of P ranks: references first, then queries (or shared when self)
    uint32_t P;                 // row pitch = max |R| + 1
    const uint32_t *ref_n;      // hashes per reference row (all of them: n_hashes <= P - 1)
    const uint32_t *qry_n;      // min(n_hashes, P) per query row
    uint64_t ref_row0, qry_row0;
    uint32_t n_ref;
    uint32_t q_begin, q_count;
    uint32_t q_per_cta;         // within_kernel: queries handled by one CTA (grid.y slices the query range)
    double max_error;           // pass = error <= max_error
    uint32_t *common; uint32_t *examined; double *score; double *error; uint8_t *pass;   // outputs, (q - q_begin) * n_ref + r
};

// Epilogue of containSketches (CommandContain.cpp:261-264).  Division and square root are IEEE (correctly rounded) in double on
// the device, as on the host: the values are bit-identical to the reference's for j > 0.  j == 0 gives 0.0 / 0 there, which on
// x86 is the default NaN with the sign bit set (printed "-nan"); the same bit pattern is written here.
__device__ __forceinline__ void within_emit(const WithinArgs &a, uint32_t q, uint32_t r, uint32_t common, uint32_t j)
{
    const uint64_t o = (uint64_t)(q - a.q_begin) * a.n_ref + r;
    const double error = 1.0 / sqrt((double)j);
    if (a.common) a.common[o] = common;
    if (a.examined) a.examined[o] = j;
    if (a.score) a.score[o] = j ? (double)common / (double)j : __longlong_as_double((long long)0xFFF8000000000000ull);
    if (a.error) a.error[o] = error;
    if (a.pass) a.pass[o] = error <= a.max_error ? 1 : 0;
}

// Tiled lockstep kernel.  The reference tile and the query staging are dist_kernel's (dict.cuh); the step is the reference's loop
// with its two stop conditions as per-lane predicates: a lane whose pair has stopped keeps issuing the step with everything
// predicated off until the whole warp is done (a vote every 8 steps).  A lane stops at the end of R (i == |R|, its pointer reaches
// the tile slot after its last rank) or once j reaches denom.
__global__ void __launch_bounds__(DIST_THREADS, 1) within_kernel(const WithinArgs a)
{
    extern __shared__ __align__(16) uint32_t smem[];
    const uint32_t qpitch = dist_qpitch(a.P);
    uint32_t *s_ref = smem;                                  // [P][32]
    uint32_t *s_qry = smem + (((size_t)a.P * DIST_TILE_R + 3) & ~(size_t)3);      // [DIST_WARPS][DIST_ILP][qpitch]
    uint64_t *s_bar = reinterpret_cast<uint64_t *>(s_qry + (size_t)DIST_WARPS * DIST_ILP * qpitch);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const uint32_t r0 = blockIdx.x * DIST_TILE_R;
    const uint32_t r = r0 + lane;
    const bool r_ok = r < a.n_ref;
    if ((uint64_t)blockIdx.y * a.q_per_cta >= a.q_count) return;

    stage_ref_tile(s_ref, a.ranks, a.ref_row0, a.P, r0, a.n_ref);
    __syncthreads();
    const uint32_t nR = r_ok ? a.ref_n[r] : 0;
    const uint32_t sref_base = (uint32_t)__cvta_generic_to_shared(s_ref) + lane * 4;
    const uint32_t sref_end = sref_base + nR * (DIST_TILE_R * 4);
    uint32_t *my_q = s_qry + (size_t)warp * DIST_ILP * qpitch;
    const uint32_t bar = warp_bar_init(s_bar + warp);
    uint32_t phase = 0;

    const uint32_t q_lo = a.q_begin + blockIdx.y * a.q_per_cta;
    const uint32_t q_hi = (uint32_t)min((uint64_t)a.q_begin + a.q_count, (uint64_t)q_lo + a.q_per_cta);
    for (uint32_t qb = q_lo + warp * DIST_ILP; qb < q_hi; qb += DIST_WARPS * DIST_ILP) {
        uint32_t skew[DIST_ILP], bytes[DIST_ILP], total = 0;
        const uint32_t *src[DIST_ILP];
#pragma unroll
        for (int c = 0; c < DIST_ILP; c++) {
            skew[c] = 0; bytes[c] = 0; src[c] = nullptr;
            if (qb + c < q_hi) {
                bytes[c] = bulk_span(a.ranks + (a.qry_row0 + qb + c) * (uint64_t)a.P, a.P, src[c], skew[c]);
                total += bytes[c];
            }
        }
        __builtin_assume(total != 0);          // slot 0 holds query qb < q_hi
        bulk_copy_wait(src, bytes, total, my_q, qpitch, bar, phase);
        uint32_t pa[DIST_ILP], pb[DIST_ILP], pb0[DIST_ILP], pb_end[DIST_ILP], va[DIST_ILP], vb[DIST_ILP], common[DIST_ILP];
#pragma unroll
        for (int c = 0; c < DIST_ILP; c++) {
            const uint32_t nQ = qb + c < q_hi ? a.qry_n[qb + c] : 0;
            pa[c] = sref_base;
            pb0[c] = pb[c] = (uint32_t)__cvta_generic_to_shared(my_q + (size_t)c * qpitch) + skew[c];
            pb_end[c] = pb0[c] + min(nR, nQ) * 4;
            va[c] = lds32(pa[c]);
            vb[c] = lds32(pb[c]);
            common[c] = 0;
        }
        // one step: go = j < denom && i < |R|;  R[i] <= Q[j] -> i++;  Q[j] <= R[i] -> j++;  both (a tie) -> common++
        for (;;) {
            bool live = false;
#pragma unroll
            for (int c = 0; c < DIST_ILP; c++) live |= pb[c] < pb_end[c] && pa[c] < sref_end;
            if (!__any_sync(0xFFFFFFFFu, live)) break;
#pragma unroll 8
            for (int t = 0; t < 8; t++) {
#pragma unroll
                for (int c = 0; c < DIST_ILP; c++) {
                    asm volatile("{\n\t.reg .pred go, pa, pb, pt;\n\t"
                                 "setp.lt.u32 go, %3, %5;\n\t"
                                 "setp.lt.and.u32 go, %2, %6, go;\n\t"
                                 "setp.le.and.u32 pa, %0, %1, go;\n\t"
                                 "setp.ge.and.u32 pb, %0, %1, go;\n\t"
                                 "and.pred pt, pa, pb;\n\t"
                                 "@pa add.u32 %2, %2, 128;\n\t"
                                 "@pb add.u32 %3, %3, 4;\n\t"
                                 "@pt add.u32 %4, %4, 1;\n\t"
                                 "@pa ld.shared.u32 %0, [%2];\n\t"
                                 "@pb ld.shared.u32 %1, [%3];\n\t}"
                                 : "+r"(va[c]), "+r"(vb[c]), "+r"(pa[c]), "+r"(pb[c]), "+r"(common[c]) : "r"(pb_end[c]), "r"(sref_end));
                }
            }
        }
#pragma unroll
        for (int c = 0; c < DIST_ILP; c++)
            if (qb + c < q_hi && r_ok) within_emit(a, qb + c, r, common[c], (pb[c] - pb0[c]) / 4);
        __syncwarp();
    }
}

// One warp per pair, rows read from global memory (through L1).  With the closed form the pair needs no sequential walk as a
// whole: j_end is an upper-bound search of R[|R|-1] in Q[0 .. denom) (all lanes, same addresses), then Q[0 .. j_end) is cut into
// 32 runs of odd length and lane l counts the ties of run l: one lower-bound search of its first element in R, then a walk
// (every Q[j] of the run is <= R[|R|-1], so the walk stays inside R).  Pairs are enumerated in 32 x 32 blocks (query-major
// blocks, reference-major inside) so that the rows of the pairs in flight stay in L2.
constexpr int WPAIR_WARPS = 8;
constexpr uint64_t WITHIN_CHUNK_PAIRS = 1ull << 24;     // mashgpu_within_run: pairs per device output chunk (~420 MB of outputs)

__global__ void __launch_bounds__(WPAIR_WARPS * 32) within_pair_kernel(const WithinArgs a)
{
    const int lane = threadIdx.x & 31;
    const uint64_t warps = (uint64_t)gridDim.x * (blockDim.x >> 5);
    const uint32_t q_blocks = (a.q_count + 31) / 32, r_blocks = (a.n_ref + 31) / 32;
    const uint64_t total = (uint64_t)q_blocks * r_blocks * 1024;
    for (uint64_t idx = (uint64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5); idx < total; idx += warps) {
        const uint64_t blk = idx >> 10;
        const uint32_t in = (uint32_t)(idx & 1023);
        const uint32_t qi = (uint32_t)(blk / r_blocks) * 32 + (in & 31), r = (uint32_t)(blk % r_blocks) * 32 + (in >> 5);
        if (qi >= a.q_count || r >= a.n_ref) continue;
        const uint32_t q = a.q_begin + qi;
        const uint32_t *R = a.ranks + (a.ref_row0 + r) * (uint64_t)a.P, *Q = a.ranks + (a.qry_row0 + q) * (uint64_t)a.P;
        const uint32_t nR = a.ref_n[r], denom = min(nR, a.qry_n[q]);
        uint32_t j_end = 0;
        if (denom) {
            const uint32_t last = R[nR - 1];
            uint32_t lo = 0, hi = denom;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (Q[mid] <= last) lo = mid + 1; else hi = mid;
            }
            j_end = lo;
        }
        uint32_t run = (j_end + 31) / 32;
        if (run > 1) run |= 1u;
        const uint32_t jb = min((uint32_t)lane * run, j_end), je = min(jb + run, j_end);
        uint32_t common = 0;
        if (jb < je) {
            uint32_t v = Q[jb], lo = 0, hi = nR;
            while (lo < hi) {
                const uint32_t mid = (lo + hi) >> 1;
                if (R[mid] < v) lo = mid + 1; else hi = mid;
            }
            uint32_t i = lo, j = jb;
            for (;;) {
                uint32_t w = R[i];
                while (w < v) w = R[++i];
                if (w == v) { common++; i++; }
                if (++j == je) break;
                v = Q[j];
            }
        }
        common = __reduce_add_sync(0xFFFFFFFFu, common);
        if (lane == 0) within_emit(a, q, r, common, j_end);
    }
}

}  // namespace mashgpu

using namespace mashgpu;

struct mashgpu_within_job {
    mashgpu_ctx *ctx = nullptr;
    uint64_t n_ref = 0, n_qry = 0;
    uint64_t qry_row0 = 0;
    uint32_t P = 0;
    double max_error = 0;
    bool tiled = true;
    DevBuf<uint32_t> ranks, n_eff;
};

namespace {

// n_hashes of a set in host memory (copied back when the set lives on the device); refuses rows longer than the stride
int set_counts(mashgpu_ctx *ctx, const mashgpu_sketch_set *s, const char *what, std::vector<uint32_t> &n)
{
    n.resize(s->n);
    if (s->n == 0) return MASHGPU_OK;
    if (s->on_device) MG_CUDA(ctx, cudaMemcpy(n.data(), s->n_hashes, s->n * 4, cudaMemcpyDeviceToHost));
    else std::memcpy(n.data(), s->n_hashes, s->n * 4);
    for (uint64_t i = 0; i < s->n; i++)
        if (n[i] > s->stride)
            return fail(ctx, MASHGPU_ERR_INVALID, "%s row %llu has %u hashes, more than the stride %llu", what, (unsigned long long)i, n[i],
                        (unsigned long long)s->stride);
    return MASHGPU_OK;
}

}  // namespace

extern "C" int mashgpu_within_open(mashgpu_ctx *ctx, const mashgpu_sketch_set *ref, const mashgpu_sketch_set *qry, double max_error,
                                   mashgpu_within_job **job_out)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!job_out) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    MG_TRY(check_set(ctx, ref, "reference", false));
    const bool self = (qry == nullptr || qry == ref);
    if (!self) MG_TRY(check_set(ctx, qry, "query", false));
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    std::vector<uint32_t> nr, nq;
    MG_TRY(set_counts(ctx, ref, "reference", nr));
    if (!self) MG_TRY(set_counts(ctx, qry, "query", nq));
    uint64_t r_max = 0;
    for (uint32_t v : nr) r_max = std::max<uint64_t>(r_max, v);
    if (r_max > 0x7FFFFFF0ull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "reference sketches of more than 2^31 hashes");

    std::unique_ptr<mashgpu_within_job> job(new mashgpu_within_job());
    job->ctx = ctx; job->max_error = max_error;
    job->n_ref = ref->n; job->n_qry = self ? ref->n : qry->n;
    job->qry_row0 = self ? 0 : job->n_ref;
    const uint32_t P = (uint32_t)r_max + 1;
    job->P = P;
    const uint64_t rows = job->n_ref + (self ? 0 : job->n_qry);
    if (rows * P >= 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^31 dictionary slots (%llu rows x %u)", (unsigned long long)rows, P);
    SetOnDevice dr, dq;
    MG_TRY(stage_set(ctx, ref, dr, st, false));
    if (!self) MG_TRY(stage_set(ctx, qry, dq, st, false));
    if (job->ranks.alloc(rows * P) != cudaSuccess || job->n_eff.alloc(rows) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (rank rows)");
    MG_TRY(encode_rows(ctx, dr, job->n_ref, ref->stride, self ? nullptr : &dq, job->n_qry, self ? 0 : qry->stride, P, job->ranks.p,
                       job->n_eff.p, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));      // the staged sets go out of scope
    job->tiled = dist_smem_bytes(P) <= 227 * 1024;
    if (job->tiled) MG_CUDA(ctx, cudaFuncSetAttribute(within_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024));
    *job_out = job.release();
    return MASHGPU_OK;
}

extern "C" int mashgpu_within_run_dev(mashgpu_within_job *job, uint64_t q_begin, uint64_t q_count, uint32_t *d_common, uint32_t *d_examined,
                                      double *d_score, double *d_error, uint8_t *d_pass, void *stream)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (q_begin + q_count > job->n_qry)
        return fail(ctx, MASHGPU_ERR_INVALID, "query range [%llu, %llu) exceeds %llu", (unsigned long long)q_begin,
                    (unsigned long long)(q_begin + q_count), (unsigned long long)job->n_qry);
    if (q_count == 0 || job->n_ref == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = stream ? (cudaStream_t)stream : ctx->stream;
    WithinArgs a{};
    a.ranks = job->ranks.p; a.P = job->P;
    a.ref_n = job->n_eff.p; a.qry_n = job->n_eff.p + job->qry_row0; a.ref_row0 = 0; a.qry_row0 = job->qry_row0;
    a.n_ref = (uint32_t)job->n_ref; a.q_begin = (uint32_t)q_begin; a.q_count = (uint32_t)q_count;
    a.max_error = job->max_error;
    a.common = d_common; a.examined = d_examined; a.score = d_score; a.error = d_error; a.pass = d_pass;
    time_begin(ctx, ctx->dist_events, st);
    if (job->tiled) {
        const dim3 grid = dense_grid((uint32_t)((job->n_ref + DIST_TILE_R - 1) / DIST_TILE_R), q_count, ctx->sm_count, a.q_per_cta);
        within_kernel<<<grid, DIST_THREADS, dist_smem_bytes(a.P), st>>>(a);
    } else {
        within_pair_kernel<<<ctx->sm_count * 8, WPAIR_WARPS * 32, 0, st>>>(a);
    }
    MG_CUDA(ctx, cudaGetLastError());
    time_end(ctx, ctx->dist_events, st);
    ctx->kernel_launches++;
    ctx->dist_launches++;
    return MASHGPU_OK;
}

extern "C" int mashgpu_within_run(mashgpu_within_job *job, uint64_t q_begin, uint64_t q_count, uint32_t *common, uint32_t *examined,
                                  double *score, double *error, uint8_t *pass)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (q_begin + q_count > job->n_qry) return fail(ctx, MASHGPU_ERR_INVALID, "query range exceeds query count");
    if (q_count == 0 || job->n_ref == 0) return MASHGPU_OK;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    // bound the device outputs: chunks of queries
    const uint64_t n_ref = job->n_ref;
    const uint64_t q_chunk = std::min(q_count, std::max<uint64_t>(1, WITHIN_CHUNK_PAIRS / n_ref));
    const HostOut out[] = {{common, 4 * n_ref}, {examined, 4 * n_ref}, {score, 8 * n_ref}, {error, 8 * n_ref}, {pass, n_ref}};
    return run_host_chunks(ctx, out, q_count, q_chunk, false, "pair outputs", [&](uint64_t q, uint64_t qc, void *const *d) {
        return mashgpu_within_run_dev(job, q_begin + q, qc, (uint32_t *)d[0], (uint32_t *)d[1], (double *)d[2], (double *)d[3], (uint8_t *)d[4],
                                      ctx->stream);
    });
}

extern "C" int mashgpu_within_close(mashgpu_within_job *job)
{
    if (!job) return MASHGPU_ERR_INVALID;
    cudaSetDevice(job->ctx->device);
    cudaStreamSynchronize(job->ctx->stream);
    delete job;
    return MASHGPU_OK;
}
