// dict.cuh -- pieces shared by the two merge translation units, dist.cu (compareSketches) and within.cu (containSketches):
// the order-preserving 32-bit dictionary that turns every sketch into a row of ranks, the staging of a sketch set in device
// memory, the shared-memory geometry of the tiled lockstep merge and the staging of rows into it (DESIGN.md 3.1, 3.2, 3.6), and
// the launch grid and host output chunks of a run.
#pragma once
#include <algorithm>

#include "common.cuh"

namespace mashgpu {

constexpr uint32_t RANK_PAD = 0xFFFFFFFFu;     // padding code after the ranks of a row (above every rank)
constexpr int DIST_WARPS = 12;
constexpr int DIST_ILP = 2;
constexpr int DIST_THREADS = DIST_WARPS * 32;
constexpr int DIST_TILE_R = 32;
static_assert(DIST_TILE_R * 4 == 128, "the merge step's PTX hard-codes the 128-byte stride of the interleaved reference tile");

__device__ __forceinline__ uint32_t lds32(uint32_t addr)
{
    uint32_t v;
    asm volatile("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(addr));
    return v;
}

// The query rows are staged by the TMA engine (bulk_span, bulk_copy_wait below).  A row of P ranks starts at a 4-byte aligned address (pitch
// P words), the bulk copy needs 16: the copy covers the 16-byte aligned span around the row and the merge starts `skew` bytes
// into the warp's buffer.
__host__ __device__ __forceinline__ uint32_t dist_qpitch(uint32_t P) { return (P + 4u + 3u) & ~3u; }

// The warp's mbarrier for bulk_copy_wait (one arrival per phase: lane 0's); returns its shared address.
__device__ __forceinline__ uint32_t warp_bar_init(uint64_t *slot)
{
    const uint32_t bar = (uint32_t)__cvta_generic_to_shared(slot);
    if ((threadIdx.x & 31) == 0) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" :: "r"(bar));
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    __syncwarp();
    return bar;
}

// A row of n > 0 ranks at `row` (4-byte aligned) as a bulk copy source: the 16-byte aligned span around it starts at `lo` and
// the row `skew` bytes into it; returns the span's bytes.
__device__ __forceinline__ uint32_t bulk_span(const uint32_t *row, uint32_t n, const uint32_t *&lo, uint32_t &skew)
{
    const uintptr_t p = (uintptr_t)row, l = p & ~(uintptr_t)15;
    lo = reinterpret_cast<const uint32_t *>(l);
    skew = (uint32_t)(p - l);
    return (uint32_t)(((p + (uintptr_t)n * 4 + 15) & ~(uintptr_t)15) - l);
}

// Copies up to N spans (bulk_span) into a warp's shared buffers dst + c * pitch, one bulk copy per span of bytes[c] > 0, with
// completion on the warp's mbarrier `bar`, and waits for all of them; `total` is the sum of bytes[].  Nothing is copied or
// waited for when it is 0; `phase` is the barrier's parity and flips with every wait.  Called by the whole warp, after the
// lanes' last reads of the buffers; the warp may read them when it returns.
template <int N>
__device__ __forceinline__ void bulk_copy_wait(const uint32_t *const (&lo)[N], const uint32_t (&bytes)[N], uint32_t total, uint32_t *dst,
                                               uint32_t pitch, uint32_t bar, uint32_t &phase)
{
    __syncwarp();                       // the lanes' reads of the previous rows precede the async writes
    if ((threadIdx.x & 31) == 0 && total) {
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(total) : "memory");
#pragma unroll
        for (int c = 0; c < N; c++)
            if (bytes[c])
                asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                             :: "r"((uint32_t)__cvta_generic_to_shared(dst + (size_t)c * pitch)), "l"(lo[c]), "r"(bytes[c]), "r"(bar) : "memory");
    }
    if (total) {
        // (braces scope the label: the helper may be inlined more than once into one kernel)
        asm volatile("{\n\t.reg .pred p;\n\tBULK_WAIT:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@!p bra BULK_WAIT;\n\t}"
                     :: "r"(bar), "r"(phase) : "memory");
        phase ^= 1;
    }
    __syncwarp();
}

// The reference tile of the tiled merges, element-interleaved so that lane l only ever touches bank l: element i of reference
// r0 + l at s_ref[i * 32 + l], RANK_PAD for references past n_ref.  The caller synchronises the CTA before reading it.
__device__ __forceinline__ void stage_ref_tile(uint32_t *s_ref, const uint32_t *ranks, uint64_t ref_row0, uint32_t P, uint32_t r0, uint32_t n_ref)
{
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const bool r_ok = r0 + lane < n_ref;
    const uint32_t *row = ranks + (ref_row0 + (r_ok ? r0 + lane : r0)) * (uint64_t)P;
    for (uint32_t i = warp; i < P; i += DIST_WARPS) s_ref[i * DIST_TILE_R + lane] = r_ok ? row[i] : RANK_PAD;
}

// Dynamic shared memory of the tiled merge for rows of P ranks: the reference tile (P x 32, element-interleaved), DIST_WARPS x
// DIST_ILP query buffers and one mbarrier per warp.  Row pitches for which it exceeds 227 KB (P > 1035) are not tiled.
inline size_t dist_smem_bytes(uint32_t P)
{
    return ((((size_t)P * DIST_TILE_R + 3) & ~(size_t)3) + (size_t)DIST_WARPS * DIST_ILP * dist_qpitch(P)) * 4 + DIST_WARPS * 8;
}

inline unsigned blocks_for(uint64_t n, unsigned tb = 256) { return (unsigned)std::max<uint64_t>(1, (n + tb - 1) / tb); }

// Grid of a tiled merge over every (query, reference tile) combination: the query range is sliced so that about 2 waves of CTAs
// cover the machine, at least one full round of warps each.  Sets the queries per CTA.
inline dim3 dense_grid(uint32_t r_tiles, uint64_t q_count, int sm_count, uint32_t &q_per_cta)
{
    const uint32_t round = DIST_WARPS * DIST_ILP;
    const uint32_t want_slices = std::max(1u, (uint32_t)(2 * sm_count + r_tiles - 1) / r_tiles);
    q_per_cta = (uint32_t)((q_count + want_slices - 1) / want_slices);
    q_per_cta = std::max(round, ((q_per_cta + round - 1) / round) * round);
    return dim3(r_tiles, (uint32_t)((q_count + q_per_cta - 1) / q_per_cta));
}

// A host call's output: its array (NULL: not wanted) and its bytes per query.
struct HostOut { void *host; uint64_t per_query; };

// Runs a host call in chunks of q_chunk queries through device buffers: one per wanted output, allocated once.  Per chunk
// [q, q + qc) the buffers are zeroed when `zero` is set, run(q, qc, d) enqueues the device call on ctx->stream (d[i]: the
// buffer of output i, NULL when it is not wanted), and every wanted output is copied back before the stream is synchronised.
template <int N, class Run>
int run_host_chunks(mashgpu_ctx *ctx, const HostOut (&out)[N], uint64_t q_count, uint64_t q_chunk, bool zero, const char *what, Run run)
{
    DevBuf<uint8_t> buf[N];
    void *d[N];
    for (int i = 0; i < N; i++) {
        d[i] = nullptr;
        if (!out[i].host) continue;
        if (buf[i].alloc(q_chunk * out[i].per_query) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (%s)", what);
        d[i] = buf[i].p;
    }
    cudaStream_t st = ctx->stream;
    for (uint64_t q = 0; q < q_count; q += q_chunk) {
        const uint64_t qc = std::min(q_chunk, q_count - q);
        for (int i = 0; i < N; i++)
            if (zero && d[i]) MG_CUDA(ctx, cudaMemsetAsync(d[i], 0, qc * out[i].per_query, st));
        MG_TRY(run(q, qc, d));
        for (int i = 0; i < N; i++)
            if (d[i]) MG_CUDA(ctx, cudaMemcpyAsync((uint8_t *)out[i].host + q * out[i].per_query, d[i], qc * out[i].per_query, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
    }
    return MASHGPU_OK;
}

// device copies of a sketch set's arrays (uploaded when the set lives in host memory)
struct SetOnDevice {
    const uint64_t *hashes = nullptr; const uint32_t *n_hashes = nullptr; const uint64_t *length = nullptr;
    DevBuf<uint64_t> h, l; DevBuf<uint32_t> n;
};

int stage_set(mashgpu_ctx *ctx, const mashgpu_sketch_set *s, SetOnDevice &d, cudaStream_t st, bool want_length = true);
int check_set(mashgpu_ctx *ctx, const mashgpu_sketch_set *s, const char *what, bool want_length = true);

// Valid hashes of a device-resident set -> keys[out0 ...] / slots[out0 ...] (compacted, row order); n_eff[row0 + row] =
// min(n_hashes, P, stride) filled.  Returns the number of entries through *n_out (synchronises the stream once to read it).
int dict_gather(mashgpu_ctx *ctx, const SetOnDevice &d, uint64_t n_rows, uint64_t stride, uint32_t P, uint64_t row0, uint32_t *n_eff,
                uint64_t out0, uint64_t *keys, uint32_t *slots, uint64_t *n_out, cudaStream_t st);

// out[vals[t]] = rank of keys[t] among the distinct keys (keys in any order; `keys` and `vals` are clobbered).
// *n_distinct is read back (synchronises the stream).
int dict_rank(mashgpu_ctx *ctx, uint64_t *keys, uint32_t *vals, uint64_t n, uint32_t *out, uint64_t *n_distinct, cudaStream_t st);

// The rank rows of a job: rows [0, n_ref) from the reference set, then (qry != NULL) rows [n_ref, n_ref + n_qry) from the query
// set, each of pitch P: the first n_eff = min(n_hashes, P, stride) slots hold the ranks of the row's hashes among all distinct
// hashes of both sets, every other slot RANK_PAD.  `ranks` holds (n_ref + n_qry) * P words, `n_eff` n_ref + n_qry.
int encode_rows(mashgpu_ctx *ctx, const SetOnDevice &ref, uint64_t n_ref, uint64_t ref_stride, const SetOnDevice *qry, uint64_t n_qry,
                uint64_t qry_stride, uint32_t P, uint32_t *ranks, uint32_t *n_eff, cudaStream_t st);

}  // namespace mashgpu
