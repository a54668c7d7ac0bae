// dict.cuh -- pieces shared by the two merge translation units, dist.cu (compareSketches) and within.cu (containSketches):
// the order-preserving 32-bit dictionary that turns every sketch into a row of ranks, the staging of a sketch set in device
// memory, and the shared-memory geometry of the tiled lockstep merge (DESIGN.md 3.1, 3.2, 3.6).
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

// The query rows are staged by the TMA engine (cp.async.bulk global -> shared, completion on a per-warp mbarrier).  A row of
// P ranks starts at a 4-byte aligned address (pitch P words), the bulk copy needs 16: the copy covers the 16-byte aligned
// span around the row and the merge starts `skew` bytes into the warp's buffer.
__host__ __device__ __forceinline__ uint32_t dist_qpitch(uint32_t P) { return (P + 4u + 3u) & ~3u; }

// Dynamic shared memory of the tiled merge for rows of P ranks: the reference tile (P x 32, element-interleaved), DIST_WARPS x
// DIST_ILP query buffers and one mbarrier per warp.  Row pitches for which it exceeds 227 KB (P > 1035) are not tiled.
inline size_t dist_smem_bytes(uint32_t P)
{
    return ((((size_t)P * DIST_TILE_R + 3) & ~(size_t)3) + (size_t)DIST_WARPS * DIST_ILP * dist_qpitch(P)) * 4 + DIST_WARPS * 8;
}

inline unsigned blocks_for(uint64_t n, unsigned tb = 256) { return (unsigned)std::max<uint64_t>(1, (n + tb - 1) / tb); }

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
