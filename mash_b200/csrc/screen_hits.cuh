// screen_hits.cuh -- the sparse finish of a screen job (mashgpu_screen_finish_hits), included by screen.cu.
//
// mashgpu_screen_finish reduces every reference sketch: one CTA per sketch probes each of its hashes in the table.  That is
// n_ref x s probes whatever the sample hit.  The sparse finish works from the hashes the sample did hit instead, through an
// inverted index distinct hash -> sketches that hold it, built once per job (DESIGN.md 4.3):
//
//   index    d of every (sketch, hash) pair and a count per d, an exclusive scan, and a scatter of the sketch index into d's
//            segment (taxscreen.cu's tax_pairs_kernel / tax_scatter_kernel with the sketch index as the code).
//   hits     distinct indices with cnt[d] >= 1, ascending (CUB DeviceSelect).
//   depths   a counting sort of the hit pairs by sketch: per-sketch counts over the expanded segments (= shared), a scan, and a
//            scatter of cnt[d] into the sketch's run.  Segments longer than HITS_SERIAL_MAX go to a warp, shorter ones to a thread.
//   reduce   one CTA per hit sketch, in ascending sketch order: the run sorted, its median, and the identity and p-value of
//            screen_estimates, the expressions the dense reduce uses.
//   -w       the hit sketches ranked by (shared / n desc, length desc, index asc), compared exactly by cross-multiplication;
//            best[i] = the smallest rank over hit i's segment; the depths are rebuilt from each hit's winner alone.
//
// The per-sketch counters are left at zero by the scatter that consumes them (or, for the plain count under -w, by clearing the
// rows), so no pass clears an n_ref array.

namespace mashgpu {

constexpr uint32_t HITS_SERIAL_MAX = 8;      // longer segments are walked by a warp

// cnt[d] >= 1: the sample hit distinct hash d
struct HitPred {
    const uint32_t *cnt;
    __device__ __forceinline__ bool operator()(uint32_t d) const { return cnt[d] >= 1; }
};

// ref_cnt[r] > 0: sketch r holds a hit pair
struct RefPred {
    const uint32_t *ref_cnt;
    __device__ __forceinline__ bool operator()(uint32_t r) const { return ref_cnt[r] > 0; }
};

// -w order of the hit sketches: the identity estimate (shared / n)^(1/k) descending, then genome length descending, then index.
// x^(1/k) is increasing, so the order of the estimates is the order of the exact fractions (DESIGN.md 4.3: distinct fractions with
// n <= 2^15 stay apart after the root and its rounding); a * d vs c * b fits 64 bits because every term is <= 2^15.
struct WinnerOrder {
    const uint32_t *ref_start, *n_hashes;
    const uint64_t *len;
    __device__ __forceinline__ bool operator()(uint32_t a, uint32_t b) const
    {
        const uint64_t sa = ref_start[a + 1] - ref_start[a], sb = ref_start[b + 1] - ref_start[b];
        const uint64_t x = sa * n_hashes[b], y = sb * n_hashes[a];
        if (x != y) return x > y;
        if (len[a] != len[b]) return len[a] > len[b];
        return a < b;
    }
};

// One thread per hit (position i of hit_d): the pairs of a short segment; longer segments are queued for the warp kernel when
// `queue` is set (the first pass of a finish), and skipped otherwise (the queue is already built).
//   SCATTER = false: ref_cnt[r]++ for every sketch r of the segment
//   SCATTER = true:  cnt[d] goes to a free place of r's run (ref_cnt counts down to 0)
template <bool SCATTER>
__global__ void __launch_bounds__(SCR_THREADS) hits_pairs_kernel(
    const uint32_t *__restrict__ hit_d, uint32_t n_hit, const uint32_t *__restrict__ seg_start, const uint32_t *__restrict__ seg_ref,
    const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ ref_start, uint32_t *__restrict__ ref_cnt, uint32_t *__restrict__ depths,
    uint32_t *__restrict__ long_list, uint32_t *__restrict__ n_long, bool queue)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_hit) return;
    const uint32_t d = hit_d[i];
    const uint32_t a = seg_start[d], n = seg_start[d + 1] - a;
    if (n > HITS_SERIAL_MAX) {
        if (queue) long_list[atomicAdd(n_long, 1u)] = i;
        return;
    }
    const uint32_t c = cnt[d];
    for (uint32_t j = 0; j < n; j++) {
        const uint32_t r = seg_ref[a + j];
        if (SCATTER) depths[ref_start[r] + atomicSub(&ref_cnt[r], 1u) - 1] = c;
        else atomicAdd(&ref_cnt[r], 1u);
    }
}

// one warp per queued hit: the lanes stride over the segment
template <bool SCATTER>
__global__ void __launch_bounds__(SCR_THREADS) hits_pairs_long_kernel(
    const uint32_t *__restrict__ hit_d, const uint32_t *__restrict__ seg_start, const uint32_t *__restrict__ seg_ref,
    const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ ref_start, uint32_t *__restrict__ ref_cnt, uint32_t *__restrict__ depths,
    const uint32_t *__restrict__ long_list, const uint32_t *__restrict__ n_long)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n_warps = gridDim.x * (SCR_THREADS / 32);
    const uint32_t total = *n_long;
    for (uint32_t w = blockIdx.x * (SCR_THREADS / 32) + threadIdx.x / 32; w < total; w += n_warps) {
        const uint32_t d = hit_d[long_list[w]];
        const uint32_t a = seg_start[d], n = seg_start[d + 1] - a;
        const uint32_t c = cnt[d];
        for (uint32_t j = lane; j < n; j += 32) {
            const uint32_t r = seg_ref[a + j];
            if (SCATTER) depths[ref_start[r] + atomicSub(&ref_cnt[r], 1u) - 1] = c;
            else atomicAdd(&ref_cnt[r], 1u);
        }
    }
}

// rank of every hit sketch in the -w order: prio[order[i]] = i
__global__ void hits_rank_kernel(const uint32_t *__restrict__ order, uint32_t n, uint32_t *__restrict__ prio)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) prio[order[i]] = i;
}

// -w: best[i] = the smallest rank over hit i's segment (every sketch in it is a hit sketch, so its rank is set).  One thread per
// short segment; long ones by a warp (hits_best_long_kernel).
__global__ void __launch_bounds__(SCR_THREADS) hits_best_kernel(
    const uint32_t *__restrict__ hit_d, uint32_t n_hit, const uint32_t *__restrict__ seg_start, const uint32_t *__restrict__ seg_ref,
    const uint32_t *__restrict__ prio, uint32_t *__restrict__ best)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_hit) return;
    const uint32_t d = hit_d[i];
    const uint32_t a = seg_start[d], n = seg_start[d + 1] - a;
    if (n > HITS_SERIAL_MAX) return;
    uint32_t b = 0xFFFFFFFFu;
    for (uint32_t j = 0; j < n; j++) b = min(b, prio[seg_ref[a + j]]);
    best[i] = b;
}

__global__ void __launch_bounds__(SCR_THREADS) hits_best_long_kernel(
    const uint32_t *__restrict__ hit_d, const uint32_t *__restrict__ seg_start, const uint32_t *__restrict__ seg_ref,
    const uint32_t *__restrict__ prio, const uint32_t *__restrict__ long_list, const uint32_t *__restrict__ n_long, uint32_t *__restrict__ best)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n_warps = gridDim.x * (SCR_THREADS / 32);
    const uint32_t total = *n_long;
    for (uint32_t w = blockIdx.x * (SCR_THREADS / 32) + threadIdx.x / 32; w < total; w += n_warps) {
        const uint32_t i = long_list[w];
        const uint32_t d = hit_d[i];
        const uint32_t a = seg_start[d], n = seg_start[d + 1] - a;
        uint32_t b = 0xFFFFFFFFu;
        for (uint32_t j = lane; j < n; j += 32) b = min(b, prio[seg_ref[a + j]]);
        b = __reduce_min_sync(0xFFFFFFFFu, b);
        if (lane == 0) best[i] = b;
    }
}

// -w: each hit counts for its winner order[best[i]] alone.  SCATTER = false counts, SCATTER = true places cnt[d] in the run.
template <bool SCATTER>
__global__ void hits_winner_kernel(const uint32_t *__restrict__ hit_d, uint32_t n_hit, const uint32_t *__restrict__ best, const uint32_t *__restrict__ order,
                                   const uint32_t *__restrict__ cnt, const uint32_t *__restrict__ ref_start, uint32_t *__restrict__ ref_cnt,
                                   uint32_t *__restrict__ depths)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_hit) return;
    const uint32_t r = order[best[i]];
    if (SCATTER) depths[ref_start[r] + atomicSub(&ref_cnt[r], 1u) - 1] = cnt[hit_d[i]];
    else atomicAdd(&ref_cnt[r], 1u);
}

// One CTA per row: sketch rows_ref[i]'s run of depths, sorted in shared memory -> median; identity and p-value as the dense reduce.
// Runs hold at most SCREEN_MAX_REF_HASHES depths (mashgpu_screen_open refuses larger sketches).
__global__ void __launch_bounds__(SCR_THREADS) hits_reduce_kernel(
    const uint32_t *__restrict__ rows_ref, const uint32_t *__restrict__ ref_start, const uint32_t *__restrict__ depths_in,
    const uint32_t *__restrict__ n_hashes, uint64_t set_size, int kmer_size, double kmer_space,
    uint64_t *__restrict__ shared_out, uint64_t *__restrict__ median_out, double *__restrict__ identity_out, double *__restrict__ pvalue_out)
{
    extern __shared__ uint32_t depths[];
    const uint32_t i = blockIdx.x;
    const uint32_t r = rows_ref[i];
    const uint32_t a = ref_start[r], shared = ref_start[r + 1] - a;
    uint32_t N = 2;
    while (N < shared) N <<= 1;
    for (uint32_t j = threadIdx.x; j < N; j += SCR_THREADS) depths[j] = j < shared ? depths_in[a + j] : 0xFFFFFFFFu;
    __syncthreads();
    for (uint32_t size = 2; size <= N; size <<= 1)
        for (uint32_t st = size >> 1; st > 0; st >>= 1) {
            for (uint32_t t = threadIdx.x; t < N / 2; t += SCR_THREADS) {
                uint32_t lo = 2 * t - (t & (st - 1)), hi = lo + st;
                bool up = (lo & size) == 0;
                uint32_t x = depths[lo], y = depths[hi];
                if ((x > y) == up) { depths[lo] = y; depths[hi] = x; }
            }
            __syncthreads();
        }
    if (threadIdx.x == 0) {
        shared_out[i] = shared;
        median_out[i] = depths[shared / 2];
        screen_estimates(shared, n_hashes[r], set_size, kmer_size, kmer_space, &identity_out[i], &pvalue_out[i]);
    }
}

// a[list[i]] = 0: the hit counters at a reset after finish_hits (list = the hits), the per-sketch counters of the plain -w count
__global__ void clear_listed_kernel(const uint32_t *__restrict__ list, uint32_t n, uint32_t *__restrict__ a)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) a[list[i]] = 0;
}

}  // namespace mashgpu
