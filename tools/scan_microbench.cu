// scan_microbench.cu -- standalone timing harness for scan_kernel<21, canonical, ASCII> variants (kernel tuning only).
//
// It runs the sketch scan at the shape of bench.py's sketch leg: U units of L bases back to back in HBM, the per-unit
// threshold and table geometry of plan_unit (3 s expected survivors, 2.7 slots per survivor), and per-tile coarse thresholds
// and first units by tile_tmax_kernel's rule (the largest threshold of the units a tile touches).  Every repetition starts from empty tables,
// as a sketch step does, and only the scan kernel is timed (CUDA events).  After the last repetition it prints an
// order-independent checksum of the candidate tables (key, count and unit of every occupied slot, plus the overflow and
// 2^64-1 counters), so two variants can be shown to produce the same candidates.
//
// Cost accounting (DESIGN.md §2.4): scan.cuh's SCAN_MB_* switches build variants without the survivor path
// (-DSCAN_MB_NO_SURVIVORS=1), with each warp's tile staged once and hashed again (-DSCAN_MB_STAGE_ONCE=1), or with clock64()
// around each tile's hot loop (-DSCAN_MB_CLOCK=1: reports the loop's cycles per warp per 256 windows, i.e. per 8 windows per
// lane; the hot-path instruction count of tools/sass_excerpt.py over it is a warp's issue rate inside the loop).  Their
// checksums differ from the kernel's by design.  -DSCAN_MB_EXTRA_FMA=n / -DSCAN_MB_EXTRA_ALU=n add a chain of n IMADs / n
// ALU instructions to every window's filter word (the checksum stays the kernel's); the kernel's time over n tells which pipe
// binds the hot loop.
//
// Variants of the kernel itself, whose checksums must all agree: -DSCAN_PREFETCH_SMEM=0 (next tile prefetched into
// registers instead of the shared landing buffer), -DSCAN_RESOLVE_INLINE=1 (the per-tile resolution of the pass masks
// inlined instead of called), -DSCAN_MIN_BLOCKS=n (resident CTAs per SM requested from ptxas).  SCAN_VOTE_GROUP applies to
// the FULL kernels only and does not change the kernel timed here.
//
// Build one binary per variant and run them alternately, e.g.
//   nvcc -std=c++17 -gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -DSCAN_MIN_BLOCKS=3 -I mash_b200/csrc \
//        tools/scan_microbench.cu -o tools/mb_mb3
//   tools/mb_mb3 [units=2000] [unit_len=5000000] [reps=5]
#include <algorithm>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
#include <cuda_runtime.h>
#include "scan.cuh"
using namespace mashgpu;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

__global__ void fill_kernel(uint8_t *p, uint64_t n, uint64_t seed)
{
    uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    for (; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        uint64_t x = (i + seed) * 0x9E3779B97F4A7C15ULL; x ^= x >> 29; x *= 0xBF58476D1CE4E5B9ULL; x ^= x >> 32;
        p[i] = "ACGT"[x & 3];
    }
}

// order-independent digest of the occupied slots of every unit's table
__global__ void checksum_kernel(const uint64_t *keys, const uint32_t *cnt, uint32_t n_units, uint32_t log2c, unsigned long long *out)
{
    const uint64_t n = (uint64_t)n_units << log2c;
    unsigned long long acc = 0, occ = 0;
    for (uint64_t i = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x; i < n; i += (uint64_t)gridDim.x * blockDim.x) {
        if (keys[i] == EMPTY_KEY) continue;
        uint64_t x = keys[i] ^ ((i >> log2c) * 0xD6E8FEB86659FD93ULL) ^ ((uint64_t)cnt[i] << 40);
        x ^= x >> 31; x *= 0xBF58476D1CE4E5B9ULL; x ^= x >> 29;
        acc += x; occ++;
    }
    atomicAdd(out, acc);
    atomicAdd(out + 1, occ);
}

int main(int argc, char **argv)
{
    const uint32_t n_units = argc > 1 ? (uint32_t)strtoul(argv[1], 0, 10) : 2000u;
    const uint64_t unit_len = argc > 2 ? strtoull(argv[2], 0, 10) : 5000000ull;
    const int reps = argc > 3 ? atoi(argv[3]) : 5;
    const uint64_t n = (uint64_t)n_units * unit_len;
    const uint32_t s = 1000;
    int sms = 0; CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0));
    uint8_t *d; CK(cudaMalloc(&d, n + 64));
    fill_kernel<<<sms * 8, 256>>>(d, n, 12345);

    // plan_unit (sketch.cu) for k=21, s=1000, 64-bit hashes: t = 3 s / L * 2^64, 2^ceil_log2(2.7 * 3 s + 2) slots
    const uint64_t t = (uint64_t)(3.0 * s / (double)unit_len * 18446744073709551616.0);
    uint32_t lg = 4;
    while ((1ull << lg) < (uint64_t)(2.7 * 3.0 * s) + 2) lg++;
    const uint64_t cap = 1ull << lg, slots = cap * n_units;
    std::vector<uint64_t> h_start(n_units + 1), h_t(n_units, t), h_off(n_units);
    std::vector<uint32_t> h_log2(n_units, lg);
    for (uint32_t u = 0; u <= n_units; u++) h_start[u] = u * unit_len;
    for (uint32_t u = 0; u < n_units; u++) h_off[u] = u * cap;
    const uint64_t ntiles = (n + SCAN_TILE - 1) / SCAN_TILE;
    std::vector<uint64_t> h_tmax(ntiles);
    std::vector<uint32_t> h_unit(ntiles);
    for (uint64_t tile = 0; tile < ntiles; tile++) {      // tile_tmax_kernel's rule
        const uint64_t first = tile * SCAN_TILE, last = std::min(first + SCAN_TILE, n) - 1;
        uint64_t m = 0;
        for (uint64_t u = first / unit_len; u < n_units && h_start[u] <= last; u++) m = std::max(m, h_t[u]);
        h_tmax[tile] = m;
        h_unit[tile] = (uint32_t)(first / unit_len);
    }

    uint64_t *unit_start, *unit_t, *tab_off, *keys, *tmax; uint32_t *log2c, *cnt, *flags, *maxh, *tunit; unsigned long long *sum;
    CK(cudaMalloc(&unit_start, (n_units + 1) * 8ull)); CK(cudaMalloc(&unit_t, n_units * 8ull)); CK(cudaMalloc(&tab_off, n_units * 8ull));
    CK(cudaMalloc(&log2c, n_units * 4ull)); CK(cudaMalloc(&flags, n_units * 4ull)); CK(cudaMalloc(&maxh, n_units * 4ull));
    CK(cudaMalloc(&keys, slots * 8)); CK(cudaMalloc(&cnt, slots * 4)); CK(cudaMalloc(&tmax, ntiles * 8)); CK(cudaMalloc(&sum, 16));
    CK(cudaMalloc(&tunit, ntiles * 4));
    CK(cudaMemcpy(unit_start, h_start.data(), (n_units + 1) * 8ull, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(unit_t, h_t.data(), n_units * 8ull, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(tab_off, h_off.data(), n_units * 8ull, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(log2c, h_log2.data(), n_units * 4ull, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(tmax, h_tmax.data(), ntiles * 8, cudaMemcpyHostToDevice));
    CK(cudaMemcpy(tunit, h_unit.data(), ntiles * 4, cudaMemcpyHostToDevice));

    ScanArgs a; memset(&a, 0, sizeof a);
    a.stream = d; a.stream_len = n; a.tile_begin = 0; a.tile_end = ntiles; a.tile_tmax = tmax; a.tile_unit = tunit; a.coarse_t = t;
    a.seed = 42; a.use64 = 1; a.mode = SCAN_SKETCH; a.unit_start = unit_start; a.n_units = n_units; a.unit_t = unit_t; a.tab_off = tab_off;
    a.tab_log2 = log2c; a.tab_keys = keys; a.tab_cnt = cnt; a.unit_flags = flags; a.unit_maxhash = maxh; a.only_unit = -1; a.min_copies = 1;
    auto kern = scan_kernel<21, true, false, false>;
    int per_sm = 0; CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, SCAN_THREADS, 0));
    cudaFuncAttributes fa; CK(cudaFuncGetAttributes(&fa, kern));
    const uint64_t need = (ntiles * (SCAN_TILE / SCAN_WARP_TILE) + SCAN_WARPS - 1) / SCAN_WARPS;   // as scan_inst.cu's launcher
    const int grid = (int)std::min<uint64_t>((uint64_t)per_sm * sms, need);
    // sink of the SCAN_MB_* variants: one word per thread, then one per warp
    const uint64_t sink_n = (uint64_t)grid * SCAN_THREADS + (uint64_t)grid * SCAN_WARPS;
    uint64_t *sink; CK(cudaMalloc(&sink, sink_n * 8)); CK(cudaMemset(sink, 0, sink_n * 8));
    a.out_hash = sink;
    auto reset = [&] {
        CK(cudaMemset(keys, 0xFF, slots * 8)); CK(cudaMemset(cnt, 0, slots * 4));
        CK(cudaMemset(flags, 0, n_units * 4ull)); CK(cudaMemset(maxh, 0, n_units * 4ull));
    };
    cudaEvent_t e0, e1; CK(cudaEventCreate(&e0)); CK(cudaEventCreate(&e1));
    for (int i = 0; i < 2; i++) { reset(); kern<<<grid, SCAN_THREADS>>>(a); }
    std::vector<float> ms(reps);
    for (int i = 0; i < reps; i++) {
        reset();
        CK(cudaEventRecord(e0)); kern<<<grid, SCAN_THREADS>>>(a); CK(cudaEventRecord(e1)); CK(cudaEventSynchronize(e1));
        CK(cudaEventElapsedTime(&ms[i], e0, e1));
    }
    CK(cudaGetLastError());
    CK(cudaMemset(sum, 0, 16));
    checksum_kernel<<<sms * 4, 256>>>(keys, cnt, n_units, lg, sum);
    unsigned long long h_sum[2];
    CK(cudaMemcpy(h_sum, sum, 16, cudaMemcpyDeviceToHost));
    std::vector<uint32_t> hf(n_units), hm(n_units);
    CK(cudaMemcpy(hf.data(), flags, n_units * 4ull, cudaMemcpyDeviceToHost)); CK(cudaMemcpy(hm.data(), maxh, n_units * 4ull, cudaMemcpyDeviceToHost));
    uint64_t nflag = 0, nmax = 0;
    for (uint32_t u = 0; u < n_units; u++) { nflag += hf[u] != 0; nmax += hm[u]; }
    // SCAN_MB_CLOCK: the warps' in-loop cycles (of the last repetition) per 256 windows
    std::vector<uint64_t> wcyc((size_t)grid * SCAN_WARPS);
    CK(cudaMemcpy(wcyc.data(), sink + (uint64_t)grid * SCAN_THREADS, wcyc.size() * 8, cudaMemcpyDeviceToHost));
    double cyc = 0;
    for (uint64_t c : wcyc) cyc += (double)c;
    const double loop_cycles_256 = cyc / ((double)ntiles * (SCAN_TILE / SCAN_WARP_TILE) * (SCAN_WARP_TILE / 256));
    std::vector<float> sorted = ms; std::sort(sorted.begin(), sorted.end());
    const float med = sorted[reps / 2];
    // SCAN_VOTE_GROUP only shapes the FULL kernels (k <= 16, screen); the kernel timed here resolves per-lane pass masks per tile
    printf("{\"variant\": \"%s\", \"min_blocks\": %d, \"prefetch_smem\": %d, \"resolve_inline\": %d, \"vote_group_full_kernels_only\": %d, "
           "\"extra_fma\": %d, \"extra_alu\": %d, \"regs\": %d, \"local_bytes\": %zu, \"occupancy\": %d, "
           "\"units\": %u, \"bases\": %llu, \"ms_median\": %.3f, \"ms_min\": %.3f, \"ms_max\": %.3f, \"gbps_median\": %.1f, "
           "\"checksum\": \"%016llx\", \"candidates\": %llu, \"overflowed_units\": %llu, \"maxhash\": %llu, \"warps_per_scheduler\": %d, "
           "\"loop_cycles_per_256_windows_per_warp\": %.1f, \"gbps_min\": %.1f, \"gbps_max\": %.1f}\n",
#ifdef VARIANT
           VARIANT,
#else
           "default",
#endif
           SCAN_MIN_BLOCKS, SCAN_PREFETCH_SMEM, SCAN_RESOLVE_INLINE, SCAN_VOTE_GROUP, SCAN_MB_EXTRA_FMA, SCAN_MB_EXTRA_ALU, fa.numRegs, (size_t)fa.localSizeBytes, per_sm, n_units, (unsigned long long)n, med,
           sorted[0], sorted[reps - 1], n / med / 1e6, h_sum[0], h_sum[1], (unsigned long long)nflag, (unsigned long long)nmax,
           per_sm * SCAN_WARPS / 4, SCAN_MB_CLOCK ? loop_cycles_256 : 0.0, n / sorted[reps - 1] / 1e6, n / sorted[0] / 1e6);
    return 0;
}
