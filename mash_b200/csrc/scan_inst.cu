// scan_inst.cu -- explicit instantiations of scan_kernel<K, CANON, PACKED, FULL> for K in [SCAN_K_LO, SCAN_K_HI].
// Compiled several times with different -DSCAN_K_LO/-DSCAN_K_HI/-DSCAN_PART so the parts build in parallel.
#include "scan.cuh"

#ifndef SCAN_K_LO
#error "compile with -DSCAN_K_LO=.. -DSCAN_K_HI=.. -DSCAN_PART=.."
#endif

namespace mashgpu {

// grid <= 0: size the persistent grid to the resident CTAs (occupancy x SM count, queried once per kernel)
template <int K, bool CANON, bool PACKED, bool FULL>
static void launch_scan_kernel(const ScanArgs &a, int grid, cudaStream_t stream)
{
    static int resident = 0;
    if (resident == 0) {
        int per_sm = 0, dev = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, scan_kernel<K, CANON, PACKED, FULL>, SCAN_THREADS, 0);
        resident = (per_sm > 0 ? per_sm : 1) * (sms > 0 ? sms : 1);
    }
    const uint64_t warp_tiles = (a.tile_end - a.tile_begin) * (SCAN_TILE / SCAN_WARP_TILE);
    const uint64_t need = (warp_tiles + SCAN_WARPS - 1) / SCAN_WARPS;
    int g = grid > 0 ? grid : resident;
    if ((uint64_t)g > need) g = (int)need;
    if (g < 1) g = 1;
    scan_kernel<K, CANON, PACKED, FULL><<<g, SCAN_THREADS, 0, stream>>>(a);
}

// k > 16: the screen probes the reference table with every lane's full hash; every other mode only needs the filter word
template <int K, bool CANON, bool PACKED>
static void launch_scan(const ScanArgs &a, int grid, cudaStream_t stream)
{
    if constexpr (K <= 16) launch_scan_kernel<K, CANON, PACKED, true>(a, grid, stream);
    else if (a.mode == SCAN_SCREEN) launch_scan_kernel<K, CANON, PACKED, true>(a, grid, stream);
    else launch_scan_kernel<K, CANON, PACKED, false>(a, grid, stream);
}

template <int K>
static scan_launch_fn pick(int k, bool canonical, bool packed)
{
    if constexpr (K > SCAN_K_HI) {
        return nullptr;
    } else {
        if (k == K) {
            if (packed) return canonical ? &launch_scan<K, true, true> : &launch_scan<K, false, true>;
            return canonical ? &launch_scan<K, true, false> : &launch_scan<K, false, false>;
        }
        return pick<K + 1>(k, canonical, packed);
    }
}

template <int K>
static void launch_bytes(const ScanArgs &a, int grid, cudaStream_t stream)
{
    static int resident = 0;
    if (resident == 0) {
        int per_sm = 0, dev = 0, sms = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
        cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, scan_bytes_kernel<K>, SCAN_THREADS, 0);
        resident = (per_sm > 0 ? per_sm : 1) * (sms > 0 ? sms : 1);
    }
    const uint64_t warp_tiles = (a.tile_end - a.tile_begin) * (SCAN_TILE / SCAN_WARP_TILE);
    const uint64_t need = (warp_tiles + SCAN_WARPS - 1) / SCAN_WARPS;
    int g = grid > 0 ? grid : resident;
    if ((uint64_t)g > need) g = (int)need;
    if (g < 1) g = 1;
    scan_bytes_kernel<K><<<g, SCAN_THREADS, 0, stream>>>(a);
}

template <int K>
static scan_launch_fn pick_bytes(int k)
{
    if constexpr (K > SCAN_K_HI) {
        return nullptr;
    } else {
        if (k == K) return &launch_bytes<K>;
        return pick_bytes<K + 1>(k);
    }
}

#define CAT_(a, b) a##b
#define CAT(a, b) CAT_(a, b)
scan_launch_fn CAT(get_scan_launcher_part, SCAN_PART)(int k, bool canonical, bool packed)
{
    if (k < SCAN_K_LO || k > SCAN_K_HI) return nullptr;
    return pick<SCAN_K_LO>(k, canonical, packed);
}

scan_launch_fn CAT(get_bytes_launcher_part, SCAN_PART)(int k)
{
    if (k < SCAN_K_LO || k > SCAN_K_HI) return nullptr;
    return pick_bytes<SCAN_K_LO>(k);
}

}  // namespace mashgpu
