// common.cuh -- context, error handling and small device-buffer helpers shared by the C-ABI translation units.
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <string>
#include <vector>
#include <utility>

#include "../../include/mashgpu.h"

namespace mashgpu {

struct EventPair { cudaEvent_t a, b; };

}  // namespace mashgpu

namespace mashgpu {
// grow-only buffer owned by the context (no allocation on the hot path after warm-up); growing discards the contents
template <cudaError_t (*Alloc)(void **, size_t), cudaError_t (*Free)(void *)>
struct GrowBuf {
    void *p = nullptr;
    size_t bytes = 0;
    ~GrowBuf() { if (p) Free(p); }
    template <typename T>
    T *get(size_t count)
    {
        size_t need = count * sizeof(T);
        if (need == 0) need = 16;
        if (need > bytes) {
            if (p) Free(p);
            p = nullptr; bytes = 0;
            size_t want = need + need / 8;
            if (Alloc(&p, want) != cudaSuccess) {
                cudaGetLastError();
                if (Alloc(&p, need) != cudaSuccess) { cudaGetLastError(); p = nullptr; return nullptr; }
                want = need;
            }
            bytes = want;
        }
        return reinterpret_cast<T *>(p);
    }
};
using Scratch = GrowBuf<cudaMalloc, cudaFree>;              // device memory
using PinnedScratch = GrowBuf<cudaMallocHost, cudaFreeHost>;  // page-locked host memory
}  // namespace mashgpu

struct mashgpu_ctx {
    int device = 0;
    int sm_count = 132;
    cudaStream_t stream = nullptr;       // compute
    cudaStream_t copy_stream = nullptr;  // H2D staging
    std::string err;
    bool attr_dist = false, attr_merge = false, attr_select = false;
    // instrumentation
    bool timing = false;
    uint64_t kernel_launches = 0;
    uint64_t scan_launches = 0, dist_launches = 0, exact_reruns = 0, translate_launches = 0;
    double scan_ms = 0, dist_ms = 0, translate_ms = 0, tax_ms = 0;
    std::vector<mashgpu::EventPair> scan_events, dist_events, translate_events, tax_events;
    uint64_t reads_events = 0, reads_peak_bytes = 0;   // reads jobs: events replayed; device footprint of the last job
    double reads_replay_ms = 0;
    uint64_t unit_stages = 0, unit_peak_bytes = 0;     // unit jobs: stages merged; device footprint of the last job
    // sketch_stream_core scratch
    mashgpu::Scratch sc_start, sc_t, sc_off, sc_log2, sc_flags, sc_maxhash, sc_keys, sc_cnt, sc_tmax, sc_tunit, sc_first, sc_last, sc_qtarget, sc_qtstar;
    // mashgpu_sketch_batch: wave stream buffers and outputs
    mashgpu::Scratch sc_wave[2], sc_inval[2], sc_runs[2], sc_out_hashes, sc_out_n, sc_out_counts;
    mashgpu::Scratch sc_sep[2], sc_codes[2];
    mashgpu::Scratch sc_big_units, sc_big_n, sc_big_off, sc_big_bounds, sc_big_comp, sc_big_sorted, sc_big_tmp;   // select of tables > 2^14 slots
    mashgpu::PinnedScratch pinned[2], pinned_sep[2];   // ASCII feed path: staged small records, separator list
    mashgpu::PinnedScratch pinned_codes[2];         // packed feed path: host code buffers
    cudaEvent_t pack_copied[2] = {nullptr, nullptr};
    mashgpu::PinnedScratch flags_pinned;            // per-unit status flags of the sketch pass in flight (sketch.cu)
    cudaStream_t pack_stream = nullptr;             // packed uploads (next to the ASCII copies on copy_stream)
    // screen: chunk staging buffers and the finish() outputs outlive a job (cudaMalloc of a few hundred MB inside a timed pass cost
    // 1-50 ms depending on the box); scr_stage_owner = the job using the staging pair, others allocate their own
    mashgpu::Scratch scr_stage[2], scr_out;
    const void *scr_stage_owner = nullptr;
    mashgpu::PinnedScratch scr_pinned[2];           // packed host feed of screen: pinned codes + mask per slot (with scr_stage)
    cudaEvent_t wave_copied[2] = {nullptr, nullptr};
};

namespace mashgpu {

inline int fail(mashgpu_ctx *ctx, int code, const char *fmt, ...)
{
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    if (ctx) ctx->err = buf;
    return code;
}

#define MG_CUDA(ctx, call)                                                                          \
    do {                                                                                            \
        cudaError_t e__ = (call);                                                                   \
        if (e__ != cudaSuccess)                                                                     \
            return mashgpu::fail((ctx), MASHGPU_ERR_CUDA, "%s failed: %s (%s:%d)", #call,           \
                                 cudaGetErrorString(e__), __FILE__, __LINE__);                      \
    } while (0)

#define MG_TRY(expr)                      \
    do {                                  \
        int rc__ = (expr);                \
        if (rc__ != MASHGPU_OK) return rc__; \
    } while (0)

// RAII device buffer (freed on scope exit)
template <typename T>
struct DevBuf {
    T *p = nullptr;
    size_t n = 0;
    DevBuf() = default;
    DevBuf(const DevBuf &) = delete;
    DevBuf &operator=(const DevBuf &) = delete;
    ~DevBuf() { release(); }
    void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
    cudaError_t alloc(size_t count)
    {
        release();
        const cudaError_t e = cudaMalloc((void **)&p, (count ? count : 1) * sizeof(T));
        if (e != cudaSuccess) { p = nullptr; cudaGetLastError(); return e; }    // n stays 0: a later `n < need` test re-allocates
        n = count;
        return e;
    }
    // grow-only: keeps the buffer when it already holds `count` entries
    cudaError_t reserve(size_t count) { return (p && n >= count) ? cudaSuccess : alloc(count + count / 4); }
};

template <typename T>
struct PinnedBuf {
    T *p = nullptr;
    size_t n = 0;
    PinnedBuf() = default;
    PinnedBuf(const PinnedBuf &) = delete;
    PinnedBuf &operator=(const PinnedBuf &) = delete;
    ~PinnedBuf() { release(); }
    void release() { if (p) cudaFreeHost(p); p = nullptr; n = 0; }
    cudaError_t alloc(size_t count)
    {
        release();
        const cudaError_t e = cudaMallocHost((void **)&p, (count ? count : 1) * sizeof(T));
        if (e != cudaSuccess) { p = nullptr; cudaGetLastError(); return e; }
        n = count;
        return e;
    }
};

inline uint32_t ceil_log2(uint64_t x)
{
    uint32_t l = 0;
    while ((1ull << l) < x) l++;
    return l;
}

// Begin/end a timed region for one of the dominant kernels (no-ops unless ctx->timing).
inline void time_begin(mashgpu_ctx *ctx, std::vector<EventPair> &list, cudaStream_t s)
{
    if (!ctx->timing) return;
    EventPair ev;
    cudaEventCreate(&ev.a);
    cudaEventCreate(&ev.b);
    cudaEventRecord(ev.a, s);
    list.push_back(ev);
}
inline void time_end(mashgpu_ctx *ctx, std::vector<EventPair> &list, cudaStream_t s)
{
    if (!ctx->timing) return;
    cudaEventRecord(list.back().b, s);
}

}  // namespace mashgpu
