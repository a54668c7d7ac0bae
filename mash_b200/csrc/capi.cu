// capi.cu -- context management and instrumentation of the C ABI (include/mashgpu.h).
#include <cstring>
#include <mutex>

#include "common.cuh"

using namespace mashgpu;

static std::string g_create_error;
static std::mutex g_mutex;

extern "C" int mashgpu_device_count(void)
{
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess) { cudaGetLastError(); return 0; }
    return n;
}

extern "C" int mashgpu_create(int device, mashgpu_ctx **out)
{
    if (!out) return MASHGPU_ERR_INVALID;
    *out = nullptr;
    auto bad = [&](int code, const std::string &msg) {
        std::lock_guard<std::mutex> lock(g_mutex);
        g_create_error = msg;
        return code;
    };
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0)
        return bad(MASHGPU_ERR_CUDA, std::string("no CUDA device available (") + cudaGetErrorString(e) + "); this engine has no CPU path");
    if (device < 0 || device >= n) return bad(MASHGPU_ERR_INVALID, "device index out of range");
    if ((e = cudaSetDevice(device)) != cudaSuccess) return bad(MASHGPU_ERR_CUDA, std::string("cudaSetDevice: ") + cudaGetErrorString(e));
    cudaDeviceProp prop;
    if ((e = cudaGetDeviceProperties(&prop, device)) != cudaSuccess) return bad(MASHGPU_ERR_CUDA, std::string("cudaGetDeviceProperties: ") + cudaGetErrorString(e));
    if (prop.major != 9 || prop.minor != 0)
        return bad(MASHGPU_ERR_UNSUPPORTED, std::string("device '") + prop.name + "' is not sm_90 (this library carries sm_90a code only)");
    mashgpu_ctx *ctx = new mashgpu_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    if ((e = cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking)) != cudaSuccess ||
        (e = cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking)) != cudaSuccess) {
        delete ctx;
        return bad(MASHGPU_ERR_CUDA, std::string("cudaStreamCreate: ") + cudaGetErrorString(e));
    }
    *out = ctx;
    return MASHGPU_OK;
}

extern "C" void mashgpu_destroy(mashgpu_ctx *ctx)
{
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    for (auto *list : {&ctx->scan_events, &ctx->dist_events, &ctx->tax_events})
        for (auto &ev : *list) { cudaEventDestroy(ev.a); cudaEventDestroy(ev.b); }
    for (int b = 0; b < 2; b++) {
        if (ctx->wave_copied[b]) cudaEventDestroy(ctx->wave_copied[b]);
        if (ctx->pack_copied[b]) cudaEventDestroy(ctx->pack_copied[b]);
    }
    if (ctx->pack_stream) cudaStreamDestroy(ctx->pack_stream);
    if (ctx->stream) cudaStreamDestroy(ctx->stream);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    delete ctx;
}

extern "C" const char *mashgpu_last_error(const mashgpu_ctx *ctx)
{
    if (ctx) return ctx->err.c_str();
    std::lock_guard<std::mutex> lock(g_mutex);
    return g_create_error.c_str();
}

extern "C" int mashgpu_set_timing(mashgpu_ctx *ctx, int timing)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    ctx->timing = timing != 0;
    return MASHGPU_OK;
}

static void drain(std::vector<EventPair> &list, double &acc)
{
    for (auto &ev : list) {
        cudaEventSynchronize(ev.b);
        float ms = 0;
        if (cudaEventElapsedTime(&ms, ev.a, ev.b) == cudaSuccess) acc += ms;
        cudaEventDestroy(ev.a);
        cudaEventDestroy(ev.b);
    }
    list.clear();
}

extern "C" int mashgpu_get_stats(mashgpu_ctx *ctx, mashgpu_stats *out, int reset)
{
    if (!ctx || !out) return MASHGPU_ERR_INVALID;
    cudaSetDevice(ctx->device);
    drain(ctx->scan_events, ctx->scan_ms);
    drain(ctx->dist_events, ctx->dist_ms);
    drain(ctx->translate_events, ctx->translate_ms);
    drain(ctx->tax_events, ctx->tax_ms);
    out->kernel_launches = ctx->kernel_launches;
    out->scan_kernel_ms = ctx->scan_ms;
    out->scan_kernel_launches = ctx->scan_launches;
    out->dist_kernel_ms = ctx->dist_ms;
    out->dist_kernel_launches = ctx->dist_launches;
    out->exact_reruns = ctx->exact_reruns;
    out->translate_kernel_ms = ctx->translate_ms;
    out->translate_kernel_launches = ctx->translate_launches;
    out->taxonomy_ms = ctx->tax_ms;
    out->reads_events = ctx->reads_events;
    out->reads_replay_ms = ctx->reads_replay_ms;
    out->reads_peak_device_bytes = ctx->reads_peak_bytes;
    out->unit_stages = ctx->unit_stages;
    out->unit_peak_device_bytes = ctx->unit_peak_bytes;
    if (reset) {
        ctx->kernel_launches = ctx->scan_launches = ctx->dist_launches = ctx->exact_reruns = ctx->translate_launches = 0;
        ctx->scan_ms = ctx->dist_ms = ctx->translate_ms = ctx->tax_ms = 0;
        ctx->reads_events = 0;
        ctx->unit_stages = 0;
        ctx->reads_replay_ms = 0;
    }
    return MASHGPU_OK;
}
