// screen.cu -- hot path 3: streaming containment screen (C-ABI: mashgpu_screen_*).
//
// Replaces hashSequence (reference CommandScreen.cpp:484-599) and the reduce that follows it
// (CommandScreen.cpp:288-355, 409-455, 463-482, 601-615).  The reference keeps a robin_hood map
// hash -> atomic<uint32_t> (:93-114); here it is an open-addressing table of the distinct reference hashes in
// HBM with a parallel uint32 counter array.  Each fed chunk runs the same scan kernel as sketching in
// SCAN_SCREEN mode: k-mer hashes <= the largest reference hash probe the table and bump the counter on a hit,
// and the chunk's bottom-s candidates are merged into the running bottom-s of the whole mixture (the
// reference merges per-thread MinHashHeaps the same way, :288-302; bottom-s of a union is order independent).
//
// Protein sketches switch the job to the translated screen (:120, 516-530): every fed chunk is first translated in six
// frames by translate.cu into a peptide stream (stops and invalid codons as 0 bytes) and the byte scan kernel runs over
// that stream.  The result does not depend on how the reads are cut into chunks (DESIGN.md 4.1), so chunk joining, the
// two-buffer pipeline and the exact re-run work unchanged.  Other non-nucleotide alphabets (-z) are screened as byte
// k-mers, untranslated (:541).
#include <algorithm>
#include <cmath>
#include <cstring>
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_merge_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include <chrono>
#include <vector>
#include <algorithm>
#include "common.cuh"
#include "scan.cuh"
#include "pack.h"
#include "sketch_core.cuh"
#include "binom.cuh"
#include "screen_view.cuh"

namespace mashgpu {

constexpr int SCR_THREADS = 256;
constexpr uint32_t SCREEN_MAX_REF_HASHES = 1u << 15;      // per reference sketch: the reduce sorts its depths in 128 KB of shared memory

// valid hashes of all reference sketches -> dense list (order irrelevant: sorted next)
__global__ void screen_gather_kernel(const uint64_t *hashes, uint64_t stride, const uint32_t *n_hashes, uint64_t n_rows, int use64,
                                     uint64_t *out, unsigned long long *out_n, uint32_t *err)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_rows * stride) return;
    const uint64_t row = t / stride, i = t % stride;
    if (i >= n_hashes[row]) return;
    const uint64_t key = hashes[t];
    if (key == EMPTY_KEY) { atomicOr(err, 1u); return; }   // 2^64-1 cannot be a table key (probability 2^-64 per hash)
    // a 32-bit job's k-mers hash below 2^32: a larger key is another sketch's hash, and it would index the bitmap (built from
    // the top bits of a 32-bit value) far past its end
    if (!use64 && (key >> 32)) { atomicOr(err, 2u); return; }
    out[atomicAdd(out_n, 1ull)] = key;
}

// distinct keys (ascending) -> open-addressing table; slot_idx[slot] = index of the key in the sorted list, so that the
// counter array (indexed by key index) has the same layout on every rank however the insertion races resolve
__global__ void screen_insert_kernel(const uint64_t *distinct, uint64_t n_distinct, uint64_t *keys, uint32_t *slot_idx, uint32_t log2cap)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_distinct) return;
    const uint64_t key = distinct[t];
    const uint32_t mask = (1u << log2cap) - 1;
    uint32_t slot = slot_hash(key, log2cap);
    for (;;) {
        unsigned long long prev = atomicCAS((unsigned long long *)&keys[slot], (unsigned long long)EMPTY_KEY, (unsigned long long)key);
        if (prev == EMPTY_KEY) { slot_idx[slot] = (uint32_t)t; return; }
        slot = (slot + 1) & mask;
    }
}

// presence bitmap over the distinct reference hashes, indexed by the top bits of the value (scan.cuh, screen_probe_lanes)
__global__ void screen_bitmap_kernel(const uint64_t *distinct, uint64_t n_distinct, uint32_t shift, uint32_t *bitmap)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n_distinct) return;
    const uint64_t b = distinct[t] >> shift;
    atomicOr(&bitmap[b >> 5], 1u << (b & 31));
}

// {number of hashes, largest hash} of the running mixture list -> two words the host reads back with one copy
__global__ void screen_mix_top_kernel(const uint64_t *mix, const uint32_t *mix_n, uint64_t *out)
{
    const uint32_t n = *mix_n;
    out[0] = n;
    out[1] = n ? mix[n - 1] : 0;
}

// merge ascending distinct lists -> ascending distinct, truncated to s, in `mix`: the running mixture (a) with n_lists more
// lists (list i = lists[i * stride ...], list_n[i] entries; 1 list = a fed chunk, G lists = the ranks' mixtures).
// Single CTA, bitonic sort of the concatenation in shared memory ((n_lists + 1) * s <= 2^14 entries).
__global__ void __launch_bounds__(SCR_THREADS) merge_bottom_s_kernel(uint64_t *mix, uint32_t *mix_n, const uint64_t *lists, const uint32_t *list_n,
                                                                     uint32_t n_lists, uint64_t stride, uint32_t s)
{
    extern __shared__ uint64_t sk[];
    __shared__ uint32_t s_off[66];
    if (threadIdx.x == 0) {
        uint32_t o = min(*mix_n, s);
        s_off[0] = o;
        for (uint32_t i = 0; i < n_lists; i++) { o += min(list_n[i], s); s_off[i + 1] = o; }
    }
    __syncthreads();
    const uint32_t na = s_off[0], n = s_off[n_lists];
    uint32_t N = 2;
    while (N < n) N <<= 1;
    for (uint32_t i = threadIdx.x; i < N; i += SCR_THREADS) {
        uint64_t v = EMPTY_KEY;
        if (i < na) v = mix[i];
        else if (i < n) {
            uint32_t l = 0;
            while (i >= s_off[l + 1]) l++;
            v = lists[(uint64_t)l * stride + (i - s_off[l])];
        }
        sk[i] = v;
    }
    __syncthreads();
    for (uint32_t size = 2; size <= N; size <<= 1)
        for (uint32_t stride2 = size >> 1; stride2 > 0; stride2 >>= 1) {
            for (uint32_t t = threadIdx.x; t < N / 2; t += SCR_THREADS) {
                uint32_t lo = 2 * t - (t & (stride2 - 1)), hi = lo + stride2;
                bool up = (lo & size) == 0;
                uint64_t a = sk[lo], b = sk[hi];
                if ((a > b) == up) { sk[lo] = b; sk[hi] = a; }
            }
            __syncthreads();
        }
    // unique + truncate: rank of each first occurrence = number of distinct predecessors (serial scan by one thread is fine: n <= 2^14)
    if (threadIdx.x == 0) {
        uint32_t m = 0;
        for (uint32_t i = 0; i < n && m < s; i++)
            if (i == 0 || sk[i] != sk[i - 1]) mix[m++] = sk[i];
        *mix_n = m;
    }
}

// identity and p-value of a sketch of n hashes with `shared` of them seen; the dense and the sparse reduce both call this, so
// their values are the same bits
__device__ __forceinline__ void screen_estimates(uint32_t shared, uint32_t n, uint64_t set_size, int kmer_size, double kmer_space,
                                                 double *identity_out, double *pvalue_out)
{
    double identity;                                                             // estimateIdentity, :463-482
    if (shared == n) identity = 1.;
    else if (shared == 0) identity = 0.;
    else identity = pow((double)shared / (double)n, 1. / kmer_size);
    *identity_out = identity;
    // pValueWithin, :601-615
    *pvalue_out = shared == 0 ? 1.0 : binomial_upper_tail(shared, (double)set_size / kmer_space, n);
}

// One CTA per reference sketch: shared count, sorted depths -> median, identity, p-value.
__global__ void __launch_bounds__(SCR_THREADS) screen_reduce_kernel(
    const uint64_t *hashes, uint64_t stride, const uint32_t *n_hashes, const uint64_t *keys, const uint32_t *slot_idx, const uint32_t *cnt, uint32_t log2cap,
    uint64_t set_size, int kmer_size, double kmer_space,
    uint64_t *shared_out, uint64_t *median_out, double *identity_out, double *pvalue_out,
    const uint32_t *best, const uint32_t *prio)     // -w: count a hash only for the sketch that won it (best[key] == prio[r])
{
    extern __shared__ uint32_t depths[];
    __shared__ uint32_t n_s;
    const uint64_t r = blockIdx.x;
    const uint32_t n = n_hashes[r];
    if (threadIdx.x == 0) n_s = 0;
    __syncthreads();
    const uint32_t mask = (1u << log2cap) - 1;
    for (uint32_t i = threadIdx.x; i < n; i += SCR_THREADS) {
        const uint64_t key = hashes[r * stride + i];
        uint32_t slot = slot_hash(key, log2cap), c = 0;
        for (;;) {
            uint64_t k = keys[slot];
            if (k == key) {
                const uint32_t d = slot_idx[slot];
                c = cnt[d];
                if (best && best[d] != prio[r]) c = 0;        // reallocated to another sketch (CommandScreen.cpp:366-404)
                break;
            }
            if (k == EMPTY_KEY) break;
            slot = (slot + 1) & mask;
        }
        if (c >= 1) depths[atomicAdd(&n_s, 1u)] = c;        // minCov == 1 (CommandScreen.cpp:152, 333-337)
    }
    __syncthreads();
    const uint32_t shared = n_s;
    uint32_t N = 2;
    while (N < shared) N <<= 1;
    for (uint32_t i = shared + threadIdx.x; i < N; i += SCR_THREADS) depths[i] = 0xFFFFFFFFu;
    __syncthreads();
    for (uint32_t size = 2; size <= N; size <<= 1)
        for (uint32_t st = size >> 1; st > 0; st >>= 1) {
            for (uint32_t t = threadIdx.x; t < N / 2; t += SCR_THREADS) {
                uint32_t lo = 2 * t - (t & (st - 1)), hi = lo + st;
                bool up = (lo & size) == 0;
                uint32_t a = depths[lo], b = depths[hi];
                if ((a > b) == up) { depths[lo] = b; depths[hi] = a; }
            }
            __syncthreads();
        }
    if (threadIdx.x == 0) {
        shared_out[r] = shared;
        median_out[r] = shared > 0 ? depths[shared / 2] : 0;                      // :436
        screen_estimates(shared, n, set_size, kmer_size, kmer_space, &identity_out[r], &pvalue_out[r]);
    }
}

// `-w`, CommandScreen.cpp:375-404: every reference hash seen in the mixture goes to the containing sketch with the best
// (identity estimate, genome length) -- prio[r] is the rank of sketch r in that order (0 = best), so the winner of a
// hash is the minimum prio over the sketches that hold it.
__global__ void __launch_bounds__(SCR_THREADS) screen_winner_kernel(
    const uint64_t *hashes, uint64_t stride, const uint32_t *n_hashes, const uint64_t *keys, const uint32_t *slot_idx, const uint32_t *cnt,
    uint32_t log2cap, const uint32_t *prio, uint32_t *best)
{
    const uint64_t r = blockIdx.x;
    const uint32_t n = n_hashes[r];
    const uint32_t mask = (1u << log2cap) - 1;
    const uint32_t pr = prio[r];
    for (uint32_t i = threadIdx.x; i < n; i += SCR_THREADS) {
        const uint64_t key = hashes[r * stride + i];
        uint32_t slot = slot_hash(key, log2cap);
        for (;;) {
            uint64_t k = keys[slot];
            if (k == key) {
                const uint32_t d = slot_idx[slot];
                if (cnt[d] >= 1) atomicMin(&best[d], pr);
                break;
            }
            if (k == EMPTY_KEY) break;
            slot = (slot + 1) & mask;
        }
    }
}

}  // namespace mashgpu

#include "screen_hits.cuh"

using namespace mashgpu;

struct mashgpu_screen_job {
    mashgpu_ctx *ctx = nullptr;
    mashgpu_sketch_params params{};
    uint64_t n_ref = 0, stride = 0;
    const uint64_t *ref_hashes = nullptr; const uint32_t *ref_n = nullptr;   // device
    DevBuf<uint64_t> own_hashes; DevBuf<uint32_t> own_n;
    DevBuf<uint64_t> keys; DevBuf<uint32_t> slot_idx, cnt;      // table slots; counters indexed by distinct-key index
    uint64_t n_distinct = 0;
    uint32_t log2cap = 4;
    uint64_t hmax = 0;
    DevBuf<uint64_t> mix, chunk_hashes; DevBuf<uint32_t> mix_n, chunk_n;
    uint32_t h_mix_n = 0; uint64_t h_mix_top = 0;
    DevBuf<uint32_t> bitmap; uint32_t bitmap_shift = 0;      // value-indexed presence bitmap (built when the table is large)
    // host-chunk pipeline: two device staging buffers; the kernels of chunk i run while chunk i+1 crosses PCIe
    DevBuf<uint8_t> stage[2];
    PinnedBuf<uint64_t> h_pack[2];       // packed host feed: codes, then the invalid mask, of the chunk being uploaded from this slot
    int host_pack = -1;                  // -1 not decided yet, 0 ASCII copies, 1 host 2-bit packer (screen_feed_host)
    int pack_threads = 1;
    cudaEvent_t copied[2] = {nullptr, nullptr};
    int next_buf = 0;
    SketchTicket ticket;
    bool pending = false;            // a chunk's kernels are in flight (ticket + mixture read-back not yet collected)
    DevBuf<uint64_t> d_mix_top; PinnedBuf<uint64_t> h_mix_top2;      // {n, top} of the mixture after the chunk in flight
    PinnedBuf<uint8_t> acc; uint64_t acc_len = 0;                    // small host chunks are joined here before they are fed
    ~mashgpu_screen_job()
    {
        for (int b = 0; b < 2; b++) if (copied[b]) cudaEventDestroy(copied[b]);
        for (int b = 0; b < 2; b++) if (hit_ev[b]) cudaEventDestroy(hit_ev[b]);
    }
    bool winner = false;     // -w
    std::vector<uint64_t> h_len;      // Reference::length per sketch (tie break of -w), zeros when the caller gave none
    std::vector<uint32_t> h_n;        // hashes per sketch
    uint32_t max_n = 0;               // largest of them (<= SCREEN_MAX_REF_HASHES): sizes the reduce's shared array
    // translated screen (protein sketches): each chunk is translated in six frames into pep[slot] and the peptide stream is
    // scanned; a slot's buffer stays untouched until its chunk is collected (the exact re-run reads it again)
    bool translate = false;
    DevBuf<uint8_t> pep[2];
    // sparse finish (screen_hits.cuh): the inverted index distinct hash -> sketches, built at the first finish_hits, and scratch
    // sized then for a sample that hits every pair
    bool index_built = false;
    uint64_t n_pairs = 0;
    DevBuf<uint32_t> seg_start, seg_ref;                 // index: seg_ref[seg_start[d] .. seg_start[d + 1]) = sketches holding d
    DevBuf<uint32_t> hit_d, long_list, best;             // per hit (n_distinct)
    DevBuf<uint32_t> ref_cnt, ref_start, rows_ref, order, prio;      // per sketch (n_ref + 1)
    DevBuf<uint32_t> depths;                             // per pair
    DevBuf<uint32_t> hit_n;                              // {hits, long segments, rows}
    DevBuf<uint64_t> d_len, out_shared, out_median;
    DevBuf<double> out_ident, out_pv;
    DevBuf<uint8_t> hit_tmp; size_t hit_tmp_bytes = 0;
    PinnedBuf<uint32_t> h_hit;                           // read-backs: n_hit, rows, pairs
    cudaEvent_t hit_ev[2] = {nullptr, nullptr};
    double index_ms = 0, finish_ms = 0;
    uint64_t last_hits = 0, last_pairs = 0;
    bool hits_valid = false;         // hit_d[0 .. last_hits) lists every nonzero counter (no feed since the last finish_hits)
};

namespace {

// The reference switches `mash screen` to translated mode exactly when the sketch alphabet is alphabetProtein
// (CommandScreen.cpp:120); setAlphabetFromString sorts the letters, so this is equality of the letter sets.
bool is_protein_alphabet(const mashgpu_sketch_params *p)
{
    static const char prot[] = "ACDEFGHIKLMNPQRSTVWY";
    uint8_t want[256] = {0};
    for (const char *c = prot; *c; c++) want[(unsigned char)*c] = 1;
    for (int i = 0; i < 256; i++)
        if ((p->alphabet[i] != 0) != (want[i] != 0)) return false;
    return true;
}

}  // namespace

extern "C" int mashgpu_screen_open(mashgpu_ctx *ctx, const mashgpu_sketch_params *params, const mashgpu_sketch_set *refs,
                                   mashgpu_screen_job **job_out)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    MG_TRY(validate_sketch_params(ctx, params));
    if (!refs || !job_out) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    if (refs->n && (!refs->hashes || !refs->n_hashes)) return fail(ctx, MASHGPU_ERR_INVALID, "reference set has NULL arrays");
    if (params->sketch_size > (1u << 13)) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "screen supports sketch_size <= 8192");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->stream;
    mashgpu_screen_job *job = new mashgpu_screen_job();
    job->ctx = ctx; job->params = *params; job->n_ref = refs->n; job->stride = refs->stride;
    // protein sketch: translated screen; any other non-nucleotide alphabet (-z): byte k-mers, untranslated (CommandScreen.cpp:541).
    // Both take ASCII copies: the 2-bit packer only carries {A,C,G,T} and cannot tell 'U' (a base on the reverse strand) from 'N'
    job->translate = is_protein_alphabet(params);
    if (!is_dna_alphabet(params)) job->host_pack = 0;
    auto bail = [&](int rc) { delete job; return rc; };
    // the row lengths first: the kernels below trust them (gather, reduce and winner read n_hashes[r] entries of row r)
    job->h_n.assign(refs->n, 0); job->h_len.assign(refs->n, 0);
    if (refs->n) {
        if (refs->on_device) {
            cudaError_t e = cudaMemcpy(job->h_n.data(), refs->n_hashes, refs->n * 4, cudaMemcpyDeviceToHost);
            if (e == cudaSuccess && refs->length) e = cudaMemcpy(job->h_len.data(), refs->length, refs->n * 8, cudaMemcpyDeviceToHost);
            if (e != cudaSuccess) return bail(fail(ctx, MASHGPU_ERR_CUDA, "reading the reference set's n_hashes failed: %s", cudaGetErrorString(e)));
        } else {
            memcpy(job->h_n.data(), refs->n_hashes, refs->n * 4);
            if (refs->length) memcpy(job->h_len.data(), refs->length, refs->n * 8);
        }
    }
    for (uint32_t v : job->h_n) job->max_n = std::max(job->max_n, v);
    if (job->max_n > refs->stride)
        return bail(fail(ctx, MASHGPU_ERR_INVALID, "a reference sketch holds %u hashes in rows of %llu", job->max_n, (unsigned long long)refs->stride));
    if (job->max_n > SCREEN_MAX_REF_HASHES)
        return bail(fail(ctx, MASHGPU_ERR_UNSUPPORTED, "reference sketches larger than %u hashes", SCREEN_MAX_REF_HASHES));
    const uint64_t total = refs->n * refs->stride;
    if (refs->on_device) { job->ref_hashes = refs->hashes; job->ref_n = refs->n_hashes; }
    else {
        if (job->own_hashes.alloc(total) != cudaSuccess || job->own_n.alloc(refs->n) != cudaSuccess) return bail(fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (reference sketches)"));
        if (total) cudaMemcpyAsync(job->own_hashes.p, refs->hashes, total * 8, cudaMemcpyHostToDevice, st);
        if (refs->n) cudaMemcpyAsync(job->own_n.p, refs->n_hashes, refs->n * 4, cudaMemcpyHostToDevice, st);
        job->ref_hashes = job->own_hashes.p; job->ref_n = job->own_n.p;
    }
    job->log2cap = std::max(4u, ceil_log2(2 * total + 2));
    if (job->log2cap > 31) return bail(fail(ctx, MASHGPU_ERR_UNSUPPORTED, "reference table too large"));
    const uint64_t cap = 1ull << job->log2cap;
    const uint32_t s = params->sketch_size;
    DevBuf<unsigned long long> d_count; DevBuf<uint32_t> d_err;
    DevBuf<uint64_t> gathered, sorted, distinct; DevBuf<uint8_t> tmp; DevBuf<uint64_t> d_nsel;
    if (job->keys.alloc(cap) != cudaSuccess || job->slot_idx.alloc(cap) != cudaSuccess || job->mix.alloc(s) != cudaSuccess || job->chunk_hashes.alloc(s) != cudaSuccess ||
        job->mix_n.alloc(1) != cudaSuccess || job->chunk_n.alloc(1) != cudaSuccess || d_count.alloc(1) != cudaSuccess || d_err.alloc(1) != cudaSuccess ||
        job->d_mix_top.alloc(2) != cudaSuccess || job->h_mix_top2.alloc(2) != cudaSuccess ||
        gathered.alloc(total) != cudaSuccess || sorted.alloc(total) != cudaSuccess || distinct.alloc(total) != cudaSuccess || d_nsel.alloc(1) != cudaSuccess)
        return bail(fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (screen table of %llu slots)", (unsigned long long)cap));
    cudaMemsetAsync(job->keys.p, 0xFF, cap * 8, st);
    cudaMemsetAsync(job->mix_n.p, 0, 4, st);
    cudaMemsetAsync(d_count.p, 0, 8, st);
    cudaMemsetAsync(d_err.p, 0, 4, st);
    unsigned long long n_valid = 0; uint32_t err = 0; uint64_t n_distinct = 0; unsigned long long hmax = 0;
    if (total) {
        screen_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(job->ref_hashes, refs->stride, job->ref_n, refs->n, params->use64,
                                                                                 gathered.p, d_count.p, d_err.p);
        cudaMemcpyAsync(&n_valid, d_count.p, 8, cudaMemcpyDeviceToHost, st);
        cudaMemcpyAsync(&err, d_err.p, 4, cudaMemcpyDeviceToHost, st);
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return bail(fail(ctx, MASHGPU_ERR_CUDA, "screen table build failed: %s", cudaGetErrorString(e)));
        if (err & 1) return bail(fail(ctx, MASHGPU_ERR_UNSUPPORTED, "reference sketch contains the hash value 2^64-1"));
        if (err & 2) return bail(fail(ctx, MASHGPU_ERR_INVALID, "reference hash >= 2^32 in a 32-bit sketch (k-mer space <= 2^32)"));
        if (n_valid >= 0x7FFFFFFFull) return bail(fail(ctx, MASHGPU_ERR_UNSUPPORTED, "more than 2^31 reference hashes"));
        if (n_valid) {
            size_t tb1 = 0, tb2 = 0;
            cub::DeviceRadixSort::SortKeys(nullptr, tb1, gathered.p, sorted.p, (int)n_valid, 0, 64, st);
            cub::DeviceSelect::Unique(nullptr, tb2, sorted.p, distinct.p, d_nsel.p, (int)n_valid, st);
            if (tmp.alloc(std::max(tb1, tb2)) != cudaSuccess) return bail(fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sort scratch)"));
            cub::DeviceRadixSort::SortKeys(tmp.p, tb1, gathered.p, sorted.p, (int)n_valid, 0, 64, st);
            cub::DeviceSelect::Unique(tmp.p, tb2, sorted.p, distinct.p, d_nsel.p, (int)n_valid, st);
            cudaMemcpyAsync(&n_distinct, d_nsel.p, 8, cudaMemcpyDeviceToHost, st);
            e = cudaStreamSynchronize(st);
            if (e != cudaSuccess) return bail(fail(ctx, MASHGPU_ERR_CUDA, "screen table sort failed: %s", cudaGetErrorString(e)));
            screen_insert_kernel<<<(unsigned)((n_distinct + 255) / 256), 256, 0, st>>>(distinct.p, n_distinct, job->keys.p, job->slot_idx.p, job->log2cap);
            cudaMemcpyAsync(&hmax, distinct.p + (n_distinct - 1), 8, cudaMemcpyDeviceToHost, st);     // ascending: the last one is the largest
            ctx->kernel_launches += 12;
            // value-indexed bitmap, ~4 bits per key, 2^20 .. 2^27 bits (16 MB: a third of the H100's 50 MB L2, which it shares
            // with the read stream and the table probes).
            // Reference hashes crowd the low end of the range (a sketch of a genome of length L reaches up to ~2^64 s/L): that
            // region is all ones, while the long sparse tail contributed by small genomes is rejected here without a table probe.
            const char *env_bm = getenv("MASHGPU_SCREEN_BITMAP");
            if (!(env_bm && env_bm[0] == '0')) {
                const uint32_t bits_log2 = std::min(27u, std::max(20u, ceil_log2(4 * n_distinct)));
                job->bitmap_shift = (params->use64 ? 64u : 32u) - bits_log2;
                if (job->bitmap.alloc((size_t)1 << (bits_log2 - 5)) != cudaSuccess) return bail(fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (screen bitmap)"));
                cudaMemsetAsync(job->bitmap.p, 0, (size_t)4 << (bits_log2 - 5), st);
                screen_bitmap_kernel<<<(unsigned)((n_distinct + 255) / 256), 256, 0, st>>>(distinct.p, n_distinct, job->bitmap_shift, job->bitmap.p);
                ctx->kernel_launches++;
            }
        }
    }
    job->n_distinct = n_distinct;
    if (job->cnt.alloc(n_distinct) != cudaSuccess) return bail(fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (hit counters)"));
    cudaMemsetAsync(job->cnt.p, 0, std::max<uint64_t>(1, n_distinct) * 4, st);
    {
        cudaError_t e = cudaStreamSynchronize(st);
        if (e != cudaSuccess) return bail(fail(ctx, MASHGPU_ERR_CUDA, "screen table build failed: %s", cudaGetErrorString(e)));
    }
    job->hmax = hmax;
    if (!ctx->attr_merge) {   // per context: function attributes are per device
        cudaFuncSetAttribute(merge_bottom_s_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 128 * 1024);
        ctx->attr_merge = true;
    }
    *job_out = job;
    return MASHGPU_OK;
}

namespace {

constexpr uint64_t SCREEN_SMALL_CHUNK = 4ull << 20;     // host chunks below this are joined before they are fed ...
constexpr uint64_t SCREEN_FLUSH_BYTES = 32ull << 20;    // ... until this much has accumulated (the reference feeds 1 MiB HashInputs)

// kernels of one chunk: scan (+ table probe) -> chunk bottom-s -> merge into the running mixture -> {n, top} read-back.  No sync.
// Translated jobs first turn the chunk into its six-frame peptide stream in pep[slot] and scan that instead.
int screen_enqueue(mashgpu_screen_job *job, int slot, const void *d_chunk, uint64_t len, const uint64_t *d_codes = nullptr, const uint32_t *d_inval = nullptr,
                   cudaEvent_t data_ready = nullptr)
{
    mashgpu_ctx *ctx = job->ctx;
    cudaStream_t st = ctx->stream;
    const uint32_t s = job->params.sketch_size;
    if (job->translate) {
        const uint64_t pep_len = translated_length(len);
        if (job->pep[slot].reserve(pep_len + 16) != cudaSuccess)
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (peptide stream of %llu B)", (unsigned long long)pep_len);
        if (data_ready) { MG_CUDA(ctx, cudaStreamWaitEvent(st, data_ready, 0)); data_ready = nullptr; }
        MG_TRY(translate_enqueue(ctx, d_chunk, len, job->params.preserve_case, job->pep[slot].p, st));
        d_chunk = job->pep[slot].p;
        len = pep_len;
    }
    uint64_t unit_start[2] = {0, len};
    SketchStream S;
    S.d_stream = d_chunk; S.d_codes = d_codes; S.d_inval = d_inval; S.unit_start = unit_start; S.n_units = 1; S.data_ready = data_ready;
    if (job->h_mix_n == s) { S.t_cap = true; S.t_cap_value = job->h_mix_top; }   // nothing above the running s-th smallest can matter
    ScreenProbe probe{job->keys.p, job->slot_idx.p, job->cnt.p, job->log2cap, job->hmax, job->bitmap.p, job->bitmap_shift};
    job->hits_valid = false;
    MG_CUDA(ctx, cudaMemsetAsync(job->chunk_n.p, 0, 4, st));      // an overflowing chunk leaves an empty list until its exact re-run
    MG_TRY(sketch_stream_enqueue(ctx, &job->params, S, job->chunk_hashes.p, nullptr, job->chunk_n.p, st, &probe, job->ticket));
    uint32_t N = 2;
    while (N < 2 * s) N <<= 1;
    // merged optimistically: if the chunk turns out to need an exact re-run, the list merged here is a subset of the chunk's real
    // hashes (harmless in a bottom-s of the union) and the exact list is merged again after the re-run (screen_collect)
    merge_bottom_s_kernel<<<1, SCR_THREADS, (size_t)N * 8, st>>>(job->mix.p, job->mix_n.p, job->chunk_hashes.p, job->chunk_n.p, 1, s, s);
    screen_mix_top_kernel<<<1, 1, 0, st>>>(job->mix.p, job->mix_n.p, job->d_mix_top.p);
    ctx->kernel_launches += 2;
    MG_CUDA(ctx, cudaGetLastError());
    MG_CUDA(ctx, cudaMemcpyAsync(job->h_mix_top2.p, job->d_mix_top.p, 16, cudaMemcpyDeviceToHost, st));
    job->pending = true;
    return MASHGPU_OK;
}

// waits for the chunk in flight, re-runs it exactly if it was flagged, and takes over the mixture's {n, top}
int screen_collect(mashgpu_screen_job *job)
{
    if (!job->pending) return MASHGPU_OK;
    job->pending = false;
    mashgpu_ctx *ctx = job->ctx;
    cudaStream_t st = ctx->stream;
    const uint64_t reruns_before = ctx->exact_reruns;
    MG_TRY(sketch_stream_finalize(ctx, job->ticket));              // synchronises the stream
    if (ctx->exact_reruns != reruns_before) {
        const uint32_t s = job->params.sketch_size;
        uint32_t N = 2;
        while (N < 2 * s) N <<= 1;
        merge_bottom_s_kernel<<<1, SCR_THREADS, (size_t)N * 8, st>>>(job->mix.p, job->mix_n.p, job->chunk_hashes.p, job->chunk_n.p, 1, s, s);
        screen_mix_top_kernel<<<1, 1, 0, st>>>(job->mix.p, job->mix_n.p, job->d_mix_top.p);
        ctx->kernel_launches += 2;
        MG_CUDA(ctx, cudaGetLastError());
        MG_CUDA(ctx, cudaMemcpyAsync(job->h_mix_top2.p, job->d_mix_top.p, 16, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
    }
    job->h_mix_n = (uint32_t)job->h_mix_top2.p[0];
    job->h_mix_top = job->h_mix_top2.p[1];
    return MASHGPU_OK;
}

// host chunk -> staging buffer (async) while the previous chunk's kernels finish; returns once the caller's buffer is free
// Host chunk, packed on the way: this thread's pool turns the chunk into 2-bit codes + an invalid bit mask in pinned memory
// (pack.cpp; 0.375 B per base cross PCIe instead of 1), the upload and the kernels are enqueued behind it and the call returns --
// the caller's buffer is free as soon as it has been read by the packer.  Packing chunk i+1 overlaps the upload of chunk i and
// the kernels of chunk i-1.
int screen_feed_host_packed(mashgpu_screen_job *job, const void *chunk, uint64_t len)
{
    mashgpu_ctx *ctx = job->ctx;
    const int b = job->next_buf;
    job->next_buf ^= 1;
    // the scan kernel reads whole tiles of the packed stream plus a halo without looking at the stream length: everything from the
    // end of the chunk to the end of the tile-padded allocation must read as invalid (sketch.cu pads its packed waves the same way)
    const uint64_t groups = ((len + SCAN_TILE - 1) / SCAN_TILE) * (SCAN_TILE / 32) + 64;
    const uint64_t bytes = groups * 12;
    static const bool trace = getenv("MASHGPU_TRACE_FEED") != nullptr;
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = now();
    if (!job->copied[b]) MG_CUDA(ctx, cudaEventCreateWithFlags(&job->copied[b], cudaEventDisableTiming));
    else MG_CUDA(ctx, cudaEventSynchronize(job->copied[b]));        // the upload that last used this slot's pinned buffer (two chunks ago)
    const double t1 = now();
    uint8_t *stage;
    uint64_t *h_codes;
    if (!ctx->scr_stage_owner || ctx->scr_stage_owner == job) {     // the context's buffers (kept across jobs)
        ctx->scr_stage_owner = job;
        stage = ctx->scr_stage[b].get<uint8_t>(ctx->scr_stage[b].bytes < bytes ? bytes + (bytes >> 2) : bytes);
        if (!stage) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (chunk of %llu B)", (unsigned long long)len);
        h_codes = ctx->scr_pinned[b].get<uint64_t>((bytes + 7) / 8);
        if (!h_codes) return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory (packed chunk of %llu B)", (unsigned long long)len);
    } else {
        if (job->stage[b].n < bytes && job->stage[b].alloc(bytes + (bytes >> 2)) != cudaSuccess)
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (chunk of %llu B)", (unsigned long long)len);
        stage = job->stage[b].p;
        if (job->h_pack[b].n * 8 < bytes && job->h_pack[b].alloc((bytes + (bytes >> 2)) / 8 + 1) != cudaSuccess)
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory (packed chunk of %llu B)", (unsigned long long)len);
        h_codes = job->h_pack[b].p;
    }
    uint32_t *h_inval = reinterpret_cast<uint32_t *>(h_codes + groups);
    const uint64_t real = (len + 31) / 32;
    pack_chunk_mask(static_cast<const uint8_t *>(chunk), len, job->params.preserve_case, job->pack_threads, h_codes, h_inval);
    for (uint64_t g = real; g < groups; g++) { h_codes[g] = 0; h_inval[g] = 0xFFFFFFFFu; }
    uint64_t *d_codes = reinterpret_cast<uint64_t *>(stage);
    uint32_t *d_inval = reinterpret_cast<uint32_t *>(d_codes + groups);
    const double t2 = now();
    MG_CUDA(ctx, cudaMemcpyAsync(d_codes, h_codes, groups * 12, cudaMemcpyHostToDevice, ctx->copy_stream));
    MG_CUDA(ctx, cudaEventRecord(job->copied[b], ctx->copy_stream));
    MG_TRY(screen_collect(job));                                    // the chunk before this one: its kernels overlapped the packing
    const double t3 = now();
    const int rc = screen_enqueue(job, b, nullptr, len, d_codes, d_inval, job->copied[b]);      // the scan kernel waits for the upload, this thread does not
    if (trace) fprintf(stderr, "[mashgpu] screen packed feed %llu B: wait %.2f, alloc + pack %.2f (%d threads), collect previous %.2f, enqueue %.2f ms\n",
                       (unsigned long long)len, t1 - t0, t2 - t1, job->pack_threads, t3 - t2, now() - t3);
    return rc;
}

int screen_feed_host(mashgpu_screen_job *job, const void *chunk, uint64_t len)
{
    mashgpu_ctx *ctx = job->ctx;
    if (job->host_pack < 0) {
        // MASHGPU_SCREEN_HOST_PACK = 1 selects the packer.  It pays off when the process may run enough threads to out-pack the
        // PCIe-ASCII rate (6-8 GB/s per thread); with a 16-thread quota it did not, so ASCII copies stay the default
        // (bench.py reports both as screen.e2e)
        job->pack_threads = host_pack_threads();
        const char *e = getenv("MASHGPU_SCREEN_HOST_PACK");
        job->host_pack = e ? (atoi(e) != 0) : 0;
    }
    if (job->host_pack) return screen_feed_host_packed(job, chunk, len);
    const int b = job->next_buf;
    job->next_buf ^= 1;
    const uint64_t padded = ((len + 15) / 16) * 16;
    uint8_t *stage;
    if (!ctx->scr_stage_owner || ctx->scr_stage_owner == job) {     // the context's staging pair (kept across jobs)
        ctx->scr_stage_owner = job;
        // (buffer b was last read by the chunk before the one in flight, which has been collected: it may move)
        stage = ctx->scr_stage[b].get<uint8_t>(ctx->scr_stage[b].bytes < padded ? padded + (padded >> 2) : padded);
        if (!stage) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (chunk of %llu B)", (unsigned long long)len);
    } else {
        if (job->stage[b].n < padded && job->stage[b].alloc(padded + (padded >> 2)) != cudaSuccess)
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (chunk of %llu B)", (unsigned long long)len);
        stage = job->stage[b].p;
    }
    if (!job->copied[b]) MG_CUDA(ctx, cudaEventCreateWithFlags(&job->copied[b], cudaEventDisableTiming));
    MG_CUDA(ctx, cudaMemcpyAsync(stage, chunk, len, cudaMemcpyHostToDevice, ctx->copy_stream));
    MG_CUDA(ctx, cudaEventRecord(job->copied[b], ctx->copy_stream));
    MG_TRY(screen_collect(job));                                    // the chunk before this one: its kernels overlapped the copy above
    MG_CUDA(ctx, cudaEventSynchronize(job->copied[b]));
    return screen_enqueue(job, b, stage, len);
}

int screen_flush_acc(mashgpu_screen_job *job)
{
    if (job->acc_len == 0) return MASHGPU_OK;
    const uint64_t n = job->acc_len;
    job->acc_len = 0;
    return screen_feed_host(job, job->acc.p, n);
}

}  // namespace

extern "C" int mashgpu_screen_feed_dev(mashgpu_screen_job *job, const void *d_chunk, uint64_t len)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (len == 0) return MASHGPU_OK;
    if (!d_chunk) return fail(ctx, MASHGPU_ERR_INVALID, "chunk is NULL");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_TRY(screen_collect(job));
    if (!job->translate && ((uintptr_t)d_chunk & 15)) {
        // the scan kernels load their stream as aligned 16-byte vectors: a chunk at any other address is scanned from an aligned
        // copy (a translated job reads the chunk with byte loads and scans its own peptide buffer)
        if (job->stage[0].reserve((len + 15) / 16 * 16) != cudaSuccess)
            return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (chunk of %llu B)", (unsigned long long)len);
        MG_CUDA(ctx, cudaMemcpyAsync(job->stage[0].p, d_chunk, len, cudaMemcpyDeviceToDevice, ctx->stream));
        d_chunk = job->stage[0].p;
    }
    MG_TRY(screen_enqueue(job, 0, d_chunk, len));
    return screen_collect(job);          // the caller's device buffer is free again when this returns
}

extern "C" int mashgpu_screen_feed(mashgpu_screen_job *job, const char *chunk, uint64_t len)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (len == 0) return MASHGPU_OK;
    if (!chunk) return fail(ctx, MASHGPU_ERR_INVALID, "chunk is NULL");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    if (len >= SCREEN_SMALL_CHUNK) return screen_feed_host(job, chunk, len);
    // small chunk: join it to the pending ones with a separator byte (any byte outside the alphabet separates reads,
    // CommandScreen.cpp:254-258 uses '*'); one kernel pass per ~32 MiB instead of one per 1 MiB HashInput
    if (job->acc.n < SCREEN_FLUSH_BYTES + SCREEN_SMALL_CHUNK + 16 && job->acc.alloc(SCREEN_FLUSH_BYTES + SCREEN_SMALL_CHUNK + 16) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of pinned host memory (chunk accumulator)");
    memcpy(job->acc.p + job->acc_len, chunk, len);
    job->acc.p[job->acc_len + len] = 0;
    job->acc_len += len + 1;
    if (job->acc_len >= SCREEN_FLUSH_BYTES) return screen_flush_acc(job);
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_finish(mashgpu_screen_job *job, uint64_t *shared, uint64_t *median, double *identity,
                                     double *pvalue, uint64_t *set_size_out, uint64_t *mixture_hashes, uint32_t *mixture_n)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    const bool trace = getenv("MASHGPU_TRACE") != nullptr;
    auto now = [] { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count(); };
    const double t0 = now();
    MG_TRY(screen_flush_acc(job));
    MG_TRY(screen_collect(job));
    const double t1 = now();
    cudaStream_t st = ctx->stream;
    const int k = job->params.kmer_size;
    int asize = 0;
    for (int i = 0; i < 256; i++) asize += job->params.alphabet[i] != 0;
    const double kmer_space = std::pow((double)asize, (double)k);
    // estimateSetSize (reference MinHashHeap.h:45), cast to uint64_t as in CommandScreen.cpp:322
    uint64_t set_size = 0;
    if (job->h_mix_n)
        set_size = (uint64_t)(std::pow(2.0, job->params.use64 ? 64.0 : 32.0) * (double)job->h_mix_n / (double)job->h_mix_top);
    if (set_size_out) *set_size_out = set_size;
    if (mixture_n) *mixture_n = job->h_mix_n;
    if (mixture_hashes && job->h_mix_n)
        MG_CUDA(ctx, cudaMemcpyAsync(mixture_hashes, job->mix.p, job->h_mix_n * 8ull, cudaMemcpyDeviceToHost, st));
    const uint64_t n = job->n_ref;
    if (n) {
        struct { uint64_t *p; } d_shared, d_median; struct { double *p; } d_ident, d_p;        // four n-element arrays in the context's scratch
        uint64_t *outs = ctx->scr_out.get<uint64_t>(4 * n);
        if (!outs) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (screen outputs)");
        d_shared.p = outs; d_median.p = outs + n;
        d_ident.p = reinterpret_cast<double *>(outs + 2 * n); d_p.p = reinterpret_cast<double *>(outs + 3 * n);
        uint32_t N = 2;
        while (N < job->max_n) N <<= 1;         // <= SCREEN_MAX_REF_HASHES (refused at open): 128 KB
        if ((size_t)N * 4 > 48 * 1024)
            MG_CUDA(ctx, cudaFuncSetAttribute(screen_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)N * 4)));
        screen_reduce_kernel<<<(unsigned)n, SCR_THREADS, (size_t)N * 4, st>>>(job->ref_hashes, job->stride, job->ref_n, job->keys.p, job->slot_idx.p, job->cnt.p, job->log2cap,
                                                                            set_size, k, kmer_space, d_shared.p, d_median.p, d_ident.p, d_p.p, nullptr, nullptr);
        ctx->kernel_launches++;
        MG_CUDA(ctx, cudaGetLastError());
        if (job->winner) {
            // scores[] = estimateIdentity of the plain shared counts (CommandScreen.cpp:361-364), evaluated with the host libm as
            // the reference does; order the sketches by (score desc, length desc, index asc) and let every seen hash go to the
            // best sketch that holds it; then rebuild shared / depths from the assignments (:366-404) with the same reduce kernel
            std::vector<uint64_t> h_shared(n);
            MG_CUDA(ctx, cudaMemcpyAsync(h_shared.data(), d_shared.p, n * 8, cudaMemcpyDeviceToHost, st));
            MG_CUDA(ctx, cudaStreamSynchronize(st));
            std::vector<double> score(n);
            for (uint64_t i = 0; i < n; i++) {
                const uint64_t common = h_shared[i], denom = job->h_n[i];
                score[i] = common == denom ? 1. : (common == 0 ? 0. : std::pow((double)common / (double)denom, 1. / k));
            }
            std::vector<uint32_t> order(n), prio(n);
            for (uint64_t i = 0; i < n; i++) order[i] = (uint32_t)i;
            std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) {
                if (score[a] != score[b]) return score[a] > score[b];
                if (job->h_len[a] != job->h_len[b]) return job->h_len[a] > job->h_len[b];
                return a < b;
            });
            for (uint64_t i = 0; i < n; i++) prio[order[i]] = (uint32_t)i;
            DevBuf<uint32_t> d_prio, d_best;
            if (d_prio.alloc(n) != cudaSuccess || d_best.alloc(job->n_distinct) != cudaSuccess) return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (winner table)");
            MG_CUDA(ctx, cudaMemcpyAsync(d_prio.p, prio.data(), n * 4, cudaMemcpyHostToDevice, st));
            MG_CUDA(ctx, cudaMemsetAsync(d_best.p, 0xFF, std::max<uint64_t>(1, job->n_distinct) * 4, st));
            screen_winner_kernel<<<(unsigned)n, SCR_THREADS, 0, st>>>(job->ref_hashes, job->stride, job->ref_n, job->keys.p, job->slot_idx.p, job->cnt.p, job->log2cap, d_prio.p, d_best.p);
            screen_reduce_kernel<<<(unsigned)n, SCR_THREADS, (size_t)N * 4, st>>>(job->ref_hashes, job->stride, job->ref_n, job->keys.p, job->slot_idx.p, job->cnt.p, job->log2cap,
                                                                                set_size, k, kmer_space, d_shared.p, d_median.p, d_ident.p, d_p.p, d_best.p, d_prio.p);
            ctx->kernel_launches += 2;
            MG_CUDA(ctx, cudaGetLastError());
            MG_CUDA(ctx, cudaStreamSynchronize(st));      // d_prio / d_best go out of scope below
        }
        const double t2 = now();
        if (trace) { cudaStreamSynchronize(st); fprintf(stderr, "[mashgpu] screen_finish: collect %.2f ms, alloc+reduce %.2f ms (reduce done %.2f)\n", t1 - t0, t2 - t1, now() - t1); }
        if (shared) MG_CUDA(ctx, cudaMemcpyAsync(shared, d_shared.p, n * 8, cudaMemcpyDeviceToHost, st));
        if (median) MG_CUDA(ctx, cudaMemcpyAsync(median, d_median.p, n * 8, cudaMemcpyDeviceToHost, st));
        if (identity) MG_CUDA(ctx, cudaMemcpyAsync(identity, d_ident.p, n * 8, cudaMemcpyDeviceToHost, st));
        if (pvalue) MG_CUDA(ctx, cudaMemcpyAsync(pvalue, d_p.p, n * 8, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
        if (trace) fprintf(stderr, "[mashgpu] screen_finish: total %.2f ms\n", now() - t0);
    } else {
        MG_CUDA(ctx, cudaStreamSynchronize(st));
    }
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_set_winner(mashgpu_screen_job *job, int on)
{
    if (!job) return MASHGPU_ERR_INVALID;
    job->winner = on != 0;
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_counters(mashgpu_screen_job *job, uint32_t **d_counters, uint64_t *n_slots)
{
    if (!job || !d_counters || !n_slots) return MASHGPU_ERR_INVALID;
    cudaSetDevice(job->ctx->device);
    MG_TRY(screen_flush_acc(job));
    MG_TRY(screen_collect(job));
    cudaStreamSynchronize(job->ctx->stream);
    job->hits_valid = false;         // the caller may write the counters
    *d_counters = job->cnt.p;
    *n_slots = job->n_distinct;
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_merge_mixture(mashgpu_screen_job *job, const uint64_t *hashes, uint32_t n)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    const uint32_t s = job->params.sketch_size;
    if (n > s) return fail(ctx, MASHGPU_ERR_INVALID, "a mixture list holds at most sketch_size hashes");
    if (n == 0) return MASHGPU_OK;
    if (!hashes) return fail(ctx, MASHGPU_ERR_INVALID, "hashes is NULL");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_TRY(screen_flush_acc(job));
    MG_TRY(screen_collect(job));
    cudaStream_t st = ctx->stream;
    MG_CUDA(ctx, cudaMemcpyAsync(job->chunk_hashes.p, hashes, n * 8ull, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(job->chunk_n.p, &n, 4, cudaMemcpyHostToDevice, st));
    uint32_t N = 2;
    while (N < 2 * s) N <<= 1;
    merge_bottom_s_kernel<<<1, SCR_THREADS, (size_t)N * 8, st>>>(job->mix.p, job->mix_n.p, job->chunk_hashes.p, job->chunk_n.p, 1, s, s);
    ctx->kernel_launches++;
    MG_CUDA(ctx, cudaGetLastError());
    MG_CUDA(ctx, cudaMemcpyAsync(&job->h_mix_n, job->mix_n.p, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    if (job->h_mix_n) {
        MG_CUDA(ctx, cudaMemcpyAsync(&job->h_mix_top, job->mix.p + (job->h_mix_n - 1), 8, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
    }
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_mixture_dev(mashgpu_screen_job *job, uint64_t **d_mix, uint32_t **d_mix_n)
{
    if (!job || !d_mix || !d_mix_n) return MASHGPU_ERR_INVALID;
    cudaSetDevice(job->ctx->device);
    MG_TRY(screen_flush_acc(job));
    MG_TRY(screen_collect(job));
    cudaStreamSynchronize(job->ctx->stream);
    *d_mix = job->mix.p;
    *d_mix_n = job->mix_n.p;
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_merge_mixtures_dev(mashgpu_screen_job *job, const uint64_t *d_hashes, const uint32_t *d_n, uint32_t n_lists, uint64_t stride)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    const uint32_t s = job->params.sketch_size;
    if (n_lists == 0) return MASHGPU_OK;
    if (!d_hashes || !d_n) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    if (stride < s) return fail(ctx, MASHGPU_ERR_INVALID, "stride must be at least sketch_size");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_TRY(screen_flush_acc(job));
    MG_TRY(screen_collect(job));
    cudaStream_t st = ctx->stream;
    // as many lists per launch as the shared-memory sort holds (2^14 keys): all of them for 8 ranks x s = 1000
    const uint32_t per_launch = std::max<uint32_t>(1, std::min<uint32_t>(64, (1u << 14) / s > 1 ? (1u << 14) / s - 1 : 1));
    for (uint32_t l0 = 0; l0 < n_lists; l0 += per_launch) {
        const uint32_t nl = std::min(per_launch, n_lists - l0);
        uint32_t N = 2;
        while (N < (nl + 1) * s) N <<= 1;
        merge_bottom_s_kernel<<<1, SCR_THREADS, (size_t)N * 8, st>>>(job->mix.p, job->mix_n.p, d_hashes + (uint64_t)l0 * stride, d_n + l0, nl, stride, s);
        ctx->kernel_launches++;
        MG_CUDA(ctx, cudaGetLastError());
    }
    MG_CUDA(ctx, cudaMemcpyAsync(&job->h_mix_n, job->mix_n.p, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    if (job->h_mix_n) {
        MG_CUDA(ctx, cudaMemcpyAsync(&job->h_mix_top, job->mix.p + (job->h_mix_n - 1), 8, cudaMemcpyDeviceToHost, st));
        MG_CUDA(ctx, cudaStreamSynchronize(st));
    }
    return MASHGPU_OK;
}

int mashgpu::screen_table_view(mashgpu_screen_job *job, ScreenTableView *v)
{
    mashgpu_ctx *ctx = job->ctx;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_TRY(screen_flush_acc(job));
    MG_TRY(screen_collect(job));
    MG_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
    *v = ScreenTableView{ctx, job->n_ref, job->stride, job->ref_hashes, job->ref_n, job->h_n.data(), job->keys.p, job->slot_idx.p, job->cnt.p,
                         job->log2cap, job->n_distinct};
    return MASHGPU_OK;
}

namespace {

// The inverted index and the per-sample scratch of the sparse finish, once per job.  The counting sort runs over every (sketch,
// hash) pair; seg_start is 32-bit, so a job of 2^32 or more pairs is refused.  Device memory: 4 B per pair for the index and 4 B per
// pair for the depth runs, 4 B per distinct hash for seg_start plus 12 B for the hit lists, about 60 B per sketch, and 8 B per pair
// of build temporaries.
int screen_build_index(mashgpu_screen_job *job)
{
    mashgpu_ctx *ctx = job->ctx;
    cudaStream_t st = ctx->stream;
    const uint64_t n = job->n_ref, nd = job->n_distinct;
    uint64_t n_pairs = 0;
    std::vector<uint64_t> off(n);
    std::vector<uint32_t> iota(n);
    for (uint64_t r = 0; r < n; r++) { off[r] = n_pairs; iota[r] = (uint32_t)r; n_pairs += job->h_n[r]; }
    if (n_pairs >= 0xFFFFFFFFull || n >= 0x7FFFFFFFull)
        return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "sparse screen finish: 2^32 or more (sketch, hash) pairs");
    size_t tb[4] = {0, 0, 0, 0};
    thrust::counting_iterator<uint32_t> it(0);
    MG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(nullptr, tb[0], job->seg_start.p, job->seg_start.p, (int)std::max<uint64_t>(nd, n) + 1, st));
    MG_CUDA(ctx, cub::DeviceSelect::If(nullptr, tb[1], it, job->hit_d.p, job->hit_n.p, (int)nd, HitPred{job->cnt.p}, st));
    MG_CUDA(ctx, cub::DeviceSelect::If(nullptr, tb[2], it, job->rows_ref.p, job->hit_n.p, (int)n, RefPred{job->ref_cnt.p}, st));
    MG_CUDA(ctx, cub::DeviceMergeSort::SortKeys(nullptr, tb[3], job->order.p, (int)n, WinnerOrder{nullptr, nullptr, nullptr}, st));
    job->hit_tmp_bytes = *std::max_element(tb, tb + 4);
    DevBuf<uint32_t> d_iota, pair_d, seg_n; DevBuf<uint64_t> d_off;
    if (job->seg_start.alloc(nd + 1) != cudaSuccess || job->seg_ref.alloc(n_pairs) != cudaSuccess || job->hit_d.alloc(nd) != cudaSuccess ||
        job->long_list.alloc(nd) != cudaSuccess || job->best.alloc(nd) != cudaSuccess || job->ref_cnt.alloc(n + 1) != cudaSuccess ||
        job->ref_start.alloc(n + 1) != cudaSuccess || job->rows_ref.alloc(n) != cudaSuccess || job->order.alloc(n) != cudaSuccess ||
        job->prio.alloc(n) != cudaSuccess || job->depths.alloc(n_pairs) != cudaSuccess || job->hit_n.alloc(3) != cudaSuccess ||
        job->d_len.alloc(n) != cudaSuccess || job->out_shared.alloc(n) != cudaSuccess || job->out_median.alloc(n) != cudaSuccess ||
        job->out_ident.alloc(n) != cudaSuccess || job->out_pv.alloc(n) != cudaSuccess || job->hit_tmp.alloc(job->hit_tmp_bytes) != cudaSuccess ||
        job->h_hit.alloc(4) != cudaSuccess ||
        d_iota.alloc(n) != cudaSuccess || d_off.alloc(n) != cudaSuccess || pair_d.alloc(n_pairs) != cudaSuccess || seg_n.alloc(nd + 1) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (sparse screen index: %llu pairs, %llu hashes)", (unsigned long long)n_pairs, (unsigned long long)nd);
    for (int b = 0; b < 2; b++)
        if (!job->hit_ev[b]) MG_CUDA(ctx, cudaEventCreate(&job->hit_ev[b]));
    MG_CUDA(ctx, cudaEventRecord(job->hit_ev[0], st));
    MG_CUDA(ctx, cudaMemcpyAsync(d_iota.p, iota.data(), n * 4, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(d_off.p, off.data(), n * 8, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemcpyAsync(job->d_len.p, job->h_len.data(), n * 8, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemsetAsync(seg_n.p, 0, (nd + 1) * 4, st));
    MG_CUDA(ctx, cudaMemsetAsync(job->ref_cnt.p, 0, (n + 1) * 4, st));       // kept at zero from here on (screen_hits.cuh)
    if (n_pairs) {
        tax_pairs_kernel<<<(unsigned)n, SCR_THREADS, 0, st>>>(job->ref_hashes, job->stride, job->ref_n, d_iota.p, d_off.p, job->keys.p, job->slot_idx.p,
                                                            job->log2cap, pair_d.p, seg_n.p);
        MG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(job->hit_tmp.p, job->hit_tmp_bytes, seg_n.p, job->seg_start.p, (int)(nd + 1), st));
        tax_scatter_kernel<<<(unsigned)n, SCR_THREADS, 0, st>>>(job->ref_n, d_iota.p, d_iota.p, d_off.p, pair_d.p, job->seg_start.p, seg_n.p, job->seg_ref.p);
        ctx->kernel_launches += 3;
    }
    MG_CUDA(ctx, cudaGetLastError());
    MG_CUDA(ctx, cudaEventRecord(job->hit_ev[1], st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));                 // the temporaries go out of scope
    float ms = 0;
    MG_CUDA(ctx, cudaEventElapsedTime(&ms, job->hit_ev[0], job->hit_ev[1]));
    job->index_ms = ms;
    job->n_pairs = n_pairs;
    job->index_built = true;
    return MASHGPU_OK;
}

// ExclusiveSum of ref_cnt[0 .. n] -> ref_start, then the sketches with ref_cnt > 0 -> rows_ref (ascending) and their number and the
// pair total to the host
int screen_hits_runs(mashgpu_screen_job *job, uint32_t *n_rows, uint32_t *n_pairs)
{
    mashgpu_ctx *ctx = job->ctx;
    cudaStream_t st = ctx->stream;
    const uint64_t n = job->n_ref;
    thrust::counting_iterator<uint32_t> it(0);
    size_t tb = job->hit_tmp_bytes;
    MG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(job->hit_tmp.p, tb, job->ref_cnt.p, job->ref_start.p, (int)(n + 1), st));
    tb = job->hit_tmp_bytes;
    MG_CUDA(ctx, cub::DeviceSelect::If(job->hit_tmp.p, tb, it, job->rows_ref.p, job->hit_n.p + 2, (int)n, RefPred{job->ref_cnt.p}, st));
    MG_CUDA(ctx, cudaMemcpyAsync(job->h_hit.p, job->hit_n.p + 2, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaMemcpyAsync(job->h_hit.p + 1, job->ref_start.p + n, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    *n_rows = job->h_hit.p[0];
    *n_pairs = job->h_hit.p[1];
    return MASHGPU_OK;
}

}  // namespace

extern "C" int mashgpu_screen_finish_hits(mashgpu_screen_job *job, uint32_t *ref, uint64_t *shared, uint64_t *median, double *identity,
                                          double *pvalue, uint64_t *n_rows, uint64_t *set_size_out)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    if (!n_rows) return fail(ctx, MASHGPU_ERR_INVALID, "n_rows is NULL");
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_TRY(screen_flush_acc(job));
    MG_TRY(screen_collect(job));
    cudaStream_t st = ctx->stream;
    const int k = job->params.kmer_size;
    int asize = 0;
    for (int i = 0; i < 256; i++) asize += job->params.alphabet[i] != 0;
    const double kmer_space = std::pow((double)asize, (double)k);
    uint64_t set_size = 0;             // as mashgpu_screen_finish
    if (job->h_mix_n)
        set_size = (uint64_t)(std::pow(2.0, job->params.use64 ? 64.0 : 32.0) * (double)job->h_mix_n / (double)job->h_mix_top);
    if (set_size_out) *set_size_out = set_size;
    *n_rows = 0;
    job->last_hits = job->last_pairs = 0;
    job->finish_ms = 0;
    const uint64_t n = job->n_ref, nd = job->n_distinct;
    if (n == 0 || nd == 0) { job->hits_valid = true; return MASHGPU_OK; }
    if (!job->index_built) MG_TRY(screen_build_index(job));
    MG_CUDA(ctx, cudaEventRecord(job->hit_ev[0], st));
    // hits: every distinct index with cnt >= 1, ascending
    thrust::counting_iterator<uint32_t> it(0);
    size_t tb = job->hit_tmp_bytes;
    MG_CUDA(ctx, cub::DeviceSelect::If(job->hit_tmp.p, tb, it, job->hit_d.p, job->hit_n.p, (int)nd, HitPred{job->cnt.p}, st));
    MG_CUDA(ctx, cudaMemsetAsync(job->hit_n.p + 1, 0, 4, st));
    MG_CUDA(ctx, cudaMemcpyAsync(job->h_hit.p, job->hit_n.p, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    const uint32_t n_hit = job->h_hit.p[0];
    uint32_t rows = 0, pairs = 0;
    if (n_hit) {
        const unsigned blocks = (n_hit + SCR_THREADS - 1) / SCR_THREADS, long_blocks = (unsigned)ctx->sm_count * 8;
        const uint32_t *hit_d = job->hit_d.p, *seg_start = job->seg_start.p, *seg_ref = job->seg_ref.p, *cnt = job->cnt.p;
        uint32_t *ref_cnt = job->ref_cnt.p, *ref_start = job->ref_start.p, *depths = job->depths.p, *long_list = job->long_list.p, *n_long = job->hit_n.p + 1;
        // per-sketch counts over the hit segments (queueing the long ones), runs, and the depths scattered into them
        hits_pairs_kernel<false><<<blocks, SCR_THREADS, 0, st>>>(hit_d, n_hit, seg_start, seg_ref, cnt, ref_start, ref_cnt, depths, long_list, n_long, true);
        hits_pairs_long_kernel<false><<<long_blocks, SCR_THREADS, 0, st>>>(hit_d, seg_start, seg_ref, cnt, ref_start, ref_cnt, depths, long_list, n_long);
        ctx->kernel_launches += 2;
        MG_CUDA(ctx, cudaGetLastError());
        MG_TRY(screen_hits_runs(job, &rows, &pairs));
        job->last_pairs = pairs;
        if (job->winner) {
            // rank the hit sketches by their plain counts, give each hit to the best-ranked sketch holding it, and count again
            MG_CUDA(ctx, cudaMemcpyAsync(job->order.p, job->rows_ref.p, rows * 4ull, cudaMemcpyDeviceToDevice, st));
            tb = job->hit_tmp_bytes;
            MG_CUDA(ctx, cub::DeviceMergeSort::SortKeys(job->hit_tmp.p, tb, job->order.p, (int)rows, WinnerOrder{ref_start, job->ref_n, job->d_len.p}, st));
            hits_rank_kernel<<<(rows + SCR_THREADS - 1) / SCR_THREADS, SCR_THREADS, 0, st>>>(job->order.p, rows, job->prio.p);
            hits_best_kernel<<<blocks, SCR_THREADS, 0, st>>>(hit_d, n_hit, seg_start, seg_ref, job->prio.p, job->best.p);
            hits_best_long_kernel<<<long_blocks, SCR_THREADS, 0, st>>>(hit_d, seg_start, seg_ref, job->prio.p, long_list, n_long, job->best.p);
            // the plain runs are not needed: their counters go back to 0, then the winners are counted
            clear_listed_kernel<<<(rows + SCR_THREADS - 1) / SCR_THREADS, SCR_THREADS, 0, st>>>(job->rows_ref.p, rows, ref_cnt);
            hits_winner_kernel<false><<<blocks, SCR_THREADS, 0, st>>>(hit_d, n_hit, job->best.p, job->order.p, cnt, ref_start, ref_cnt, depths);
            ctx->kernel_launches += 6;
            MG_CUDA(ctx, cudaGetLastError());
            uint32_t winner_pairs = 0;
            MG_TRY(screen_hits_runs(job, &rows, &winner_pairs));
            hits_winner_kernel<true><<<blocks, SCR_THREADS, 0, st>>>(hit_d, n_hit, job->best.p, job->order.p, cnt, ref_start, ref_cnt, depths);
        } else {
            hits_pairs_kernel<true><<<blocks, SCR_THREADS, 0, st>>>(hit_d, n_hit, seg_start, seg_ref, cnt, ref_start, ref_cnt, depths, long_list, n_long, false);
            hits_pairs_long_kernel<true><<<long_blocks, SCR_THREADS, 0, st>>>(hit_d, seg_start, seg_ref, cnt, ref_start, ref_cnt, depths, long_list, n_long);
            ctx->kernel_launches++;
        }
        ctx->kernel_launches++;
        uint32_t N = 2;
        while (N < job->max_n) N <<= 1;         // <= SCREEN_MAX_REF_HASHES (refused at open): 128 KB
        if ((size_t)N * 4 > 48 * 1024)
            MG_CUDA(ctx, cudaFuncSetAttribute(hits_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)N * 4)));
        if (rows) {
            hits_reduce_kernel<<<rows, SCR_THREADS, (size_t)N * 4, st>>>(job->rows_ref.p, ref_start, depths, job->ref_n, set_size, k, kmer_space,
                                                                        job->out_shared.p, job->out_median.p, job->out_ident.p, job->out_pv.p);
            ctx->kernel_launches++;
        }
        MG_CUDA(ctx, cudaGetLastError());
    }
    MG_CUDA(ctx, cudaEventRecord(job->hit_ev[1], st));
    if (rows) {
        if (ref) MG_CUDA(ctx, cudaMemcpyAsync(ref, job->rows_ref.p, rows * 4ull, cudaMemcpyDeviceToHost, st));
        if (shared) MG_CUDA(ctx, cudaMemcpyAsync(shared, job->out_shared.p, rows * 8ull, cudaMemcpyDeviceToHost, st));
        if (median) MG_CUDA(ctx, cudaMemcpyAsync(median, job->out_median.p, rows * 8ull, cudaMemcpyDeviceToHost, st));
        if (identity) MG_CUDA(ctx, cudaMemcpyAsync(identity, job->out_ident.p, rows * 8ull, cudaMemcpyDeviceToHost, st));
        if (pvalue) MG_CUDA(ctx, cudaMemcpyAsync(pvalue, job->out_pv.p, rows * 8ull, cudaMemcpyDeviceToHost, st));
    }
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    float ms = 0;
    MG_CUDA(ctx, cudaEventElapsedTime(&ms, job->hit_ev[0], job->hit_ev[1]));
    job->finish_ms = ms;
    job->last_hits = n_hit;
    job->hits_valid = true;
    *n_rows = rows;
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_hits_stats(mashgpu_screen_job *job, uint64_t *hit_hashes, uint64_t *hit_pairs, double *index_ms, double *finish_ms)
{
    if (!job) return MASHGPU_ERR_INVALID;
    if (hit_hashes) *hit_hashes = job->last_hits;
    if (hit_pairs) *hit_pairs = job->last_pairs;
    if (index_ms) *index_ms = job->index_ms;
    if (finish_ms) *finish_ms = job->finish_ms;
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_reset(mashgpu_screen_job *job)
{
    if (!job) return MASHGPU_ERR_INVALID;
    mashgpu_ctx *ctx = job->ctx;
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    MG_TRY(screen_flush_acc(job));               // the joined small chunks belong to the sample being closed
    MG_TRY(screen_collect(job));
    cudaStream_t st = ctx->stream;
    if (job->hits_valid) {
        if (job->last_hits) {
            clear_listed_kernel<<<(unsigned)((job->last_hits + SCR_THREADS - 1) / SCR_THREADS), SCR_THREADS, 0, st>>>(job->hit_d.p, (uint32_t)job->last_hits, job->cnt.p);
            ctx->kernel_launches++;
            MG_CUDA(ctx, cudaGetLastError());
        }
    } else if (job->n_distinct) {
        MG_CUDA(ctx, cudaMemsetAsync(job->cnt.p, 0, job->n_distinct * 4, st));
    }
    MG_CUDA(ctx, cudaMemsetAsync(job->mix_n.p, 0, 4, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    job->h_mix_n = 0;
    job->h_mix_top = 0;
    job->hits_valid = false;
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_close(mashgpu_screen_job *job)
{
    if (!job) return MASHGPU_ERR_INVALID;
    cudaSetDevice(job->ctx->device);
    job->acc_len = 0;
    screen_collect(job);                 // never leave a chunk in flight behind
    cudaStreamSynchronize(job->ctx->stream);
    cudaStreamSynchronize(job->ctx->copy_stream);
    if (job->ctx->scr_stage_owner == job) job->ctx->scr_stage_owner = nullptr;     // the staging pair stays with the context for the next job
    delete job;
    return MASHGPU_OK;
}
