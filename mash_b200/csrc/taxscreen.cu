// taxscreen.cu -- `mash taxscreen` after the stream: lowest-common-ancestor (LCA) taxon of every distinct reference hash,
// per-taxon hash counts and their roll-up over the tree (C-ABI: mashgpu_taxonomy_*, mashgpu_screen_taxonomy).
//
// Replaces the reference's single-threaded pass over the hash table (CommandTaxScreen.cpp:415-471, with
// TaxDB::getLowestCommonAncestor, taxdb.hpp:158-190).  It runs on the screen job's table as the stream left it: the keys,
// slot_idx, the hit counters and the reference sketches, all already in device memory.
//
//   pairs    one CTA per reference sketch with a taxon code: every hash is looked up in the table (as screen_winner_kernel
//            does) and its distinct index d is written next to the pair's position; seg_n[d] counts the sketches holding d.
//   group    exclusive scan of seg_n -> seg_start; a second pass scatters each sketch's code into d's segment (a counting
//            sort by d; the order inside a segment is irrelevant because the fold below is commutative).
//   fold     the reference's fold of getLowestCommonAncestor over the sketches holding d (in hash-set order) equals the
//            order-free rule below (DESIGN.md 4.2; tests/test_taxscreen_model.py pins it to the reference's own fold):
//              no sketch -> taxon 0;  one sketch -> its code, known or not;
//              two or more -> 1 if any code is unknown, if the known taxa have no common ancestor, or if that ancestor is a
//                             root; otherwise the LCA.
//            Segments of up to TAX_SERIAL_MAX codes are folded by one thread, longer ones (hashes shared by thousands of
//            near-identical genomes) by a warp with shuffles.  The LCA walks parent[] by depth[]; nothing bounds the depth.
//   count    per taxon slot: hashes assigned (taxHashCount) and those seen in the reads (taxCount), warp-aggregated atomics.
//   roll-up  every taxonomy node that got hashes adds its two counts to itself and every ancestor (cladeCount,
//            cladeHashCount), once each.
//   compact  rows for the keys of the reference's `counts` map: every node with a nonzero clade hash count and every
//            other slot (unknown taxIDs, taxon 0 or 1 outside the taxonomy) that got hashes.
#include <algorithm>
#include <vector>
#include <cub/device/device_scan.cuh>
#include <cub/device/device_select.cuh>
#include <thrust/iterator/counting_iterator.h>

#include "common.cuh"
#include "scan.cuh"
#include "screen_view.cuh"

namespace mashgpu {

constexpr int TAX_THREADS = 256;
constexpr uint32_t TAX_EMPTY = 0xFFFFFFFFu;      // fold state: no known taxon yet
constexpr uint32_t TAX_DISJOINT = 0xFFFFFFFEu;   // fold state: known taxa under different LCA roots
constexpr uint32_t TAX_SERIAL_MAX = 8;           // longer segments go to the warp fold

// LCA of two fold states over the tree: depth[] counts the edges to the node's LCA root (depth 0), parent[] is only followed
// from nodes of depth > 0
__device__ __forceinline__ uint32_t tax_lca(uint32_t a, uint32_t b, const uint32_t *__restrict__ parent, const uint32_t *__restrict__ depth)
{
    if (a == TAX_EMPTY || a == b) return b;
    if (b == TAX_EMPTY) return a;
    if (a == TAX_DISJOINT || b == TAX_DISJOINT) return TAX_DISJOINT;
    uint32_t da = __ldg(&depth[a]), db = __ldg(&depth[b]);
    while (da > db) { a = __ldg(&parent[a]); da--; }
    while (db > da) { b = __ldg(&parent[b]); db--; }
    while (a != b) {
        if (da == 0) return TAX_DISJOINT;
        a = __ldg(&parent[a]); b = __ldg(&parent[b]); da--;
    }
    return a;
}

// result of a segment of two or more codes
__device__ __forceinline__ uint32_t tax_finish(uint32_t acc, bool unknown, const uint32_t *__restrict__ depth, uint32_t one_slot)
{
    if (unknown || acc >= TAX_DISJOINT || __ldg(&depth[acc]) == 0) return one_slot;
    return acc;
}

__device__ __forceinline__ uint32_t tax_find(const uint64_t *__restrict__ keys, const uint32_t *__restrict__ slot_idx, uint32_t log2cap, uint64_t key)
{
    const uint32_t mask = (1u << log2cap) - 1;
    uint32_t slot = slot_hash(key, log2cap);
    for (;;) {
        const uint64_t k = keys[slot];
        if (k == key) return slot_idx[slot];
        if (k == EMPTY_KEY) return 0xFFFFFFFFu;       // cannot happen: the table holds every reference hash
        slot = (slot + 1) & mask;
    }
}

// one CTA per coded sketch (refs[b]): d of every hash -> pair_d[pair_off[b] + i], seg_n[d]++
__global__ void __launch_bounds__(TAX_THREADS) tax_pairs_kernel(
    const uint64_t *__restrict__ hashes, uint64_t stride, const uint32_t *__restrict__ n_hashes, const uint32_t *__restrict__ refs,
    const uint64_t *__restrict__ pair_off, const uint64_t *__restrict__ keys, const uint32_t *__restrict__ slot_idx, uint32_t log2cap,
    uint32_t *__restrict__ pair_d, uint32_t *__restrict__ seg_n)
{
    const uint64_t r = refs[blockIdx.x];
    const uint32_t n = n_hashes[r];
    const uint64_t off = pair_off[blockIdx.x];
    for (uint32_t i = threadIdx.x; i < n; i += TAX_THREADS) {
        const uint32_t d = tax_find(keys, slot_idx, log2cap, hashes[r * stride + i]);
        pair_d[off + i] = d;
        atomicAdd(&seg_n[d], 1u);
    }
}

// same grid: the sketch's code goes to a free place of d's segment (seg_n counts down to 0)
__global__ void __launch_bounds__(TAX_THREADS) tax_scatter_kernel(
    const uint32_t *__restrict__ n_hashes, const uint32_t *__restrict__ refs, const uint32_t *__restrict__ ref_code,
    const uint64_t *__restrict__ pair_off, const uint32_t *__restrict__ pair_d, const uint32_t *__restrict__ seg_start,
    uint32_t *__restrict__ seg_n, uint32_t *__restrict__ seg_code)
{
    const uint32_t r = refs[blockIdx.x];
    const uint32_t n = n_hashes[r], code = ref_code[r];
    const uint64_t off = pair_off[blockIdx.x];
    for (uint32_t i = threadIdx.x; i < n; i += TAX_THREADS) {
        const uint32_t d = pair_d[off + i];
        seg_code[seg_start[d] + atomicSub(&seg_n[d], 1u) - 1] = code;
    }
}

// one thread per distinct hash; segments longer than TAX_SERIAL_MAX are queued for tax_fold_long_kernel
__global__ void __launch_bounds__(TAX_THREADS) tax_fold_kernel(
    const uint32_t *__restrict__ seg_start, const uint32_t *__restrict__ seg_code, uint64_t n_distinct, uint32_t n_nodes,
    const uint32_t *__restrict__ parent, const uint32_t *__restrict__ depth, uint32_t none_slot, uint32_t one_slot,
    uint32_t *__restrict__ out_slot, uint32_t *__restrict__ long_list, uint32_t *__restrict__ n_long, uint8_t *__restrict__ unknown_in_lca)
{
    const uint64_t d = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (d >= n_distinct) return;
    const uint32_t a = seg_start[d], n = seg_start[d + 1] - a;
    if (n > TAX_SERIAL_MAX) { long_list[atomicAdd(n_long, 1u)] = (uint32_t)d; return; }
    if (n <= 1) { out_slot[d] = n ? seg_code[a] : none_slot; return; }
    uint32_t acc = TAX_EMPTY;
    bool unknown = false;
    for (uint32_t j = 0; j < n; j++) {
        const uint32_t c = seg_code[a + j];
        if (c >= n_nodes) { unknown = true; unknown_in_lca[c - n_nodes] = 1; }
        else if (!unknown) acc = tax_lca(acc, c, parent, depth);
    }
    out_slot[d] = tax_finish(acc, unknown, depth, one_slot);
}

// one warp per queued segment: strided lane folds, then a shuffle tree of LCAs (the rule is associative and commutative)
__global__ void __launch_bounds__(TAX_THREADS) tax_fold_long_kernel(
    const uint32_t *__restrict__ seg_start, const uint32_t *__restrict__ seg_code, uint32_t n_nodes,
    const uint32_t *__restrict__ parent, const uint32_t *__restrict__ depth, uint32_t one_slot,
    const uint32_t *__restrict__ long_list, const uint32_t *__restrict__ n_long, uint32_t *__restrict__ out_slot, uint8_t *__restrict__ unknown_in_lca)
{
    const uint32_t lane = threadIdx.x & 31;
    const uint32_t n_warps = gridDim.x * (TAX_THREADS / 32);
    const uint32_t total = *n_long;
    for (uint32_t w = blockIdx.x * (TAX_THREADS / 32) + threadIdx.x / 32; w < total; w += n_warps) {
        const uint32_t d = long_list[w];
        const uint32_t a = seg_start[d], n = seg_start[d + 1] - a;
        uint32_t acc = TAX_EMPTY;
        bool unknown = false;
        for (uint32_t j = lane; j < n; j += 32) {
            const uint32_t c = seg_code[a + j];
            if (c >= n_nodes) { unknown = true; unknown_in_lca[c - n_nodes] = 1; }
            else acc = tax_lca(acc, c, parent, depth);
        }
        unknown = __any_sync(0xFFFFFFFFu, unknown);
        if (!unknown)
            for (int o = 16; o > 0; o >>= 1) acc = tax_lca(acc, __shfl_xor_sync(0xFFFFFFFFu, acc, o), parent, depth);
        if (lane == 0) out_slot[d] = tax_finish(acc, unknown, depth, one_slot);
    }
}

// per taxon slot: taxHashCount += 1 per hash, taxCount += 1 per hash seen at least once (minCov 1, CommandTaxScreen.cpp:227)
__global__ void __launch_bounds__(TAX_THREADS) tax_count_kernel(const uint32_t *__restrict__ out_slot, const uint32_t *__restrict__ cnt, uint64_t n_distinct,
                                                                unsigned long long *__restrict__ tax_hash, unsigned long long *__restrict__ tax_count)
{
    const uint64_t d = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    const bool active = d < n_distinct;
    const uint32_t slot = active ? out_slot[d] : 0xFFFFFFFFu;
    const uint32_t seen = __ballot_sync(0xFFFFFFFFu, active && cnt[d] >= 1);
    const uint32_t peers = __match_any_sync(0xFFFFFFFFu, slot);
    if (!active || (threadIdx.x & 31) != (uint32_t)(__ffs(peers) - 1)) return;
    atomicAdd(&tax_hash[slot], (unsigned long long)__popc(peers));
    const uint32_t c = __popc(peers & seen);
    if (c) atomicAdd(&tax_count[slot], (unsigned long long)c);
}

// one thread per taxonomy node: a node that got hashes adds its counts to itself and to every ancestor up to its root
__global__ void __launch_bounds__(TAX_THREADS) tax_rollup_kernel(const uint32_t *__restrict__ parent, uint32_t n_nodes,
                                                                 const unsigned long long *__restrict__ tax_hash, const unsigned long long *__restrict__ tax_count,
                                                                 unsigned long long *__restrict__ clade_hash, unsigned long long *__restrict__ clade_count)
{
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_nodes) return;
    const unsigned long long th = tax_hash[s], tc = tax_count[s];
    if (th == 0) return;
    for (uint32_t v = s;;) {
        atomicAdd(&clade_hash[v], th);
        if (tc) atomicAdd(&clade_count[v], tc);
        const uint32_t p = parent[v];
        if (p == v) break;
        v = p;
    }
}

// keys of the reference's counts map: nodes with clade hashes, other slots with hashes of their own
__global__ void tax_flag_kernel(uint32_t n_slots, uint32_t n_nodes, const unsigned long long *__restrict__ tax_hash,
                                const unsigned long long *__restrict__ clade_hash, uint8_t *__restrict__ flag)
{
    const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
    if (s >= n_slots) return;
    flag[s] = (s < n_nodes ? clade_hash[s] : tax_hash[s]) > 0;
}

__global__ void tax_gather_kernel(const uint32_t *__restrict__ sel, const uint32_t *__restrict__ n_sel, uint32_t n_nodes,
                                  const unsigned long long *__restrict__ tax_hash, const unsigned long long *__restrict__ tax_count,
                                  const unsigned long long *__restrict__ clade_hash, const unsigned long long *__restrict__ clade_count,
                                  mashgpu_tax_row *__restrict__ rows)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= *n_sel) return;
    const uint32_t s = sel[i];
    mashgpu_tax_row r;
    r.taxid = s;                         // the host replaces the slot by its taxID
    r.tax_count = tax_count[s];
    r.tax_hash_count = tax_hash[s];
    r.clade_count = s < n_nodes ? clade_count[s] : 0;
    r.clade_hash_count = s < n_nodes ? clade_hash[s] : 0;
    rows[i] = r;
}

}  // namespace mashgpu

using namespace mashgpu;

struct mashgpu_taxonomy {
    mashgpu_ctx *ctx = nullptr;
    uint32_t n_nodes = 0;
    std::vector<uint64_t> taxid;
    int64_t node_of[2] = {-1, -1};          // nodes with taxID 0 and 1
    DevBuf<uint32_t> parent, depth;
};

extern "C" int mashgpu_taxonomy_open(mashgpu_ctx *ctx, uint64_t n_nodes, const uint32_t *parent, const uint64_t *taxid, mashgpu_taxonomy **out)
{
    if (!ctx) return MASHGPU_ERR_INVALID;
    if (!out || (n_nodes && (!parent || !taxid))) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    if (n_nodes >= 0x7FFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "taxonomy of 2^31 or more nodes");
    for (uint64_t i = 0; i < n_nodes; i++)
        if (parent[i] >= n_nodes) return fail(ctx, MASHGPU_ERR_INVALID, "parent of node %llu out of range", (unsigned long long)i);
    // depth over the tree the LCA walks: a node is an LCA root when it is its own parent or has taxID 0 or 1 (the reference's
    // walks stop there, taxdb.hpp:176, 183); the roll-up follows parent[] through taxID 0 and 1 to the real root
    const uint32_t n = (uint32_t)n_nodes;
    std::vector<uint32_t> depth(n, 0xFFFFFFFFu), stack;
    std::vector<uint8_t> state(n, 0);            // cycle check on parent[]: 0 new, 1 on the current path, 2 done
    for (uint32_t i = 0; i < n; i++) {
        uint32_t v = i;
        while (state[v] == 0) { state[v] = 1; stack.push_back(v); if (parent[v] == v) break; v = parent[v]; }
        if (state[v] == 1 && parent[v] != v)
            return fail(ctx, MASHGPU_ERR_INVALID, "taxonomy has a parent cycle through taxID %llu", (unsigned long long)taxid[v]);
        for (uint32_t u : stack) state[u] = 2;
        stack.clear();
    }
    for (uint32_t i = 0; i < n; i++) {
        uint32_t v = i;
        while (depth[v] == 0xFFFFFFFFu && !(parent[v] == v || taxid[v] <= 1)) { stack.push_back(v); v = parent[v]; }
        if (depth[v] == 0xFFFFFFFFu) depth[v] = 0;
        uint32_t dd = depth[v];
        while (!stack.empty()) { depth[stack.back()] = ++dd; stack.pop_back(); }
    }
    MG_CUDA(ctx, cudaSetDevice(ctx->device));
    mashgpu_taxonomy *tax = new mashgpu_taxonomy();
    tax->ctx = ctx;
    tax->n_nodes = n;
    tax->taxid.assign(taxid, taxid + n);
    for (uint32_t i = 0; i < n; i++)
        if (taxid[i] <= 1 && tax->node_of[taxid[i]] < 0) tax->node_of[taxid[i]] = i;
    if (tax->parent.alloc(n) != cudaSuccess || tax->depth.alloc(n) != cudaSuccess) {
        delete tax;
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (taxonomy of %u nodes)", n);
    }
    cudaError_t e = cudaSuccess;
    if (n) {
        e = cudaMemcpy(tax->parent.p, parent, n * 4ull, cudaMemcpyHostToDevice);
        if (e == cudaSuccess) e = cudaMemcpy(tax->depth.p, depth.data(), n * 4ull, cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) { delete tax; return fail(ctx, MASHGPU_ERR_CUDA, "taxonomy upload failed: %s", cudaGetErrorString(e)); }
    *out = tax;
    return MASHGPU_OK;
}

extern "C" int mashgpu_taxonomy_close(mashgpu_taxonomy *tax)
{
    if (!tax) return MASHGPU_ERR_INVALID;
    cudaSetDevice(tax->ctx->device);
    delete tax;
    return MASHGPU_OK;
}

extern "C" int mashgpu_screen_taxonomy(mashgpu_screen_job *job, const mashgpu_taxonomy *tax, const uint32_t *ref_code,
                                       uint32_t n_unknown, const uint64_t *unknown_taxid,
                                       mashgpu_tax_row *rows, uint64_t capacity, uint64_t *n_rows,
                                       uint64_t *total_count, uint64_t *total_hash_count,
                                       uint64_t *hash_taxid, uint8_t *unknown_in_lca)
{
    if (!job || !tax) return MASHGPU_ERR_INVALID;
    ScreenTableView v;
    MG_TRY(screen_table_view(job, &v));
    mashgpu_ctx *ctx = v.ctx;
    if (tax->ctx != ctx) return fail(ctx, MASHGPU_ERR_INVALID, "taxonomy and screen job belong to different contexts");
    if (!n_rows || (v.n_ref && !ref_code) || (n_unknown && !unknown_taxid) || (capacity && !rows)) return fail(ctx, MASHGPU_ERR_INVALID, "NULL argument");
    const uint32_t n_nodes = tax->n_nodes;
    if ((uint64_t)n_nodes + n_unknown + 2 >= TAX_DISJOINT) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "too many taxon slots");
    // slots: [0, n_nodes) nodes, n_nodes + u unknown taxID u, then taxID 0 and taxID 1 when they are neither
    const uint32_t n_slots = n_nodes + n_unknown + 2;
    std::vector<uint64_t> slot_taxid(tax->taxid);
    slot_taxid.insert(slot_taxid.end(), unknown_taxid, unknown_taxid + n_unknown);
    slot_taxid.push_back(0); slot_taxid.push_back(1);
    uint32_t special[2] = {n_nodes + n_unknown, n_nodes + n_unknown + 1};
    for (int t = 0; t < 2; t++)
        if (tax->node_of[t] >= 0) special[t] = (uint32_t)tax->node_of[t];
    for (uint32_t u = 0; u < n_unknown; u++) {
        if (unknown_taxid[u] == 0) return fail(ctx, MASHGPU_ERR_INVALID, "taxID 0 cannot be an unknown taxon (it means none)");
        if (unknown_taxid[u] == 1 && tax->node_of[1] < 0) special[1] = n_nodes + u;
    }
    std::vector<uint32_t> refs;
    std::vector<uint64_t> off;
    uint64_t n_pairs = 0;
    for (uint64_t r = 0; r < v.n_ref; r++) {
        if (ref_code[r] == MASHGPU_TAX_NONE) continue;
        if (ref_code[r] >= n_nodes + n_unknown) return fail(ctx, MASHGPU_ERR_INVALID, "code of sketch %llu out of range", (unsigned long long)r);
        refs.push_back((uint32_t)r);
        off.push_back(n_pairs);
        n_pairs += v.h_ref_n[r];
    }
    if (n_pairs >= 0xFFFFFFFFull) return fail(ctx, MASHGPU_ERR_UNSUPPORTED, "2^32 or more (sketch, hash) pairs with a taxon");
    const uint64_t nd = v.n_distinct;
    cudaStream_t st = ctx->stream;
    DevBuf<uint32_t> d_refs, d_code, pair_d, seg_n, seg_start, seg_code, out_slot, long_list, n_long, sel, n_sel;
    DevBuf<uint64_t> d_off;
    DevBuf<unsigned long long> counts;       // tax_hash, tax_count, clade_hash, clade_count: n_slots each
    DevBuf<uint8_t> unk, flag, tmp;
    DevBuf<mashgpu_tax_row> d_rows;
    size_t tb_scan = 0, tb_sel = 0;
    thrust::counting_iterator<uint32_t> slots_it(0);
    cub::DeviceScan::ExclusiveSum(nullptr, tb_scan, seg_n.p, seg_start.p, (int)(nd + 1), st);
    cub::DeviceSelect::Flagged(nullptr, tb_sel, slots_it, flag.p, sel.p, n_sel.p, (int)n_slots, st);
    if (d_refs.alloc(refs.size()) != cudaSuccess || d_off.alloc(refs.size()) != cudaSuccess || d_code.alloc(v.n_ref) != cudaSuccess ||
        pair_d.alloc(n_pairs) != cudaSuccess || seg_code.alloc(n_pairs) != cudaSuccess || seg_n.alloc(nd + 1) != cudaSuccess ||
        seg_start.alloc(nd + 1) != cudaSuccess || out_slot.alloc(nd) != cudaSuccess || long_list.alloc(nd) != cudaSuccess ||
        n_long.alloc(1) != cudaSuccess || sel.alloc(n_slots) != cudaSuccess || n_sel.alloc(1) != cudaSuccess ||
        counts.alloc(4ull * n_slots) != cudaSuccess || unk.alloc(n_unknown) != cudaSuccess || flag.alloc(n_slots) != cudaSuccess ||
        tmp.alloc(std::max(tb_scan, tb_sel)) != cudaSuccess || d_rows.alloc(n_slots) != cudaSuccess)
        return fail(ctx, MASHGPU_ERR_NOMEM, "out of device memory (taxonomy step: %llu pairs, %llu hashes)", (unsigned long long)n_pairs, (unsigned long long)nd);
    unsigned long long *tax_hash = counts.p, *tax_count = counts.p + n_slots, *clade_hash = counts.p + 2ull * n_slots, *clade_count = counts.p + 3ull * n_slots;
    time_begin(ctx, ctx->tax_events, st);
    if (!refs.empty()) {
        MG_CUDA(ctx, cudaMemcpyAsync(d_refs.p, refs.data(), refs.size() * 4, cudaMemcpyHostToDevice, st));
        MG_CUDA(ctx, cudaMemcpyAsync(d_off.p, off.data(), off.size() * 8, cudaMemcpyHostToDevice, st));
    }
    if (v.n_ref) MG_CUDA(ctx, cudaMemcpyAsync(d_code.p, ref_code, v.n_ref * 4, cudaMemcpyHostToDevice, st));
    MG_CUDA(ctx, cudaMemsetAsync(seg_n.p, 0, (nd + 1) * 4, st));
    MG_CUDA(ctx, cudaMemsetAsync(n_long.p, 0, 4, st));
    MG_CUDA(ctx, cudaMemsetAsync(counts.p, 0, 4ull * n_slots * 8, st));
    if (n_unknown) MG_CUDA(ctx, cudaMemsetAsync(unk.p, 0, n_unknown, st));
    const uint32_t fold_blocks = (uint32_t)((nd + TAX_THREADS - 1) / TAX_THREADS);
    if (!refs.empty() && n_pairs) {
        tax_pairs_kernel<<<(unsigned)refs.size(), TAX_THREADS, 0, st>>>(v.ref_hashes, v.stride, v.ref_n, d_refs.p, d_off.p, v.keys, v.slot_idx, v.log2cap,
                                                                      pair_d.p, seg_n.p);
        ctx->kernel_launches++;
    }
    if (nd) {
        MG_CUDA(ctx, cub::DeviceScan::ExclusiveSum(tmp.p, tb_scan, seg_n.p, seg_start.p, (int)(nd + 1), st));
        if (!refs.empty() && n_pairs) {
            tax_scatter_kernel<<<(unsigned)refs.size(), TAX_THREADS, 0, st>>>(v.ref_n, d_refs.p, d_code.p, d_off.p, pair_d.p, seg_start.p, seg_n.p, seg_code.p);
            ctx->kernel_launches++;
        }
        tax_fold_kernel<<<fold_blocks, TAX_THREADS, 0, st>>>(seg_start.p, seg_code.p, nd, n_nodes, tax->parent.p, tax->depth.p, special[0], special[1],
                                                             out_slot.p, long_list.p, n_long.p, unk.p);
        tax_fold_long_kernel<<<(unsigned)ctx->sm_count * 8, TAX_THREADS, 0, st>>>(seg_start.p, seg_code.p, n_nodes, tax->parent.p, tax->depth.p, special[1],
                                                                                 long_list.p, n_long.p, out_slot.p, unk.p);
        tax_count_kernel<<<fold_blocks, TAX_THREADS, 0, st>>>(out_slot.p, v.cnt, nd, tax_hash, tax_count);
        ctx->kernel_launches += 4;
    }
    if (n_nodes) {
        tax_rollup_kernel<<<(n_nodes + TAX_THREADS - 1) / TAX_THREADS, TAX_THREADS, 0, st>>>(tax->parent.p, n_nodes, tax_hash, tax_count, clade_hash, clade_count);
        ctx->kernel_launches++;
    }
    tax_flag_kernel<<<(n_slots + TAX_THREADS - 1) / TAX_THREADS, TAX_THREADS, 0, st>>>(n_slots, n_nodes, tax_hash, clade_hash, flag.p);
    MG_CUDA(ctx, cub::DeviceSelect::Flagged(tmp.p, tb_sel, slots_it, flag.p, sel.p, n_sel.p, (int)n_slots, st));
    tax_gather_kernel<<<(n_slots + TAX_THREADS - 1) / TAX_THREADS, TAX_THREADS, 0, st>>>(sel.p, n_sel.p, n_nodes, tax_hash, tax_count, clade_hash, clade_count, d_rows.p);
    ctx->kernel_launches += 4;
    time_end(ctx, ctx->tax_events, st);
    MG_CUDA(ctx, cudaGetLastError());
    uint32_t h_n_sel = 0;
    MG_CUDA(ctx, cudaMemcpyAsync(&h_n_sel, n_sel.p, 4, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    std::vector<mashgpu_tax_row> h_rows(h_n_sel);
    if (h_n_sel) MG_CUDA(ctx, cudaMemcpyAsync(h_rows.data(), d_rows.p, h_n_sel * sizeof(mashgpu_tax_row), cudaMemcpyDeviceToHost, st));
    std::vector<uint32_t> h_slot(hash_taxid ? nd : 0);
    if (hash_taxid && nd) MG_CUDA(ctx, cudaMemcpyAsync(h_slot.data(), out_slot.p, nd * 4, cudaMemcpyDeviceToHost, st));
    if (unknown_in_lca && n_unknown) MG_CUDA(ctx, cudaMemcpyAsync(unknown_in_lca, unk.p, n_unknown, cudaMemcpyDeviceToHost, st));
    MG_CUDA(ctx, cudaStreamSynchronize(st));
    uint64_t tc = 0, thc = 0;
    for (auto &r : h_rows) {
        tc += r.tax_count; thc += r.tax_hash_count;
        r.taxid = slot_taxid[r.taxid];
    }
    *n_rows = h_n_sel;
    if (h_n_sel <= capacity && h_n_sel) std::copy(h_rows.begin(), h_rows.end(), rows);
    if (total_count) *total_count = tc;
    if (total_hash_count) *total_hash_count = thc;
    if (hash_taxid)
        for (uint64_t d = 0; d < nd; d++) hash_taxid[d] = slot_taxid[h_slot[d]];
    return MASHGPU_OK;
}
