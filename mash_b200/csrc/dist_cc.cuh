// dist_cc.cuh -- connected components of a dist run (mashgpu_dist_components, DESIGN.md 3.8): the device side.
//
// The component graph of a self job has one vertex per sketch and an edge {q, r} (r < q) for every pair of the lower triangle
// that passes (-d / -v) and shares a hash: the hit rule of the best runs.  No edge list is kept: dist_emit and dist_fix_kernel,
// the two places that know a pair's final pass flag, union its two sketches into a forest of one uint32 per sketch, and
// cc_flatten_kernel turns the forest into labels after the last run.  The union-find follows ECL-CC (Jaiganesh & Burtscher,
// 2018): find with path halving, hooking by atomicCAS on the root.  The larger root is always hooked under the smaller one, so the
// root of every tree is its smallest member and label[i] = smallest index of i's component, whatever order the unions ran in.
// The reference has no counterpart (its users cluster the output of `mash triangle -E` with a script).
#pragma once
#include <cstdint>

namespace mashgpu {

// Parent reads and the halving writes go through L2 (relaxed, device scope): a plain load may be served from a stale L1 line
// inside the retry loop of a hook.
__device__ __forceinline__ uint32_t cc_load(const uint32_t *p)
{
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

__device__ __forceinline__ void cc_store(uint32_t *p, uint32_t v)
{
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}

// Root of x, halving the path on the way: every other node is pointed at its grandparent.  A node that is not a root never becomes
// one again and its parent only ever moves to an ancestor, so a halving write (grandparent, an ancestor) cannot undo a hook.
__device__ __forceinline__ uint32_t cc_find(uint32_t *parent, uint32_t x)
{
    uint32_t p = cc_load(parent + x);
    while (p != x) {
        const uint32_t g = cc_load(parent + p);
        if (g == p) return p;
        cc_store(parent + x, g);
        x = g;
        p = cc_load(parent + x);
    }
    return x;
}

// Joins the trees of x and y: the larger root is hooked under the smaller one.  Shared by the component runs and the spanning
// forest's rounds (dist_msf.cuh).
__device__ __forceinline__ void cc_join(uint32_t *parent, uint32_t x, uint32_t y)
{
    uint32_t a = cc_find(parent, x), b = cc_find(parent, y);
    while (a != b) {
        if (a < b) { const uint32_t t = a; a = b; b = t; }         // hook the larger root a under the smaller b
        const uint32_t old = atomicCAS(parent + a, a, b);
        if (old == a) break;
        a = cc_find(parent, old);                                   // a was hooked meanwhile: retry from its new root
        b = cc_find(parent, b);
    }
}

// Joins the components of q and r (r_global: the reference's row in the query numbering, tri_r0 + r) in the forest `parent`
// (parent[i] <= i, parent[i] == i at a root; indexed by query row) and counts the edge in `edges` (every unordered pair once: the
// run enumerates the lower triangle).  Called through the not-inlined dist_graph_hit (dist_msf.cuh).
__device__ __forceinline__ void dist_cc_union(uint32_t *parent, unsigned long long *edges, uint32_t q, uint32_t r_global)
{
    const unsigned peers = __activemask();          // one counter update per warp for the lanes that report an edge together
    if ((int)(threadIdx.x & 31) == __ffs(peers) - 1) atomicAdd(edges, (unsigned long long)__popc(peers));
    cc_join(parent, q, r_global);
}

__global__ void cc_init_kernel(uint32_t *parent, uint64_t n)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t < n) parent[t] = (uint32_t)t;
}

// After every run: label[i] = root of i, in place.  The walk to the root only reads (as ECL-CC's flatten does): a halving write
// here could land on another thread's entry after that thread stored its root there, and leave it pointing at an ancestor below
// the root.  Each thread writes its own entry only, and only the root: every entry any walk reads is an ancestor of the node it
// belongs to, before and after that write, so every walk still ends at the root.
__global__ void cc_flatten_kernel(uint32_t *parent, uint64_t n)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n) return;
    uint32_t x = (uint32_t)t, p = cc_load(parent + x);
    while (p != x) {
        x = p;
        p = cc_load(parent + x);
    }
    if (x != (uint32_t)t) cc_store(parent + t, x);
}

}  // namespace mashgpu
