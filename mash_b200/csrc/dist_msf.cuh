// dist_msf.cuh -- minimum spanning forest of a dist run (mashgpu_dist_spanning_forest, DESIGN.md 3.9): the device side.
//
// The graph is the component graph of dist_cc.cuh: one vertex per sketch, an edge {i, j} (j < i) for every pair of the lower
// triangle that passes (-d / -v) and shares a hash.  Edges are ordered by the strict total order (distance, j, i), so the forest is
// unique.  It is built in Boruvka rounds without an edge list.  In a round every pair's capture offers its edge to the cheapest-edge
// slot of both endpoints' components (dist_graph_hit in dist_greedy.cuh, at the places where dist_cc_union is called); msf_hook_kernel
// then adds each component's cheapest edge to the forest and joins the two components with dist_cc.cuh's union-find, and
// cc_flatten_kernel turns the forest into the next round's labels.  The edge values are recomputed for the <= n - 1 forest edges after the last round.
// The reference has no counterpart (its users build single linkage from the output of `mash triangle -E`).
#pragma once
#include <cstdint>

#include "dist_cc.cuh"

namespace mashgpu {

// An edge as a 128-bit key that orders like (distance, j, i): hi = the bits of the distance (a non-negative double orders like its
// bit pattern; -0.0 is stored as +0.0), lo = j << 32 | i.  All ones = no edge.
struct __align__(16) MsfKey { unsigned long long lo, hi; };

constexpr unsigned long long MSF_NONE = ~0ull;

__device__ __forceinline__ bool msf_less(const MsfKey &x, const MsfKey &y)
{
    return x.hi < y.hi || (x.hi == y.hi && x.lo < y.lo);
}

// Capture target of the graph runs inside DistArgs; forest == nullptr outside them.  One struct for every kind of run: the hit is
// one not-inlined call with as few argument registers as possible (see dist_graph_hit, dist_greedy.cuh).  The kind follows from
// which of edges and best are set: component runs set edges, spanning-forest rounds set best, greedy runs set neither.
struct GraphCapture {
    uint32_t *forest;               // component runs: the union-find forest (dist_cc.cuh); spanning-forest rounds: the component
                                    // (root) of every vertex, read-only during the round; greedy runs: their GreedyRun header
    unsigned long long *edges;      // component runs: the edge counter; nullptr otherwise
    MsfKey *best;                   // spanning-forest rounds: per component root, the cheapest edge offered to it; nullptr otherwise
};

__device__ __forceinline__ unsigned long long msf_load_u64(const unsigned long long *p)
{
    unsigned long long v;
    asm volatile("ld.relaxed.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
    return v;
}

// best = min(best, k).  Slots only ever decrease, so a candidate whose distance word exceeds the one read is done after one 64-bit
// load.  Otherwise a 128-bit CAS loop; the first expected value is made of two loads and may be torn, so it is only trusted once a
// CAS has confirmed it (a CAS that finds it and is not lower writes the same value back).
__device__ __forceinline__ void msf_lower(MsfKey *slot, const MsfKey k)
{
    const unsigned long long hi = msf_load_u64(&slot->hi);
    if (k.hi > hi) return;
    MsfKey cur{msf_load_u64(&slot->lo), hi};
    for (bool known = false;; known = true) {
        const bool lower = msf_less(k, cur);
        if (!lower && known) return;
        const MsfKey old = atomicCAS(slot, cur, lower ? k : cur);
        if (old.lo == cur.lo && old.hi == cur.hi) return;
        cur = old;
    }
}

// The key of the edge {i, j}, j < i, at distance `dist`
__device__ __forceinline__ MsfKey msf_key(uint32_t i, uint32_t j, double dist)
{
    return MsfKey{((unsigned long long)j << 32) | i, dist == 0.0 ? 0ull : (unsigned long long)__double_as_longlong(dist)};
}


// One thread per vertex; the roots act.  A root's cheapest edge joins it to another component o.  When o picked the same edge (a
// mutual pick) only the smaller of the two roots records it.  Under a strict order the picked edges form a forest, every one of them
// belongs to the minimum spanning forest, and each joins two different trees of `parent`.  The slots are not reset here: other
// threads of this kernel read them.
__global__ void msf_hook_kernel(const uint32_t *label, const MsfKey *best, uint32_t *parent, unsigned long long *count,
                                unsigned long long *f_lo, unsigned long long *f_hi, uint64_t capacity, uint64_t n)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t >= n || label[t] != (uint32_t)t) return;
    const uint32_t v = (uint32_t)t;
    const MsfKey k = best[v];
    if (k.hi == MSF_NONE) return;                               // no edge leaves this component
    const uint32_t i = (uint32_t)k.lo, j = (uint32_t)(k.lo >> 32);
    const uint32_t li = label[i];
    const uint32_t o = li == v ? label[j] : li;
    if (o < v) {
        const MsfKey ko = best[o];
        if (ko.lo == k.lo && ko.hi == k.hi) return;
    }
    const unsigned long long at = atomicAdd(count, 1ull);
    if (at < capacity) { f_lo[at] = k.lo; f_hi[at] = k.hi; }   // the host refuses a count above n - 1
    cc_join(parent, v, o);
}

}  // namespace mashgpu
