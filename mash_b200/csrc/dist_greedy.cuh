// dist_greedy.cuh -- greedy dereplication of a dist run (mashgpu_dist_representatives, DESIGN.md 3.12): the device side.
//
// The graph is the component graph of dist_cc.cuh: an edge {i, j} (j < i) for every pair of the lower triangle that passes (-d / -v)
// and shares a hash.  The greedy order is the index order: sketch v is a representative iff no representative u < v has an edge
// {u, v} -- the lexicographically first maximal independent set (the rule of CD-HIT and of galah's and skDER's greedy clustering).
//
// Pass 1 decides it in blocks of consecutive query rows [q0, q0 + rows), strictly in order, one lower-triangle run per block.  Sketch 0
// has no earlier sketch and is a representative before the first block, which starts at row 1.  The capture (dist_greedy_hit) handles
// a hit (i, j) of the block's run in one of two ways: j < q0 is final, and a representative j covers i; j >= q0 sets bit (i - q0, j - q0)
// of the block's rows x rows bit matrix.  greedy_resolve_kernel then decides the block's rows in the rounds of Blelloch, Fineman and Shun
// ("Greedy sequential maximal independent set and matching are parallel on average", SPAA 2012): covered rows are out, and in every
// round each undecided row v looks at its earlier neighbours in the block -- one of them in: v is out; all of them out: v is in;
// otherwise v waits.  A round reads the sets of the round before (two buffers), so the number of rounds does not depend on timing.  The
// smallest undecided row has only decided neighbours, so every round decides at least one row: more rounds than rows is an error.
//
// Pass 2 is one more lower-triangle run.  Every edge between a representative and a member is offered to the member's slot under the
// spanning forest's key (distance, j, i) with msf_lower, and greedy_values_kernel (dist.cu) recomputes each member's pair.
//
// Device state: the status word and the 16-byte slot of every sketch, and one block's bit matrix (rows x ceil(rows / 32) words).
// The reference has no counterpart (its users dereplicate the output of `mash triangle -E` with a script).
#pragma once
#include <cstdint>
#include <cooperative_groups.h>

#include "dist_cc.cuh"
#include "dist_msf.cuh"

namespace mashgpu {

constexpr uint32_t GREEDY_REP = 1;          // status: a representative (final once its block is resolved)
constexpr uint32_t GREEDY_COVERED = 2;      // status during its block's run: the row has an edge to a representative of an earlier block
constexpr uint32_t GREEDY_MAX_BLOCK = 32768;        // rows of a pass-1 block at most: a 128 MiB bit matrix
constexpr int GREEDY_THREADS = 256;

// The header a greedy run's GraphCapture::forest points at (edges == best == nullptr): one per pass-1 block, one for pass 2.
struct __align__(16) GreedyRun {
    uint32_t *status;           // per sketch: GREEDY_REP, GREEDY_COVERED or 0
    uint32_t *bits;             // pass 1: the block's bit matrix, row i - q0 at bits + (i - q0) * pitch; nullptr in pass 2
    MsfKey *slot;               // pass 2: per sketch, the least key of an edge to a representative; nullptr in pass 1
    uint32_t q0, pitch;         // pass 1: the block's first row, words per matrix row
};

// status[0] = GREEDY_REP, every other 0
__global__ void greedy_init_kernel(uint32_t *status, uint64_t n)
{
    const uint64_t t = blockIdx.x * (uint64_t)blockDim.x + threadIdx.x;
    if (t < n) status[t] = t == 0 ? GREEDY_REP : 0u;
}

// The resolve step of one pass-1 block.  Mask word w holds rows 32 w .. 32 w + 31 of the block, bit l = row 32 w + l.
struct GreedyResolve {
    const uint32_t *bits;
    uint32_t pitch, rows, q0;
    uint32_t *status;
    uint32_t *in, *und;         // two buffers of pitch words each: round r reads buffer r & 1 and writes the other
    uint32_t *lo, *hi;          // per row: the first matrix word that may hold a neighbour not yet out, one past the last nonzero word
    int *ctl;                   // live[3]: round r sets live[r % 3] when a row waits; top[3]: the highest mask word with a row in,
                                // top[r % 3] for round r's sets (-1: none).  Zeroed and -1 by the host before the launch.
    unsigned long long *counters;       // [0] += rounds, [2] |= 1 when the rounds exceed the rows
};

// One cooperative launch per block: the extents and starting sets, then the rounds, each closed by a grid barrier, then the rows'
// final status.  A warp owns mask words; in a round lane l evaluates row 32 w + l against its matrix row, and the warp's ballots are the
// next sets' word.  The sets are read through L2 (cc_load): other SMs wrote them in the round before.
__global__ void __launch_bounds__(GREEDY_THREADS, 1) greedy_resolve_kernel(const GreedyResolve p)
{
    namespace cg = cooperative_groups;
    cg::grid_group grid = cg::this_grid();
    const int lane = threadIdx.x & 31;
    const uint32_t warp0 = (uint32_t)((blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5);
    const uint32_t warps = (uint32_t)(((uint64_t)gridDim.x * blockDim.x) >> 5);
    const uint32_t words = (p.rows + 31) / 32;
    int *live = p.ctl, *top = p.ctl + 3;

    for (uint32_t w = warp0; w < words; w += warps) {
        uint32_t und = 0;
        for (int l = 0; l < 32 && w * 32 + l < p.rows; l++) {
            const uint32_t v = w * 32 + l, n_words = (v + 31) / 32;       // the bits j < v
            const uint32_t *row = p.bits + (uint64_t)v * p.pitch;
            uint32_t first = n_words, last = 0;
            for (uint32_t k0 = 0; k0 < n_words; k0 += 32) {
                const uint32_t k = k0 + lane;
                const unsigned nz = __ballot_sync(0xFFFFFFFFu, k < n_words && row[k] != 0);
                if (nz && first == n_words) first = k0 + __ffs(nz) - 1;
                if (nz) last = k0 + 32 - __clz(nz);
            }
            if (lane == 0) { p.lo[v] = first; p.hi[v] = last; }
            if (!(p.status[p.q0 + v] & GREEDY_COVERED)) und |= 1u << l;
        }
        if (lane == 0) {
            cc_store(p.in + w, 0u);
            cc_store(p.und + w, und);
            if (und) cc_store(reinterpret_cast<uint32_t *>(live + 2), 1u);
        }
    }
    grid.sync();

    uint32_t r = 0;
    for (;; r++) {
        if (cc_load(reinterpret_cast<const uint32_t *>(live + (r + 2) % 3)) == 0) break;
        if (r == p.rows) {                          // cannot happen: every round decides the smallest undecided row
            if (blockIdx.x == 0 && threadIdx.x == 0) atomicOr(p.counters + 2, 1ull);
            break;
        }
        const uint32_t *in_c = p.in + (r & 1) * p.pitch, *und_c = p.und + (r & 1) * p.pitch;
        uint32_t *in_n = p.in + ((r + 1) & 1) * p.pitch, *und_n = p.und + ((r + 1) & 1) * p.pitch;
        const int in_top = (int)cc_load(reinterpret_cast<const uint32_t *>(top + r % 3));
        if (blockIdx.x == 0 && threadIdx.x == 0) {      // the flags of the rounds after this one; neither is read or written now
            cc_store(reinterpret_cast<uint32_t *>(live + (r + 1) % 3), 0u);
            cc_store(reinterpret_cast<uint32_t *>(top + (r + 2) % 3), 0xFFFFFFFFu);
        }
        for (uint32_t w = warp0; w < words; w += warps) {
            const uint32_t u = cc_load(und_c + w), iw = cc_load(in_c + w);
            bool in = false, wait = false;
            if ((u >> lane) & 1u) {
                const uint32_t v = w * 32 + lane;
                const uint32_t *row = p.bits + (uint64_t)v * p.pitch;
                uint32_t k = p.lo[v];
                const uint32_t end = p.hi[v];
                while (k < end && !(row[k] & (cc_load(in_c + k) | cc_load(und_c + k)))) k++;       // out neighbours stay out
                p.lo[v] = k;
                bool out = false, seen = false;
                for (; k < end; k++) {
                    const uint32_t b = row[k];
                    if (b & cc_load(in_c + k)) { out = true; break; }
                    if (b & cc_load(und_c + k)) {
                        seen = true;
                        if ((int)k >= in_top) break;            // no row in past this word: v waits
                    }
                }
                in = !out && !seen;
                wait = !out && seen;
            }
            const unsigned b_in = __ballot_sync(0xFFFFFFFFu, in), b_wait = __ballot_sync(0xFFFFFFFFu, wait);
            if (lane == 0) {
                cc_store(in_n + w, iw | b_in);
                cc_store(und_n + w, b_wait);
                if (b_wait) cc_store(reinterpret_cast<uint32_t *>(live + r % 3), 1u);
                if (iw | b_in) atomicMax(top + (r + 1) % 3, (int)w);
            }
        }
        grid.sync();
    }

    const uint32_t *in_f = p.in + (r & 1) * p.pitch;
    for (uint32_t w = warp0; w < words; w += warps) {
        const uint32_t v = w * 32 + lane;
        if (v < p.rows) p.status[p.q0 + v] = (cc_load(in_f + w) >> lane) & 1u ? GREEDY_REP : 0u;
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) p.counters[0] += r;
}

// A hit (pass, shared hash) of a component run, a spanning-forest round or a greedy run.  Not inlined, like dist_best_append: the
// merge kernels' epilogues keep their register allocation.  One call for every kind of run: a second call site in dist_emit, or a
// second capture among the arguments, costs dist_kernel registers beyond its allocation granule.  For the same reason the spanning
// forest's offer and the greedy assignment share one pair of msf_lower calls.
//   spanning-forest round: the edge goes to the slots of both endpoints' components, unless they are one component;
//   greedy pass 1 (GreedyRun::bits set; j < i = q): the status of rows before the block's first row q0 is final, so only
//     representatives are read there, and only the block's own rows are written (a plain store: every writer stores the same value);
//   greedy pass 2: an edge between a representative and a member goes to the member's slot.
__device__ __noinline__ void dist_graph_hit(const GraphCapture g, uint32_t q, uint32_t r_global, double dist)
{
    if (g.edges) { dist_cc_union(g.forest, g.edges, q, r_global); return; }
    MsfKey *first, *second = nullptr;
    if (g.best) {
        const uint32_t a = __ldg(g.forest + q), b = __ldg(g.forest + r_global);
        if (a == b) return;
        first = g.best + a; second = g.best + b;
    } else {
        const GreedyRun *run = reinterpret_cast<const GreedyRun *>(g.forest);
        uint32_t *status = run->status, *bits = run->bits;
        if (bits) {
            const uint32_t q0 = run->q0;
            if (r_global < q0) {
                if (status[r_global] & GREEDY_REP) status[q] = GREEDY_COVERED;
            } else {
                const uint32_t row = q - q0, col = r_global - q0;
                atomicOr(bits + (uint64_t)row * run->pitch + (col >> 5), 1u << (col & 31));
            }
            return;
        }
        const bool rep_q = status[q] & GREEDY_REP;
        if (rep_q == (bool)(status[r_global] & GREEDY_REP)) return;
        first = run->slot + (rep_q ? r_global : q);
    }
    const MsfKey k = msf_key(q, r_global, dist);
    msf_lower(first, k);
    if (second) msf_lower(second, k);
}

}  // namespace mashgpu
