// screen_view.cuh -- read-only view of a screen job's device table for the passes that run after the stream
// (taxscreen.cu).  The job itself stays private to screen.cu.
#pragma once
#include <cstdint>

#include "common.cuh"

namespace mashgpu {

struct ScreenTableView {
    mashgpu_ctx *ctx;
    uint64_t n_ref, stride;
    const uint64_t *ref_hashes;          // device: n_ref rows of `stride` slots
    const uint32_t *ref_n;               // device: hashes per row
    const uint32_t *h_ref_n;             // host: hashes per row
    const uint64_t *keys;                // device: open-addressing table of the distinct reference hashes
    const uint32_t *slot_idx;            // device: table slot -> index of its key in ascending order
    const uint32_t *cnt;                 // device: hit counter per distinct hash (ascending hash order)
    uint32_t log2cap;
    uint64_t n_distinct;
};

// Flushes and collects every chunk fed so far, then fills *v.
int screen_table_view(mashgpu_screen_job *job, ScreenTableView *v);

// The counting sort of (sketch, hash) pairs by distinct hash index (defined in taxscreen.cu, 256 threads, one CTA per entry of
// refs): tax_pairs_kernel looks up each pair's d and counts seg_n[d]; after an exclusive scan of seg_n into seg_start,
// tax_scatter_kernel writes ref_code[r] into a free place of d's segment, counting seg_n back down to 0.  The sparse screen
// finish (screen_hits.cuh) builds its inverted index with them, the sketch index as the code.
__global__ void tax_pairs_kernel(const uint64_t *hashes, uint64_t stride, const uint32_t *n_hashes, const uint32_t *refs,
                                 const uint64_t *pair_off, const uint64_t *keys, const uint32_t *slot_idx, uint32_t log2cap,
                                 uint32_t *pair_d, uint32_t *seg_n);
__global__ void tax_scatter_kernel(const uint32_t *n_hashes, const uint32_t *refs, const uint32_t *ref_code, const uint64_t *pair_off,
                                   const uint32_t *pair_d, const uint32_t *seg_start, uint32_t *seg_n, uint32_t *seg_code);

}  // namespace mashgpu
