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

}  // namespace mashgpu
