// pfnav_repair_kernel.cuh -- the seeds of N_FlowFieldUpdateToNearestPathable (field.c:2247) built inside the CTA that
// applies the repair (k_repair_chain, pfnav_fields.cu). Kept in its own header so that tests/emu/repair_emu.cpp can run
// the same source on CPU threads against the host's breadth-first search (pfnav_repair_seeds).
//
// The host search starts at the non-passable start tile, walks the 4-connected non-passable tiles and collects the
// passable tiles it reaches: the passable tiles 4-adjacent to the start tile's 4-connected non-passable component
// (field_passable_frontier, field.c:1441). That set does not depend on the visit order, so a bit-row flood yields it
// exactly: row r of the component grows by its own row (shifted left and right) and its neighbour rows, masked to the
// non-passable tiles, until nothing changes; the seeds are the component dilated by one tile, masked to the passable
// tiles. Passable here is cost != 0xFF && blockers == 0, as on the host (not the faction rule of the integration).
#pragma once
#include <stdint.h>
#include <stddef.h>

struct repair_seed_smem {
    uint64_t np[64];      // non-passable tiles of the chunk, one row per word (bit c = column c)
    uint64_t comp[64];    // the start tile's 4-connected non-passable component
    int changed;
};

// Every thread of the CTA calls this (blockDim.x >= 64); rows are owned by threads 0..63. cost / blk: the layer's
// row-major images from `lbase`, W64 tiles wide. seed: 64 words, written by threads 0..63 before the final barrier.
__device__ inline void repair_nearest_pathable_seeds(const uint8_t *__restrict__ cost, const uint16_t *__restrict__ blk,
                                                     size_t lbase, int W64, int chunk_r, int chunk_c, int start,
                                                     repair_seed_smem &s, uint64_t *seed)
{
    const int tid = threadIdx.x;
    if (tid < 64) {
        const size_t off = lbase + (size_t)(chunk_r * 64 + tid) * W64 + (size_t)chunk_c * 64;
        uint64_t np = 0;
        for (int c = 0; c < 64; c++)
            if (cost[off + c] == 0xFF || blk[off + c] != 0) np |= 1ull << c;
        s.np[tid] = np;
        s.comp[tid] = tid == (start >> 6) ? (1ull << (start & 63)) & np : 0;
    }
    for (;;) {
        __syncthreads();
        if (tid == 0) s.changed = 0;
        uint64_t nx = 0;
        if (tid < 64) {
            const uint64_t np = s.np[tid];
            uint64_t x = s.comp[tid];
            if (tid > 0) x |= s.comp[tid - 1] & np;
            if (tid < 63) x |= s.comp[tid + 1] & np;
            for (uint64_t y = 0; y != x;) { y = x; x |= ((x << 1) | (x >> 1)) & np; }     // fill along the row
            nx = x;
        }
        __syncthreads();
        if (tid < 64 && nx != s.comp[tid]) { s.comp[tid] = nx; s.changed = 1; }
        __syncthreads();
        if (!s.changed) break;
    }
    if (tid < 64) {
        const uint64_t c = s.comp[tid];
        uint64_t d = c | (c << 1) | (c >> 1);
        if (tid > 0) d |= s.comp[tid - 1];
        if (tid < 63) d |= s.comp[tid + 1];
        seed[tid] = d & ~s.np[tid];
    }
    __syncthreads();
}
