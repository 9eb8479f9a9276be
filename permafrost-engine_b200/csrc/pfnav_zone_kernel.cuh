// pfnav_zone_kernel.cuh -- the device code of k_zone_seed_bits (the TARGET_ZONE seed flood), kept in a header of its own
// so that tests/emu can run the SAME source on CPU threads (tests/emu/zone_emu.cpp defines the CUDA keywords and warp
// intrinsics it uses as plain C++); pfnav_region.cu includes it inside its anonymous namespace.
// Needs: <stdint.h>, uint4.
#pragma once

// One flood: the padded window of one chunk field, in the reference's arithmetic (field_update_zone, field.c:1810)
struct zone_job {
    int32_t layer, centre_r, centre_c;      // absolute nav tile of the zone centre
    int32_t base_r, base_c;                 // the window's first tile (chunk_region_base)
    int32_t budget;                         // (size_t)(M_PI * r * r + 0.5), capped at dim * dim (field.c:1843)
};

// heap words: priority dr^2 + dc^2 (< 2 * 127^2 < 2^15, exact in the reference's float) above the window-relative tile
// index (< 2^14); comparisons look at the priority alone
#define ZONE_TILE_BITS 14
#define ZONE_PRIO(w) ((w) >> ZONE_TILE_BITS)

__device__ __forceinline__ bool zone_bit(const uint32_t *bm, int i) { return (bm[i >> 5] >> (i & 31)) & 1u; }
__device__ __forceinline__ void zone_set(uint32_t *bm, int i) { bm[i >> 5] |= 1u << (i & 31); }

// lib/public/pqueue.h:109-208 as zone_heap restates it: 1-indexed (h[0] unused), `size` elements; push with strict `>`,
// pop moves the last element to the root and sifts it down with `target` starting at its own slot and strict `<` for
// both children
__device__ __forceinline__ void zone_push(uint32_t *h, uint32_t &size, uint32_t w)
{
    uint32_t curr = ++size, parent = curr >> 1;
    const uint32_t p = ZONE_PRIO(w);
    while (curr > 1 && ZONE_PRIO(h[parent]) > p) { h[curr] = h[parent]; curr = parent; parent >>= 1; }
    h[curr] = w;
}

__device__ __forceinline__ uint32_t zone_pop(uint32_t *h, uint32_t &size)
{
    const uint32_t top = h[1], n = size - 1;          // n: the size after the pop; h[n + 1] is the element sifted down
    const uint32_t last = h[n + 1], pl = ZONE_PRIO(last);
    uint32_t root = 1;
    while (root != n + 1) {
        uint32_t target = n + 1, tv = last, pt = pl;
        const uint32_t l = root * 2, r = l + 1;
        if (l <= n) { const uint32_t v = h[l]; if (ZONE_PRIO(v) < pt) { target = l; tv = v; pt = ZONE_PRIO(v); } }
        if (r <= n) { const uint32_t v = h[r]; if (ZONE_PRIO(v) < pt) { target = r; tv = v; } }
        h[root] = tv;
        root = target;
    }
    size = n;
    return top;
}

// field_zone_initial_frontier (field.c:1683) over one window, tiles relative to it. pass: the window's "exists and
// passable" bits (field_tile_passable, field.c:117), vis: all zero on entry. Phase one: a best-first search from the
// centre through any tile of the map until the first passable tile is popped; returns it, or -1.
__device__ __forceinline__ int zone_flood_start(const uint32_t *pass, uint32_t *vis, uint32_t *h, int dim, int H64, int W64,
                                                const zone_job &j)
{
    const int er[8] = {0, 0, -1, 1, -1, -1, 1, 1}, ec[8] = {-1, 1, 0, 0, -1, 1, -1, 1};
    const int cdr = j.centre_r - j.base_r, cdc = j.centre_c - j.base_c;
    uint32_t size = 0;
    zone_set(vis, cdr * dim + cdc);
    zone_push(h, size, (uint32_t)(cdr * dim + cdc));
    while (size > 0) {
        const int t = (int)(zone_pop(h, size) & ((1u << ZONE_TILE_BITS) - 1));
        if (zone_bit(pass, t)) return t;
        const int r = t / dim, c = t - r * dim;
        for (int e = 0; e < 8; e++) {
            const int nr = r + er[e], nc = c + ec[e];
            const int ar = j.base_r + nr, ac = j.base_c + nc;
            if (ar < 0 || ar >= H64 || ac < 0 || ac >= W64) continue;
            if (nr < 0 || nr >= dim || nc < 0 || nc >= dim) continue;
            const int i = nr * dim + nc;
            if (zone_bit(vis, i)) continue;
            zone_set(vis, i);
            const int dr = nr - cdr, dc = nc - cdc;
            zone_push(h, size, ((uint32_t)(dr * dr + dc * dc) << ZONE_TILE_BITS) | (uint32_t)i);
        }
    }
    return -1;
}

// phase two: a best-first search through passable tiles from `start` (vis all zero again); the first `budget` pops are
// the seeds
__device__ __forceinline__ void zone_flood_seeds(const uint32_t *pass, uint32_t *vis, uint32_t *h, uint32_t *seed, int dim,
                                                 int H64, int W64, const zone_job &j, int start)
{
    const int er[8] = {0, 0, -1, 1, -1, -1, 1, 1}, ec[8] = {-1, 1, 0, 0, -1, 1, -1, 1};
    const int cdr = j.centre_r - j.base_r, cdc = j.centre_c - j.base_c;
    uint32_t size = 0;
    zone_set(vis, start);
    zone_push(h, size, (uint32_t)start);
    int ret = 0;
    while (size > 0 && ret < j.budget) {
        const int t = (int)(zone_pop(h, size) & ((1u << ZONE_TILE_BITS) - 1));
        if (zone_bit(pass, t)) { zone_set(seed, t); ret++; }
        const int r = t / dim, c = t - r * dim;
        for (int e = 0; e < 8; e++) {
            const int nr = r + er[e], nc = c + ec[e];
            const int ar = j.base_r + nr, ac = j.base_c + nc;
            if (ar < 0 || ar >= H64 || ac < 0 || ac >= W64) continue;
            if (nr < 0 || nr >= dim || nc < 0 || nc >= dim) continue;
            const int i = nr * dim + nc;
            if (zone_bit(vis, i)) continue;
            zone_set(vis, i);
            if (!zone_bit(pass, i)) continue;
            const int dr = nr - cdr, dc = nc - cdc;
            zone_push(h, size, ((uint32_t)(dr * dr + dc * dc) << ZONE_TILE_BITS) | (uint32_t)i);
        }
    }
}

// one 32-tile word of the window's pass bits: the window's base column and the map width are multiples of 32, so a word
// lies wholly inside or wholly outside the map, and its 32 cost bytes / 64 blocker bytes are 16-byte aligned
__device__ __forceinline__ uint32_t zone_pass_word(const uint8_t *cost, const uint16_t *blk, int H64, int W64, const zone_job &j,
                                                   int dim, int w)
{
    const int wpr = dim >> 5, r = w / wpr, c0 = (w - r * wpr) * 32;
    const int ar = j.base_r + r, ac = j.base_c + c0;
    if (ar < 0 || ar >= H64 || ac < 0 || ac + 32 > W64) return 0;
    const size_t off = ((size_t)j.layer * H64 + ar) * W64 + ac;
    const uint4 *cv = reinterpret_cast<const uint4 *>(cost + off), *bv = reinterpret_cast<const uint4 *>(blk + off);
    uint32_t word = 0;
#pragma unroll
    for (int q = 0; q < 2; q++) {
        const uint4 c4 = cv[q];
        const uint32_t cw[4] = {c4.x, c4.y, c4.z, c4.w};
#pragma unroll
        for (int h = 0; h < 2; h++) {
            const uint4 b4 = bv[q * 2 + h];
            const uint32_t bw[4] = {b4.x, b4.y, b4.z, b4.w};
#pragma unroll
            for (int k = 0; k < 8; k++) {            // tile q * 16 + h * 8 + k
                const uint32_t cb = (cw[h * 2 + (k >> 2)] >> ((k & 3) * 8)) & 0xFFu;
                const uint32_t bb = (bw[k >> 1] >> ((k & 1) * 16)) & 0xFFFFu;
                if (cb != 0xFFu && bb == 0) word |= 1u << (q * 16 + h * 8 + k);
            }
        }
    }
    return word;
}

#define ZONE_FULL 0xFFFFFFFFu

// One warp per field: the warp stages the window's pass bits, lane 0 replays the flood, the warp writes the field's
// dim x dim seed bitmap (row-major, dim * dim / 32 words, the layout k_region_fields reads through seed_bits). Shared
// memory: the heap (dim * dim + 1 words: each phase pushes a tile at most once) and three bitmaps.
__global__ void __launch_bounds__(32) k_zone_seed_bits(const uint8_t *__restrict__ cost, const uint16_t *__restrict__ blk, int H64,
                                                       int W64, int dim, const zone_job *__restrict__ jobs, int n,
                                                       uint32_t *__restrict__ bits_out)
{
    extern __shared__ uint32_t zs_smem[];
    const int N = dim * dim, nw = N >> 5, lane = threadIdx.x & 31;
    uint32_t *heap = zs_smem, *pass = heap + N + 1, *vis = pass + nw, *seed = vis + nw;
    for (int f = blockIdx.x; f < n; f += gridDim.x) {
        const zone_job j = jobs[f];
        uint32_t *out = bits_out + (size_t)f * nw;
        const int cdr = j.centre_r - j.base_r, cdc = j.centre_c - j.base_c;
        if (cdr < 0 || cdr >= dim || cdc < 0 || cdc >= dim || j.budget <= 0) {     // no seeds
            for (int i = lane; i < nw; i += 32) out[i] = 0;
            continue;
        }
        for (int i = lane; i < nw; i += 32) { pass[i] = zone_pass_word(cost, blk, H64, W64, j, dim, i); vis[i] = 0; seed[i] = 0; }
        __syncwarp();
        int start = -1;
        if (lane == 0) start = zone_flood_start(pass, vis, heap, dim, H64, W64, j);
        start = __shfl_sync(ZONE_FULL, start, 0);
        __syncwarp();                               // orders lane 0's phase-one stores to `vis` before the clear
        if (start >= 0) {
            for (int i = lane; i < nw; i += 32) vis[i] = 0;
            __syncwarp();
            if (lane == 0) zone_flood_seeds(pass, vis, heap, seed, dim, H64, W64, j, start);
            __syncwarp();
        }
        for (int i = lane; i < nw; i += 32) out[i] = seed[i];
        __syncwarp();
    }
}
