// pfnav_fields.cu -- context, device map state, flow-field and LOS-field kernels.
//
// Replaces (reference file:line):
//   N_FlowFieldInit / N_FlowFieldUpdate TARGET_TILE | TARGET_PORTAL   src/navigation/field.c:2020-2083
//     field_build_integration :539, field_build_flow/field_flow_dir :734/:355,
//     field_portal_initial_frontier :1160, field_fixup_portal_edges :830
//   N_LOSFieldCreate                                                   src/navigation/field.c:2085-2245
//     field_neighbours_grid_los :304, field_is_los_corner :435,
//     field_create_wavefront_blocked_line :463, field_pad_wavefront :519, pqueue.h:109-208
//
// Design: the nav grids live in HBM as row-major images per layer so that any 64x64
// window is one TMA box (cp.async.bulk.tensor.3d, coordinates {x, y, layer}).
//   * K1 flow field, unit-cost chunks (the only costs a finished map holds are 1 and 0xFF,
//     nav.c:339-342): ONE WARP PER FIELD, bit-parallel multi-source BFS. A row of 64 tiles is one
//     64-bit word, a lane owns two rows, a BFS level is a handful of shifts/ORs plus two warp
//     shuffles for the rows above/below; the flow direction of every tile reached at level d is
//     derived in the same step from the level d-1 / d-2 frontiers (the integration field is
//     never materialised). The reference's float Dijkstra sums small integers exactly, so the
//     distance field is unique and any correct SSSP is bit-exact (SURVEY.md 8a-1).
//   * K1g general costs (transient 0-cost tiles, nav.c:359): one CTA per field, Bellman-Ford
//     relaxation on u32 distances in shared memory, then the reference's 8-neighbour rule.
//   * K3 LOS field: order-dependent (heap pop order among equal priorities is observable,
//     SURVEY.md 8a-2). k_los_level runs the wavefront level by level across the warp and checks,
//     per level, a certificate that the reference's pop order cannot have changed the result;
//     a field whose certificate fails is rebuilt by lane 0 replaying the reference's binary heap
//     exactly in shared memory (k_los_b's replay) while the whole warp stages, pads and stores.
#include "pfnav_internal.cuh"
#include <stdarg.h>
#include <string.h>
#include <algorithm>

// ------------------------------------------------------------------------------------------
// error plumbing
// ------------------------------------------------------------------------------------------
static thread_local char g_err[512] = "";

void pfnav_set_error(const char *fmt, ...)
{
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_err, sizeof(g_err), fmt, ap);
    va_end(ap);
}

extern "C" const char *pfnav_last_error(void) { return g_err; }
extern "C" int pfnav_version(void) { return PFNAV_VERSION; }
extern "C" uint64_t pfnav_launch_count(const pfnav_ctx *ctx) { return ctx ? ctx->launches : 0; }

// ------------------------------------------------------------------------------------------
// small PTX wrappers (mbarrier + TMA)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void *p)
{
    return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint64_t *bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, uint32_t parity)
{
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "WAIT_LOOP:\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
        "@p bra WAIT_DONE;\n\t"
        "bra WAIT_LOOP;\n\t"
        "WAIT_DONE:\n\t"
        "}" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
__device__ __forceinline__ void fence_barrier_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_load_3d(void *dst, const CUtensorMap *map, uint64_t *bar, int x, int y,
                                            int z)
{
    asm volatile(
        "cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
        ::"r"(smem_u32(dst)),
        "l"(map), "r"(smem_u32(bar)), "r"(x), "r"(y), "r"(z)
        : "memory");
}

#include "pfnav_los_kernel.cuh"   // bit helpers, FlowGrids, k_los_b, k_los_level
#include "pfnav_repair_kernel.cuh"   // kind-0 repair seeds of k_repair_chain

// ------------------------------------------------------------------------------------------
// Map-state kernels
// ------------------------------------------------------------------------------------------
// chunk-blocked [chunk][64][64] -> image [H64][W64]
template <typename T>
__global__ void k_deblock(const T *__restrict__ src, T *__restrict__ dst, int chunk_w, int chunk_h)
{
    const int W64 = chunk_w * 64;
    size_t total = (size_t)chunk_w * chunk_h * 4096;
    for (size_t i = blockIdx.x * (size_t)blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
        size_t chunk = i >> 12;
        int t = (int)(i & 4095);
        int cr = (int)(chunk / chunk_w), cc = (int)(chunk % chunk_w);
        dst[(size_t)(cr * 64 + (t >> 6)) * W64 + cc * 64 + (t & 63)] = src[i];
    }
}

// ------------------------------------------------------------------------------------------
// Tile attributes -> cost_base image (n_set_cost_for_tile nav.c:267-344 + n_make_cliff_edges
// nav.c:431-475). One thread per MAP tile (= 2x2 nav tiles); tiles are packed char4
// {pathable, type, base_height, ramp_height} in a global row-major [H32][W32] image.
// M_Tile_HeightAtPos (map/tile.c:249) is only consulted at the four corners of corner tiles,
// where it returns 4*corner_height up to float rounding that the int conversion + compare
// against -1 erase, so the integer corner height (tile.c:117-180) is used directly.
__device__ __forceinline__ bool tile_corner_raised(int type, int sr, int sc)
{
    // bit i set = tile type i raises this corner (tile.c:117-180); order NW, NE, SW, SE
    const unsigned raised[4] = {
        (1u<<1)|(1u<<3)|(1u<<6)|(1u<<8)|(1u<<7)|(1u<<12),
        (1u<<1)|(1u<<4)|(1u<<6)|(1u<<5)|(1u<<8)|(1u<<10),
        (1u<<2)|(1u<<3)|(1u<<8)|(1u<<10)|(1u<<11)|(1u<<12),
        (1u<<2)|(1u<<4)|(1u<<6)|(1u<<12)|(1u<<9)|(1u<<10)};
    const int k = sr * 2 + sc;
    const unsigned m = k == 0 ? raised[0] : k == 1 ? raised[1] : k == 2 ? raised[2] : raised[3];
    return (m >> type) & 1u;
}

__device__ __forceinline__ bool tile_path_bit(int type, int sr, int sc)
{
    // "tile_path_map" of n_set_cost_for_tile (nav.c:276-322): the one passable quarter of a corner tile
    const unsigned bl = (1u<<5)|(1u<<12), br = (1u<<7)|(1u<<10), tl = (1u<<9)|(1u<<8), tr = (1u<<11)|(1u<<6);
    const unsigned m = sr ? (sc ? br : bl) : (sc ? tr : tl);
    return (m >> type) & 1u;
}

__global__ void k_cost_from_tiles(const char4 *__restrict__ tiles, uint8_t *__restrict__ cost, int W32, int H32,
                                  int group)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    const int r = blockIdx.y * blockDim.y + threadIdx.y;
    if (c >= W32 || r >= H32) return;
    const char4 t = tiles[(size_t)r * W32 + c];
    const int path = t.x != 0, type = t.y, base = t.z, ramp = t.w;
    bool pathable;
    if (group == 0)      pathable = path && base >= -1 && !(type != 0 && ramp > 1);   // n_tile_pathable nav.c:215
    else if (group == 1) pathable = path && !(base + ramp > -1);                       // n_tile_water_pathable :226
    else                 pathable = true;
    // cliff edges between FLAT tiles of different base height (nav.c:420-475); n_set_cost_edge blocks the
    // half where its map is ZERO (nav.c:415): EDGE_BOT -> top sub-row, EDGE_TOP -> bottom sub-row,
    // EDGE_LEFT -> right sub-column, EDGE_RIGHT -> left sub-column.
    bool cb = false, ct = false, cl = false, crt = false;
    if (type == 0) {
        if (r + 1 < H32) { char4 o = tiles[(size_t)(r + 1) * W32 + c]; cb = o.y == 0 && o.z != base; }
        if (r > 0)       { char4 o = tiles[(size_t)(r - 1) * W32 + c]; ct = o.y == 0 && o.z != base; }
        if (c > 0)       { char4 o = tiles[(size_t)r * W32 + c - 1];   cl = o.y == 0 && o.z != base; }
        if (c + 1 < W32) { char4 o = tiles[(size_t)r * W32 + c + 1];   crt = o.y == 0 && o.z != base; }
    }
    const int W64 = W32 * 2;
#pragma unroll
    for (int sr = 0; sr < 2; sr++) {
        uint8_t v[2];
#pragma unroll
        for (int sc = 0; sc < 2; sc++) {
            const int h = (tile_corner_raised(type, sr, sc) ? base + ramp : base) * 4;   // Y_COORDS_PER_TILE
            const bool hp = group == 1 ? (h <= -1) : group == 2 ? true : (h >= -1);      // n_height_pathable :258
            uint8_t x = pathable ? 1 : (tile_path_bit(type, sr, sc) && hp) ? 1 : 0xFF;
            if ((cb && sr == 0) || (ct && sr == 1) || (cl && sc == 1) || (crt && sc == 0)) x = 0xFF;
            v[sc] = x;
        }
        *(uint16_t *)(cost + (size_t)(2 * r + sr) * W64 + 2 * c) = (uint16_t)(v[0] | (v[1] << 8));
    }
}

// per-chunk flag: 1 if every passable tile has cost 1. One warp per chunk.
__global__ void k_unit_flags(const uint8_t *__restrict__ cost, uint8_t *__restrict__ unit, int chunk_w, int chunk_h)
{
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    if (warp >= chunk_w * chunk_h) return;
    int cr = warp / chunk_w, cc = warp % chunk_w;
    const int W64 = chunk_w * 64;
    bool bad = false;
    for (int t = lane; t < 4096; t += 32) {
        uint8_t c = cost[(size_t)(cr * 64 + (t >> 6)) * W64 + cc * 64 + (t & 63)];
        bad |= (c != 1 && c != 0xFF);
    }
    bad = __any_sync(0xffffffffu, bad);
    if (lane == 0) unit[warp] = bad ? 0 : 1;
}

// ------------------------------------------------------------------------------------------
// K1: flow field, unit-cost fast path. One warp per field.
// ------------------------------------------------------------------------------------------
// field_tile_passable_no_enemies (field.c:179): a blocked tile stays passable for an "attacking" request when
// every faction holding a refcount on it is an enemy of the requesting faction
__device__ __forceinline__ bool blocked_for(const FlowGrids &g, int faction_id, size_t off)
{
    if (g.blk[off] == 0) return false;
    if (faction_id == PFNAV_FACTION_ID_NONE) return true;
    return (g.fmask[off] & ~g.enemies[faction_id & 0xF]) != 0;
}

#define FLOW_WARPS_PER_CTA 8
#define FLOW_SMEM_PER_WARP 12288   // cost tile 4096 + blockers tile 8192

// Load the passable masks of the lane's two rows (rows 2*lane, 2*lane+1).
// P bit c = cost != 0xFF && blockers == 0 (field_tile_passable, field.c:117).
template <bool USE_TMA>
__device__ __forceinline__ void load_pass_rows(const FlowGrids &g, const CUtensorMap *tm_cost,
                                               const CUtensorMap *tm_blk, uint8_t *sm, uint64_t *bar,
                                               uint32_t &phase, int layer, int chunk_r, int chunk_c,
                                               uint32_t lane, uint64_t &P0, uint64_t &P1, bool &nonunit)
{
    uint64_t P[2] = {0, 0};
    uint32_t nu = 0;
    if (USE_TMA) {
        if (lane == 0) {
            mbar_expect_tx(bar, FLOW_SMEM_PER_WARP);
            tma_load_3d(sm, tm_cost, bar, chunk_c * 64, chunk_r * 64, layer);
            tma_load_3d(sm + 4096, tm_blk, bar, chunk_c * 64, chunk_r * 64, layer);
        }
        mbar_wait(bar, phase);
        phase ^= 1;
        // lane's cost bytes: 128 contiguous bytes at lane*128 (8 x 16B); rotate the chunk order by
        // lane so the 8 lanes of a quarter-warp hit distinct bank groups.
        const uint4 *sc = reinterpret_cast<const uint4 *>(sm + lane * 128);
#pragma unroll
        for (int k = 0; k < 8; k++) {
            int q = (k + lane) & 7;
            uint32_t imp, n1;
            cost16_bits(sc[q], imp, n1);
            uint32_t pass = (~imp) & 0xFFFFu;
            nu |= n1 & pass;
            const uint64_t val = (uint64_t)pass << ((q & 3) * 16);
            if (q >> 2) P[1] |= val; else P[0] |= val;
        }
        const uint4 *sb = reinterpret_cast<const uint4 *>(sm + 4096 + lane * 256);
#pragma unroll
        for (int k = 0; k < 16; k++) {
            int q = (k + lane) & 15;
            const uint64_t b = (uint64_t)blk8_bits(sb[q]) << ((q & 7) * 8);
            if (q >> 3) P[1] &= ~b; else P[0] &= ~b;
        }
    } else {
#pragma unroll
        for (int rr = 0; rr < 2; rr++) {
            int row = 2 * lane + rr;
            size_t off = ((size_t)layer * g.H64 + chunk_r * 64 + row) * g.W64 + chunk_c * 64;
            const uint4 *pc = reinterpret_cast<const uint4 *>(g.cost + off);
            const uint4 *pb = reinterpret_cast<const uint4 *>(g.blk + off);
            uint4 c4[4], b4[8];
#pragma unroll
            for (int k = 0; k < 4; k++) c4[k] = __ldg(pc + k);
#pragma unroll
            for (int k = 0; k < 8; k++) b4[k] = __ldg(pb + k);
            uint64_t p = 0, blocked = 0;
#pragma unroll
            for (int k = 0; k < 4; k++) {
                uint32_t imp, n1;
                cost16_bits(c4[k], imp, n1);
                uint32_t pass = (~imp) & 0xFFFFu;
                nu |= n1 & pass;
                p |= (uint64_t)pass << (16 * k);
            }
#pragma unroll
            for (int k = 0; k < 8; k++) blocked |= (uint64_t)blk8_bits(b4[k]) << (8 * k);
            P[rr] = p & ~blocked;
        }
    }
    P0 = P[0];
    P1 = P[1];
    nonunit = nu != 0;
}

// Seeds of a TARGET_PORTAL field (field_portal_initial_frontier, field.c:1160 +
// field_tile_adjacent_to_next_iid :1131). Returns the seed masks of the lane's two rows.
__device__ __forceinline__ void portal_seeds(const FlowGrids &g, const pfnav_field_req &q, uint32_t lane,
                                             uint64_t P0, uint64_t P1, uint64_t &S0, uint64_t &S1)
{
    S0 = 0; S1 = 0;
    const int nr = q.port_r1 - q.port_r0 + 1, nc = q.port_c1 - q.port_c0 + 1;
    const int ntiles = nr * nc;
    const size_t lbase = (size_t)q.layer * g.H64 * g.W64;
    for (int base = 0; base < ntiles; base += 32) {
        int i = base + (int)lane;
        int r = -1, c = -1;
        bool ok = false;
        if (i < ntiles) {
            r = q.port_r0 + i / nc;
            c = q.port_c0 + i % nc;
            ok = true;
            if (q.port_iid != PFNAV_ISLAND_NONE) {
                uint16_t li = g.liid[lbase + (size_t)(q.chunk_r * 64 + r) * g.W64 + q.chunk_c * 64 + c];
                ok = (li == q.port_iid);
            }
            if (ok) {
                // adjacency to a tile of the next portal whose local island is next_iid
                const int gr = q.chunk_r * 64 + r, gc = q.chunk_c * 64 + c;
                const int dr[4] = {-1, 1, 0, 0}, dc[4] = {0, 0, -1, 1};
                bool adj = false;
#pragma unroll
                for (int k = 0; k < 4; k++) {
                    int ngr = gr + dr[k], ngc = gc + dc[k];
                    if (ngr < 0 || ngc < 0 || ngr >= g.H64 || ngc >= g.W64) continue;
                    if ((ngr >> 6) != q.next_chunk_r || (ngc >> 6) != q.next_chunk_c) continue;
                    int tr = ngr & 63, tc = ngc & 63;
                    if (tr < q.next_r0 || tr > q.next_r1 || tc < q.next_c0 || tc > q.next_c1) continue;
                    uint16_t li = g.liid[lbase + (size_t)ngr * g.W64 + ngc];
                    if (li == q.next_iid) adj = true;
                }
                ok = adj;
            }
        }
        // route each accepted tile to the lane that owns its row
#pragma unroll 1
        for (int src = 0; src < 32; src++) {
            int rr = __shfl_sync(0xffffffffu, r, src);
            int cc = __shfl_sync(0xffffffffu, c, src);
            int oo = __shfl_sync(0xffffffffu, (int)ok, src);
            if (oo && (rr >> 1) == (int)lane) {
                if (rr & 1) S1 |= 1ull << cc; else S0 |= 1ull << cc;
            }
        }
    }
    // only passable tiles seed the frontier (field.c:1186-1193)
    S0 &= P0;
    S1 &= P1;
}

// Expand one row (4 bit planes + reached mask) into 64 dir bytes and store them.
__device__ __forceinline__ void store_row(uint8_t *dst_row, uint64_t b0, uint64_t b1, uint64_t b2, uint64_t b3,
                                          uint64_t reached, bool init)
{
    uint4 *dst = reinterpret_cast<uint4 *>(dst_row);
#pragma unroll
    for (int k = 0; k < 4; k++) {      // 16 tiles per uint4
        uint32_t w[4];
#pragma unroll
        for (int j = 0; j < 4; j++) {  // 4 tiles per u32
            int sh = k * 16 + j * 4;
            uint32_t x0 = (uint32_t)(b0 >> sh), x1 = (uint32_t)(b1 >> sh), x2 = (uint32_t)(b2 >> sh),
                     x3 = (uint32_t)(b3 >> sh);
            w[j] = spread4(x0) | (spread4(x1) << 1) | (spread4(x2) << 2) | (spread4(x3) << 3);
        }
        if (!init) {
            // tiles the integration never reached keep their previous direction (field.c:744-745)
            uint4 old = dst[k];
            uint32_t o[4] = {old.x, old.y, old.z, old.w};
#pragma unroll
            for (int j = 0; j < 4; j++) {
                int sh = k * 16 + j * 4;
                uint32_t keep = spread4((uint32_t)(~reached >> sh)) * 0xFFu;
                w[j] = (w[j] & ~keep) | (o[j] & keep);
            }
        }
        dst[k] = make_uint4(w[0], w[1], w[2], w[3]);
    }
}

template <bool USE_TMA>
__global__ void __launch_bounds__(FLOW_WARPS_PER_CTA * 32)
k_flow_unit(const __grid_constant__ CUtensorMap tm_cost, const __grid_constant__ CUtensorMap tm_blk, FlowGrids g,
            const pfnav_field_req *__restrict__ reqs, int n, uint8_t *__restrict__ fields,
            const int32_t *__restrict__ out_slot)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    uint8_t *sm = smem + warp * FLOW_SMEM_PER_WARP;
    uint64_t *bar = reinterpret_cast<uint64_t *>(smem + FLOW_WARPS_PER_CTA * FLOW_SMEM_PER_WARP) + warp;
    uint32_t phase = 0;
    if (USE_TMA) {
        if (lane == 0) {
            mbar_init(bar, 1);
            fence_barrier_init();
        }
        __syncwarp();
    }
    const int total_warps = gridDim.x * FLOW_WARPS_PER_CTA;
    for (int i = blockIdx.x * FLOW_WARPS_PER_CTA + warp; i < n; i += total_warps) {
        const pfnav_field_req q = reqs[i];
        // the general-cost kernel owns chunks that hold a passable cost other than 1
        if (!g.unit[(size_t)q.layer * g.chunk_w * g.chunk_h + q.chunk_r * g.chunk_w + q.chunk_c]) continue;
        // ... and the faction-aware ("attacking") requests, whose passability is per request
        if (q.faction_id != PFNAV_FACTION_ID_NONE) continue;

        uint64_t P0, P1;
        bool nonunit;
        if (USE_TMA) { fence_proxy_async(); __syncwarp(); }
        load_pass_rows<USE_TMA>(g, &tm_cost, &tm_blk, sm, bar, phase, q.layer, q.chunk_r, q.chunk_c, lane, P0, P1,
                                nonunit);

        // ---- seeds (field_initial_frontier, field.c:1372) ----
        uint64_t S0 = 0, S1 = 0;
        if (q.target_type == PFNAV_TARGET_TILE) {
            if ((q.tile_r >> 1) == (int)lane) {
                if (q.tile_r & 1) S1 = (1ull << q.tile_c) & P1; else S0 = (1ull << q.tile_c) & P0;
            }
        } else {
            portal_seeds(g, q, lane, P0, P1, S0, S1);
        }

        // ---- bit-parallel BFS with on-the-fly direction derivation ----
        const uint64_t Pu = shfl_up64(P1, lane), Pd = shfl_down64(P0, lane);
        uint64_t V0 = S0, V1 = S1, F0 = S0, F1 = S1, G0 = 0, G1 = 0, Gu = 0, Gd = 0;
        uint64_t D00 = 0, D01 = 0, D02 = 0, D03 = 0, D10 = 0, D11 = 0, D12 = 0, D13 = 0;
        const uint64_t P0l = P0 << 1, P0r = P0 >> 1, P1l = P1 << 1, P1r = P1 >> 1;
        while (true) {
            const uint64_t Fu = shfl_up64(F1, lane), Fd = shfl_down64(F0, lane);
            const uint64_t N0 = ((F0 << 1) | (F0 >> 1) | Fu | F1) & P0 & ~V0;
            const uint64_t N1 = ((F1 << 1) | (F1 >> 1) | F0 | Fd) & P1 & ~V1;
            if (!__any_sync(0xffffffffu, (N0 | N1) != 0)) break;
            {   // row 0: above = lane-1's row 1 (Fu/Gu/Pu), below = own row 1
                const uint64_t dNW = (Gu << 1) & Pu & P0l, dNE = (Gu >> 1) & Pu & P0r;
                const uint64_t dSW = (G1 << 1) & P1 & P0l, dSE = (G1 >> 1) & P1 & P0r;
                const uint64_t anyd = (dNW | dNE | dSW | dSE) & N0;
                // min_cost is d-2 where an admissible diagonal exists; the selection then takes the
                // first neighbour EQUAL to min_cost without re-checking admissibility (field.c:405-428)
                uint64_t t;
                const uint64_t m1 = (Gu << 1) & anyd;            t = m1;
                const uint64_t m3 = (Gu >> 1) & anyd & ~t;       t |= m3;
                const uint64_t m6 = (G1 << 1) & anyd & ~t;       t |= m6;
                const uint64_t m8 = (G1 >> 1) & anyd & ~t;
                const uint64_t card = N0 & ~anyd;
                const uint64_t m2 = Fu & card;                   t = m2;
                const uint64_t m7 = F1 & card & ~t;              t |= m7;
                const uint64_t m5 = (F0 >> 1) & card & ~t;       t |= m5;
                const uint64_t m4 = (F0 << 1) & card & ~t;
                D00 |= m1 | m3 | m5 | m7;
                D01 |= m2 | m3 | m6 | m7;
                D02 |= m4 | m5 | m6 | m7;
                D03 |= m8;
            }
            {   // row 1: above = own row 0, below = lane+1's row 0 (Fd/Gd/Pd)
                const uint64_t dNW = (G0 << 1) & P0 & P1l, dNE = (G0 >> 1) & P0 & P1r;
                const uint64_t dSW = (Gd << 1) & Pd & P1l, dSE = (Gd >> 1) & Pd & P1r;
                const uint64_t anyd = (dNW | dNE | dSW | dSE) & N1;
                uint64_t t;
                const uint64_t m1 = (G0 << 1) & anyd;            t = m1;
                const uint64_t m3 = (G0 >> 1) & anyd & ~t;       t |= m3;
                const uint64_t m6 = (Gd << 1) & anyd & ~t;       t |= m6;
                const uint64_t m8 = (Gd >> 1) & anyd & ~t;
                const uint64_t card = N1 & ~anyd;
                const uint64_t m2 = F0 & card;                   t = m2;
                const uint64_t m7 = Fd & card & ~t;              t |= m7;
                const uint64_t m5 = (F1 >> 1) & card & ~t;       t |= m5;
                const uint64_t m4 = (F1 << 1) & card & ~t;
                D10 |= m1 | m3 | m5 | m7;
                D11 |= m2 | m3 | m6 | m7;
                D12 |= m4 | m5 | m6 | m7;
                D13 |= m8;
            }
            G0 = F0; G1 = F1; Gu = Fu; Gd = Fd;
            F0 = N0; F1 = N1;
            V0 |= N0; V1 |= N1;
        }

        // ---- portal fixup: seeds point across the border (field_fixup_portal_edges, field.c:830) ----
        if (q.target_type == PFNAV_TARGET_PORTAL) {
            const bool up = q.next_chunk_r < q.chunk_r, down = q.next_chunk_r > q.chunk_r;
            const bool left = q.next_chunk_c < q.chunk_c;
            // FD_N = 2, FD_S = 7, FD_W = 4, FD_E = 5
            const uint32_t code = up ? 2u : down ? 7u : left ? 4u : 5u;
            if (code & 1) { D00 |= S0; D10 |= S1; }
            if (code & 2) { D01 |= S0; D11 |= S1; }
            if (code & 4) { D02 |= S0; D12 |= S1; }
        }

        uint8_t *dst = fields + (size_t)(out_slot ? out_slot[i] : i) * 4096 + lane * 128;
        store_row(dst, D00, D01, D02, D03, V0, q.init != 0);
        store_row(dst + 64, D10, D11, D12, D13, V1, q.init != 0);
    }
}

// ------------------------------------------------------------------------------------------
// The integration and direction pass of the CTA-per-field kernels (k_flow_general, k_repair_chain), 128 threads.
// Every thread calls it once dist / cost / dom hold the field's start state: dom 0 = outside the integration, 1 = relaxed
// (edge weight = cost of the tile entered, field_build_integration, field.c:556-563), 2 = seed (dist 0). The relaxation
// runs to the unique shortest-distance fixpoint, so the order tiles are visited in cannot change a result. The
// directions then go to dst (4096 bytes) by the 8-neighbour rule; both exceptions key on the distance value, since a
// zero-cost tile (the transient 0 of nav.c:359) next to a seed reaches 0 without being one:
//   unreached tiles get 0 when zero_unreached and keep their byte otherwise;
//   tiles at distance 0 get the portal fix-up (field_fixup_portal_edges, field.c:830) or 0 when set_dist0, and keep
//   their byte otherwise.
// Returns after a barrier: the caller may reuse the arrays and read dst.
// ------------------------------------------------------------------------------------------
#define FLOWG_THREADS 128
__device__ __forceinline__ void flow_integrate(uint32_t *dist, const uint8_t *cost, const uint8_t *dom, int &changed,
                                               const pfnav_field_req &q, bool zero_unreached, bool set_dist0,
                                               uint8_t *__restrict__ dst)
{
    const int tid = threadIdx.x;
    do {
        __syncthreads();
        if (tid == 0) changed = 0;
        __syncthreads();
        bool ch = false;
        for (int t = tid; t < 4096; t += FLOWG_THREADS) {
            if (dom[t] != 1) continue;
            const int r = t >> 6, cc = t & 63;
            uint32_t m = 0xFFFFFFFFu;
            if (r > 0)   m = min(m, dist[t - 64]);
            if (r < 63)  m = min(m, dist[t + 64]);
            if (cc > 0)  m = min(m, dist[t - 1]);
            if (cc < 63) m = min(m, dist[t + 1]);
            if (m != 0xFFFFFFFFu && m + cost[t] < dist[t]) { dist[t] = m + cost[t]; ch = true; }
        }
        if (ch) changed = 1;
        __syncthreads();
    } while (changed);

    const bool up = q.next_chunk_r < q.chunk_r, down = q.next_chunk_r > q.chunk_r;
    const bool left = q.next_chunk_c < q.chunk_c;
    const uint8_t fix = up ? 2 : down ? 7 : left ? 4 : 5;
    for (int t = tid; t < 4096; t += FLOWG_THREADS) {
        const uint32_t d = dist[t];
        if (d == 0xFFFFFFFFu) { if (zero_unreached) dst[t] = 0; continue; }
        if (d == 0) { if (set_dist0) dst[t] = (q.target_type == PFNAV_TARGET_PORTAL) ? fix : 0; continue; }
        const int r = t >> 6, c = t & 63;
        const uint32_t INF = 0xFFFFFFFFu;
        const uint32_t dn = r > 0 ? dist[t - 64] : INF, ds = r < 63 ? dist[t + 64] : INF;
        const uint32_t dw = c > 0 ? dist[t - 1] : INF, de = c < 63 ? dist[t + 1] : INF;
        const uint32_t dnw = (r > 0 && c > 0) ? dist[t - 65] : INF, dne = (r > 0 && c < 63) ? dist[t - 63] : INF;
        const uint32_t dsw = (r < 63 && c > 0) ? dist[t + 63] : INF, dse = (r < 63 && c < 63) ? dist[t + 65] : INF;
        uint32_t m = min(min(dn, ds), min(dw, de));
        if (dn != INF && dw != INF) m = min(m, dnw);
        if (dn != INF && de != INF) m = min(m, dne);
        if (ds != INF && dw != INF) m = min(m, dsw);
        if (ds != INF && de != INF) m = min(m, dse);
        uint8_t dir;   // field.c:405-428 priority N,S,E,W,NW,NE,SW,SE
        if (dn == m) dir = 2; else if (ds == m) dir = 7; else if (de == m) dir = 5; else if (dw == m) dir = 4;
        else if (dnw == m) dir = 1; else if (dne == m) dir = 3; else if (dsw == m) dir = 6; else dir = 8;
        dst[t] = dir;
    }
    __syncthreads();
}

// ------------------------------------------------------------------------------------------
// K1g: flow field, general u8 costs. One CTA (128 threads) per field.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FLOWG_THREADS)
k_flow_general(FlowGrids g, const pfnav_field_req *__restrict__ reqs, int n, uint8_t *__restrict__ fields,
               const int32_t *__restrict__ out_slot, int only_nonunit)
{
    __shared__ uint32_t dist[4096];
    __shared__ uint8_t cost[4096];       // 0xFF = impassable or blocked
    __shared__ uint8_t dom[4096];        // flow_integrate's domain: 0 = impassable, 1 = passable, 2 = seed
    __shared__ int changed;
    const int tid = threadIdx.x;
    for (int i = blockIdx.x; i < n; i += gridDim.x) {
        const pfnav_field_req q = reqs[i];
        if (only_nonunit && q.faction_id == PFNAV_FACTION_ID_NONE &&
            g.unit[(size_t)q.layer * g.chunk_w * g.chunk_h + q.chunk_r * g.chunk_w + q.chunk_c])
            continue;
        const size_t lbase = (size_t)q.layer * g.H64 * g.W64;
        for (int t = tid; t < 4096; t += FLOWG_THREADS) {
            size_t off = lbase + (size_t)(q.chunk_r * 64 + (t >> 6)) * g.W64 + q.chunk_c * 64 + (t & 63);
            uint8_t c = g.cost[off];
            if (blocked_for(g, q.faction_id, off)) c = 0xFF;
            cost[t] = c;
            dist[t] = 0xFFFFFFFFu;
            dom[t] = c != 0xFF;
        }
        __syncthreads();
        if (q.target_type == PFNAV_TARGET_TILE) {
            if (tid == 0) {
                int t = q.tile_r * 64 + q.tile_c;
                if (cost[t] != 0xFF) { dom[t] = 2; dist[t] = 0; }
            }
        } else {
            const int nc = q.port_c1 - q.port_c0 + 1, ntiles = (q.port_r1 - q.port_r0 + 1) * nc;
            for (int k = tid; k < ntiles; k += FLOWG_THREADS) {
                int r = q.port_r0 + k / nc, c = q.port_c0 + k % nc;
                if (cost[r * 64 + c] == 0xFF) continue;
                if (q.port_iid != PFNAV_ISLAND_NONE &&
                    g.liid[lbase + (size_t)(q.chunk_r * 64 + r) * g.W64 + q.chunk_c * 64 + c] != q.port_iid)
                    continue;
                const int gr = q.chunk_r * 64 + r, gc = q.chunk_c * 64 + c;
                const int dr[4] = {-1, 1, 0, 0}, dc[4] = {0, 0, -1, 1};
                bool adj = false;
                for (int e = 0; e < 4; e++) {
                    int ngr = gr + dr[e], ngc = gc + dc[e];
                    if (ngr < 0 || ngc < 0 || ngr >= g.H64 || ngc >= g.W64) continue;
                    if ((ngr >> 6) != q.next_chunk_r || (ngc >> 6) != q.next_chunk_c) continue;
                    int tr = ngr & 63, tc = ngc & 63;
                    if (tr < q.next_r0 || tr > q.next_r1 || tc < q.next_c0 || tc > q.next_c1) continue;
                    if (g.liid[lbase + (size_t)ngr * g.W64 + ngc] == q.next_iid) adj = true;
                }
                if (adj) { dom[r * 64 + c] = 2; dist[r * 64 + c] = 0; }
            }
        }
        flow_integrate(dist, cost, dom, changed, q, q.init != 0, true, fields + (size_t)(out_slot ? out_slot[i] : i) * 4096);
    }
}

// ------------------------------------------------------------------------------------------
// K1c: the repair chain of N_DesiredPointSeekVelocity (nav.c:3508-3554) on cached fields, in place. One CTA per field
// slot that has items in the launch; it walks the slot's items in order and applies an item only if the tile it names
// still has no direction when the item's turn comes, or always when the item says so (pfnav_flow_fields_repair, the
// serial pfnav_pool_repair, the surround variant on a blocked tile): the serial loop's read-back before the repair,
// answered where the byte lives.
//   kind 0 = N_FlowFieldUpdateToNearestPathable (field.c:2247): seeds flooded in the CTA (pfnav_repair_kernel.cuh); the
//            integration runs over NON-passable tiles only (field_build_integration_nonpass, field.c:643; edge weight =
//            raw cost_base of the tile entered) and distance-0 tiles keep their byte.
//   kind 1 = N_FlowFieldUpdateIslandToNearest (field.c:2307): seeds from the host; ordinary integration / flow / portal
//            fix-up from the substitute frontier.
// count: the repairs applied are added to it when given.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(FLOWG_THREADS)
k_repair_chain(FlowGrids g, const pf_chain_item *__restrict__ items, const int32_t *__restrict__ group_off, int ngroups,
               const uint64_t *__restrict__ host_masks, uint8_t *__restrict__ fields, uint32_t *__restrict__ count)
{
    __shared__ uint32_t dist[4096];
    __shared__ uint8_t cost[4096];       // raw cost_base
    __shared__ uint8_t dom[4096];        // 1 = tile takes part in the integration, 2 = seed
    __shared__ uint64_t seed[64];
    __shared__ repair_seed_smem ss;
    __shared__ int changed, apply;
    const int tid = threadIdx.x;
    for (int gi = blockIdx.x; gi < ngroups; gi += gridDim.x) {
        for (int it = group_off[gi]; it < group_off[gi + 1]; it++) {
            const pf_chain_item item = items[it];
            const pfnav_field_req q = item.q;
            const int kind = item.kind;
            uint8_t *dst = fields + (size_t)item.slot * 4096;
            __syncthreads();
            if (tid == 0) apply = item.always || (dst[item.tile] & 0xF) == 0;
            __syncthreads();
            if (!apply) continue;
            const size_t lbase = (size_t)q.layer * g.H64 * g.W64;
            if (kind == 0)       // arg = start_r << 8 | start_c
                repair_nearest_pathable_seeds(g.cost, g.blk, lbase, g.W64, q.chunk_r, q.chunk_c,
                                              ((item.arg >> 8) << 6) | (item.arg & 63), ss, seed);
            else if (tid < 64) seed[tid] = host_masks[(size_t)item.mask * 64 + tid];
            __syncthreads();
            for (int t = tid; t < 4096; t += FLOWG_THREADS) {
                const size_t off = lbase + (size_t)(q.chunk_r * 64 + (t >> 6)) * g.W64 + q.chunk_c * 64 + (t & 63);
                const uint8_t c = g.cost[off];
                const bool pass = c != 0xFF && !blocked_for(g, q.faction_id, off);
                const bool sd = (seed[t >> 6] >> (t & 63)) & 1;
                cost[t] = c;
                dom[t] = sd ? 2 : (kind == 0 ? !pass : pass) ? 1 : 0;
                dist[t] = sd ? 0u : 0xFFFFFFFFu;
            }
            flow_integrate(dist, cost, dom, changed, q, false, kind == 1, dst);     // the next item reads the bytes after it
            if (tid == 0 && count) atomicAdd(count, 1u);
        }
    }
}

static FlowGrids grids_of(const pfnav_ctx *ctx);

int pfnav_repair_chain_launch(pfnav_ctx *ctx, cudaStream_t st, const std::vector<pf_chain_item> &items,
                              const std::vector<uint64_t> &masks, uint8_t *fields, size_t host_fields, uint32_t *d_count)
{
    if (items.empty()) return PFNAV_OK;
    // group by slot, serial order inside a group (a stable sort)
    std::vector<int32_t> order(items.size());
    for (size_t i = 0; i < items.size(); i++) order[i] = (int32_t)i;
    std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return items[a].slot < items[b].slot; });
    std::vector<pf_chain_item> sorted(items.size());
    std::vector<int32_t> off;
    for (size_t k = 0; k < order.size(); k++) {
        sorted[k] = items[order[k]];
        if (k == 0 || sorted[k].slot != sorted[k - 1].slot) off.push_back((int32_t)k);
    }
    off.push_back((int32_t)sorted.size());
    const int ngroups = (int)off.size() - 1;
    const size_t b_item = sorted.size() * sizeof(pf_chain_item), b_mask = masks.size() * 8, b_off = off.size() * 4;
    const size_t b_f = host_fields * 4096;
    const size_t a_mask = (b_item + 15) & ~(size_t)15, a_off = a_mask + b_mask, a_f = (a_off + b_off + 15) & ~(size_t)15;
    const size_t total = a_f + b_f;
    pf_stage S;
    int rc = pf_stage_begin(ctx, st, total, total, false, &S);
    if (rc) return rc;
    memcpy(S.host, sorted.data(), b_item);
    if (b_mask) memcpy(S.host + a_mask, masks.data(), b_mask);
    memcpy(S.host + a_off, off.data(), b_off);
    if (b_f) memcpy(S.host + a_f, fields, b_f);
    if ((rc = pf_stage_upload(ctx, st, S, total))) return rc;
    uint8_t *dev = S.dev;
    k_repair_chain<<<(unsigned)std::min(ngroups, ctx->sm_count * 8), FLOWG_THREADS, 0, st>>>(
        grids_of(ctx), (const pf_chain_item *)dev, (const int32_t *)(dev + a_off), ngroups, (const uint64_t *)(dev + a_mask),
        b_f ? dev + a_f : fields, d_count);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    if (b_f) PF_CUDA(cudaMemcpyAsync(fields, dev + a_f, b_f, cudaMemcpyDeviceToHost, st));
    return pf_stage_done(ctx, st);
}

// ------------------------------------------------------------------------------------------
// K3: LOS field, bit-row replay (k_los). One warp per field; lane 0 replays the reference heap exactly. The byte-state
// replay k_los_b and the default, level-parallel k_los_level are in pfnav_los_kernel.cuh.
// ------------------------------------------------------------------------------------------
struct __align__(16) LosSmem {
    uint64_t pass[64];       // cost != 0xFF && blockers == 0
    uint64_t open[64];       // pass && cost <= 1  (neighbour_costs[i] > 1 test, field.c:2211)
    uint64_t assigned[64];   // integration_field < INF
    uint64_t blk[64];
    uint8_t  visb[4096];     // `visible`, one byte per tile: the serial loop only ever stores 1 (no read-modify-write)
    uint16_t heap[4104];     // 1-indexed; entry = r << 6 | c (size keeps the struct a multiple of 16 B)
};

static_assert(sizeof(LosSmem) % 16 == 0, "LosSmem must keep 16-byte alignment per warp");

// field_create_wavefront_blocked_line (field.c:463-517)
__device__ void los_blocked_line(LosSmem &s, const LosMapInfo mi, int tgt_cr, int tgt_cc, int tgt_r, int tgt_c,
                                 int cr, int cc, int r, int c)
{
    // M_Tile_Bounds (tile.c:356): x decreases with the column, z increases with the row
    const float tbx = (mi.map_x - (float)(tgt_cc * 256)) - (float)(tgt_c * 4);
    const float tbz = (mi.map_z + (float)(tgt_cr * 256)) + (float)(tgt_r * 4);
    const float cbx = (mi.map_x - (float)(cc * 256)) - (float)(c * 4);
    const float cbz = (mi.map_z + (float)(cr * 256)) + (float)(r * 4);
    const float tcx = tbx - 4.0f / 2.0f, tcz = tbz + 4.0f / 2.0f;
    const float ccx = cbx - 4.0f / 2.0f, ccz = cbz + 4.0f / 2.0f;
    float sx_ = tcx - ccx, sz_ = tcz - ccz;
    const float len = sqrtf(sx_ * sx_ + sz_ * sz_);   // PFM_Vec2_Len: float sum, correctly rounded sqrt
    sx_ = sx_ / len;
    sz_ = sz_ / len;
    if (!(len > 0.0f)) {
        // The line starts ON the target tile (a blocked / impassable destination seen as a corner by its neighbour):
        // the slope is 0/0 = NaN, (int)(NaN * 1000) is INT_MIN on x86-64 (cvttss2si), abs() and the negation leave it
        // there, err = dx + dy wraps to 0 (the engine is built with -fwrapv) and every step takes the `e2 >= dy` branch
        // only: with sx = -1 (NaN > 0 is false) the reference marks the row from the tile to column 0.
        or_row(&s.blk[r], (c == 63) ? ~0ull : ((2ull << c) - 1));
        return;
    }
    int dx = abs((int)(sx_ * 1000));
    int dy = -abs((int)(sz_ * 1000));
    const int sx = sx_ > 0.0f ? 1 : -1;
    const int sy = sz_ < 0.0f ? 1 : -1;
    int err = dx + dy, e2;
    int rr = r, c2 = c;
    // bits of the row being walked accumulate in a register and are OR-ed into shared memory with a
    // fire-and-forget reduction when the walk leaves the row: no load-use stall per step
    int acc_row = rr;
    uint64_t acc = 0;
    do {
        if (rr != acc_row) { or_row(&s.blk[acc_row], acc); acc_row = rr; acc = 0; }
        acc |= 1ull << c2;
        e2 = 2 * err;
        if (e2 >= dy) { err += dy; c2 += sx; }
        if (e2 <= dx) { err += dx; rr += sy; }
    } while (rr >= 0 && rr < 64 && c2 >= 0 && c2 < 64);
    or_row(&s.blk[acc_row], acc);
}

// field_is_los_corner (field.c:435)
__device__ __forceinline__ bool los_is_corner(const LosSmem &s, int r, int c)
{
    if (r > 0 && r < 63) {
        bool a = !((s.pass[r - 1] >> c) & 1), b = !((s.pass[r + 1] >> c) & 1);
        if (a ^ b) return true;
    }
    if (c > 0 && c < 63) {
        bool a = !((s.pass[r] >> (c - 1)) & 1), b = !((s.pass[r] >> (c + 1)) & 1);
        if (a ^ b) return true;
    }
    return false;
}

// The reference's binary heap (pqueue.h:109-208), 1-indexed, entries = prio2 << 12 | r << 6 | c.
// A unit-cost wavefront only ever holds two adjacent priorities (d and d+1), so priorities are kept
// modulo 4 and compared through their difference; and a push (always priority d+1, i.e. >= every
// priority in the heap) never sifts up: it is an append.
// (Restructurings of this loop that were measured and rejected as slower than this plain form: a sift path
//  from a "holds priority d" bit per slot, lane 0 only; the same with the pop loop in lockstep on 32 lanes and
//  the neighbours on 4 lanes; one state byte per tile in a padded array + bit-derived sift path; that plus a
//  resumable lane-0 loop handing every wavefront-blocked line to the whole warp (closed-form line positions).
//  The loop is bound by the dependent chain of one thread (SURVEY.md 8a-2), not by memory. What did pay was
//  cutting the instruction count of a pop: the byte-state kernel k_los_b below; a per-slot priority-bit sift
//  on top of it bought nothing.)
__device__ __forceinline__ bool heap_lt(uint16_t a, uint16_t b) { return (((b >> 12) - (a >> 12)) & 3) == 1; }

// pq_coord_pop + _pq_balance (pqueue.h:109-130, 190-200). Only two adjacent priorities are ever in the heap,
// so "a < b" is "a holds the lower one (that of the root being popped) and b does not": the sift of the
// former last element X runs only if X is of the higher priority, and follows the children that hold the
// lower one, left before right -- exactly what the strict comparisons of _pq_balance select.
__device__ __forceinline__ uint16_t heap_pop(uint16_t *h, int &size)
{
    const uint16_t out = h[1];
    const uint16_t x = h[size];
    size--;
    const uint32_t lowp = out >> 12;                 // the root holds the minimum priority
    int root = 1;
    if ((uint32_t)(x >> 12) != lowp) {
        const uint32_t *h2 = reinterpret_cast<const uint32_t *>(h);      // children 2k, 2k+1 share one aligned word
        while (true) {
            const int l = root * 2;
            if (l > size) break;
            const uint32_t two = h2[root];
            const bool dl = ((two >> 12) & 0xFu) == lowp, dr = l < size && (two >> 28) == lowp;
            if (!(dl || dr)) break;
            h[root] = (uint16_t)(dl ? two : two >> 16);
            root = dl ? l : l + 1;
        }
    }
    h[root] = x;
    return out;
}

__global__ void __launch_bounds__(LOS_WARPS_PER_CTA * 32)
k_los(FlowGrids g, LosMapInfo mi, const pfnav_los_req *__restrict__ reqs, int n,
      uint8_t *fields, const int32_t *__restrict__ out_slot, unsigned *counter, int *done,
      unsigned long long *trace)
{
    extern __shared__ __align__(16) uint8_t smem_raw[];
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    LosSmem &s = reinterpret_cast<LosSmem *>(smem_raw)[warp];
    // Dependency-driven scheduling: requests are sorted so that a request's prev_index is smaller than
    // its own index; warps take indices in order from a global counter and wait (only) for the one
    // field they depend on. No barrier between dependency levels: the LOS phase costs the slowest
    // chain, not the sum over levels of the slowest field of each level.
    for (;;) {
        int i = 0;
        if (lane == 0) i = (int)atomicAdd(counter, 1u);
        i = __shfl_sync(0xffffffffu, i, 0);
        if (i >= n) break;
        const pfnav_los_req q = reqs[i];
        unsigned long long t_take = 0, t_ready = 0;
        if (trace && lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_take));
        if (q.prev_index >= 0) {
            if (lane == 0) {
                volatile int *flag = done + q.prev_index;
                while (*flag == 0) __nanosleep(100);
            }
            __syncwarp();
            __threadfence();
        }
        if (trace && lane == 0) asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_ready));
        // A chunk other than the destination whose shared edge with the previous chunk carries no
        // `visible` and no `wavefront_blocked` tile starts with an empty frontier and draws no line
        // (field.c:2157-2195): the field is all zero. Most chunks far from the goal end here.
        if (!(q.chunk_r == q.tgt_chunk_r && q.chunk_c == q.tgt_chunk_c)) {
            const uint8_t *prev = fields + (size_t)(q.prev_index >= 0 ? (out_slot ? out_slot[q.prev_index] : q.prev_index) : q._pad) * 4096;
            int pe; bool horiz;
            if (q.prev_chunk_r < q.chunk_r)      { horiz = false; pe = 63; }
            else if (q.prev_chunk_r > q.chunk_r) { horiz = false; pe = 0;  }
            else if (q.prev_chunk_c < q.chunk_c) { horiz = true;  pe = 63; }
            else                                 { horiz = true;  pe = 0;  }
            uint32_t any = 0;
            for (int e = lane; e < 64; e += 32) any |= LOS_PREV_LOAD(horiz ? prev + e * 64 + pe : prev + pe * 64 + e);
            if (!__any_sync(0xffffffffu, any != 0)) {
                uint4 *d4 = reinterpret_cast<uint4 *>(fields + (size_t)(out_slot ? out_slot[i] : i) * 4096);
                for (int j = lane; j < 256; j += 32) d4[j] = make_uint4(0, 0, 0, 0);
                __threadfence();
                __syncwarp();
                if (lane == 0) {
                    *(volatile int *)(done + i) = 1;
                    if (trace) {
                        unsigned long long t_done; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_done));
                        trace[4 * (size_t)i] = t_take; trace[4 * (size_t)i + 1] = t_ready; trace[4 * (size_t)i + 2] = t_done; trace[4 * (size_t)i + 3] = (unsigned long long)(unsigned)(q.prev_index + 1) << 32;
                    }
                }
                continue;
            }
        }
        // ---- stage tile -> bit rows (2 rows per lane) ----
#pragma unroll
        for (int rr = 0; rr < 2; rr++) {
            const int row = 2 * lane + rr;
            const size_t off = ((size_t)q.layer * g.H64 + q.chunk_r * 64 + row) * g.W64 + q.chunk_c * 64;
            const uint4 *pc = reinterpret_cast<const uint4 *>(g.cost + off);
            const uint4 *pb = reinterpret_cast<const uint4 *>(g.blk + off);
            uint64_t p = 0, blocked = 0, gt1 = 0;
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint4 v = __ldg(pc + j);
                uint32_t imp, n1;
                cost16_bits(v, imp, n1);
                p |= (uint64_t)((~imp) & 0xFFFFu) << (16 * j);
                // cost > 1  <=>  cost not in {0, 1}
                const uint32_t w[4] = {v.x, v.y, v.z, v.w};
                uint32_t g1 = 0;
#pragma unroll
                for (int e = 0; e < 4; e++)
                    g1 |= bytemask_to_bits(__vcmpgtu4(w[e], 0x01010101u)) << (4 * e);
                gt1 |= (uint64_t)g1 << (16 * j);
            }
#pragma unroll
            for (int j = 0; j < 8; j++) blocked |= (uint64_t)blk8_bits(__ldg(pb + j)) << (8 * j);
            // an "attacking" request (dest_id carries a faction, field.c:2095) walks over tiles blocked only by its
            // enemies (field_tile_passable_no_enemies, field.c:179); the corner test keeps the plain rule (field.c:435)
            uint64_t blocked_f = blocked;
            if (q.faction_id != PFNAV_FACTION_ID_NONE && blocked) {
                const uint16_t en = g.enemies[q.faction_id & 0xF];
                const uint16_t *pf = g.fmask + off;
                for (uint64_t rest = blocked; rest; rest &= rest - 1) {
                    const int c = __ffsll((long long)rest) - 1;
                    if ((pf[c] & ~en) == 0) blocked_f &= ~(1ull << c);
                }
            }
            s.pass[row] = p & ~blocked;
            s.open[row] = p & ~blocked_f & ~gt1;
            s.assigned[row] = 0;
            s.blk[row] = 0;
            uint4 *vz = reinterpret_cast<uint4 *>(s.visb + row * 64);
            vz[0] = make_uint4(0, 0, 0, 0); vz[1] = make_uint4(0, 0, 0, 0); vz[2] = make_uint4(0, 0, 0, 0); vz[3] = make_uint4(0, 0, 0, 0);
        }
        __syncwarp();

        unsigned npops = 0;
        if (lane == 0) {
            uint16_t *h = s.heap;
            int size = 0;
            const bool dest_chunk = (q.chunk_r == q.tgt_chunk_r && q.chunk_c == q.tgt_chunk_c);
            if (dest_chunk) {
                h[++size] = (uint16_t)((q.tgt_tile_r << 6) | q.tgt_tile_c);
                s.assigned[q.tgt_tile_r] |= 1ull << q.tgt_tile_c;
            } else {
                // carry the shared edge over from the previous chunk's field (field.c:2122-2196)
                const uint8_t *prev = fields + (size_t)(q.prev_index >= 0 ? (out_slot ? out_slot[q.prev_index] : q.prev_index) : q._pad) * 4096;
                bool horizontal; int curr_edge, prev_edge;
                if (q.prev_chunk_r < q.chunk_r)      { horizontal = false; curr_edge = 0;  prev_edge = 63; }
                else if (q.prev_chunk_r > q.chunk_r) { horizontal = false; curr_edge = 63; prev_edge = 0;  }
                else if (q.prev_chunk_c < q.chunk_c) { horizontal = true;  curr_edge = 0;  prev_edge = 63; }
                else                                 { horizontal = true;  curr_edge = 63; prev_edge = 0;  }
                for (int e = 0; e < 64; e++) {
                    const int r = horizontal ? e : curr_edge, c = horizontal ? curr_edge : e;
                    const uint8_t pv = LOS_PREV_LOAD(horizontal ? prev + e * 64 + prev_edge : prev + prev_edge * 64 + e);
                    const uint64_t bit = 1ull << c;
                    // struct assignment overwrites both flags of the edge tile
                    s.visb[r * 64 + c] = pv & 1;
                    s.blk[r] = (s.blk[r] & ~bit) | ((pv & 2) ? bit : 0);
                    if (pv & 2)
                        los_blocked_line(s, mi, q.tgt_chunk_r, q.tgt_chunk_c, q.tgt_tile_r, q.tgt_tile_c,
                                         q.chunk_r, q.chunk_c, r, c);
                    if (pv & 1) {
                        h[++size] = (uint16_t)((r << 6) | c);     // priority 0: an append, all seeds are equal
                        s.assigned[r] |= bit;
                    }
                }
            }
            while (size > 0) {
                npops++;
                const uint16_t cur = heap_pop(h, size);
                const int r = (cur >> 6) & 63, c = cur & 63;
                const uint16_t nprio = (uint16_t)((((cur >> 12) + 1) & 3) << 12);
                // every bitmap row this pop can read, loaded together (one shared-memory round trip):
                // rows r-1..r+1 of blocked/open/assigned, rows r-2..r+2 of passable (corner tests)
                const int rm = max(r - 1, 0), rp = min(r + 1, 63), rmm = max(r - 2, 0), rpp = min(r + 2, 63);
                const uint64_t b_m = s.blk[rm], b_0 = s.blk[r], b_p = s.blk[rp];
                const uint64_t o_m = s.open[rm], o_0 = s.open[r], o_p = s.open[rp];
                const uint64_t a_m = s.assigned[rm], a_0 = s.assigned[r], a_p = s.assigned[rp];
                // neighbour order of field_neighbours_grid_los: (-1,0) (0,-1) (0,+1) (+1,0). The list
                // (incl. the wavefront_blocked filter) is collected before any neighbour is processed
                // (field.c:2205): a line drawn for an earlier neighbour of this pop must not hide a later one.
                // The four neighbours are distinct tiles, so their tests are independent of each other: they are
                // evaluated branch-free side by side (this loop is one thread's dependent chain -- ILP is all
                // there is); only the rare corner / blocked-line case branches.
                const int cl = (c + 63) & 63, cg = (c + 1) & 63;          // c-1 / c+1 as shift counts
                const bool t0 = r > 0 && !((b_m >> c) & 1), t1 = c > 0 && !((b_0 >> cl) & 1);
                const bool t2 = c < 63 && !((b_0 >> cg) & 1), t3 = r < 63 && !((b_p >> c) & 1);
                const bool o0 = (o_m >> c) & 1, o1 = (o_0 >> cl) & 1, o2 = (o_0 >> cg) & 1, o3 = (o_p >> c) & 1;
                const bool v0 = t0 && o0, v1 = t1 && o1, v2 = t2 && o2, v3 = t3 && o3;     // become visible
                const bool p0 = v0 && !((a_m >> c) & 1), p1 = v1 && !((a_0 >> cl) & 1);
                const bool p2 = v2 && !((a_0 >> cg) & 1), p3 = v3 && !((a_p >> c) & 1);    // first visit: push
                const uint64_t bitc = 1ull << c;
                if (v0) s.visb[(r - 1) * 64 + c] = 1;
                if (v1) s.visb[r * 64 + cl] = 1;
                if (v2) s.visb[r * 64 + cg] = 1;
                if (v3) s.visb[(r + 1) * 64 + c] = 1;
                if (p0) s.assigned[r - 1] = a_m | bitc;
                if (p1 || p2) s.assigned[r] = a_0 | (p1 ? 1ull << cl : 0ull) | (p2 ? 1ull << cg : 0ull);
                if (p3) s.assigned[r + 1] = a_p | bitc;
                const uint16_t base0 = (uint16_t)(nprio | (r << 6) | c);
                int sz = size;
                if (p0) h[++sz] = (uint16_t)(base0 - 64);
                if (p1) h[++sz] = (uint16_t)(base0 - 1);
                if (p2) h[++sz] = (uint16_t)(base0 + 1);
                if (p3) h[++sz] = (uint16_t)(base0 + 64);
                size = sz;
                if ((t0 && !o0) | (t1 && !o1) | (t2 && !o2) | (t3 && !o3)) {
                    // an impassable (or cost > 1) neighbour that is not wavefront-blocked: field_is_los_corner
                    // (field.c:435) on the passable rows r-2..r+2, then the blocked line
                    const uint64_t p_mm = s.pass[rmm], p_m = s.pass[rm], p_0 = s.pass[r], p_p = s.pass[rp], p_pp = s.pass[rpp];
#pragma unroll
                    for (int e = 0; e < 4; e++) {
                        const bool k = e == 0 ? (t0 && !o0) : e == 1 ? (t1 && !o1) : e == 2 ? (t2 && !o2) : (t3 && !o3);
                        if (!k) continue;
                        const int rr = e == 0 ? r - 1 : e == 3 ? r + 1 : r, cc = e == 1 ? c - 1 : e == 2 ? c + 1 : c;
                        const uint64_t up = e == 0 ? p_mm : e == 3 ? p_0 : p_m;     // row rr-1
                        const uint64_t dn = e == 0 ? p_0 : e == 3 ? p_pp : p_p;     // row rr+1
                        const uint64_t me = e == 0 ? p_m : e == 3 ? p_p : p_0;      // row rr
                        bool corner = false;
                        if (rr > 0 && rr < 63) corner = (((up >> cc) ^ (dn >> cc)) & 1) != 0;
                        if (!corner && cc > 0 && cc < 63) corner = (((me >> (cc - 1)) ^ (me >> (cc + 1))) & 1) != 0;
                        if (!corner) continue;
                        los_blocked_line(s, mi, q.tgt_chunk_r, q.tgt_chunk_c, q.tgt_tile_r, q.tgt_tile_c,
                                         q.chunk_r, q.chunk_c, rr, cc);
                    }
                }
            }
        }
        __syncwarp();
        // ---- field_pad_wavefront (field.c:519): clear `visible` within 1 tile of a blocked tile ----
        uint8_t *dst = fields + (size_t)(out_slot ? out_slot[i] : i) * 4096;
#pragma unroll
        for (int rr = 0; rr < 2; rr++) {
            const int row = 2 * lane + rr;
            uint64_t b = s.blk[row];
            if (row > 0) b |= s.blk[row - 1];
            if (row < 63) b |= s.blk[row + 1];
            b = b | (b << 1) | (b >> 1);
            const uint64_t keep = ~b, w = s.blk[row];
            uint4 *d4 = reinterpret_cast<uint4 *>(dst + row * 64);
            const uint4 *v4 = reinterpret_cast<const uint4 *>(s.visb + row * 64);
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint4 vv = v4[j];
                const uint32_t vw[4] = {vv.x, vv.y, vv.z, vv.w};
                uint32_t o[4];
#pragma unroll
                for (int e = 0; e < 4; e++) {
                    const int sh = j * 16 + e * 4;
                    o[e] = (vw[e] & spread4((uint32_t)(keep >> sh))) | (spread4((uint32_t)(w >> sh)) << 1);
                }
                d4[j] = make_uint4(o[0], o[1], o[2], o[3]);
            }
        }
        __threadfence();
        __syncwarp();
        if (lane == 0) {
            *(volatile int *)(done + i) = 1;
            if (trace) {
                unsigned long long t_done; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t_done));
                trace[4 * (size_t)i] = t_take; trace[4 * (size_t)i + 1] = t_ready; trace[4 * (size_t)i + 2] = t_done; trace[4 * (size_t)i + 3] = ((unsigned long long)(unsigned)(q.prev_index + 1) << 32) | (npops + 1);
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// Host side: context + map state
// ------------------------------------------------------------------------------------------
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                    CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                    CUtensorMapFloatOOBfill);

static int make_tensor_maps(pfnav_ctx *ctx)
{
    ctx->tma_ok = false;
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres);
    if (e != cudaSuccess || !fn || qres != cudaDriverEntryPointSuccess) {
        cudaGetLastError();
        return 0;
    }
    PFN_encodeTiled enc = (PFN_encodeTiled)fn;
    cuuint64_t dims[3] = {(cuuint64_t)ctx->W64, (cuuint64_t)ctx->H64, (cuuint64_t)ctx->nlayers};
    cuuint32_t box[3] = {64, 64, 1}, estr[3] = {1, 1, 1};
    cuuint64_t str8[2] = {(cuuint64_t)ctx->W64, (cuuint64_t)ctx->W64 * ctx->H64};
    cuuint64_t str16[2] = {(cuuint64_t)ctx->W64 * 2, (cuuint64_t)ctx->W64 * ctx->H64 * 2};
    CUresult r1 = enc(&ctx->tmap_cost, CU_TENSOR_MAP_DATA_TYPE_UINT8, 3, ctx->d_cost, dims, str8, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    CUresult r2 = enc(&ctx->tmap_blk, CU_TENSOR_MAP_DATA_TYPE_UINT16, 3, ctx->d_blk, dims, str16, box, estr,
                      CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B,
                      CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    ctx->tma_ok = (r1 == CUDA_SUCCESS && r2 == CUDA_SUCCESS);
    return 0;
}

extern "C" int pfnav_create(int device, pfnav_ctx **out)
{
    if (!out) { pfnav_set_error("pfnav_create: out == NULL"); return PFNAV_ERR_ARG; }
    *out = nullptr;
    int ndev = 0;
    cudaError_t e = cudaGetDeviceCount(&ndev);
    if (e != cudaSuccess || ndev <= 0) {
        pfnav_set_error("pfnav_create: no CUDA device (%s); this library has no CPU fallback",
                        e != cudaSuccess ? cudaGetErrorString(e) : "device count 0");
        cudaGetLastError();
        return PFNAV_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= ndev) { pfnav_set_error("pfnav_create: device %d out of range", device); return PFNAV_ERR_ARG; }
    PF_CUDA(cudaSetDevice(device));
    cudaDeviceProp prop;
    PF_CUDA(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {      // sm_90a code runs on compute capability 9.0 and nothing else
        pfnav_set_error("pfnav_create: device %d is sm_%d%d; libpfnav is built for sm_90a (H100) only", device,
                        prop.major, prop.minor);
        return PFNAV_ERR_NO_DEVICE;
    }
    pfnav_ctx *ctx = new pfnav_ctx();
    ctx->device = device;
    ctx->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->tick_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&ctx->field_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaStreamCreateWithFlags(&ctx->flow_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->ev_flow, cudaEventDisableTiming) != cudaSuccess ||
        cudaEventCreate(&ctx->ev_fork) != cudaSuccess || cudaEventCreate(&ctx->ev_los) != cudaSuccess ||
        cudaEventCreate(&ctx->ev_vel0) != cudaSuccess || cudaEventCreate(&ctx->ev_vel1) != cudaSuccess ||
        cudaEventCreateWithFlags(&ctx->tick_done, cudaEventDisableTiming) != cudaSuccess) {
        pfnav_set_error("pfnav_create: stream/event creation failed");
        delete ctx;
        return PFNAV_ERR_CUDA;
    }
    int rc = pfnav_fields_init(ctx);
    if (!rc) rc = pfnav_agents_init(ctx);
    if (rc) { delete ctx; return rc; }
    *out = ctx;
    return PFNAV_OK;
}

// Host-only context: holds the host mirrors of the map so that the HOST-side structure code
// (local islands, portals, routing) can be exercised on a machine without a GPU. It has NO compute
// path: every entry point that would launch a kernel fails with PFNAV_ERR_NO_DEVICE.
extern "C" int pfnav_create_hostonly(pfnav_ctx **out)
{
    if (!out) { pfnav_set_error("pfnav_create_hostonly: out == NULL"); return PFNAV_ERR_ARG; }
    pfnav_ctx *ctx = new pfnav_ctx();
    ctx->device = -1;
    *out = ctx;
    return PFNAV_OK;
}

int pfnav_fields_init(pfnav_ctx *ctx)
{
    PF_CUDA(cudaFuncSetAttribute(k_flow_unit<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 FLOW_WARPS_PER_CTA * FLOW_SMEM_PER_WARP + 128));
    PF_CUDA(cudaFuncSetAttribute(k_los_b, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(LOS_WARPS_PER_CTA * sizeof(LosSmemB))));
    PF_CUDA(cudaFuncSetAttribute(k_los_level, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(LOS_WARPS_PER_CTA * sizeof(LosSmemB))));
    PF_CUDA(cudaFuncSetAttribute(k_los, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)(LOS_WARPS_PER_CTA * sizeof(LosSmem))));
    return 0;
}

static void free_map(pfnav_ctx *ctx)
{
    cudaFree(ctx->d_cost); cudaFree(ctx->d_blk); cudaFree(ctx->d_liid); cudaFree(ctx->d_unit); cudaFree(ctx->d_fmask);
    ctx->d_fmask = nullptr; ctx->h_fac.clear(); ctx->h_fmask.clear();
    ctx->d_cost = nullptr; ctx->d_blk = nullptr; ctx->d_liid = nullptr; ctx->d_unit = nullptr;
}

void pfnav_fields_free(pfnav_ctx *ctx)
{
    free_map(ctx);
    pf_pool_free(ctx);
    if (ctx->ev_los_sched) { cudaEventDestroy(ctx->ev_los_sched); ctx->ev_los_sched = nullptr; }
}

void pfnav_route_forget(pfnav_ctx *ctx);
void pfnav_route_invalidate_layer(pfnav_ctx *ctx, int layer);
void pfnav_blockers_forget(pfnav_ctx *ctx);

extern "C" void pfnav_destroy(pfnav_ctx *ctx)
{
    if (!ctx) return;
    pfnav_route_forget(ctx);
    pfnav_blockers_forget(ctx);
    pf_planner_destroy(ctx);
    if (ctx->device < 0) { delete ctx; return; }
    cudaSetDevice(ctx->device);
    cudaDeviceSynchronize();
    pf_stage_free(ctx);
    pfnav_fields_free(ctx);
    pfnav_agents_free(ctx);
    pf_events_free(ctx);
    pf_digest_free(ctx);
    if (ctx->tick_done) cudaEventDestroy(ctx->tick_done);
    if (ctx->tick_stream) cudaStreamDestroy(ctx->tick_stream);
    if (ctx->ev_vel0) cudaEventDestroy(ctx->ev_vel0);
    if (ctx->ev_vel1) cudaEventDestroy(ctx->ev_vel1);
    if (ctx->ev_fork) cudaEventDestroy(ctx->ev_fork);
    if (ctx->ev_los) cudaEventDestroy(ctx->ev_los);
    if (ctx->field_stream) cudaStreamDestroy(ctx->field_stream);
    if (ctx->ev_flow) cudaEventDestroy(ctx->ev_flow);
    if (ctx->flow_stream) cudaStreamDestroy(ctx->flow_stream);
    delete ctx;
}

// Per-kernel-group device timings, for bench.py's roofline line. ms_out/count_out: PF_PROF_SLOTS (8)
// entries: 0 flow, 1 LOS, 2 index build, 3 desired velocity, 4 cohesion, 5 agent velocity.
extern "C" int pfnav_profile_enable(pfnav_ctx *ctx, int enable)
{
    PF_ARG(ctx, "ctx");
    ctx->profiling = enable != 0;
    return PFNAV_OK;
}

extern "C" int pfnav_profile_read(pfnav_ctx *ctx, float *ms_out, uint32_t *count_out)
{
    PF_ARG(ctx && ms_out && count_out, "args");
    PF_CUDA(cudaSetDevice(ctx->device));
    for (int i = 0; i < PF_PROF_SLOTS; i++) { ms_out[i] = 0.f; count_out[i] = 0; }
    for (auto &r : ctx->prof_pending) {
        float ms = 0.f;
        cudaEventSynchronize(r.b);
        if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) { ms_out[r.slot] += ms; count_out[r.slot]++; }
        cudaEventDestroy(r.a); cudaEventDestroy(r.b);
    }
    ctx->prof_pending.clear();
    cudaGetLastError();
    return PFNAV_OK;
}

extern "C" int pfnav_profile_read_host(pfnav_ctx *ctx, double *ms_out, uint32_t *count_out)
{
    PF_ARG(ctx && ms_out && count_out, "args");
    for (int i = 0; i < PF_HPROF_SLOTS; i++) {
        ms_out[i] = ctx->host_ms[i]; count_out[i] = ctx->host_count[i];
        ctx->host_ms[i] = 0.0; ctx->host_count[i] = 0;
    }
    return PFNAV_OK;
}

extern "C" int pfnav_set_tma(pfnav_ctx *ctx, int enable)
{
    PF_ARG(ctx, "ctx");
    ctx->use_tma = enable != 0;
    return PFNAV_OK;
}

extern "C" int pfnav_map_create(pfnav_ctx *ctx, int chunk_w, int chunk_h, int nlayers, float map_x, float map_z)
{
    PF_ARG(ctx, "ctx");
    PF_ARG(chunk_w > 0 && chunk_h > 0 && chunk_w <= 64 && chunk_h <= 64, "chunk_w/chunk_h must be in 1..64 (dest_id has 6 bits per chunk coordinate, nav.c:841)");
    PF_ARG(nlayers > 0 && nlayers <= PFNAV_NAV_LAYER_MAX, "nlayers");
    ctx->map_epoch++;
    // structures derived from the previous map (dirty sets, routes, per-faction counts) do not carry over
    pfnav_route_forget(ctx);
    pfnav_blockers_forget(ctx);
    ctx->h_fac.clear(); ctx->h_fmask.clear();
    // the field pool is sized ndests x (chunks of the OLD map): it does not carry over either
    if (int rc = pf_pool_free(ctx)) return rc;
    ctx->aux.clear();
    ctx->chunk_w = chunk_w; ctx->chunk_h = chunk_h; ctx->nlayers = nlayers;
    ctx->W64 = chunk_w * 64; ctx->H64 = chunk_h * 64;
    ctx->map_x = map_x; ctx->map_z = map_z;
    const size_t tiles = (size_t)ctx->W64 * ctx->H64 * nlayers;
    if (ctx->device < 0) {
        ctx->d_cost = reinterpret_cast<uint8_t *>(1);      // "map created" marker; never dereferenced
        ctx->h_unit.assign((size_t)chunk_w * chunk_h * nlayers, 1);
        ctx->h_cost.assign(tiles, 0xFF); ctx->h_blk.assign(tiles, 0); ctx->h_liid.assign(tiles, 0xFFFF);
        ctx->portals.assign(nlayers, {});
        return PFNAV_OK;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    free_map(ctx);
    PF_CUDA(cudaMalloc(&ctx->d_cost, tiles));
    PF_CUDA(cudaMalloc(&ctx->d_blk, tiles * 2));
    PF_CUDA(cudaMalloc(&ctx->d_liid, tiles * 2));
    PF_CUDA(cudaMalloc(&ctx->d_unit, (size_t)chunk_w * chunk_h * nlayers));
    PF_CUDA(cudaMemset(ctx->d_cost, 0xFF, tiles));
    PF_CUDA(cudaMemset(ctx->d_blk, 0, tiles * 2));
    PF_CUDA(cudaMemset(ctx->d_liid, 0xFF, tiles * 2));
    PF_CUDA(cudaMalloc(&ctx->d_fmask, tiles * 2));
    PF_CUDA(cudaMemset(ctx->d_fmask, 0, tiles * 2));
    PF_CUDA(cudaMemset(ctx->d_unit, 1, (size_t)chunk_w * chunk_h * nlayers));
    ctx->h_unit.assign((size_t)chunk_w * chunk_h * nlayers, 1);
    ctx->h_cost.assign(tiles, 0xFF);
    ctx->h_blk.assign(tiles, 0);
    ctx->h_liid.assign(tiles, 0xFFFF);
    ctx->portals.assign(nlayers, {});
    make_tensor_maps(ctx);
    return PFNAV_OK;
}

extern "C" int pfnav_map_set_pos(pfnav_ctx *ctx, float map_x, float map_z)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    if (ctx->map_x != map_x || ctx->map_z != map_z) { ctx->map_x = map_x; ctx->map_z = map_z; ctx->map_epoch++; ctx->arrival_valid = false; }
    return PFNAV_OK;
}

static int refresh_unit_flags(pfnav_ctx *ctx, int layer)
{
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
    k_unit_flags<<<(chunks * 32 + 127) / 128, 128>>>(ctx->d_cost + ltiles * layer, ctx->d_unit + (size_t)chunks * layer,
                                                     ctx->chunk_w, ctx->chunk_h);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaMemcpy(ctx->h_unit.data() + (size_t)chunks * layer, ctx->d_unit + (size_t)chunks * layer, chunks,
                       cudaMemcpyDeviceToHost));
    return 0;
}

extern "C" int pfnav_map_upload_layer(pfnav_ctx *ctx, int layer, const uint8_t *cost_base, const uint16_t *blockers,
                                      const uint16_t *local_islands)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG(cost_base, "cost_base");
    { int rc = pfnav_blockers_flush(ctx); if (rc) return rc; }     // queued refcount operations come first
    ctx->map_epoch++;
    // new costs: the portal edges / travel index / global islands built from the old ones are void. (The structural
    // build re-uploads the layer from the mirrors themselves: same costs, tables stay.)
    if (cost_base != ctx->h_cost.data() + (size_t)ctx->W64 * ctx->H64 * layer) pfnav_route_invalidate_layer(ctx, layer);
    const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
    if (ctx->device < 0) {
        memmove(ctx->h_cost.data() + ltiles * layer, cost_base, ltiles);
        if (blockers) memmove(ctx->h_blk.data() + ltiles * layer, blockers, ltiles * 2);
        else std::fill(ctx->h_blk.begin() + ltiles * layer, ctx->h_blk.begin() + ltiles * (layer + 1), 0);
        if (local_islands) memmove(ctx->h_liid.data() + ltiles * layer, local_islands, ltiles * 2);
        return PFNAV_OK;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());     // the kernels below run on the default stream: nothing may still read the old grids
    int rc = ctx->d_stage.reserve(ltiles * 2);
    if (rc) return rc;
    const int nblk = std::min<size_t>((ltiles + 255) / 256, (size_t)ctx->sm_count * 8);
    memmove(ctx->h_cost.data() + ltiles * layer, cost_base, ltiles);      // callers may pass the mirrors themselves
    if (blockers) memmove(ctx->h_blk.data() + ltiles * layer, blockers, ltiles * 2);
    else std::fill(ctx->h_blk.begin() + ltiles * layer, ctx->h_blk.begin() + ltiles * (layer + 1), 0);
    if (local_islands) memmove(ctx->h_liid.data() + ltiles * layer, local_islands, ltiles * 2);
    PF_CUDA(cudaMemcpy(ctx->d_stage, cost_base, ltiles, cudaMemcpyHostToDevice));
    k_deblock<uint8_t><<<nblk, 256>>>((const uint8_t *)ctx->d_stage.p, ctx->d_cost + ltiles * layer, ctx->chunk_w, ctx->chunk_h);
    ctx->launches++;
    if (blockers) {
        PF_CUDA(cudaMemcpy(ctx->d_stage, blockers, ltiles * 2, cudaMemcpyHostToDevice));
        k_deblock<uint16_t><<<nblk, 256>>>((const uint16_t *)ctx->d_stage.p, ctx->d_blk + ltiles * layer, ctx->chunk_w, ctx->chunk_h);
        ctx->launches++;
    } else {
        PF_CUDA(cudaMemset(ctx->d_blk + ltiles * layer, 0, ltiles * 2));
    }
    if (local_islands) {
        PF_CUDA(cudaMemcpy(ctx->d_stage, local_islands, ltiles * 2, cudaMemcpyHostToDevice));
        k_deblock<uint16_t><<<nblk, 256>>>((const uint16_t *)ctx->d_stage.p, ctx->d_liid + ltiles * layer, ctx->chunk_w, ctx->chunk_h);
        ctx->launches++;
    }
    PF_CUDA(cudaGetLastError());
    return refresh_unit_flags(ctx, layer);
}

// N_NewCtxForMapData's cost pass for one layer (nav.c:2311-2336), on the device.
extern "C" int pfnav_map_cost_from_tiles(pfnav_ctx *ctx, int layer, int ref_layer, const void *const *chunk_tiles,
                                         size_t tile_stride)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG(ref_layer >= 0 && ref_layer < PFNAV_NAV_LAYER_MAX, "ref_layer");
    PF_ARG(chunk_tiles && tile_stride >= 16, "chunk_tiles / tile_stride");
    { int rc = pfnav_blockers_flush(ctx); if (rc) return rc; }     // queued refcount operations come first
    PF_CUDA(cudaSetDevice(ctx->device));
    const int W32 = ctx->chunk_w * 32, H32 = ctx->chunk_h * 32;
    const size_t ntiles = (size_t)W32 * H32, ltiles = (size_t)ctx->W64 * ctx->H64;
    // pack the head of the engine's `struct tile` (tile.h:101: bool pathable @0, enum type @4,
    // int base_height @8, int ramp_height @12) into 4-byte records, de-blocking the chunks
    std::vector<char4> packed(ntiles);
    for (int cr = 0; cr < ctx->chunk_h; cr++)
        for (int cc = 0; cc < ctx->chunk_w; cc++) {
            const uint8_t *base = (const uint8_t *)chunk_tiles[cr * ctx->chunk_w + cc];
            PF_ARG(base, "chunk_tiles[i] is NULL");
            for (int t = 0; t < 1024; t++) {
                const uint8_t *rec = base + (size_t)t * tile_stride;
                int32_t type, bh, rh;
                memcpy(&type, rec + 4, 4); memcpy(&bh, rec + 8, 4); memcpy(&rh, rec + 12, 4);
                PF_ARG(type >= 0 && type <= 12, "tile type outside enum tiletype (tile.h:58-73)");
                PF_ARG(bh >= -128 && bh <= 127 && rh >= -128 && rh <= 127, "tile height outside int8 range");
                packed[(size_t)(cr * 32 + (t >> 5)) * W32 + cc * 32 + (t & 31)] =
                    make_char4((char)(rec[0] != 0), (char)type, (char)bh, (char)rh);
            }
        }
    int rc = ctx->d_stage.reserve(std::max(ntiles * 4, ltiles * 2));
    if (rc) return rc;
    ctx->map_epoch++;
    PF_CUDA(cudaMemcpy(ctx->d_stage, packed.data(), ntiles * 4, cudaMemcpyHostToDevice));
    dim3 blk(32, 8), grd((W32 + 31) / 32, (H32 + 7) / 8);
    k_cost_from_tiles<<<grd, blk>>>((const char4 *)ctx->d_stage.p, ctx->d_cost + ltiles * layer, W32, H32, ref_layer / 4);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaMemset(ctx->d_blk + ltiles * layer, 0, ltiles * 2));       // nav.c:2332
    std::fill(ctx->h_blk.begin() + ltiles * layer, ctx->h_blk.begin() + ltiles * (layer + 1), 0);
    // host mirror (chunk-blocked) for the route planner
    std::vector<uint8_t> img(ltiles);
    PF_CUDA(cudaMemcpy(img.data(), ctx->d_cost + ltiles * layer, ltiles, cudaMemcpyDeviceToHost));
    uint8_t *hc = ctx->h_cost.data() + ltiles * layer;
    for (int cr = 0; cr < ctx->chunk_h; cr++)
        for (int cc = 0; cc < ctx->chunk_w; cc++)
            for (int r = 0; r < 64; r++)
                memcpy(hc + ((size_t)cr * ctx->chunk_w + cc) * 4096 + r * 64,
                       img.data() + (size_t)(cr * 64 + r) * ctx->W64 + cc * 64, 64);
    return refresh_unit_flags(ctx, layer);
}

// Packed read-back of one layer's DEVICE grids (N_CopyCostBasePacked / N_CopyBlockersPacked layout,
// nav.c:2432, 2462). Any pointer may be NULL.
extern "C" int pfnav_map_get_layer(pfnav_ctx *ctx, int layer, uint8_t *cost_base, uint16_t *blockers,
                                   uint16_t *local_islands)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    { int rc = pfnav_blockers_flush(ctx); if (rc) return rc; }
    PF_CUDA(cudaSetDevice(ctx->device));
    const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
    std::vector<uint16_t> img(ltiles);
    auto reblock = [&](auto *dst, const auto *src) {
        for (int cr = 0; cr < ctx->chunk_h; cr++)
            for (int cc = 0; cc < ctx->chunk_w; cc++)
                for (int r = 0; r < 64; r++)
                    memcpy(dst + ((size_t)cr * ctx->chunk_w + cc) * 4096 + r * 64,
                           src + (size_t)(cr * 64 + r) * ctx->W64 + cc * 64, 64 * sizeof(*dst));
    };
    if (cost_base) {
        PF_CUDA(cudaMemcpy(img.data(), ctx->d_cost + ltiles * layer, ltiles, cudaMemcpyDeviceToHost));
        reblock(cost_base, (const uint8_t *)img.data());
    }
    if (blockers) {
        PF_CUDA(cudaMemcpy(img.data(), ctx->d_blk + ltiles * layer, ltiles * 2, cudaMemcpyDeviceToHost));
        reblock(blockers, (const uint16_t *)img.data());
    }
    if (local_islands) {
        PF_CUDA(cudaMemcpy(img.data(), ctx->d_liid + ltiles * layer, ltiles * 2, cudaMemcpyDeviceToHost));
        reblock(local_islands, (const uint16_t *)img.data());
    }
    return PFNAV_OK;
}

// chunk->factions (nav_data.h): direct upload of the per-faction blocker refcounts of one layer,
// [chunk][15][64][64] u8 (what N_BlockersIncref accumulates, nav.c:1032).
extern "C" int pfnav_map_upload_factions(pfnav_ctx *ctx, int layer, const uint8_t *factions)
{
    PF_ARG(ctx && ctx->d_cost && factions, "map not created / null");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    { int rc = pfnav_blockers_flush(ctx); if (rc) return rc; }     // queued refcount operations come first
    const size_t chunks = (size_t)ctx->chunk_w * ctx->chunk_h, ltiles = chunks * 4096;
    if (ctx->h_fac.size() < (size_t)ctx->nlayers) ctx->h_fac.resize(ctx->nlayers);
    if (ctx->h_fmask.size() < ltiles * ctx->nlayers) ctx->h_fmask.assign(ltiles * ctx->nlayers, 0);
    ctx->h_fac[layer].assign(factions, factions + ltiles * 15);
    uint16_t *fm = ctx->h_fmask.data() + ltiles * layer;
    for (size_t ch = 0; ch < chunks; ch++)
        for (int t = 0; t < 4096; t++) {
            uint16_t m = 0;
            for (int f = 0; f < 15; f++) if (factions[(ch * 15 + f) * 4096 + t]) m |= (uint16_t)(1u << f);
            fm[ch * 4096 + t] = m;
        }
    ctx->map_epoch++;
    if (ctx->device < 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    int rc = ctx->d_stage.reserve(ltiles * 2);
    if (rc) return rc;
    PF_CUDA(cudaMemcpy(ctx->d_stage, fm, ltiles * 2, cudaMemcpyHostToDevice));
    const int nblk = (int)std::min<size_t>((ltiles + 255) / 256, (size_t)ctx->sm_count * 8);
    k_deblock<uint16_t><<<nblk, 256>>>((const uint16_t *)ctx->d_stage.p, ctx->d_fmask + ltiles * layer, ctx->chunk_w, ctx->chunk_h);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaDeviceSynchronize());
    return pfnav_blockers_factions_uploaded(ctx, layer);
}

// Push the faction masks of one chunk after blocker refcount changes (called by pfnav_map_commit).
int pfnav_fmask_push_chunk(pfnav_ctx *ctx, int layer, int chunk)
{
    if (ctx->device < 0 || ctx->h_fmask.empty()) return PFNAV_OK;
    const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
    const int cr = chunk / ctx->chunk_w, cc = chunk % ctx->chunk_w;
    PF_CUDA(cudaMemcpy2D(ctx->d_fmask + ltiles * layer + (size_t)cr * 64 * ctx->W64 + cc * 64, ctx->W64 * 2,
                         ctx->h_fmask.data() + ltiles * layer + (size_t)chunk * 4096, 128, 128, 64, cudaMemcpyHostToDevice));
    return PFNAV_OK;
}

// G_GetEnemyFactions (game.h:184): the factions at war with `faction_id`, bit i = faction i.
extern "C" int pfnav_set_enemy_factions(pfnav_ctx *ctx, int faction_id, uint16_t enemies_mask)
{
    PF_ARG(ctx, "ctx");
    PF_ARG(faction_id >= 0 && faction_id < 15, "faction_id");
    ctx->enemies[faction_id] = enemies_mask;
    ctx->faction_enabled = true;
    ctx->map_epoch++;
    return PFNAV_OK;
}

extern "C" int pfnav_map_update_chunk(pfnav_ctx *ctx, int layer, int chunk_r, int chunk_c, const uint8_t *cost_base,
                                      const uint16_t *blockers, const uint16_t *local_islands)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG(chunk_r >= 0 && chunk_r < ctx->chunk_h && chunk_c >= 0 && chunk_c < ctx->chunk_w, "chunk coords");
    { int rc = pfnav_blockers_flush(ctx); if (rc) return rc; }     // queued refcount operations come first
    ctx->map_epoch++;
    const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
    const size_t off = ltiles * layer + (size_t)chunk_r * 64 * ctx->W64 + chunk_c * 64;
    const size_t hoff = ltiles * layer + ((size_t)chunk_r * ctx->chunk_w + chunk_c) * 4096;
    if (cost_base) memmove(ctx->h_cost.data() + hoff, cost_base, 4096);
    if (blockers) memmove(ctx->h_blk.data() + hoff, blockers, 8192);
    if (local_islands) memmove(ctx->h_liid.data() + hoff, local_islands, 8192);
    if (ctx->device < 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());     // synchronous copies below are not ordered against the (non-blocking) work streams
    if (cost_base)
        PF_CUDA(cudaMemcpy2D(ctx->d_cost + off, ctx->W64, cost_base, 64, 64, 64, cudaMemcpyHostToDevice));
    if (blockers)
        PF_CUDA(cudaMemcpy2D(ctx->d_blk + off, ctx->W64 * 2, blockers, 128, 128, 64, cudaMemcpyHostToDevice));
    if (local_islands)
        PF_CUDA(cudaMemcpy2D(ctx->d_liid + off, ctx->W64 * 2, local_islands, 128, 128, 64, cudaMemcpyHostToDevice));
    if (cost_base) {
        bool unit = true;
        for (int i = 0; i < 4096; i++) unit &= (cost_base[i] == 1 || cost_base[i] == 0xFF);
        const size_t idx = (size_t)ctx->chunk_w * ctx->chunk_h * layer + chunk_r * ctx->chunk_w + chunk_c;
        uint8_t u = unit ? 1 : 0;
        ctx->h_unit[idx] = u;
        PF_CUDA(cudaMemcpy(ctx->d_unit + idx, &u, 1, cudaMemcpyHostToDevice));
    }
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// Host side: flow / LOS batch APIs
// ------------------------------------------------------------------------------------------
static FlowGrids grids_of(const pfnav_ctx *ctx)
{
    FlowGrids g;
    g.cost = ctx->d_cost; g.blk = ctx->d_blk; g.liid = ctx->d_liid; g.unit = ctx->d_unit;
    g.W64 = ctx->W64; g.H64 = ctx->H64; g.chunk_w = ctx->chunk_w; g.chunk_h = ctx->chunk_h;
    g.fmask = ctx->d_fmask;
    for (int f = 0; f < 16; f++) g.enemies[f] = ctx->enemies[f];
    return g;
}

int pfnav_flow_launch(pfnav_ctx *ctx, const pfnav_field_req *d_reqs, size_t n, uint8_t *d_inout_fields,
                      const int32_t *d_out_slot, void *stream);

extern "C" int pfnav_flow_fields_update_dev(pfnav_ctx *ctx, const pfnav_field_req *d_reqs, size_t n,
                                            uint8_t *d_inout_fields, void *stream)
{
    return pfnav_flow_launch(ctx, d_reqs, n, d_inout_fields, nullptr, stream);
}

int pfnav_flow_launch(pfnav_ctx *ctx, const pfnav_field_req *d_reqs, size_t n, uint8_t *d_inout_fields,
                      const int32_t *d_out_slot, void *stream)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(d_reqs && d_inout_fields, "null buffer");
    PF_ARG(n < (1u << 30), "n");
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    const FlowGrids g = grids_of(ctx);
    pf_prof_scope prof(ctx, st, PF_PROF_FLOW);
    // persistent-style grid: a multiple of the SM count (2 CTAs of 8 warps fit per SM)
    const int ctas_needed = (int)((n + FLOW_WARPS_PER_CTA - 1) / FLOW_WARPS_PER_CTA);
    const int grid = std::max(1, std::min(ctas_needed, ctx->sm_count * 2 * 4));
    if (ctx->use_tma && ctx->tma_ok) {
        const size_t smem = FLOW_WARPS_PER_CTA * FLOW_SMEM_PER_WARP + 128;
        k_flow_unit<true><<<grid, FLOW_WARPS_PER_CTA * 32, smem, st>>>(ctx->tmap_cost, ctx->tmap_blk, g, d_reqs, (int)n,
                                                                      d_inout_fields, d_out_slot);
    } else {
        k_flow_unit<false><<<grid, FLOW_WARPS_PER_CTA * 32, 0, st>>>(ctx->tmap_cost, ctx->tmap_blk, g, d_reqs, (int)n,
                                                                    d_inout_fields, d_out_slot);
    }
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    bool any_nonunit = false;
    for (uint8_t u : ctx->h_unit) any_nonunit |= (u == 0);
    if (any_nonunit || ctx->faction_enabled) {
        const int gridg = (int)std::min<size_t>(n, (size_t)ctx->sm_count * 8);
        k_flow_general<<<gridg, FLOWG_THREADS, 0, st>>>(g, d_reqs, (int)n, d_inout_fields, d_out_slot, 1);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    return PFNAV_OK;
}

// Test hook: force every request through the general-cost kernel (cross-checks the two paths).
extern "C" int pfnav_flow_fields_update_general_dev(pfnav_ctx *ctx, const pfnav_field_req *d_reqs, size_t n,
                                                    uint8_t *d_inout_fields, void *stream)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(d_reqs && d_inout_fields, "null buffer");
    PF_ARG(n < (1u << 30), "n");
    PF_CUDA(cudaSetDevice(ctx->device));
    const int gridg = (int)std::min<size_t>(n, (size_t)ctx->sm_count * 8);
    k_flow_general<<<gridg, FLOWG_THREADS, 0, pf_stream(ctx, stream)>>>(grids_of(ctx), d_reqs, (int)n, d_inout_fields, nullptr, 0);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}

static int validate_field_reqs(const pfnav_ctx *ctx, const pfnav_field_req *reqs, size_t n)
{
    for (size_t i = 0; i < n; i++) {
        const pfnav_field_req &q = reqs[i];
        PF_ARG(q.layer >= 0 && q.layer < ctx->nlayers, "field req: layer");
        PF_ARG(q.chunk_r >= 0 && q.chunk_r < ctx->chunk_h && q.chunk_c >= 0 && q.chunk_c < ctx->chunk_w, "field req: chunk");
        PF_ARG(q.faction_id == PFNAV_FACTION_ID_NONE || (q.faction_id >= 0 && q.faction_id < 15 && ctx->faction_enabled),
               "field req: faction_id (attacking requests need pfnav_set_enemy_factions first)");
        if (q.target_type == PFNAV_TARGET_TILE) {
            PF_ARG(q.tile_r >= 0 && q.tile_r < 64 && q.tile_c >= 0 && q.tile_c < 64, "field req: tile");
        } else if (q.target_type == PFNAV_TARGET_PORTAL) {
            PF_ARG(q.port_r0 >= 0 && q.port_r0 <= q.port_r1 && q.port_r1 < 64 && q.port_c0 >= 0 && q.port_c0 <= q.port_c1 && q.port_c1 < 64, "field req: portal endpoints");
            PF_ARG(q.next_r0 >= 0 && q.next_r0 <= q.next_r1 && q.next_r1 < 64 && q.next_c0 >= 0 && q.next_c0 <= q.next_c1 && q.next_c1 < 64, "field req: next endpoints");
            PF_ARG(abs(q.next_chunk_r - q.chunk_r) + abs(q.next_chunk_c - q.chunk_c) == 1, "field req: next chunk must be adjacent");
        } else {
            PF_ARG(false, "field req: target_type");
        }
    }
    return 0;
}

extern "C" int pfnav_flow_fields_update(pfnav_ctx *ctx, const pfnav_field_req *reqs, size_t n, uint8_t *inout_fields)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(reqs && inout_fields, "null buffer");
    int rc = validate_field_reqs(ctx, reqs, n);
    if (rc) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->tick_stream;
    // staged: the requests, then the fields, which go up only when a request updates its field in place
    bool need_in = false;
    for (size_t i = 0; i < n; i++) need_in |= (reqs[i].init == 0);
    const size_t b_req = n * sizeof(pfnav_field_req), a_f = (b_req + 15) & ~(size_t)15, b_f = n * 4096;
    pf_stage S;
    if ((rc = pf_stage_begin(ctx, st, need_in ? a_f + b_f : b_req, a_f + b_f, false, &S))) return rc;
    memcpy(S.host, reqs, b_req);
    if (need_in) memcpy(S.host + a_f, inout_fields, b_f);
    if ((rc = pf_stage_upload(ctx, st, S, need_in ? a_f + b_f : b_req))) return rc;
    if ((rc = pfnav_flow_launch(ctx, (const pfnav_field_req *)S.dev, n, S.dev + a_f, nullptr, st))) return rc;
    PF_CUDA(cudaMemcpyAsync(inout_fields, S.dev + a_f, b_f, cudaMemcpyDeviceToHost, st));
    if ((rc = pf_stage_done(ctx, st))) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

// Repair chain of N_DesiredPointSeekVelocity (nav.c:3508-3554) applied to caller-held fields, in place.
extern "C" int pfnav_flow_fields_repair(pfnav_ctx *ctx, const pfnav_field_req *targets, const int32_t *kinds,
                                        const int32_t *args, size_t n, uint8_t *inout_fields)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(targets && kinds && args && inout_fields, "null buffer");
    int rc = validate_field_reqs(ctx, targets, n);
    if (rc) return rc;
    std::vector<pf_chain_item> items(n);
    std::vector<uint64_t> masks;
    for (size_t i = 0; i < n; i++) {
        PF_ARG(kinds[i] == PFNAV_REPAIR_NEAREST_PATHABLE || kinds[i] == PFNAV_REPAIR_ISLAND_TO_NEAREST, "repair kind");
        pf_chain_item &it = items[i];
        it.q = targets[i]; it.slot = (int32_t)i; it.tile = 0; it.kind = kinds[i]; it.arg = args[i]; it.always = 1;
        if ((rc = pf_chain_item_seeds(ctx, it, masks))) return rc;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->tick_stream;
    if ((rc = pfnav_repair_chain_launch(ctx, st, items, masks, inout_fields, n, nullptr))) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

// The wave arguments stay for the ABI and are only checked: the requests are dependency-sorted, and the kernel schedules
// them itself.
extern "C" int pfnav_los_fields_create_dev(pfnav_ctx *ctx, const pfnav_los_req *d_reqs, size_t n, uint8_t *d_out_fields,
                                           int n_waves, const int32_t *h_wave_offsets, void *stream)
{
    if (n) {
        PF_ARG(n_waves >= 1 && h_wave_offsets, "null buffer");
        PF_ARG(h_wave_offsets[0] == 0 && (size_t)h_wave_offsets[n_waves] == n, "wave offsets must run from 0 to n");
        for (int w = 0; w < n_waves; w++) PF_ARG(h_wave_offsets[w] <= h_wave_offsets[w + 1], "wave offsets must not decrease");
    }
    return pfnav_los_launch(ctx, d_reqs, n, d_out_fields, nullptr, stream);
}

int pfnav_los_launch(pfnav_ctx *ctx, const pfnav_los_req *d_reqs, size_t n, uint8_t *d_out_fields,
                     const int32_t *d_out_slot, void *stream)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(d_reqs && d_out_fields, "null buffer");
    PF_CUDA(cudaSetDevice(ctx->device));
    const FlowGrids g = grids_of(ctx);
    LosMapInfo mi{ctx->map_x, ctx->map_z};
    const size_t smem = LOS_WARPS_PER_CTA * (ctx->los_variant != 0 ? sizeof(LosSmemB) : sizeof(LosSmem));
    cudaStream_t st = pf_stream(ctx, stream);
    // scheduler state: [counter][done flags]. ONE buffer per context: the warps of a launch spin on its flags, so a
    // later launch (on any stream) must not reset or free it while an earlier one is still running -- every launch
    // is ordered after the previous one through ev_los_sched, and growing the buffer waits for the whole device.
    if (!ctx->ev_los_sched) PF_CUDA(cudaEventCreateWithFlags(&ctx->ev_los_sched, cudaEventDisableTiming));
    else PF_CUDA(cudaStreamWaitEvent(st, ctx->ev_los_sched, 0));
    if (int rc = ctx->d_los_sched.reserve(n + 1)) return rc;
    PF_CUDA(cudaMemsetAsync(ctx->d_los_sched, 0, (n + 1) * sizeof(int), st));
    if (ctx->los_trace_on)
        if (int rc = ctx->d_los_trace.reserve(n * 4)) return rc;
    pf_prof_scope prof(ctx, st, PF_PROF_LOS);
    // 2 persistent CTAs per SM (117 KB of shared memory): a flow CTA (98 KB) still fits beside them, so the flow
    // waves of the same batch -- and with them every later launch, the block scheduler serves grids in order --
    // are not held up until LOS CTAs retire. The makespan is one chain's latency, not a matter of warp count.
    const int grid = std::max(1, std::min((int)((n + LOS_WARPS_PER_CTA - 1) / LOS_WARPS_PER_CTA), ctx->sm_count * 2));
    if (ctx->los_variant == 2)
        k_los_level<<<grid, LOS_WARPS_PER_CTA * 32, smem, st>>>(g, mi, d_reqs, (int)n, d_out_fields, d_out_slot,
                                                                (unsigned *)ctx->d_los_sched.p, ctx->d_los_sched + 1,
                                                                ctx->los_trace_on ? ctx->d_los_trace.p : nullptr);
    else if (ctx->los_variant == 1)
        k_los_b<<<grid, LOS_WARPS_PER_CTA * 32, smem, st>>>(g, mi, d_reqs, (int)n, d_out_fields, d_out_slot,
                                                            (unsigned *)ctx->d_los_sched.p, ctx->d_los_sched + 1,
                                                            ctx->los_trace_on ? ctx->d_los_trace.p : nullptr);
    else
        k_los<<<grid, LOS_WARPS_PER_CTA * 32, smem, st>>>(g, mi, d_reqs, (int)n, d_out_fields, d_out_slot,
                                                          (unsigned *)ctx->d_los_sched.p, ctx->d_los_sched + 1,
                                                          ctx->los_trace_on ? ctx->d_los_trace.p : nullptr);
    ctx->los_trace_n = ctx->los_trace_on ? std::min(n, ctx->d_los_trace.cap / 4) : 0;
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaEventRecord(ctx->ev_los_sched, st));
    return PFNAV_OK;
}

extern "C" int pfnav_los_fields_create(pfnav_ctx *ctx, const pfnav_los_req *reqs, size_t n, uint8_t *out_fields)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(reqs && out_fields, "null buffer");
    std::vector<size_t> inplace;
    for (size_t i = 0; i < n; i++) {
        const pfnav_los_req &q = reqs[i];
        PF_ARG(q.layer >= 0 && q.layer < ctx->nlayers, "los req: layer");
        PF_ARG(q.chunk_r >= 0 && q.chunk_r < ctx->chunk_h && q.chunk_c >= 0 && q.chunk_c < ctx->chunk_w, "los req: chunk");
        PF_ARG(q.tgt_chunk_r >= 0 && q.tgt_chunk_r < ctx->chunk_h && q.tgt_chunk_c >= 0 && q.tgt_chunk_c < ctx->chunk_w, "los req: target chunk");
        PF_ARG(q.tgt_tile_r >= 0 && q.tgt_tile_r < 64 && q.tgt_tile_c >= 0 && q.tgt_tile_c < 64, "los req: target tile");
        PF_ARG(q.faction_id == PFNAV_FACTION_ID_NONE || (q.faction_id >= 0 && q.faction_id < 15 && ctx->faction_enabled),
               "los req: faction_id (attacking requests need pfnav_set_enemy_factions first)");
        const bool dest = (q.chunk_r == q.tgt_chunk_r && q.chunk_c == q.tgt_chunk_c);
        if (dest) { PF_ARG(q.prev_index < 0, "los req: destination chunk must not name a prev field"); }
        else if (q.prev_index == PFNAV_LOS_PREV_INPLACE) {
            // N_LOSFieldCreate(..., prev) with a caller-held previous field: its bytes arrive in out_fields[i]
            PF_ARG(abs(q.prev_chunk_r - q.chunk_r) + abs(q.prev_chunk_c - q.chunk_c) == 1, "los req: prev chunk must be adjacent");
            inplace.push_back(i);
        } else {
            PF_ARG(q.prev_index >= 0 && (size_t)q.prev_index < i, "los req: prev_index must name an earlier request");
            PF_ARG(abs(q.prev_chunk_r - q.chunk_r) + abs(q.prev_chunk_c - q.chunk_c) == 1, "los req: prev chunk must be adjacent");
        }
    }
    // requests go to the device in dependency order (pfnav_waves_host.h). Staged: the packed requests, then the field
    // blocks: the caller-held previous fields first, named like pool slots (-2), then request i's output in block k + i
    const size_t k = inplace.size();
    pf_wave_pack W;
    for (size_t i = 0, j = 0; i < n; i++) {
        if (j < k && inplace[j] == i) W.los_kept(reqs[i], (int32_t)(k + i), (int32_t)j++);
        else W.los(reqs[i], (int32_t)(k + i));
    }
    const size_t a_f = W.layout(), b_in = a_f + k * 4096;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->tick_stream;
    pf_stage S;
    int rc = pf_stage_begin(ctx, st, b_in, b_in + n * 4096, false, &S);
    if (rc) return rc;
    W.pack(S.host);
    for (size_t j = 0; j < k; j++) memcpy(S.host + a_f + j * 4096, out_fields + inplace[j] * 4096, 4096);
    if ((rc = pf_stage_upload(ctx, st, S, b_in))) return rc;
    if ((rc = pfnav_los_launch(ctx, (const pfnav_los_req *)(S.dev + W.out.o_lr), n, S.dev + a_f,
                               (const int32_t *)(S.dev + W.out.o_ls), st)))
        return rc;
    PF_CUDA(cudaMemcpyAsync(out_fields, S.dev + b_in, n * 4096, cudaMemcpyDeviceToHost, st));
    if ((rc = pf_stage_done(ctx, st))) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

// Per-field trace of the last LOS launch (debug / profiling aid): for request i, out[4i..4i+3] =
// {taken, dependency satisfied, finished} in %globaltimer ns, and (prev_index + 1) << 32 | (1 + heap pops; 0 = zero-filled early out),
// the low half OR-ed with LOS_TRACE_REPLAYED (bit 31) when k_los_level's certificate failed and the field was replayed.
extern "C" int pfnav_los_trace(pfnav_ctx *ctx, int enable, unsigned long long *out, size_t cap, size_t *out_n)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_CUDA(cudaSetDevice(ctx->device));
    if (out && out_n) {
        PF_CUDA(cudaDeviceSynchronize());
        const size_t n = std::min(cap, ctx->los_trace_n);
        if (n) PF_CUDA(cudaMemcpy(out, ctx->d_los_trace, n * 4 * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
        *out_n = n;
    }
    ctx->los_trace_on = enable != 0;
    return PFNAV_OK;
}

// Test / tuning hook: 0 = bit-row LOS kernel (k_los), 1 = byte-state LOS kernel (k_los_b), 2 = level-parallel LOS
// kernel with the replay as fallback (k_los_level, the default). Same results.
extern "C" int pfnav_set_los_variant(pfnav_ctx *ctx, int variant)
{
    PF_ARG(ctx && variant >= 0 && variant <= 2, "variant");
    ctx->los_variant = variant;
    return PFNAV_OK;
}
