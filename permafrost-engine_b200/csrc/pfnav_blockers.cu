// pfnav_blockers.cu -- dynamic obstacles: host-side restatement of the blocker reference counting and
// of N_Update, pushing only the chunks that changed to the device (deltas, not whole-state re-uploads
// as the reference's GLSL path does every tick, src/game/movement.c:3894-3900).
//
// Restates (reference file:line):
//   N_BlockersIncref / N_BlockersDecref                src/navigation/nav.c:4663-4683
//   n_update_blockers_circle_{ground,water,air}        src/navigation/nav.c:1051-1127
//   n_update_blockers                                  src/navigation/nav.c:1017-1049
//   M_Tile_AllUnderCircle / M_Tile_Contour             src/map/tile.c:687-718, 759-852
//   C_CircleRectIntersection, C_PointInsideRect2D, C_LineCircleIntersection
//                                                      src/phys/collision.c:997-1027, 756-768, 960-996
//   N_Update + N_ApplyDeferredInvalidations            src/navigation/nav.c:2119-2223
//   N_FC_InvalidateAllAtChunk / ...ThroughChunk        src/navigation/fieldcache.c:460-472, 481-545
#include "pfnav_internal.cuh"
#include "pfnav_scan.cuh"
#include <algorithm>
#include <limits.h>
#include <math.h>
#include <set>
#include <string.h>
#include <unordered_map>

int pfnav_route_refresh_edges(pfnav_ctx *ctx, int layer, int chunk);      // pfnav_route.cu; -1 if routing not built

namespace {

#include "pfnav_tile_geom.cuh"

static geom geom_of(const pfnav_ctx *ctx) { return geom{ctx->map_x, ctx->map_z, ctx->chunk_w, ctx->chunk_h}; }
static bool desc_for_point(const pfnav_ctx *ctx, float px, float pz, td *out) { return desc_for_point(geom_of(ctx), px, pz, out); }

// M_Tile_AllUnderCircle (tile.c:687)
static size_t tiles_under_circle(const pfnav_ctx *ctx, v2f c, float radius, td *out, size_t maxout)
{
    const geom g = geom_of(ctx);
    td tile;
    if (!desc_for_point(g, c.x, c.z, &tile)) return 0;
    const int ntiles = (int)ceil(radius / 4);
    size_t ret = 0;
    for (int dr = -ntiles; dr <= ntiles; dr++)
        for (int dc = -ntiles; dc <= ntiles; dc++) {
            const int ar = tile.chunk_r * 64 + tile.tile_r + dr, ac = tile.chunk_c * 64 + tile.tile_c + dc;
            if (ar < 0 || ar >= ctx->chunk_h * 64 || ac < 0 || ac >= ctx->chunk_w * 64) continue;
            if (!tile_under_circle(g, ar, ac, c, radius)) continue;
            out[ret++] = {ar / 64, ac / 64, ar % 64, ac % 64};
            if (ret == maxout) return ret;
        }
    return ret;
}

// M_Tile_LineSupercoverTilesSorted (tile.c:430), for a segment that STARTS inside the map (the only
// case pfnav_blockers_*_obb accepts): Amanatides-Woo traversal in the reference's float arithmetic.
static size_t line_supercover(const pfnav_ctx *ctx, float ax, float az, float bx, float bz, td *out, size_t maxout)
{
    size_t ret = 0;
    if (maxout == 0) return 0;
    float dx = bx - ax, dz = bz - az;
    const float len = (float)sqrt(dx * dx + dz * dz);
    dx = dx / len; dz = dz / len;                                  // PFM_Vec2_Normal
    td cur;
    if (!desc_for_point(ctx, ax, az, &cur)) return 0;
    const int step_c = dx <= 0.0f ? 1 : -1;
    const int step_r = dz >= 0.0f ? 1 : -1;
    const float t_delta_x = (float)fabs(4 / dx), t_delta_z = (float)fabs(4 / dz);       // TILE_X_DIM is an int
    const float bnx = (ctx->map_x - (float)(cur.chunk_c * 256)) - (float)(cur.tile_c * 4);
    const float bnz = (ctx->map_z + (float)(cur.chunk_r * 256)) + (float)(cur.tile_r * 4);
    float t_max_x = (step_c > 0) ? (float)(fabs(ax - (bnx - 4.0f)) / fabs(dx)) : (float)(fabs(ax - bnx) / fabs(dx));
    float t_max_z = (step_r > 0) ? (float)(fabs(az - (bnz + 4.0f)) / fabs(dz)) : (float)(fabs(az - bnz) / fabs(dz));
    td fin;
    const bool ends_inside = desc_for_point(ctx, bx, bz, &fin);
    do {
        out[ret++] = cur;
        int dc = 0, dr = 0;
        if (t_max_x < t_max_z) { t_max_x = t_max_x + t_delta_x; dc = step_c; }
        else                   { t_max_z = t_max_z + t_delta_z; dr = step_r; }
        if (ends_inside && cur.chunk_r == fin.chunk_r && cur.chunk_c == fin.chunk_c && cur.tile_r == fin.tile_r && cur.tile_c == fin.tile_c)
            break;
        const int ar = cur.chunk_r * 64 + cur.tile_r + dr, ac = cur.chunk_c * 64 + cur.tile_c + dc;      // M_Tile_RelativeDesc
        if (ar < 0 || ar >= ctx->chunk_h * 64 || ac < 0 || ac >= ctx->chunk_w * 64) break;
        cur = {ar / 64, ac / 64, ar % 64, ac % 64};
    } while (ret < maxout);
    return ret;
}

// M_Tile_AllUnderObj (tile.c:594): supercover of the four bottom edges (duplicates at the corners included, as
// in the reference: the refcounts see them twice) plus every tile of the bounding tile box -- upper bounds
// EXCLUDED, tile.c:656-659 -- whose centre lies inside the rectangle (C_PointInsideRect2D, collision.c:756).
// c[4] = bottom corners obb->corners[0], [1], [5], [4] as (x, z).
static size_t tiles_under_obb(const pfnav_ctx *ctx, const v2f c[4], td *out, size_t maxout)
{
    size_t ret = 0;
    int min_r = ctx->chunk_h * 64 - 1, max_r = 0, min_c = ctx->chunk_w * 64 - 1, max_c = 0;
    // the reference starts its column minimum at {chunk_w-1, chunk_w-1} (tile.c:624): reproduce it
    int min_c_init = (ctx->chunk_w - 1) * 64 + (ctx->chunk_w - 1);
    min_c = min_c_init;
    for (int i = 0; i < 4; i++) {
        const v2f a = c[i], b = c[(i + 1) & 3];
        const size_t n = line_supercover(ctx, a.x, a.z, b.x, b.z, out + ret, maxout - ret);
        const td *d = out + ret;
        ret += n;
        if (ret == maxout) return ret;
        for (size_t j = 0; j < n; j++) {
            const int ar = d[j].chunk_r * 64 + d[j].tile_r, ac = d[j].chunk_c * 64 + d[j].tile_c;
            min_r = std::min(min_r, ar); max_r = std::max(max_r, ar);
            min_c = std::min(min_c, ac); max_c = std::max(max_c, ac);
        }
    }
    const v2f ab = {c[1].x - c[0].x, c[1].z - c[0].z}, ad = {c[3].x - c[0].x, c[3].z - c[0].z};
    const float abab = ab.x * ab.x + ab.z * ab.z, adad = ad.x * ad.x + ad.z * ad.z;
    for (int r = min_r; r < max_r; r++)
        for (int cc = min_c; cc < max_c; cc++) {
            const float bx = (ctx->map_x - (float)((cc / 64) * 256)) - (float)((cc % 64) * 4);
            const float bz = (ctx->map_z + (float)((r / 64) * 256)) + (float)((r % 64) * 4);
            const v2f ctr = {bx - 4.0f / 2.0f, bz + 4.0f / 2.0f};
            const v2f ap = {ctr.x - c[0].x, ctr.z - c[0].z};
            const float apab = ap.x * ab.x + ap.z * ab.z, apad = ap.x * ad.x + ap.z * ad.z;
            if ((apab >= 0.0f && apab <= abab) && (apad >= 0.0f && apad <= adad)) {
                out[ret++] = {r / 64, cc / 64, r % 64, cc % 64};
                if (ret == maxout) return ret;
            }
        }
    return ret;
}

// M_Tile_Contour (tile.c:759)
static size_t tiles_contour(const pfnav_ctx *ctx, size_t ntds, const td *tds, td *out, size_t maxout)
{
    if (ntds == 0) return 0;
    int minr = INT_MAX, minc = INT_MAX, maxr = INT_MIN, maxc = INT_MIN;
    for (size_t i = 0; i < ntds; i++) {
        const int ar = tds[i].chunk_r * 64 + tds[i].tile_r, ac = tds[i].chunk_c * 64 + tds[i].tile_c;
        minr = std::min(minr, ar); minc = std::min(minc, ac); maxr = std::max(maxr, ar); maxc = std::max(maxc, ac);
    }
    const int dr = maxr - minr + 1, dc = maxc - minc + 1;
    const size_t width = dc + 2, height = dr + 2;
    std::vector<uint8_t> marked(width * height, 0);
    for (size_t i = 0; i < ntds; i++) {
        const int ar = tds[i].chunk_r * 64 + tds[i].tile_r, ac = tds[i].chunk_c * 64 + tds[i].tile_c;
        marked[(ar - minr + 1) * width + (ac - minc + 1)] = 1;
    }
    size_t ret = 0;
    for (int r = minr - 1; r <= maxr + 1; r++)
        for (int c = minc - 1; c <= maxc + 1; c++) {
            if (r < 0 || r >= ctx->chunk_h * 64 || c < 0 || c >= ctx->chunk_w * 64) continue;
            const int relr = r - minr + 1, relc = c - minc + 1;
            if (marked[relr * width + relc]) continue;
            if (ret == maxout) return ret;
            bool contour = false;
            if ((relr > 0 && marked[(relr - 1) * (dc + 2) + relc]) || (relr < dr && marked[(relr + 1) * (dc + 2) + relc]) ||
                (relc > 0 && marked[relr * (dc + 2) + (relc - 1)]) || (relc < dc && marked[relr * (dc + 2) + (relc + 1)]))
                contour = true;
            if ((relr > 0 && relc > 0 && marked[(relr - 1) * (dc + 2) + (relc - 1)]) ||
                (relr > 0 && relc < dc && marked[(relr - 1) * (dc + 2) + (relc + 1)]) ||
                (relr < dr && relc > 0 && marked[(relr + 1) * (dc + 2) + (relc - 1)]) ||
                (relr < dr && relc < dc && marked[(relr + 1) * (dc + 2) + (relc + 1)]))
                contour = true;
            if (contour) out[ret++] = {r / 64, c / 64, r % 64, c % 64};
        }
    return ret;
}

// dirty (layer, chunk) sets live in the context: pfnav_ctx::dirty (occupancy changed), ::fdirty (faction mask changed)

// ------------------------------------------------------------------------------------------
// Device side. On a context with a device the refcounts live in HBM: blocker operations are queued by the
// entry points and applied by pfnav_map_commit (or the first read-back) in three launches --
//   k_blockers_circles  one warp per circle: the tiles under it and its three contour rings as 31 x 31 bit rows,
//                       counted into d_blk (u16) / d_fac (u8 per faction) with word-wide compare-and-swap;
//   k_blockers_tiles    the same counting for tile lists rasterised on the host (building footprints, circles
//                       wider than the bit window);
//   k_chunks_finish     one CTA per touched (layer, chunk): faction masks from the counts, and -- when the set of
//                       passable tiles changed -- the local islands (union-find in shared memory, islands numbered
//                       by their first tile in row-major order exactly like the reference's flood fill nav.c:1213);
// then the touched chunks come back in one copy to refresh the host mirrors the route planner reads.
// "Dirty" here means the chunk's passable set changed between two commits; the reference marks a chunk on every
// 0 <-> non-zero transition of a single count (nav.c:1038), which also fires for an obstacle that leaves and
// re-enters a tile inside one tick. Both recompute identical islands / fields; ours skips the no-op rebuilds.
// ------------------------------------------------------------------------------------------
struct tile_op { int32_t layer, ar, ac, faction, delta; };

struct blk_state {
    std::vector<pfnav_blocker_op> circles;
    std::vector<tile_op> tiles;
    pf_dbuf<uint8_t> d_fac;                 // [layer][15][H64][W64] u8, allocated with the first faction-tagged op
    pf_dbuf<uint8_t> d_touched;             // touched, ftouched and res, [nlayers * chunks] each
    uint8_t *d_ftouched = nullptr, *d_res = nullptr;
    int nslots = 0;
    pf_dbuf<uint8_t> d_ops;
    pf_dbuf<uint16_t> d_out;
    uint64_t applied_ops = 0;
    // ops decided on the device (pf_blocker_ops_*): narrow ones for k_blockers_circles, wide ones for the host rasteriser,
    // d_dev_cnt = {narrow, wide} pending; dev_bound: an upper bound of either count, known without reading them
    pfnav_blocker_op *d_dev_narrow = nullptr, *d_dev_wide = nullptr; size_t dev_cap = 0, dev_bound = 0;
    uint32_t *d_dev_cnt = nullptr;
    bool dev_pending = false, dev_fac = false;
    // member of a job that shares blockers (pfnav_mgpu_share_blockers): the leading dev_sent = {narrow, wide} pending ops
    // are held by every member since the last exchange; dev_unexchanged: ops were decided after it
    uint32_t dev_sent[2] = {0, 0};
    bool dev_unexchanged = false;
    // staging of one producer launch: 2 ops + 1 descriptor per item, a count pair and an offset pair per block
    void *d_stage = nullptr; size_t stage_items = 0;
};
static_assert(CIRCLE_MAX_NT == 12, "pf_op_wide (pfnav_internal.cuh) restates the bit window of k_blockers_circles");
static blk_state *state_of(pfnav_ctx *ctx, bool create)
{
    if (!ctx->blk_state && create) ctx->blk_state = new blk_state();
    return (blk_state *)ctx->blk_state;
}

struct apply_args {
    geom g; int nlayers, W64, H64;
    uint16_t *blk; uint8_t *fac; uint8_t *touched, *ftouched;
};

__device__ __forceinline__ void atomic_add_u16(uint16_t *p, int d)
{
    unsigned *w = (unsigned *)((uintptr_t)p & ~(uintptr_t)3);
    const int sh = ((uintptr_t)p & 2) ? 16 : 0;
    unsigned old = *w, assumed;
    do {
        assumed = old;
        const unsigned v = (((assumed >> sh) & 0xFFFFu) + (unsigned)d) & 0xFFFFu;
        old = atomicCAS(w, assumed, (assumed & ~(0xFFFFu << sh)) | (v << sh));
    } while (old != assumed);
}
__device__ __forceinline__ void atomic_add_u8(uint8_t *p, int d)
{
    unsigned *w = (unsigned *)((uintptr_t)p & ~(uintptr_t)3);
    const int sh = (int)((uintptr_t)p & 3) * 8;
    unsigned old = *w, assumed;
    do {
        assumed = old;
        const unsigned v = (((assumed >> sh) & 0xFFu) + (unsigned)d) & 0xFFu;
        old = atomicCAS(w, assumed, (assumed & ~(0xFFu << sh)) | (v << sh));
    } while (old != assumed);
}

// n_update_blockers (nav.c:1017) for one tile: `times` applications of `delta` at once
__device__ __forceinline__ void apply_tile(const apply_args &a, int layer, int ar, int ac, int faction, int d)
{
    const size_t ltiles = (size_t)a.W64 * a.H64, t = (size_t)ar * a.W64 + ac;
    atomic_add_u16(a.blk + ltiles * layer + t, d);
    const int slot = layer * (a.g.chunk_w * a.g.chunk_h) + (ar >> 6) * a.g.chunk_w + (ac >> 6);
    a.touched[slot] = 1;
    if (faction >= 0 && faction < 15) {
        atomic_add_u8(a.fac + ltiles * 15 * layer + ltiles * faction + t, d);
        a.ftouched[slot] = 1;
    }
}

__global__ void __launch_bounds__(128) k_blockers_circles(const pfnav_blocker_op *__restrict__ ops, int nops, apply_args a)
{
    __shared__ unsigned rows[4][32];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int op = blockIdx.x * 4 + w;
    if (op >= nops) return;
    const pfnav_blocker_op o = ops[op];
    const v2f c = {o.x, o.z};
    td ct;
    if (!desc_for_point(a.g, o.x, o.z, &ct)) return;           // M_Tile_AllUnderCircle returns 0 tiles (tile.c:693)
    const int nt = (int)ceil(o.range / 4);
    const int win = 2 * nt + 7;
    const int r0 = ct.chunk_r * 64 + ct.tile_r - nt - 3, c0 = ct.chunk_c * 64 + ct.tile_c - nt - 3;
    rows[w][lane] = 0;
    __syncwarp();
    circle_rows(a.g, a.H64, a.W64, c, o.range, nt, r0, c0, rows[w], lane);
    const int myr = r0 + lane;
    const unsigned inmap = window_inmap(a.H64, a.W64, r0, c0, win, lane);
    const unsigned s = rows[w][lane];
    const unsigned o3 = contour_rows(s, inmap, lane), o5 = contour_rows(o3, inmap, lane), o7 = contour_rows(o5, inmap, lane);
    const bool air = (o.flags & PFNAV_FLAG_AIR) != 0;
    for (int layer = 0; layer < a.nlayers; layer++) {
        const int grp = layer >> 2, k = layer & 3;
        if (air ? grp != 2 : grp > 1) continue;                // nav.c:1051-1127: ground + water, or air
        unsigned u = s | (k >= 1 ? o3 : 0u) | (k >= 2 ? o5 : 0u) | (k >= 3 ? o7 : 0u);
        while (u) {
            const int b = __ffs(u) - 1;
            u &= u - 1;
            const int times = (int)((s >> b) & 1u) + (k >= 1 ? (int)((o3 >> b) & 1u) : 0) + (k >= 2 ? (int)((o5 >> b) & 1u) : 0) +
                              (k >= 3 ? (int)((o7 >> b) & 1u) : 0);
            apply_tile(a, layer, myr, c0 + b, o.faction_id, o.delta * times);
        }
    }
}

__global__ void k_blockers_tiles(const tile_op *__restrict__ ops, int nops, apply_args a)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nops) return;
    const tile_op o = ops[i];
    apply_tile(a, o.layer, o.ar, o.ac, o.faction, o.delta);
}

// offsets of the producer blocks behind the ops already pending; advances the pending counts
__global__ void __launch_bounds__(1024) k_ops_offsets(const unsigned long long *__restrict__ bsum, int nb, uint32_t *cnt,
                                                      unsigned long long *__restrict__ boff)
{
    __shared__ unsigned long long warp_tot[32];
    const unsigned long long base = (unsigned long long)cnt[0] | (unsigned long long)cnt[1] << 32;
    unsigned long long carry = 0;
    for (int b0 = 0; b0 < nb; b0 += 1024) {
        const int b = b0 + threadIdx.x;
        const unsigned long long v = b < nb ? bsum[b] : 0ull;
        unsigned long long tot;
        const unsigned long long ex = pf_block_excl_scan(v, warp_tot, tot);
        if (b < nb) boff[b] = base + carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) { cnt[0] = (uint32_t)(base + carry); cnt[1] = (uint32_t)((base + carry) >> 32); }
}

// move the staged ops of each item, in item order, to the narrow / wide op buffers
__global__ void __launch_bounds__(PF_OPS_BLOCK) k_ops_compact(const pfnav_blocker_op *__restrict__ ops, const uint8_t *__restrict__ desc, int n,
                                                              const unsigned long long *__restrict__ boff,
                                                              pfnav_blocker_op *__restrict__ narrow, pfnav_blocker_op *__restrict__ wide)
{
    __shared__ unsigned long long warp_tot[PF_OPS_BLOCK / 32];
    const int i = blockIdx.x * PF_OPS_BLOCK + threadIdx.x;
    const unsigned d = i < n ? desc[i] : 0u, nops = d & 3u;
    unsigned nwide = 0;
    for (unsigned k = 0; k < nops; k++) nwide += (d >> (2 + k)) & 1u;
    // one u64 scan ranks both lists: narrow counts in the low 32 bits, wide in the high (a count never reaches 2^32)
    unsigned long long tot;
    const unsigned long long off = boff[blockIdx.x] +
        pf_block_excl_scan((unsigned long long)(nops - nwide) | (unsigned long long)nwide << 32, warp_tot, tot);
    uint32_t on = (uint32_t)off, ow = (uint32_t)(off >> 32);
    for (unsigned k = 0; k < nops; k++) {
        if ((d >> (2 + k)) & 1u) wide[ow++] = ops[2 * (size_t)i + k];
        else narrow[on++] = ops[2 * (size_t)i + k];
    }
}

__device__ __forceinline__ int uf_find(volatile int *L, int x)
{
    int p = L[x];
    while (p != x) { x = p; p = L[x]; }
    return x;
}
__device__ __forceinline__ void uf_unite(int *L, int a, int b)
{
    while (true) {
        a = uf_find(L, a); b = uf_find(L, b);
        if (a == b) return;
        if (a < b) { const int t = a; a = b; b = t; }          // link the larger root under the smaller one
        const int old = atomicMin(&L[a], b);
        if (old == a) return;
        a = old;
    }
}

struct finish_args {
    int nlayers, chunk_w, chunk_h, W64, H64;
    const uint8_t *cost; const uint16_t *blk; uint16_t *liid; const uint8_t *fac; uint16_t *fmask;
    uint8_t *touched, *ftouched, *res;
};

__global__ void __launch_bounds__(256) k_chunks_finish(finish_args a)
{
    __shared__ int L[4096];
    __shared__ uint16_t ids[4096];
    __shared__ int warp_tot[8];
    const int slot = blockIdx.x, tid = threadIdx.x;
    const bool t = a.touched[slot] != 0, ft = a.ftouched[slot] != 0;
    if (!t && !ft) { if (tid == 0) a.res[slot] = 0; return; }
    const int chunks = a.chunk_w * a.chunk_h, layer = slot / chunks, chunk = slot - layer * chunks;
    const int cr = chunk / a.chunk_w, cc = chunk - cr * a.chunk_w;
    const size_t ltiles = (size_t)a.W64 * a.H64;
    const size_t base = (size_t)cr * 64 * a.W64 + cc * 64;
    int changed = 0, fchanged = 0;
    for (int i = tid; i < 4096; i += 256) {
        const size_t off = base + (size_t)(i >> 6) * a.W64 + (i & 63);
        const bool pass = a.cost[ltiles * layer + off] != 0xFF && a.blk[ltiles * layer + off] == 0;
        changed |= (int)(pass != (a.liid[ltiles * layer + off] != 0xFFFF));
        L[i] = pass ? i : -1;
        if (ft && a.fac) {
            unsigned m = 0;
            for (int f = 0; f < 15; f++) m |= (unsigned)(a.fac[ltiles * 15 * layer + ltiles * f + off] != 0) << f;
            if (a.fmask[ltiles * layer + off] != (uint16_t)m) { a.fmask[ltiles * layer + off] = (uint16_t)m; fchanged = 1; }
        }
    }
    changed = __syncthreads_or(changed);
    fchanged = __syncthreads_or(fchanged);
    if (changed) {
        // n_update_local_islands (nav.c:1213): 4-connected components of the passable tiles
        for (int i = tid; i < 4096; i += 256) {
            if (L[i] < 0) continue;
            if ((i & 63) && L[i - 1] >= 0) uf_unite(L, i, i - 1);
            if (i >= 64 && L[i - 64] >= 0) uf_unite(L, i, i - 64);
        }
        __syncthreads();
        for (int i = tid; i < 4096; i += 256) if (L[i] >= 0) { const int r = uf_find(L, i); L[i] = r; }
        __syncthreads();
        // island ids count the roots (= the first tile of each island in scan order) from 1
        int cnt = 0;
        for (int j = 0; j < 16; j++) cnt += (int)(L[tid * 16 + j] == tid * 16 + j);
        int nroots;
        int before = pf_block_excl_scan(cnt, warp_tot, nroots);
        for (int j = 0; j < 16; j++) if (L[tid * 16 + j] == tid * 16 + j) ids[tid * 16 + j] = (uint16_t)(++before);
        __syncthreads();
        for (int i = tid; i < 4096; i += 256) {
            const size_t off = base + (size_t)(i >> 6) * a.W64 + (i & 63);
            a.liid[ltiles * layer + off] = L[i] >= 0 ? ids[L[i]] : (uint16_t)0xFFFF;
        }
    }
    if (tid == 0) {
        a.res[slot] = (uint8_t)((t ? 1 : 0) | (changed ? 2 : 0) | (fchanged ? 4 : 0));
        a.touched[slot] = 0; a.ftouched[slot] = 0;
    }
}

// the touched chunks, chunk-blocked, for the host mirrors: out[e] = {blk[4096], liid[4096]}
__global__ void __launch_bounds__(256) k_chunks_gather(const int32_t *__restrict__ slots, int chunk_w, int chunk_h, int W64, int H64,
                                                       const uint16_t *__restrict__ blk, const uint16_t *__restrict__ liid,
                                                       uint16_t *__restrict__ out)
{
    const int slot = slots[blockIdx.x], chunks = chunk_w * chunk_h, layer = slot / chunks, chunk = slot - layer * chunks;
    const int cr = chunk / chunk_w, cc = chunk - cr * chunk_w;
    const size_t off0 = (size_t)W64 * H64 * layer + (size_t)cr * 64 * W64 + cc * 64;
    uint16_t *o = out + (size_t)blockIdx.x * 8192;
    for (int i = threadIdx.x; i < 4096; i += 256) {
        const size_t off = off0 + (size_t)(i >> 6) * W64 + (i & 63);
        o[i] = blk[off]; o[4096 + i] = liid[off];
    }
}

static size_t stage_blocks(size_t items) { return (items + PF_OPS_BLOCK - 1) / PF_OPS_BLOCK; }
static size_t stage_desc_off(size_t items) { return items * 2 * sizeof(pfnav_blocker_op); }
static size_t stage_bsum_off(size_t items) { return (stage_desc_off(items) + items + 7) & ~(size_t)7; }

// d_fac of one layer from the host counts ([chunk][15][4096] -> [15][H64][W64])
static int fac_push_layer(pfnav_ctx *ctx, blk_state *st, int layer)
{
    const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
    uint8_t *dst = st->d_fac + ltiles * 15 * layer;
    if ((size_t)layer >= ctx->h_fac.size() || ctx->h_fac[layer].size() != ltiles * 15) {
        PF_CUDA(cudaMemset(dst, 0, ltiles * 15));
        return 0;
    }
    std::vector<uint8_t> img(ltiles * 15);
    const uint8_t *src = ctx->h_fac[layer].data();
    const size_t chunks = (size_t)ctx->chunk_w * ctx->chunk_h;
    for (size_t ch = 0; ch < chunks; ch++) {
        const size_t cr = ch / ctx->chunk_w, cc = ch % ctx->chunk_w;
        for (int f = 0; f < 15; f++)
            for (int r = 0; r < 64; r++)
                memcpy(img.data() + ltiles * f + (cr * 64 + r) * ctx->W64 + cc * 64, src + (ch * 15 + f) * 4096 + r * 64, 64);
    }
    PF_CUDA(cudaMemcpy(dst, img.data(), ltiles * 15, cudaMemcpyHostToDevice));
    return 0;
}

static int blockers_circle(pfnav_ctx *ctx, float x, float z, float range, int faction_id, uint32_t flags, int delta);

// Apply the queued operations on the device and bring the touched chunks' mirrors up to date; fills ctx->dirty
// (passable set changed) and ctx->fdirty (a faction mask changed) for pfnav_map_commit.
static int device_flush(pfnav_ctx *ctx)
{
    blk_state *st = state_of(ctx, false);
    if (!st || ctx->device < 0 || (st->circles.empty() && st->tiles.empty() && !st->dev_pending)) return PFNAV_OK;
    if (st->dev_unexchanged && pf_mgpu_shares_blockers(ctx)) {
        // the other members would never count these ops: their copies of the map would diverge from this one
        pfnav_set_error("device blockers: ops decided since the last exchange have not been exchanged "
                        "(pfnav_mgpu_exchange_blocker_ops / pfnav_group_exchange_blocker_ops)");
        return PFNAV_ERR_STATE;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(pf_fields_sync(ctx));         // forked LOS chains still read the map that is about to change
    // ticks / field launches on the context stream or on caller streams (all non-blocking, so not ordered against
    // the default stream used below) may still read the grids
    PF_CUDA(cudaDeviceSynchronize());
    // ops decided on the device go after the host-queued ones; the counts are additive, so where they are counted does
    // not change the result. The few wider than the bit window are read back and rasterised on the host.
    uint32_t dev_cnt[2] = {0, 0};
    if (st->dev_pending) {
        PF_CUDA(cudaMemcpy(dev_cnt, st->d_dev_cnt, sizeof(dev_cnt), cudaMemcpyDeviceToHost));
        if (dev_cnt[1]) {
            std::vector<pfnav_blocker_op> wide(dev_cnt[1]);
            PF_CUDA(cudaMemcpy(wide.data(), st->d_dev_wide, wide.size() * sizeof(pfnav_blocker_op), cudaMemcpyDeviceToHost));
            for (const pfnav_blocker_op &o : wide) blockers_circle(ctx, o.x, o.z, o.range, o.faction_id, o.flags, o.delta);
        }
    }
    const int chunks = ctx->chunk_w * ctx->chunk_h, nslots = chunks * ctx->nlayers;
    const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
    int rc;
    if (st->nslots != nslots) {
        if ((rc = st->d_touched.reserve((size_t)nslots * 3))) return rc;
        PF_CUDA(cudaMemset(st->d_touched, 0, (size_t)nslots * 3));
        st->d_ftouched = st->d_touched + nslots; st->d_res = st->d_touched + 2 * (size_t)nslots;
        st->nslots = nslots;
    }
    bool need_fac = false;
    for (const auto &o : st->circles) need_fac |= (o.faction_id >= 0 && o.faction_id < 15);
    for (const auto &o : st->tiles) need_fac |= (o.faction >= 0 && o.faction < 15);
    need_fac |= dev_cnt[0] && st->dev_fac;
    if (need_fac && !st->d_fac) {
        if ((rc = st->d_fac.reserve(ltiles * 15 * ctx->nlayers))) return rc;
        for (int l = 0; l < ctx->nlayers; l++) if ((rc = fac_push_layer(ctx, st, l))) return rc;
    }
    apply_args a;
    a.g = geom_of(ctx); a.nlayers = ctx->nlayers; a.W64 = ctx->W64; a.H64 = ctx->H64;
    a.blk = ctx->d_blk; a.fac = st->d_fac; a.touched = st->d_touched; a.ftouched = st->d_ftouched;
    const size_t nc = st->circles.size(), ntl = st->tiles.size();
    if ((rc = st->d_ops.reserve(std::max(nc * sizeof(pfnav_blocker_op), std::max(ntl * sizeof(tile_op), (size_t)nslots * 4)))))
        return rc;
    if (nc) {
        PF_CUDA(cudaMemcpy(st->d_ops, st->circles.data(), nc * sizeof(pfnav_blocker_op), cudaMemcpyHostToDevice));
        k_blockers_circles<<<(unsigned)((nc + 3) / 4), 128>>>((const pfnav_blocker_op *)st->d_ops.p, (int)nc, a);
        ctx->launches++;
    }
    if (ntl) {
        PF_CUDA(cudaMemcpy(st->d_ops, st->tiles.data(), ntl * sizeof(tile_op), cudaMemcpyHostToDevice));   // after the circles kernel (same stream)
        k_blockers_tiles<<<(unsigned)((ntl + 255) / 256), 256>>>((const tile_op *)st->d_ops.p, (int)ntl, a);
        ctx->launches++;
    }
    if (dev_cnt[0]) {
        k_blockers_circles<<<(dev_cnt[0] + 3) / 4, 128>>>(st->d_dev_narrow, (int)dev_cnt[0], a);
        ctx->launches++;
    }
    if (st->dev_pending) {
        PF_CUDA(cudaMemset(st->d_dev_cnt, 0, 2 * sizeof(uint32_t)));     // done by the blocking read of the results below
        st->dev_pending = false; st->dev_fac = false; st->dev_bound = 0;
        st->dev_sent[0] = st->dev_sent[1] = 0; st->dev_unexchanged = false;
    }
    st->applied_ops += nc + ntl + dev_cnt[0];
    st->circles.clear(); st->tiles.clear();
    finish_args f;
    f.nlayers = ctx->nlayers; f.chunk_w = ctx->chunk_w; f.chunk_h = ctx->chunk_h; f.W64 = ctx->W64; f.H64 = ctx->H64;
    f.cost = ctx->d_cost; f.blk = ctx->d_blk; f.liid = ctx->d_liid; f.fac = st->d_fac; f.fmask = ctx->d_fmask;
    f.touched = st->d_touched; f.ftouched = st->d_ftouched; f.res = st->d_res;
    k_chunks_finish<<<nslots, 256>>>(f);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    std::vector<uint8_t> res(nslots);
    PF_CUDA(cudaMemcpy(res.data(), st->d_res, nslots, cudaMemcpyDeviceToHost));
    std::vector<int32_t> slots;
    for (int s = 0; s < nslots; s++) {
        if (res[s] & 1) slots.push_back(s);
        if (res[s] & 2) ctx->dirty.insert({s / chunks, s % chunks});
        if (res[s] & 4) ctx->fdirty.insert({s / chunks, s % chunks});
    }
    if (!slots.empty()) {
        if ((rc = st->d_out.reserve(slots.size() * 8192))) return rc;
        PF_CUDA(cudaMemcpy(st->d_ops, slots.data(), slots.size() * 4, cudaMemcpyHostToDevice));
        k_chunks_gather<<<(unsigned)slots.size(), 256>>>((const int32_t *)st->d_ops.p, ctx->chunk_w, ctx->chunk_h, ctx->W64, ctx->H64,
                                                         ctx->d_blk, ctx->d_liid, st->d_out);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
        std::vector<uint16_t> out(slots.size() * 8192);
        PF_CUDA(cudaMemcpy(out.data(), st->d_out, out.size() * 2, cudaMemcpyDeviceToHost));
        for (size_t e = 0; e < slots.size(); e++) {
            const size_t hoff = (size_t)slots[e] * 4096;        // [layer][chunk][4096] == slot * 4096
            memcpy(ctx->h_blk.data() + hoff, out.data() + e * 8192, 8192);
            if (res[slots[e]] & 2) memcpy(ctx->h_liid.data() + hoff, out.data() + e * 8192 + 4096, 8192);
        }
    }
    return PFNAV_OK;
}

// n_update_blockers (nav.c:1017); layers the context does not hold are skipped. With a device the tiles are queued
// for k_blockers_tiles; a host-only context counts them into its mirrors at once.
static void apply(pfnav_ctx *ctx, int layer, int faction_id, const td *tds, size_t n, int delta)
{
    if (layer >= ctx->nlayers) return;
    if (ctx->device >= 0) {
        blk_state *st = state_of(ctx, true);
        for (size_t i = 0; i < n; i++)
            st->tiles.push_back({layer, tds[i].chunk_r * 64 + tds[i].tile_r, tds[i].chunk_c * 64 + tds[i].tile_c, faction_id, delta});
        return;
    }
    const size_t chunks = (size_t)ctx->chunk_w * ctx->chunk_h, ltiles = chunks * 4096;
    const size_t lbase = (size_t)layer * ltiles;
    const bool fac = faction_id >= 0 && faction_id < 15;
    if (fac) {      // chunk->factions[faction_id] (nav.c:1032), allocated on first use
        if (ctx->h_fac.size() < (size_t)ctx->nlayers) ctx->h_fac.resize(ctx->nlayers);
        if (ctx->h_fac[layer].empty()) ctx->h_fac[layer].assign(ltiles * 15, 0);
        if (ctx->h_fmask.size() < ltiles * ctx->nlayers) ctx->h_fmask.assign(ltiles * ctx->nlayers, 0);
    }
    for (size_t i = 0; i < n; i++) {
        const int chunk = tds[i].chunk_r * ctx->chunk_w + tds[i].chunk_c;
        const int t = tds[i].tile_r * 64 + tds[i].tile_c;
        uint16_t &v = ctx->h_blk[lbase + (size_t)chunk * 4096 + t];
        const int prev = v;
        v = (uint16_t)(prev + delta);
        if (!!v != !!prev) ctx->dirty.insert({layer, chunk});
        if (fac) {
            uint8_t &fv = ctx->h_fac[layer][((size_t)chunk * 15 + faction_id) * 4096 + t];
            const int fprev = fv;
            fv = (uint8_t)(fprev + delta);
            if (!!fv != !!fprev) {
                uint16_t &m = ctx->h_fmask[lbase + (size_t)chunk * 4096 + t];
                m = fv ? (uint16_t)(m | (1u << faction_id)) : (uint16_t)(m & ~(1u << faction_id));
                ctx->fdirty.insert({layer, chunk});
            }
        }
    }
}

static int blockers_circle(pfnav_ctx *ctx, float x, float z, float range, int faction_id, uint32_t flags, int delta)
{
    if (ctx->device >= 0 && range >= 0.0f && (int)ceil(range / 4) <= CIRCLE_MAX_NT) {      // rasterised by k_blockers_circles
        state_of(ctx, true)->circles.push_back({x, z, range, faction_id, flags, delta});
        return PFNAV_OK;
    }
    td tds[1024], o3[1024], o5[1024], o7[1024];
    const size_t n = tiles_under_circle(ctx, {x, z}, range, tds, 1024);
    const size_t n3 = tiles_contour(ctx, n, tds, o3, 1024);
    const size_t n5 = tiles_contour(ctx, n3, o3, o5, 1024);
    const size_t n7 = tiles_contour(ctx, n5, o5, o7, 1024);
    // layer groups: ground 0..3, water 4..7, air 8..11 (nav.h:78-92); non-air entities block ground AND water
    const int groups[2] = {(flags & PFNAV_FLAG_AIR) ? 8 : 4, (flags & PFNAV_FLAG_AIR) ? -1 : 0};
    for (int gi = 0; gi < 2; gi++) {
        const int g = groups[gi];
        if (g < 0) continue;
        apply(ctx, g + 0, faction_id, tds, n, delta);
        apply(ctx, g + 1, faction_id, tds, n, delta); apply(ctx, g + 1, faction_id, o3, n3, delta);
        apply(ctx, g + 2, faction_id, tds, n, delta); apply(ctx, g + 2, faction_id, o3, n3, delta); apply(ctx, g + 2, faction_id, o5, n5, delta);
        apply(ctx, g + 3, faction_id, tds, n, delta); apply(ctx, g + 3, faction_id, o3, n3, delta); apply(ctx, g + 3, faction_id, o5, n5, delta); apply(ctx, g + 3, faction_id, o7, n7, delta);
    }
    return PFNAV_OK;
}

// n_update_blockers_obb_{ground,water,air} (nav.c:1135-1211)
static int blockers_obb(pfnav_ctx *ctx, const float *corners_xz, int faction_id, uint32_t flags, int delta)
{
    v2f c[4];
    for (int i = 0; i < 4; i++) {
        c[i] = {corners_xz[2 * i], corners_xz[2 * i + 1]};
        td t;
        if (!desc_for_point(ctx, c[i].x, c[i].z, &t)) {
            pfnav_set_error("pfnav_blockers_*_obb: corner %d lies outside the map (clipped boxes are not supported)", i);
            return PFNAV_ERR_ARG;
        }
    }
    td tds[1024], o3[1024], o5[1024], o7[1024];
    const size_t n = tiles_under_obb(ctx, c, tds, 1024);
    const size_t n3 = tiles_contour(ctx, n, tds, o3, 1024);
    const size_t n5 = tiles_contour(ctx, n3, o3, o5, 1024);
    const size_t n7 = tiles_contour(ctx, n5, o5, o7, 1024);
    const int groups[2] = {(flags & PFNAV_FLAG_AIR) ? 8 : 4, (flags & PFNAV_FLAG_AIR) ? -1 : 0};
    for (int gi = 0; gi < 2; gi++) {
        const int g = groups[gi];
        if (g < 0) continue;
        apply(ctx, g + 0, faction_id, tds, n, delta);
        apply(ctx, g + 1, faction_id, tds, n, delta); apply(ctx, g + 1, faction_id, o3, n3, delta);
        apply(ctx, g + 2, faction_id, tds, n, delta); apply(ctx, g + 2, faction_id, o3, n3, delta); apply(ctx, g + 2, faction_id, o5, n5, delta);
        apply(ctx, g + 3, faction_id, tds, n, delta); apply(ctx, g + 3, faction_id, o3, n3, delta); apply(ctx, g + 3, faction_id, o5, n5, delta); apply(ctx, g + 3, faction_id, o7, n7, delta);
    }
    return PFNAV_OK;
}

}   // namespace

// The tiles an entity occupies as a field target (field_entity_initial_frontier field.c:1334-1355,
// field_enemies_initial_frontier :1262-1283): circle (selection radius) or building OBB footprint, then `rings`
// contour rings, each taken around everything collected so far, all inside one 512-entry array.
// out_rc: up to 512 (r, c) pairs. Returns the count, or -1 when an OBB corner lies outside the map.
int pfnav_footprint_tiles(const pfnav_ctx *ctx, const pfnav_footprint *e, int rings, int32_t *out_rc)
{
    td tds[512];
    size_t n;
    if (e->is_building) {
        v2f c[4];
        for (int i = 0; i < 4; i++) {
            c[i] = {e->corners_xz[2 * i], e->corners_xz[2 * i + 1]};
            td t;
            if (!desc_for_point(ctx, c[i].x, c[i].z, &t)) return -1;
        }
        n = tiles_under_obb(ctx, c, tds, 512);
    } else {
        n = tiles_under_circle(ctx, {e->x, e->z}, e->sel_radius, tds, 512);
    }
    for (int k = 0; k < rings; k++) n += tiles_contour(ctx, n, tds, tds + n, 512 - n);
    for (size_t i = 0; i < n; i++) { out_rc[2 * i] = tds[i].chunk_r * 64 + tds[i].tile_r; out_rc[2 * i + 1] = tds[i].chunk_c * 64 + tds[i].tile_c; }
    return (int)n;
}

// Staging for a producer of nitems items (k_blocking_decide) and room for 2 * nitems more pending device ops. Growing
// waits for the device (the pending ops are copied over); a steady tick reuses the buffers without waiting.
// the pending op count pair, and room for `need` pending ops in each op buffer; growing waits for the device and keeps
// the pending ops
static int dev_ops_reserve(blk_state *st, size_t need)
{
    if (!st->d_dev_cnt) {
        PF_CUDA(cudaMalloc(&st->d_dev_cnt, 2 * sizeof(uint32_t)));
        PF_CUDA(cudaMemset(st->d_dev_cnt, 0, 2 * sizeof(uint32_t)));
        PF_CUDA(cudaDeviceSynchronize());
    }
    if (need > st->dev_cap) {
        const size_t cap = std::max(need, 2 * st->dev_cap);
        pfnav_blocker_op *n = nullptr, *w = nullptr;
        PF_CUDA(cudaDeviceSynchronize());
        PF_CUDA(cudaMalloc(&n, cap * sizeof(pfnav_blocker_op)));
        PF_CUDA(cudaMalloc(&w, cap * sizeof(pfnav_blocker_op)));
        if (st->dev_bound) {
            PF_CUDA(cudaMemcpy(n, st->d_dev_narrow, st->dev_bound * sizeof(pfnav_blocker_op), cudaMemcpyDeviceToDevice));
            PF_CUDA(cudaMemcpy(w, st->d_dev_wide, st->dev_bound * sizeof(pfnav_blocker_op), cudaMemcpyDeviceToDevice));
        }
        cudaFree(st->d_dev_narrow); cudaFree(st->d_dev_wide);
        st->d_dev_narrow = n; st->d_dev_wide = w; st->dev_cap = cap;
    }
    return 0;
}

int pf_blocker_ops_stage(pfnav_ctx *ctx, size_t nitems, pf_op_stage *out)
{
    PF_ARG(ctx->d_cost, "map not created");
    blk_state *st = state_of(ctx, true);
    PF_CUDA(cudaSetDevice(ctx->device));
    if (dev_ops_reserve(st, st->dev_bound + 2 * nitems)) return PFNAV_ERR_CUDA;
    if (nitems > st->stage_items) {
        const size_t items = std::max(nitems, 2 * st->stage_items);
        PF_CUDA(cudaDeviceSynchronize());
        cudaFree(st->d_stage); st->d_stage = nullptr; st->stage_items = 0;
        PF_CUDA(cudaMalloc(&st->d_stage, stage_bsum_off(items) + 2 * stage_blocks(items) * sizeof(unsigned long long)));
        st->stage_items = items;
    }
    uint8_t *base = (uint8_t *)st->d_stage;
    out->ops = (pfnav_blocker_op *)base;
    out->desc = base + stage_desc_off(st->stage_items);
    out->bsum = (unsigned long long *)(base + stage_bsum_off(st->stage_items));
    return PFNAV_OK;
}

// compact what the producer staged behind the pending device ops, on `st`
int pf_blocker_ops_append(pfnav_ctx *ctx, cudaStream_t s, size_t nitems, bool any_fac)
{
    blk_state *st = state_of(ctx, false);
    if (!nitems) return PFNAV_OK;
    uint8_t *base = (uint8_t *)st->d_stage;
    const size_t nb = stage_blocks(nitems);
    const unsigned long long *bsum = (const unsigned long long *)(base + stage_bsum_off(st->stage_items));
    unsigned long long *boff = (unsigned long long *)(base + stage_bsum_off(st->stage_items)) + stage_blocks(st->stage_items);
    k_ops_offsets<<<1, 1024, 0, s>>>(bsum, (int)nb, st->d_dev_cnt, boff);
    k_ops_compact<<<(unsigned)nb, PF_OPS_BLOCK, 0, s>>>((const pfnav_blocker_op *)base, base + stage_desc_off(st->stage_items),
                                                         (int)nitems, boff, st->d_dev_narrow, st->d_dev_wide);
    ctx->launches += 2;
    PF_CUDA(cudaGetLastError());
    st->dev_bound += 2 * nitems;
    st->dev_pending = true;
    st->dev_fac |= any_fac;
    st->dev_unexchanged = true;
    return PFNAV_OK;
}

static void ops_view_fill(const blk_state *st, pf_ops_view *out)
{
    out->narrow = st->d_dev_narrow; out->wide = st->d_dev_wide; out->d_cnt = st->d_dev_cnt;
    out->sent[0] = st->dev_sent[0]; out->sent[1] = st->dev_sent[1];
    out->fac = st->dev_fac;
}

int pf_blocker_ops_view(pfnav_ctx *ctx, pf_ops_view *out)
{
    PF_ARG(ctx->d_cost, "map not created");
    blk_state *st = state_of(ctx, true);
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());        // the ops may have been decided on any stream
    if (dev_ops_reserve(st, 0)) return PFNAV_ERR_CUDA;
    ops_view_fill(st, out);
    return PFNAV_OK;
}

int pf_blocker_ops_reserve(pfnav_ctx *ctx, size_t need, pf_ops_view *out)
{
    blk_state *st = state_of(ctx, false);
    PF_CUDA(cudaSetDevice(ctx->device));
    if (dev_ops_reserve(st, need)) return PFNAV_ERR_CUDA;
    ops_view_fill(st, out);
    return PFNAV_OK;
}

bool pf_blocker_ops_unexchanged(pfnav_ctx *ctx)
{
    const blk_state *st = state_of(ctx, false);
    return st && st->dev_unexchanged;
}

bool pf_blocker_ops_pending(pfnav_ctx *ctx)
{
    const blk_state *st = state_of(ctx, false);
    return st && st->dev_pending;
}

bool pf_map_uncommitted(pfnav_ctx *ctx)
{
    const blk_state *st = state_of(ctx, false);
    return !ctx->dirty.empty() || !ctx->fdirty.empty() || (st && (st->dev_pending || !st->circles.empty() || !st->tiles.empty()));
}

int pf_blocker_ops_exchanged(pfnav_ctx *ctx, const uint32_t cnt[2], bool any_fac)
{
    blk_state *st = state_of(ctx, false);
    PF_CUDA(cudaSetDevice(ctx->device));
    // synchronous: a producer on any stream that follows appends behind the new counts
    PF_CUDA(cudaMemcpy(st->d_dev_cnt, cnt, 2 * sizeof(uint32_t), cudaMemcpyHostToDevice));
    st->dev_bound = std::max(st->dev_bound, (size_t)std::max(cnt[0], cnt[1]));
    st->dev_pending |= cnt[0] != 0 || cnt[1] != 0;
    st->dev_fac |= any_fac;
    st->dev_sent[0] = cnt[0]; st->dev_sent[1] = cnt[1];
    st->dev_unexchanged = false;
    return PFNAV_OK;
}

// the map is going away (pfnav_map_create / pfnav_destroy): queued operations and the device-side counts with it
void pfnav_blockers_forget(pfnav_ctx *ctx)
{
    ctx->dirty.clear(); ctx->fdirty.clear();
    blk_state *st = state_of(ctx, false);
    if (!st) return;
    if (ctx->device >= 0) {
        cudaSetDevice(ctx->device);
        cudaDeviceSynchronize();
        cudaFree(st->d_dev_narrow); cudaFree(st->d_dev_wide); cudaFree(st->d_dev_cnt); cudaFree(st->d_stage);
    }
    delete st;
    ctx->blk_state = nullptr;
}

// Apply what is queued (no-op on a host-only context): called before anything that reads or overwrites the counts.
int pfnav_blockers_flush(pfnav_ctx *ctx) { return device_flush(ctx); }

// pfnav_map_upload_factions replaced the host counts of one layer: the device copy follows
int pfnav_blockers_factions_uploaded(pfnav_ctx *ctx, int layer)
{
    blk_state *st = state_of(ctx, false);
    if (!st || !st->d_fac || ctx->device < 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    return fac_push_layer(ctx, st, layer) ? PFNAV_ERR_CUDA : PFNAV_OK;
}

extern "C" int pfnav_blockers_incref(pfnav_ctx *ctx, float x, float z, float range, int faction_id, uint32_t flags)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    return blockers_circle(ctx, x, z, range, faction_id, flags, +1);
}

// N_BlockersIncrefOBB / N_BlockersDecrefOBB (nav.c:4685-4705). corners_xz: the bottom face of the box,
// obb->corners[0], [1], [5], [4] as x,z pairs (tile.c:599).
extern "C" int pfnav_blockers_incref_obb(pfnav_ctx *ctx, const float *corners_xz, int faction_id, uint32_t flags)
{
    PF_ARG(ctx && ctx->d_cost && corners_xz, "map not created / null");
    return blockers_obb(ctx, corners_xz, faction_id, flags, +1);
}

extern "C" int pfnav_blockers_decref_obb(pfnav_ctx *ctx, const float *corners_xz, int faction_id, uint32_t flags)
{
    PF_ARG(ctx && ctx->d_cost && corners_xz, "map not created / null");
    return blockers_obb(ctx, corners_xz, faction_id, flags, -1);
}

extern "C" int pfnav_blockers_decref(pfnav_ctx *ctx, float x, float z, float range, int faction_id, uint32_t flags)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    return blockers_circle(ctx, x, z, range, faction_id, flags, -1);
}

// A tick's worth of N_BlockersIncref / N_BlockersDecref calls (nav.c:4663-4683) in one call, applied in order.
extern "C" int pfnav_blockers_batch(pfnav_ctx *ctx, const pfnav_blocker_op *ops, size_t n)
{
    PF_ARG(ctx && ctx->d_cost && (n == 0 || ops), "map not created / null");
    for (size_t i = 0; i < n; i++) {
        PF_ARG(ops[i].delta == 1 || ops[i].delta == -1, "blocker op: delta must be +1 or -1");
        int rc = blockers_circle(ctx, ops[i].x, ops[i].z, ops[i].range, ops[i].faction_id, ops[i].flags, ops[i].delta);
        if (rc) return rc;
    }
    return PFNAV_OK;
}

// N_Update + N_ApplyDeferredInvalidations: recompute the local islands of every dirty chunk, refresh the
// portal edge states there, push the chunk (blockers + islands) to the device, and invalidate pool
// entries: everything AT a dirty chunk; and, when an edge state flipped, every field of every
// destination whose path runs THROUGH that chunk. *out_ndirty = number of (layer, chunk) pairs handled.
extern "C" int pfnav_map_commit(pfnav_ctx *ctx, int *out_ndirty)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    if (ctx->device >= 0) {
        PF_CUDA(cudaSetDevice(ctx->device));
        int rc = device_flush(ctx);       // counts, faction masks and local islands of the touched chunks, on the device
        if (rc) return rc;
        if (!ctx->fdirty.empty()) ctx->map_epoch++;     // faction masks only matter to attacking requests
        ctx->fdirty.clear();
    } else {
        if (!ctx->fdirty.empty()) ctx->map_epoch++;
        ctx->fdirty.clear();
    }
    int nd = 0;
    if (!ctx->dirty.empty()) {
        const int chunks = ctx->chunk_w * ctx->chunk_h;
        bool pool_touched = false;
        for (const auto &lc : ctx->dirty) {
            const int layer = lc.first, chunk = lc.second;
            if (ctx->device < 0) {      // host-only context: islands on the host mirror (the device path did them in k_chunks_finish)
                int rc = pfnav_map_refresh_chunk(ctx, layer, chunk / ctx->chunk_w, chunk % ctx->chunk_w);
                if (rc) return rc;
            }
            const int flipped = pfnav_route_refresh_edges(ctx, layer, chunk);
            nd++;
            for (int d = 0; d < ctx->pool.ndests; d++) {
                if (!ctx->pool.has_of((size_t)d * chunks + chunk)) continue;
                pool_touched = true;
                if (flipped <= 0) pf_pool_drop(ctx, d, chunk);
                else for (int c = 0; c < chunks; c++) pf_pool_drop(ctx, d, c);   // N_FC_InvalidateAllThroughChunk: the whole path goes
            }
        }
        ctx->dirty.clear();
        ctx->map_epoch++;          // the resident goal plan is not relaunched on a changed map
        if (pool_touched && ctx->device >= 0) {
            PF_CUDA(cudaSetDevice(ctx->device));
            PF_CUDA(cudaDeviceSynchronize());     // a tick on a non-blocking stream may still read the flags
            PF_CUDA(cudaMemcpy(ctx->pool.d_has, ctx->pool.has.data(), ctx->pool.max,
                               cudaMemcpyHostToDevice));
        }
    }
    if (out_ndirty) *out_ndirty = nd;
    return PFNAV_OK;
}

// Read back one layer's blocker counts ([chunk][64][64] u16) from the host mirror (parity tests).
extern "C" int pfnav_blockers_get(pfnav_ctx *ctx, int layer, uint16_t *out)
{
    PF_ARG(ctx && out && layer >= 0 && layer < ctx->nlayers, "args");
    { int rc = device_flush(ctx); if (rc) return rc; }
    const size_t ltiles = (size_t)ctx->chunk_w * ctx->chunk_h * 4096;
    memcpy(out, ctx->h_blk.data() + ltiles * layer, ltiles * 2);
    return PFNAV_OK;
}

// Read back one layer's per-faction blocker counts (nav_chunk::factions, nav_data.h: [chunk][15][64][64] u8)
// from the host mirror; all zero until a faction-tagged blocker was counted or pfnav_map_upload_factions ran.
extern "C" int pfnav_blockers_get_factions(pfnav_ctx *ctx, int layer, uint8_t *out)
{
    PF_ARG(ctx && out && layer >= 0 && layer < ctx->nlayers, "args");
    { int rc = device_flush(ctx); if (rc) return rc; }
    const size_t n = (size_t)ctx->chunk_w * ctx->chunk_h * 15 * 4096;
    if (blk_state *st = state_of(ctx, false); st && st->d_fac && ctx->device >= 0) {
        // the device holds the counts: [15][H64][W64] -> [chunk][15][4096]
        PF_CUDA(cudaSetDevice(ctx->device));
        const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
        std::vector<uint8_t> img(ltiles * 15);
        PF_CUDA(cudaMemcpy(img.data(), st->d_fac + ltiles * 15 * layer, ltiles * 15, cudaMemcpyDeviceToHost));
        const size_t chunks = (size_t)ctx->chunk_w * ctx->chunk_h;
        for (size_t ch = 0; ch < chunks; ch++) {
            const size_t cr = ch / ctx->chunk_w, cc = ch % ctx->chunk_w;
            for (int f = 0; f < 15; f++)
                for (int r = 0; r < 64; r++)
                    memcpy(out + (ch * 15 + f) * 4096 + r * 64, img.data() + ltiles * f + (cr * 64 + r) * ctx->W64 + cc * 64, 64);
        }
        return PFNAV_OK;
    }
    if ((size_t)layer < ctx->h_fac.size() && ctx->h_fac[layer].size() == n) memcpy(out, ctx->h_fac[layer].data(), n);
    else memset(out, 0, n);
    return PFNAV_OK;
}
