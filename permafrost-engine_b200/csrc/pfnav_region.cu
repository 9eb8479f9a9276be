// pfnav_region.cu -- region ("cell arrival" / "group arrival") fields, sm_90a.
//
// Reference: N_CellArrivalFieldCreate (navigation/field.c:2445), N_GroupArrivalFieldCreate (field.c:2525),
// N_CellArrivalFieldUpdateToNearestPathable (field.c:2603) and their helpers field_build_integration_region
// (:587), field_build_integration_nonpass_region (:678), field_passable_frontier (:1441), clamped_region
// (:1892), field_build_flow_unaligned (:804), field_flow_dir (:355), set_flow_cell (:790).
//
// One CTA per field. The dim x dim window (dim = 96 for formations) is gathered from the row-major layer
// images into shared memory once per pass: a cost byte and a flag byte per cell plus a 32-bit integration
// value (6 bytes per cell, 54 KB at dim 96, four CTAs per SM). The reference's Dijkstra has non-negative
// integer edge weights (cost_base of the tile entered, every sum < 2^24 so its float arithmetic is exact),
// so its result is the unique shortest-distance fixed point: the kernel reaches it by in-place relaxation
// sweeps (each thread owns a run of consecutive cells and alternates sweep direction) until no cell changes.
//
// The fix-up's flood (the passable rim of the blocked island around `start`) is a reachability fixed point as
// well -- except when the map-clamped region has fewer rows than columns: the reference indexes its visited
// array with stride region.r (visited_idx, field.c:1431), distinct tiles alias, and the outcome depends on
// the breadth-first order. That case (regions hanging over the top / bottom map edge only) is replayed
// literally by one thread, with the queue and visited array overlaid on the integration buffer.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <map>
#include "pfnav_internal.cuh"

namespace {

#include "pfnav_map_view.cuh"
#include "pfnav_region_kernel.cuh"
#include "pfnav_tile_geom.cuh"
#include "pfnav_zone_kernel.cuh"
}   // namespace

static int region_launch(pfnav_ctx *ctx, int dim, const pfnav_region_req *d_reqs, size_t n, const int32_t *d_seeds,
                         const int32_t *d_overlay, uint8_t *d_fields, cudaStream_t st, int chunk_out = 0,
                         const uint32_t *d_seed_bits = nullptr, const int32_t *d_out_slot = nullptr)
{
    RegionGrids g;
    g.cost = ctx->d_cost; g.blk = ctx->d_blk; g.fmask = ctx->d_fmask; g.W64 = ctx->W64; g.H64 = ctx->H64;
    const size_t smem = (size_t)dim * dim * 6;
    PF_CUDA(cudaFuncSetAttribute(k_region_fields, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 PFNAV_REGION_DIM_MAX * PFNAV_REGION_DIM_MAX * 6));
    const int per_sm = std::max(1, std::min(4, (int)((size_t)(227 * 1024) / (smem + 1024))));
    const int grid = (int)std::min<size_t>(n, (size_t)ctx->sm_count * per_sm);
    k_region_fields<<<grid, RG_THREADS, smem, st>>>(g, dim, d_reqs, (int)n, d_seeds, d_overlay, d_fields, chunk_out,
                                                            d_seed_bits, d_out_slot);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}

extern "C" int pfnav_region_fields_dev(pfnav_ctx *ctx, int dim, const pfnav_region_req *d_reqs, size_t n,
                                       const int32_t *d_seeds_rc, const int32_t *d_overlay_rc, uint8_t *d_inout_fields,
                                       void *stream)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(dim >= 2 && dim <= PFNAV_REGION_DIM_MAX && dim % 2 == 0, "dim must be even and <= PFNAV_REGION_DIM_MAX");
    PF_ARG(d_reqs && d_inout_fields, "null buffer");
    PF_ARG(n < (1u << 30), "n");
    PF_CUDA(cudaSetDevice(ctx->device));
    return region_launch(ctx, dim, d_reqs, n, d_seeds_rc, d_overlay_rc, d_inout_fields, pf_stream(ctx, stream));
}

// the reference asserts these (field.c:2498-2499, 1455, 1487); here they are argument errors
static int validate_region_reqs(const pfnav_ctx *ctx, int dim, const pfnav_region_req *reqs, size_t n, const int32_t *seeds,
                                size_t nseeds, size_t noverlay)
{
    const int half = dim / 2;
    for (size_t i = 0; i < n; i++) {
        const pfnav_region_req &q = reqs[i];
        PF_ARG(q.layer >= 0 && q.layer < ctx->nlayers, "region request: layer");
        PF_ARG((q.flags & (PFNAV_REGION_CREATE | PFNAV_REGION_FIXUP)) != 0, "region request: neither CREATE nor FIXUP");
        PF_ARG(q.center_r >= 0 && q.center_r < ctx->H64 && q.center_c >= 0 && q.center_c < ctx->W64, "region request: center outside the map");
        PF_ARG(q.overlay_n >= 0 && q.overlay_off >= 0 && (size_t)q.overlay_off + q.overlay_n <= noverlay, "region request: overlay range");
        if (q.flags & PFNAV_REGION_CREATE) {
            PF_ARG(q.seed_n >= 0 && q.seed_off >= 0 && (size_t)q.seed_off + q.seed_n <= nseeds, "region request: seed range");
            for (int k = 0; k < q.seed_n; k++) {
                const int32_t *s = seeds + 2 * ((size_t)q.seed_off + k);
                PF_ARG(s[0] >= 0 && s[0] < ctx->H64 && s[1] >= 0 && s[1] < ctx->W64, "region request: seed tile outside the map");
            }
            if (q.flags & PFNAV_REGION_CELL) {
                PF_ARG(q.seed_n == 1, "region request: PFNAV_REGION_CELL takes exactly one seed");
                const int32_t *s = seeds + 2 * (size_t)q.seed_off;
                PF_ARG(s[0] >= q.center_r - half && s[1] >= q.center_c - half, "region request: cell tile before the region base");
            }
        }
        if (q.flags & PFNAV_REGION_FIXUP) {
            const int cb_r = std::max(q.center_r - half, 0), cb_c = std::max(q.center_c - half, 0);
            const int ce_r = q.center_r + half < ctx->H64 ? q.center_r + half : ctx->H64 - 1;
            const int ce_c = q.center_c + half < ctx->W64 ? q.center_c + half : ctx->W64 - 1;
            PF_ARG(q.start_r >= cb_r && q.start_r < ce_r && q.start_c >= cb_c && q.start_c < ce_c,
                   "region request: fix-up start outside the clamped region");
        }
    }
    return PFNAV_OK;
}

extern "C" int pfnav_region_fields(pfnav_ctx *ctx, int dim, const pfnav_region_req *reqs, size_t n, const int32_t *seeds_rc,
                                   size_t nseeds, const int32_t *overlay_rc, size_t noverlay, uint8_t *inout_fields)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(dim >= 2 && dim <= PFNAV_REGION_DIM_MAX && dim % 2 == 0, "dim must be even and <= PFNAV_REGION_DIM_MAX");
    PF_ARG(reqs && inout_fields, "null buffer");
    PF_ARG((nseeds == 0 || seeds_rc) && (noverlay == 0 || overlay_rc), "null seed / overlay list");
    PF_ARG(n < (1u << 30), "n");
    int rc = validate_region_reqs(ctx, dim, reqs, n, seeds_rc, nseeds, noverlay);
    if (rc) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    const size_t fbytes = (size_t)dim * dim / 2;
    bool need_in = false;
    for (size_t i = 0; i < n; i++) need_in |= !(reqs[i].flags & PFNAV_REGION_CREATE);
    // staged: requests, seeds, overlay, then the fields, which go up only when a request fixes up its field in place
    const size_t b_req = n * sizeof(pfnav_region_req), b_f = n * fbytes;
    const size_t a_seed = (b_req + 15) & ~(size_t)15, a_ov = a_seed + nseeds * 8, a_f = (a_ov + noverlay * 8 + 15) & ~(size_t)15;
    const size_t b_in = need_in ? a_f + b_f : a_f;
    cudaStream_t st = ctx->tick_stream;
    pf_stage S;
    if ((rc = pf_stage_begin(ctx, st, b_in, a_f + b_f, false, &S))) return rc;
    memcpy(S.host, reqs, b_req);
    if (nseeds) memcpy(S.host + a_seed, seeds_rc, nseeds * 8);
    if (noverlay) memcpy(S.host + a_ov, overlay_rc, noverlay * 8);
    if (need_in) memcpy(S.host + a_f, inout_fields, b_f);
    if ((rc = pf_stage_upload(ctx, st, S, b_in))) return rc;
    if ((rc = region_launch(ctx, dim, (const pfnav_region_req *)S.dev, n, (const int32_t *)(S.dev + a_seed),
                            (const int32_t *)(S.dev + a_ov), S.dev + a_f, st)))
        return rc;
    PF_CUDA(cudaMemcpyAsync(inout_fields, S.dev + a_f, b_f, cudaMemcpyDeviceToHost, st));
    if ((rc = pf_stage_done(ctx, st))) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

// M_Tile_DescForPoint2D with the nav resolution (tile.c:547) -> absolute (r, c)
static bool region_tile_for_point(const pfnav_ctx *ctx, float px, float pz, int32_t *out_rc)
{
    const float width = (float)(ctx->chunk_w * 256), height = (float)(ctx->chunk_h * 256);
    if (px > ctx->map_x || px < ctx->map_x - width) return false;
    if (pz < ctx->map_z || pz > ctx->map_z + height) return false;
    int chunk_r = (int)(fabs(ctx->map_z - pz) / 256.0f), chunk_c = (int)(fabs(ctx->map_x - px) / 256.0f);
    chunk_r = std::min(std::max(chunk_r, 0), ctx->chunk_h - 1);
    chunk_c = std::min(std::max(chunk_c, 0), ctx->chunk_w - 1);
    const float bx = ctx->map_x - (chunk_c * 256.0f), bz = ctx->map_z + (chunk_r * 256.0f);
    const int tile_r = (int)(fabs(bz - pz) / 4), tile_c = (int)(fabs(bx - px) / 4);
    out_rc[0] = chunk_r * 64 + std::min(std::max(tile_r, 0), 63);
    out_rc[1] = chunk_c * 64 + std::min(std::max(tile_c, 0), 63);
    return true;
}

extern "C" int pfnav_group_arrival_field(pfnav_ctx *ctx, int layer, int dim, uint16_t enemies, const float *targets_xz,
                                         size_t ntargets, const float *center_xz, const int32_t *overlay_rc, size_t noverlay,
                                         uint8_t *out_field)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    PF_ARG(dim >= 2 && dim <= PFNAV_REGION_DIM_MAX && dim % 2 == 0, "dim must be even and <= PFNAV_REGION_DIM_MAX");
    PF_ARG(center_xz && out_field && (ntargets == 0 || targets_xz), "null buffer");
    PF_ARG(ntargets < (1u << 28), "ntargets");
    int32_t c[2];
    if (!region_tile_for_point(ctx, center_xz[0], center_xz[1], c)) {        // field.c:2552-2556
        memset(out_field, 0, (size_t)dim * dim / 2);
        return PFNAV_OK;
    }
    std::vector<int32_t> seeds;
    seeds.reserve(ntargets * 2);
    for (size_t i = 0; i < ntargets; i++) {
        int32_t t[2];
        if (region_tile_for_point(ctx, targets_xz[2 * i], targets_xz[2 * i + 1], t)) { seeds.push_back(t[0]); seeds.push_back(t[1]); }
    }
    pfnav_region_req q = {};
    q.layer = layer; q.center_r = c[0]; q.center_c = c[1];
    q.seed_off = 0; q.seed_n = (int32_t)(seeds.size() / 2);
    q.overlay_off = 0; q.overlay_n = (int32_t)noverlay;
    q.enemies = enemies; q.flags = PFNAV_REGION_CREATE;
    return pfnav_region_fields(ctx, dim, &q, 1, seeds.data(), seeds.size() / 2, overlay_rc, noverlay, out_field);
}

// ------------------------------------------------------------------------------------------
// TARGET_ZONE chunk fields: the group arrival fields (N_RequestAsyncGroupArrivalField nav.c:3921 ->
// N_FlowFieldUpdate field.c:2050 -> field_update_zone :1810) and their per-entity consumer
// N_DesiredGroupArrivalVelocity (nav.c:3561).
// ------------------------------------------------------------------------------------------
namespace {

// lib/public/pqueue.h:109-208 (1-indexed binary min-heap, hole-based sift; ties keep the reference's order)
struct zone_heap {
    struct node { float prio; int r, c; };
    std::vector<node> a{1};
    size_t size() const { return a.size() - 1; }
    void clear() { a.resize(1); }
    void push(float prio, int r, int c)
    {
        a.push_back({});
        size_t curr = a.size() - 1, parent = curr / 2;
        while (curr > 1 && a[parent].prio > prio) { a[curr] = a[parent]; curr = parent; parent /= 2; }
        a[curr] = {prio, r, c};
    }
    void pop(int *r, int *c)
    {
        *r = a[1].r; *c = a[1].c;
        const size_t n = a.size() - 2;      // size after the pop; a[n + 1], the last element, is the one being sifted
        a[1] = a[n + 1];
        size_t root = 1;
        while (root != n + 1) {             // _pq_balance: `target` starts at the sifted element's own slot
            size_t target = n + 1;
            const size_t l = root * 2, rr = l + 1;
            if (l <= n && a[l].prio < a[target].prio) target = l;
            if (rr <= n && a[rr].prio < a[target].prio) target = rr;
            a[root] = a[target];
            root = target;
        }
        a.pop_back();
    }
};

struct zone_map {
    const uint8_t *cost; const uint16_t *blk; int chunk_w, chunk_h;
    bool exists(int r, int c) const { return r >= 0 && r < chunk_h * 64 && c >= 0 && c < chunk_w * 64; }
    bool passable(int r, int c) const       // field_tile_passable (field.c:117)
    {
        const size_t off = ((size_t)(r / 64) * chunk_w + c / 64) * 4096 + (r % 64) * 64 + (c % 64);
        return cost[off] != 0xFF && blk[off] == 0;
    }
};

// field_zone_initial_frontier (field.c:1683)
void zone_initial_frontier(const zone_map &m, int centre_r, int centre_c, int base_r, int base_c, int dim, size_t budget,
                           std::vector<int32_t> &out)
{
    static const int er[8] = {0, 0, -1, 1, -1, -1, 1, 1}, ec[8] = {-1, 1, 0, 0, -1, 1, -1, 1};
    const int cdr = centre_r - base_r, cdc = centre_c - base_c;
    if (cdr < 0 || cdr >= dim || cdc < 0 || cdc >= dim) return;
    std::vector<uint8_t> visited((size_t)dim * dim, 0);
    zone_heap frontier;
    visited[cdr * dim + cdc] = 1;
    frontier.push(0.0f, centre_r, centre_c);
    int start_r = 0, start_c = 0; bool have_start = false;
    while (frontier.size() > 0) {
        int r, c; frontier.pop(&r, &c);
        if (m.passable(r, c)) { start_r = r; start_c = c; have_start = true; break; }
        for (int e = 0; e < 8; e++) {
            const int nr = r + er[e], nc = c + ec[e];
            if (!m.exists(nr, nc)) continue;
            const int dr = nr - base_r, dc = nc - base_c;
            if (dr < 0 || dr >= dim || dc < 0 || dc >= dim) continue;
            if (visited[dr * dim + dc]) continue;
            visited[dr * dim + dc] = 1;
            const int ndr = nr - centre_r, ndc = nc - centre_c;
            frontier.push((float)(ndr * ndr + ndc * ndc), nr, nc);
        }
    }
    if (!have_start) return;
    frontier.clear();
    std::fill(visited.begin(), visited.end(), 0);
    visited[(start_r - base_r) * dim + (start_c - base_c)] = 1;
    frontier.push(0.0f, start_r, start_c);
    size_t ret = 0;
    while (frontier.size() > 0 && ret < budget) {
        int r, c; frontier.pop(&r, &c);
        if (m.passable(r, c)) { out.push_back(r); out.push_back(c); ret++; }
        for (int e = 0; e < 8; e++) {
            const int nr = r + er[e], nc = c + ec[e];
            if (!m.exists(nr, nc)) continue;
            const int dr = nr - base_r, dc = nc - base_c;
            if (dr < 0 || dr >= dim || dc < 0 || dc >= dim) continue;
            if (visited[dr * dim + dc]) continue;
            visited[dr * dim + dc] = 1;
            if (!m.passable(nr, nc)) continue;
            const int ndr = nr - centre_r, ndc = nc - centre_c;
            frontier.push((float)(ndr * ndr + ndc * ndc), nr, nc);
        }
    }
}

struct ZoneView {
    const int32_t *slot; const uint8_t *flow; const uint8_t *has;     // the field pool (pfnav_pool_*)
    int chunk_w, chunk_h; float map_x, map_z;
};

// M_Tile_DescForPoint2D (tile.c:547) -> absolute (r, c); divisions by powers of two are exact in float
__device__ __forceinline__ bool zone_tile_for_point(const ZoneView &z, float px, float pz, int &ar, int &ac)
{
    const float width = (float)(z.chunk_w * 256), height = (float)(z.chunk_h * 256);
    if (px > z.map_x || px < z.map_x - width) return false;
    if (pz < z.map_z || pz > z.map_z + height) return false;
    int chunk_r = (int)(fabsf(z.map_z - pz) / 256.0f), chunk_c = (int)(fabsf(z.map_x - px) / 256.0f);
    chunk_r = min(max(chunk_r, 0), z.chunk_h - 1);
    chunk_c = min(max(chunk_c, 0), z.chunk_w - 1);
    const float bx = z.map_x - (float)chunk_c * 256.0f, bz = z.map_z + (float)chunk_r * 256.0f;
    const int tile_r = (int)(fabsf(bz - pz) / 4.0f), tile_c = (int)(fabsf(bx - px) / 4.0f);
    ar = chunk_r * 64 + min(max(tile_r, 0), 63);
    ac = chunk_c * 64 + min(max(tile_c, 0), 63);
    return true;
}

// N_DesiredGroupArrivalVelocity (nav.c:3561): one thread per position
__global__ void k_group_arrival_velocity(ZoneView z, int dest, float cx, float cz, int radius, const float2 *__restrict__ pos, int n,
                                         float2 *__restrict__ out_vel, uint8_t *__restrict__ out_flags)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float2 v = make_float2(0.0f, 0.0f);
    uint8_t fl = 0;
    int ar, ac, cr, cc;
    const float2 p = pos[i];
    if (zone_tile_for_point(z, p.x, p.y, ar, ac) && zone_tile_for_point(z, cx, cz, cr, cc)) {
        const int chunk = (ar >> 6) * z.chunk_w + (ac >> 6);
        const int slot = z.slot[(size_t)dest * z.chunk_w * z.chunk_h + chunk];
        if (slot >= 0 && (z.has[slot] & 1)) {
            const uint32_t dir = z.flow[(size_t)slot * 4096 + (ar & 63) * 64 + (ac & 63)];
            // N_FlowDir (field.c:2429): x grows to the left
            const float d = (float)(1.0 / 1.4142135623730951);      // 1.0f / sqrt(2.0f): a double division rounded to float
            switch (dir) {
            case 1: v = make_float2(d, -d); break;
            case 2: v = make_float2(0.0f, -1.0f); break;
            case 3: v = make_float2(-d, -d); break;
            case 4: v = make_float2(1.0f, 0.0f); break;
            case 5: v = make_float2(-1.0f, 0.0f); break;
            case 6: v = make_float2(d, d); break;
            case 7: v = make_float2(0.0f, 1.0f); break;
            case 8: v = make_float2(-d, d); break;
            default: break;
            }
            fl = 1;
            if (dir == 0) {
                const int dr = ar - cr, dc = ac - cc;
                if (dr * dr + dc * dc <= radius * radius) fl |= 2;
            }
        }
    }
    out_vel[i] = v; out_flags[i] = fl;
}

}   // namespace

static int zone_dim(const pfnav_ctx *ctx, int *out_dim)
{
    // field_update_zone sizes its square buffer with rdim as the row stride (field.c:1821-1828): only the
    // cases where rows == columns are defined
    if (ctx->chunk_h > 1 && ctx->chunk_w > 1) { *out_dim = 128; return PFNAV_OK; }
    if (ctx->chunk_h == 1 && ctx->chunk_w == 1) { *out_dim = 64; return PFNAV_OK; }
    pfnav_set_error("zone fields need a map with more than one chunk row AND column (or a 1 x 1 map): the reference's padded "
                    "region is indexed with one stride for both");
    return PFNAV_ERR_ARG;
}

// Padded-chunk fields from per-chunk seed lists (seed_off[i] .. seed_off[i + 1] pairs of chunk i) into out_fields, n x 4096
// direction bytes on the host; blocking. Shared by the host-array zone and entity / enemies calls (field_update_zone /
// _entity / _enemies).
static int chunk_fields(pfnav_ctx *ctx, int layer, int dim, const int32_t *chunks_rc, size_t n, const std::vector<int32_t> &seeds,
                        const std::vector<size_t> &seed_off, uint8_t *out_fields)
{
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->tick_stream;
    // staged: the requests, their seeds, then the fields
    const size_t b_req = n * sizeof(pfnav_region_req), a_seed = (b_req + 15) & ~(size_t)15;
    const size_t a_f = (a_seed + seeds.size() * 4 + 15) & ~(size_t)15;
    pf_stage S;
    int rc = pf_stage_begin(ctx, st, a_f, a_f + n * 4096, false, &S);
    if (rc) return rc;
    for (size_t i = 0; i < n; i++) {
        pfnav_region_req q = {};
        q.layer = layer; q.center_r = chunks_rc[2 * i]; q.center_c = chunks_rc[2 * i + 1];
        q.seed_off = (int32_t)seed_off[i]; q.seed_n = (int32_t)(seed_off[i + 1] - seed_off[i]);
        q.flags = PFNAV_REGION_CREATE;
        memcpy(S.host + i * sizeof(pfnav_region_req), &q, sizeof(q));
    }
    memcpy(S.host + a_seed, seeds.data(), seeds.size() * 4);
    if ((rc = pf_stage_upload(ctx, st, S, a_f))) return rc;
    const int32_t *d_seeds = (const int32_t *)(S.dev + a_seed);
    if ((rc = region_launch(ctx, dim, (const pfnav_region_req *)S.dev, n, d_seeds, d_seeds, S.dev + a_f, st, 1))) return rc;
    PF_CUDA(cudaMemcpyAsync(out_fields, S.dev + a_f, n * 4096, cudaMemcpyDeviceToHost, st));
    if ((rc = pf_stage_done(ctx, st))) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

// the padded region of chunk (cr, cc): field.c:1566-1571
static inline void chunk_region_base(int dim, int cr, int cc, int *base_r, int *base_c)
{
    *base_r = (cr > 0 && dim > 64) ? cr * 64 - 32 : cr * 64;
    *base_c = (cc > 0 && dim > 64) ? cc * 64 - 32 : cc * 64;
}

extern "C" int pfnav_zone_fields(pfnav_ctx *ctx, int layer, int centre_r, int centre_c, int radius, const int32_t *chunks_rc,
                                 size_t n, uint8_t *out_fields)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(chunks_rc && out_fields, "null buffer");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG(centre_r >= 0 && centre_r < ctx->H64 && centre_c >= 0 && centre_c < ctx->W64, "zone centre outside the map");
    PF_ARG(radius >= 0 && radius <= 0xFFFF, "radius");
    PF_ARG(n < (1u << 24), "n");
    int dim = 0;
    int rc = zone_dim(ctx, &dim);
    if (rc) return rc;
    const size_t ltiles = (size_t)ctx->chunk_w * ctx->chunk_h * 4096;
    zone_map zm = { ctx->h_cost.data() + ltiles * layer, ctx->h_blk.data() + ltiles * layer, ctx->chunk_w, ctx->chunk_h };
    size_t budget = (size_t)(M_PI * radius * radius + 0.5);             // field.c:1843
    if (budget > (size_t)dim * dim) budget = (size_t)dim * dim;
    std::vector<int32_t> seeds;
    std::vector<size_t> off(n + 1, 0);
    for (size_t i = 0; i < n; i++) {
        const int cr = chunks_rc[2 * i], cc = chunks_rc[2 * i + 1];
        PF_ARG(cr >= 0 && cr < ctx->chunk_h && cc >= 0 && cc < ctx->chunk_w, "zone field: chunk");
        int base_r, base_c;
        chunk_region_base(dim, cr, cc, &base_r, &base_c);
        zone_initial_frontier(zm, centre_r, centre_c, base_r, base_c, dim, budget, seeds);
        off[i + 1] = seeds.size() / 2;
    }
    return chunk_fields(ctx, layer, dim, chunks_rc, n, seeds, off, out_fields);
}

// the pool entries a zone batch changed: slot table entries fresh[2i] = fresh[2i + 1], `has` bytes has[slot[i]] = hasv[i]
__global__ void k_pool_scatter(const int32_t *__restrict__ fresh, int nfresh, int32_t *__restrict__ slot_table,
                               const int32_t *__restrict__ slot, const uint8_t *__restrict__ hasv, int nhas, uint8_t *__restrict__ has)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < nfresh) slot_table[fresh[2 * i]] = fresh[2 * i + 1];
    if (i < nhas) has[slot[i]] = hasv[i];
}

// A zone or entity field of a batch: request `req` writes chunk (cr, cc) of its destination into `slot` (a pool slot, or a
// staging block when a job member builds it for the job)
struct aux_field { uint32_t req; int32_t cr, cc, slot; };

// The stages of a zone batch, shared by pfnav_pool_request_zones and the job form (pf_aux_job_*). zone_validate checks
// the whole batch before anything changes: ctile[2i..] is request i's centre tile when on_map[i] (nav.c:3931), *dim the
// window of its fields.
static int zone_validate(const pfnav_ctx *ctx, const pfnav_zone_req *reqs, size_t m, std::vector<int32_t> &ctile,
                         std::vector<uint8_t> &on_map, int *dim)
{
    PF_ARG(ctx->d_cost && ctx->pool.d_slot, "map / pool not created");
    PF_ARG(m == 0 || reqs, "reqs");
    PF_ARG(m < (1u << 24), "m");
    ctile.assign(2 * m, 0);
    on_map.assign(m, 0);
    bool any_on_map = false;
    for (size_t i = 0; i < m; i++) {
        const pfnav_zone_req &q = reqs[i];
        PF_ARG(q.dest >= 0 && q.dest < ctx->pool.ndests, "dest");
        PF_ARG(q.layer >= 0 && q.layer < ctx->nlayers, "layer");
        PF_ARG(q.radius >= 0 && q.radius <= 0xFFFF, "radius");
        on_map[i] = region_tile_for_point(ctx, q.centre_x, q.centre_z, &ctile[2 * i]);      // nav.c:3931
        any_on_map |= on_map[i] != 0;
    }
    *dim = 0;
    return any_on_map ? zone_dim(ctx, dim) : PFNAV_OK;
}

// the chunks request q's footprint can reach, rows {min, max} then columns (nav.c:3945-3951; C division truncates toward zero)
static void zone_chunks(const pfnav_ctx *ctx, const pfnav_zone_req &q, const int32_t *ctile, int out[4])
{
    const int r0 = ctile[0], c0 = ctile[1], reach = 2 * q.radius;
    auto clampi = [](int v, int lo, int hi) { return std::min(std::max(v, lo), hi); };
    out[0] = clampi((r0 - reach) / 64, 0, ctx->chunk_h - 1); out[1] = clampi((r0 + reach) / 64, 0, ctx->chunk_h - 1);
    out[2] = clampi((c0 - reach) / 64, 0, ctx->chunk_w - 1); out[3] = clampi((c0 + reach) / 64, 0, ctx->chunk_w - 1);
}

// the flood of zone request q's field of chunk (cr, cc) -> its budget when the window holds the centre (what the flood
// pops; field.c:1843), else 0
static uint64_t zone_flood(const pfnav_zone_req &q, const int32_t *ctile, int dim, int cr, int cc, zone_job *j)
{
    size_t budget = (size_t)(M_PI * q.radius * q.radius + 0.5);         // field.c:1843
    if (budget > (size_t)dim * dim) budget = (size_t)dim * dim;
    j->layer = q.layer; j->centre_r = ctile[0]; j->centre_c = ctile[1]; j->budget = (int32_t)budget;
    chunk_region_base(dim, cr, cc, &j->base_r, &j->base_c);
    const int cdr = j->centre_r - j->base_r, cdc = j->centre_c - j->base_c;
    return cdr >= 0 && cdr < dim && cdc >= 0 && cdc < dim ? budget : 0;
}

// Slots request by request, in order, by the single call's rule (pf_pool_zone_take; only `has` bit 0), chunk by chunk. fresh: (slot table index, slot) of every new reservation. On
// PFNAV_ERR_NOMEM, *out_done is the request that did not fit: it keeps its reservations, unbuilt, as the single call
// leaves them.
static int zone_reserve(pfnav_ctx *ctx, const pfnav_zone_req *reqs, size_t m, const std::vector<int32_t> &ctile,
                        const std::vector<uint8_t> &on_map, std::vector<aux_field> &fields, std::vector<int32_t> &fresh,
                        int32_t *out_nfields, size_t *out_done)
{
    const int cw = ctx->chunk_w, nch = cw * ctx->chunk_h;
    int rc = PFNAV_OK;
    size_t done = 0;
    for (; done < m; done++) {
        if (!on_map[done]) continue;
        const pfnav_zone_req &q = reqs[done];
        int ch[4];
        zone_chunks(ctx, q, &ctile[2 * done], ch);
        const size_t first = fields.size();
        for (int cr = ch[0]; cr <= ch[1] && rc == PFNAV_OK; cr++)
            for (int cc = ch[2]; cc <= ch[3]; cc++) {
                const size_t si = (size_t)q.dest * nch + cr * cw + cc;
                const bool had = ctx->pool.slot_of(si) >= 0;
                const int32_t slot = pf_pool_zone_take(ctx, si);
                if (slot < 0) {
                    pfnav_set_error("pfnav_pool_request_zone: pool full (%d fields)", ctx->pool.max);
                    rc = PFNAV_ERR_NOMEM;
                    break;
                }
                if (!had) { fresh.push_back((int32_t)si); fresh.push_back(slot); }
                fields.push_back({(uint32_t)done, cr, cc, slot});
            }
        if (rc) {
            fields.resize(first);
            break;
        }
        for (size_t f = first; f < fields.size(); f++) ctx->pool.built(fields[f].slot, 1);
        if (out_nfields) out_nfields[done] = (int32_t)(fields.size() - first);
    }
    *out_done = done;
    return rc;
}

// A batch floods its zone seeds on the host when the sum of its floods' budgets is at most this many times the largest one.
// The device replays a flood on one lane, about ten times slower per popped tile than the host (H100, DESIGN.md §5), and
// a batch waits for its longest flood; the host floods one field after another.
#define PF_ZONE_HOST_POP_RATIO 10

// One flood + one integration per field of F, into block F[k].slot of d_out (the pool's flow fields, or a job's staging).
// scatter: the pool entries the batch changed (fresh, and the `has` bytes of the F slots) go to the device first;
// k_pool_scatter writes only those, since the device slot table and `has` bytes equal the host mirrors otherwise.
static int zone_build(pfnav_ctx *ctx, cudaStream_t st, const pfnav_zone_req *reqs, const std::vector<int32_t> &ctile, int dim,
                      const std::vector<aux_field> &F, const std::vector<int32_t> &fresh, bool scatter, uint8_t *d_out)
{
    std::vector<zone_job> jobs;
    std::vector<pfnav_region_req> kreq;
    std::vector<int32_t> kslot;
    uint64_t pops = 0, max_pops = 0;        // the floods' budgets: what each costs on the host / the device's critical chain
    for (const aux_field &f : F) {
        const pfnav_zone_req &q = reqs[f.req];
        zone_job j;
        const uint64_t b = zone_flood(q, &ctile[2 * f.req], dim, f.cr, f.cc, &j);
        pops += b; max_pops = std::max(max_pops, b);
        jobs.push_back(j);
        pfnav_region_req rq = {};
        rq.layer = q.layer; rq.center_r = f.cr; rq.center_c = f.cc; rq.flags = PFNAV_REGION_CREATE;
        kreq.push_back(rq); kslot.push_back(f.slot);
    }
    const size_t nk = kreq.size();
    // ---- where the floods run: a device flood is one lane's serial chain, and the batch waits for the longest one; the
    // host floods one field after another. Small batches (a few large zones) flood on the host as seed lists.
    const bool host_floods = pops <= PF_ZONE_HOST_POP_RATIO * max_pops;
    std::vector<int32_t> seeds;
    if (host_floods) {
        const size_t ltiles = (size_t)ctx->chunk_w * ctx->chunk_h * 4096;
        for (size_t k = 0; k < nk; k++) {
            const zone_job &j = jobs[k];
            const zone_map zm = { ctx->h_cost.data() + ltiles * j.layer, ctx->h_blk.data() + ltiles * j.layer, ctx->chunk_w, ctx->chunk_h };
            kreq[k].seed_off = (int32_t)(seeds.size() / 2);
            zone_initial_frontier(zm, j.centre_r, j.centre_c, j.base_r, j.base_c, dim, (size_t)j.budget, seeds);
            kreq[k].seed_n = (int32_t)(seeds.size() / 2) - kreq[k].seed_off;
        }
    }
    // the `has` bytes of the written slots (the host mirror after the batch)
    std::vector<uint8_t> hasv(scatter ? nk : 0);
    for (size_t k = 0; k < hasv.size(); k++) hasv[k] = ctx->pool.has[kslot[k]];
    // ---- the inputs, staged; the seed bitmaps follow them in the device buffer
    size_t b_in = 0;
    auto sec = [&](size_t bytes) { const size_t o = b_in; b_in = (b_in + bytes + 15) & ~(size_t)15; return o; };
    const size_t o_req = sec(nk * sizeof(pfnav_region_req)), o_slot = sec(nk * 4);
    const size_t o_jobs = sec(host_floods ? 0 : nk * sizeof(zone_job)), o_seeds = sec(seeds.size() * 4);
    const size_t o_fresh = sec(fresh.size() * 4), o_hasv = sec(hasv.size());
    const size_t o_bits = b_in, need = o_bits + (host_floods ? 0 : nk * ((size_t)dim * dim / 8)) + 16;
    pf_stage S;
    int lrc = pf_stage_begin(ctx, st, b_in, need, false, &S);
    if (lrc) return lrc;
    uint8_t *host = S.host, *dev = S.dev;
    memcpy(host + o_req, kreq.data(), nk * sizeof(pfnav_region_req));
    memcpy(host + o_slot, kslot.data(), nk * 4);
    if (!host_floods) memcpy(host + o_jobs, jobs.data(), nk * sizeof(zone_job));
    memcpy(host + o_seeds, seeds.data(), seeds.size() * 4);
    memcpy(host + o_fresh, fresh.data(), fresh.size() * 4);
    memcpy(host + o_hasv, hasv.data(), hasv.size());
    if ((lrc = pf_stage_upload(ctx, st, S, b_in))) return lrc;
    const int nscatter = (int)std::max(fresh.size() / 2, hasv.size());
    if (nscatter) {
        k_pool_scatter<<<(unsigned)((nscatter + 255) / 256), 256, 0, st>>>((const int32_t *)(dev + o_fresh), (int)(fresh.size() / 2),
                                                                            ctx->pool.d_slot, (const int32_t *)(dev + o_slot),
                                                                            (const uint8_t *)(dev + o_hasv), (int)hasv.size(),
                                                                            ctx->pool.d_has);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    if (nk && host_floods) {
        if ((lrc = region_launch(ctx, dim, (const pfnav_region_req *)(dev + o_req), nk, (const int32_t *)(dev + o_seeds),
                                 (const int32_t *)dev, d_out, st, 1, nullptr, (const int32_t *)(dev + o_slot))))
            return lrc;
    } else if (nk) {
        const pfnav_region_req *d_req = (const pfnav_region_req *)(dev + o_req);
        uint32_t *d_bits = (uint32_t *)(dev + o_bits);
        const size_t smem = ((size_t)dim * dim + 1) * 4 + 3 * ((size_t)dim * dim / 8);
        PF_CUDA(cudaFuncSetAttribute(k_zone_seed_bits, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                     (PFNAV_REGION_DIM_MAX * PFNAV_REGION_DIM_MAX + 1) * 4 + 3 * PFNAV_REGION_DIM_MAX * PFNAV_REGION_DIM_MAX / 8));
        k_zone_seed_bits<<<(unsigned)nk, 32, smem, st>>>(ctx->d_cost, ctx->d_blk, ctx->H64, ctx->W64, dim, (const zone_job *)(dev + o_jobs),
                                                          (int)nk, d_bits);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
        if ((lrc = region_launch(ctx, dim, d_req, nk, (const int32_t *)dev, (const int32_t *)dev, d_out, st, 1, d_bits,
                                 (const int32_t *)(dev + o_slot))))
            return lrc;
    }
    return pf_stage_done(ctx, st);
}

// N_RequestAsyncGroupArrivalField (nav.c:3921) for m requests, in the order of the serial calls (zone_reserve). The
// device work writes pool slots only: when several fields of the batch land in one slot (a repeated (dest, chunk)), only
// the last is flooded and integrated, which is what the serial calls leave there.
extern "C" int pfnav_pool_request_zones(pfnav_ctx *ctx, const pfnav_zone_req *reqs, size_t m, void *stream, int32_t *out_nfields,
                                        int *out_ndone)
{
    if (out_ndone) *out_ndone = 0;
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    std::vector<int32_t> ctile;
    std::vector<uint8_t> on_map;
    int dim = 0;
    int rc = zone_validate(ctx, reqs, m, ctile, on_map, &dim);
    if (rc) return rc;
    if (out_nfields) std::fill(out_nfields, out_nfields + m, 0);
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    PF_CUDA(pf_fields_join(ctx, st));
    PF_CUDA(pf_pool_refresh(ctx, st));
    std::vector<aux_field> fields;
    std::vector<int32_t> fresh;
    size_t done = 0;
    rc = zone_reserve(ctx, reqs, m, ctile, on_map, fields, fresh, out_nfields, &done);
    if (out_ndone) *out_ndone = (int)done;
    if (fields.empty() && fresh.empty()) return rc;
    // ---- one flood + one integration per slot: the last field written to it
    std::vector<int32_t> last(ctx->pool.max, -1);
    for (size_t f = 0; f < fields.size(); f++) last[fields[f].slot] = (int32_t)f;
    std::vector<aux_field> build;
    for (size_t f = 0; f < fields.size(); f++)
        if (last[fields[f].slot] == (int32_t)f) build.push_back(fields[f]);
    const int lrc = zone_build(ctx, st, reqs, ctile, dim, build, fresh, true, ctx->pool.d_flow);
    return lrc ? lrc : rc;
}

extern "C" int pfnav_pool_request_zone(pfnav_ctx *ctx, int dest, int layer, const float *centre_xz, int radius, void *stream,
                                       int *out_nfields)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(centre_xz, "centre");
    const pfnav_zone_req q = {dest, layer, centre_xz[0], centre_xz[1], radius, 0};
    int rc = pfnav_pool_request_zones(ctx, &q, 1, stream, out_nfields, nullptr);
    if (rc) return rc;
    PF_CUDA(cudaStreamSynchronize(pf_stream(ctx, stream)));      // returns once the fields are in the pool
    return PFNAV_OK;
}

// pfnav_group_arrival_velocity, and its resident form when P is not NULL: P's named positions are staged in place of
// pos_xz and written on the device by k_resident_xz, ahead of the same kernel
static int group_arrival(pfnav_ctx *ctx, int dest, const float *centre_xz, int radius, const float *pos_xz,
                         const pf_resident_points *P, size_t n, float *out_vel, uint8_t *out_flags)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->pool.d_slot, "pool not created");
    PF_ARG(dest >= 0 && dest < ctx->pool.ndests, "dest");
    if (n == 0) return PFNAV_OK;
    PF_ARG(centre_xz && (pos_xz || P) && out_vel && out_flags, "null buffer");
    PF_ARG(n < (1u << 30), "n");
    PF_ARG(radius >= 0 && radius <= 0xFFFF, "radius");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(pf_fields_sync(ctx));
    cudaStream_t st = ctx->tick_stream;
    PF_CUDA(pf_pool_refresh(ctx, st));
    // staged: the positions (the resident form: the named pairs, then room for the positions), then the velocities and
    // the flags
    const size_t o_pos = P ? (P->bytes() + 15) & ~(size_t)15 : 0, up = P ? P->bytes() : n * 8;
    pf_stage S;
    if (int rc = pf_stage_begin(ctx, st, up, o_pos + n * 17, false, &S)) return rc;
    if (P) P->pack(S.host);
    else memcpy(S.host, pos_xz, n * 8);
    if (int rc = pf_stage_upload(ctx, st, S, up)) return rc;
    const float2 *d_pos = (const float2 *)(S.dev + o_pos);
    float2 *d_vel = (float2 *)(S.dev + o_pos + n * 8);
    uint8_t *d_fl = S.dev + o_pos + n * 16;
    if (P)
        if (int rc = pf_resident_xz_launch(ctx, st, S.dev, *P, 2, 0, 0, (float *)d_pos)) return rc;
    ZoneView z = { ctx->pool.d_slot, ctx->pool.d_flow, ctx->pool.d_has, ctx->chunk_w, ctx->chunk_h,
                   ctx->map_x, ctx->map_z };
    k_group_arrival_velocity<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(z, dest, centre_xz[0], centre_xz[1], radius, d_pos, (int)n, d_vel, d_fl);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaMemcpyAsync(out_vel, d_vel, n * 8, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaMemcpyAsync(out_flags, d_fl, n, cudaMemcpyDeviceToHost, st));
    if (int rc = pf_stage_done(ctx, st)) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

extern "C" int pfnav_group_arrival_velocity(pfnav_ctx *ctx, int dest, const float *centre_xz, int radius, const float *pos_xz,
                                            size_t n, float *out_vel, uint8_t *out_flags)
{
    return group_arrival(ctx, dest, centre_xz, radius, pos_xz, nullptr, n, out_vel, out_flags);
}

extern "C" int pfnav_group_arrival_velocity_resident(pfnav_ctx *ctx, int dest, const float *centre_xz, int radius,
                                                     const uint32_t *uids, size_t n, float *out_vel, uint8_t *out_flags)
{
    PF_ARG(ctx, "ctx");
    pf_resident_points P;
    if (int rc = pf_resident_points_begin(ctx, "group arrival velocities", n, uids, false, nullptr, true, P)) return rc;
    return group_arrival(ctx, dest, centre_xz, radius, nullptr, &P, n, out_vel, out_flags);
}

// The zone's seed tiles alone (host structure code, no device needed): the first `budget` open tiles of the
// best-first flood. out_rc = (r, c) pairs, at most cap of them; *out_n = the full count.
extern "C" int pfnav_zone_seeds(pfnav_ctx *ctx, int layer, int chunk_r, int chunk_c, int centre_r, int centre_c, int radius,
                                int32_t *out_rc, size_t cap, size_t *out_n)
{
    PF_ARG(ctx && !ctx->h_cost.empty(), "map not created");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG(chunk_r >= 0 && chunk_r < ctx->chunk_h && chunk_c >= 0 && chunk_c < ctx->chunk_w, "chunk");
    PF_ARG(centre_r >= 0 && centre_r < ctx->H64 && centre_c >= 0 && centre_c < ctx->W64, "zone centre outside the map");
    PF_ARG(radius >= 0 && radius <= 0xFFFF && out_n, "radius / out_n");
    int dim = 0;
    int rc = zone_dim(ctx, &dim);
    if (rc) return rc;
    const size_t ltiles = (size_t)ctx->chunk_w * ctx->chunk_h * 4096;
    zone_map zm = { ctx->h_cost.data() + ltiles * layer, ctx->h_blk.data() + ltiles * layer, ctx->chunk_w, ctx->chunk_h };
    size_t budget = (size_t)(M_PI * radius * radius + 0.5);
    if (budget > (size_t)dim * dim) budget = (size_t)dim * dim;
    const int base_r = (chunk_r > 0 && dim > 64) ? chunk_r * 64 - 32 : chunk_r * 64, base_c = (chunk_c > 0 && dim > 64) ? chunk_c * 64 - 32 : chunk_c * 64;
    std::vector<int32_t> seeds;
    zone_initial_frontier(zm, centre_r, centre_c, base_r, base_c, dim, budget, seeds);
    *out_n = seeds.size() / 2;
    if (out_rc) memcpy(out_rc, seeds.data(), std::min(cap * 2, seeds.size()) * sizeof(int32_t));
    return PFNAV_OK;
}


// ------------------------------------------------------------------------------------------
// TARGET_ENTITY / TARGET_ENEMIES chunk fields (field_update_entity field.c:1609, field_update_enemies :1540)
// ------------------------------------------------------------------------------------------
// BG_SCALE_F (lib/public/bitmap_grid.h:196): the position index compares scaled integers, bounds inclusive (:543)
static inline int32_t bg_scale_f(float x) { return (int32_t)lrintf(x * 256.0f); }

// contour rings around a target's footprint: field_entity_initial_frontier (field.c:1317; note `layer == GROUND_3X3` for
// the first ring) and field_enemies_initial_frontier (field.c:1209)
static inline int entity_rings(int kind, int ref_layer)
{
    return kind == PFNAV_TARGET_ENTITY ? (ref_layer == 1) + (ref_layer >= 2) + (ref_layer >= 3)
                                       : (ref_layer >= 1) + (ref_layer >= 2) + (ref_layer >= 3);
}

// the scaled search rectangle of chunk (chunk_r, chunk_c), bounds inclusive: field_chunk_bounds (field.c:863) and
// field.c:1229-1243, in the reference's float arithmetic
struct search_rect { int32_t mnx, mxx, mnz, mxz; };
static search_rect enemies_search_rect(const pfnav_ctx *ctx, int chunk_r, int chunk_c)
{
    const int x_offset = -(chunk_c * 256), z_offset = chunk_r * 256;
    const float x_max = ctx->map_x + (float)x_offset, x_min = x_max - 256.0f;
    const float z_min = ctx->map_z + (float)z_offset, z_max = z_min + 256.0f;
    const float xlen = x_max - x_min, zlen = z_max - z_min;
    return {bg_scale_f(x_min - xlen / 2.0f - 16.0f), bg_scale_f(x_max + xlen / 2.0f + 16.0f),
            bg_scale_f(z_min - zlen / 2.0f - 16.0f), bg_scale_f(z_max + zlen / 2.0f + 16.0f)};
}

static int entity_seeds(const pfnav_ctx *ctx, int ref_layer, int kind, const pfnav_footprint *ents, size_t nents, int dim,
                        int chunk_r, int chunk_c, std::vector<int32_t> &out)
{
    int base_r, base_c;
    chunk_region_base(dim, chunk_r, chunk_c, &base_r, &base_c);
    int32_t tiles[512 * 2];
    const int rings = entity_rings(kind, ref_layer);
    if (kind == PFNAV_TARGET_ENTITY) {
        const int n = pfnav_footprint_tiles(ctx, &ents[0], rings, tiles);
        if (n < 0) { pfnav_set_error("entity field: a building corner lies outside the map"); return PFNAV_ERR_ARG; }
        for (int i = 0; i < n; i++) {
            const int dr = tiles[2 * i] - base_r, dc = tiles[2 * i + 1] - base_c;
            if (dr < 0 || dr >= dim || dc < 0 || dc >= dim) continue;
            out.push_back(tiles[2 * i]); out.push_back(tiles[2 * i + 1]);
        }
        return PFNAV_OK;
    }
    // field_enemies_initial_frontier (field.c:1209)
    const search_rect R = enemies_search_rect(ctx, chunk_r, chunk_c);
    std::vector<uint8_t> has((size_t)dim * dim, 0);
    for (size_t k = 0; k < nents; k++) {
        const int32_t ix = bg_scale_f(ents[k].x), iz = bg_scale_f(ents[k].z);
        if (ix < R.mnx || ix > R.mxx || iz < R.mnz || iz > R.mxz) continue;
        const int n = pfnav_footprint_tiles(ctx, &ents[k], rings, tiles);
        if (n < 0) { pfnav_set_error("enemies field: a building corner lies outside the map"); return PFNAV_ERR_ARG; }
        for (int i = 0; i < n; i++) {
            const int dr = tiles[2 * i] - base_r, dc = tiles[2 * i + 1] - base_c;
            if (dr < 0 || dr >= dim || dc < 0 || dc >= dim) continue;
            has[(size_t)dr * dim + dc] = 1;
        }
    }
    for (int r = 0; r < dim; r++)
        for (int c = 0; c < dim; c++)
            if (has[(size_t)r * dim + c]) { out.push_back(base_r + r); out.push_back(base_c + c); }
    return PFNAV_OK;
}

static int entity_args_ok(const pfnav_ctx *ctx, int ref_layer, int kind, const pfnav_footprint *ents, size_t nents)
{
    PF_ARG(ref_layer >= 0 && ref_layer < PFNAV_NAV_LAYER_MAX, "ref_layer");
    PF_ARG(kind == PFNAV_TARGET_ENTITY || kind == PFNAV_TARGET_ENEMIES, "target_kind");
    PF_ARG(nents == 0 || ents, "ents");
    PF_ARG(kind != PFNAV_TARGET_ENTITY || nents == 1, "TARGET_ENTITY takes exactly one entity");
    PF_ARG(nents < (1u << 24), "nents");
    return PFNAV_OK;
}

extern "C" int pfnav_entity_seeds(pfnav_ctx *ctx, int ref_layer, int target_kind, const pfnav_footprint *ents, size_t nents,
                                  int chunk_r, int chunk_c, int32_t *out_rc, size_t cap, size_t *out_n)
{
    PF_ARG(ctx && !ctx->h_cost.empty(), "map not created");
    PF_ARG(chunk_r >= 0 && chunk_r < ctx->chunk_h && chunk_c >= 0 && chunk_c < ctx->chunk_w && out_n, "chunk / out_n");
    int rc = entity_args_ok(ctx, ref_layer, target_kind, ents, nents);
    if (rc) return rc;
    int dim = 0;
    rc = zone_dim(ctx, &dim);
    if (rc) return rc;
    std::vector<int32_t> seeds;
    rc = entity_seeds(ctx, ref_layer, target_kind, ents, nents, dim, chunk_r, chunk_c, seeds);
    if (rc) return rc;
    *out_n = seeds.size() / 2;
    if (out_rc) memcpy(out_rc, seeds.data(), std::min(cap * 2, seeds.size()) * sizeof(int32_t));
    return PFNAV_OK;
}

extern "C" int pfnav_entity_fields(pfnav_ctx *ctx, int layer, int ref_layer, int target_kind, const pfnav_footprint *ents,
                                   size_t nents, const int32_t *chunks_rc, size_t n, uint8_t *out_fields)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    if (n == 0) return PFNAV_OK;
    PF_ARG(chunks_rc && out_fields, "null buffer");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG(n < (1u << 24), "n");
    int rc = entity_args_ok(ctx, ref_layer, target_kind, ents, nents);
    if (rc) return rc;
    int dim = 0;
    rc = zone_dim(ctx, &dim);
    if (rc) return rc;
    std::vector<int32_t> seeds;
    std::vector<size_t> off(n + 1, 0);
    for (size_t i = 0; i < n; i++) {
        const int cr = chunks_rc[2 * i], cc = chunks_rc[2 * i + 1];
        PF_ARG(cr >= 0 && cr < ctx->chunk_h && cc >= 0 && cc < ctx->chunk_w, "entity field: chunk");
        rc = entity_seeds(ctx, ref_layer, target_kind, ents, nents, dim, cr, cc, seeds);
        if (rc) return rc;
        off[i + 1] = seeds.size() / 2;
    }
    return chunk_fields(ctx, layer, dim, chunks_rc, n, seeds, off, out_fields);
}


// ------------------------------------------------------------------------------------------
// TARGET_ENEMIES / TARGET_ENTITY fields as pool destinations: what N_RequestAsyncEnemySeekField /
// N_RequestAsyncSurroundField + N_AwaitAsyncFields leave in the field cache for the chunks the seekers stand on
// (nav.c:3769-3960), consumed by N_DesiredEnemySeekVelocity / N_DesiredSurroundVelocity (k_desired_velocity).
// ------------------------------------------------------------------------------------------
//
// A batch builds its seed frontiers on the device, in three launches on the caller's stream:
//   k_footprint_rows    one warp per distinct (circle footprint, ring count) of the batch: the tiles under the circle
//                       and its contour rings as 32 bit rows, with the circle test and the dilation of the blocker
//                       rasterisation (pfnav_tile_geom.cuh);
//   k_entity_seed_bits  one CTA per field: its dim x dim seed bitmap, the union of the footprint rows inside the padded
//                       window plus the tile lists of the footprints rasterised on the host (buildings, and circles
//                       whose rings could reach the 512-tile cap of pfnav_footprint_tiles, which truncates in list order);
//   k_region_fields     (chunk_out with seed_bits and out_slot) integrates every field straight into its pool slot.
// TARGET_ENEMIES footprints are binned by chunk on the host, with the scaled-integer test of entity_seeds, so the work
// grows with footprints x 9 and not with fields x footprints. The device work only writes pool slots; when several
// fields of a batch end in the same slot (a repeated (dest, chunk), or a slot evicted and handed out again inside the
// batch) only the last is built, which is what the serial calls leave there.
namespace {

struct fp_job { float x, z, radius; int32_t rings; };

__global__ void __launch_bounds__(128) k_footprint_rows(const fp_job *__restrict__ jobs, int n, geom g, int H64, int W64,
                                                        int2 *__restrict__ org, uint32_t *__restrict__ rows_out)
{
    __shared__ unsigned rows[4][32];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, j = blockIdx.x * 4 + w;
    if (j >= n) return;
    const fp_job f = jobs[j];
    td ct;
    unsigned u = 0;
    int r0 = 0, c0 = 0;
    if (desc_for_point(g, f.x, f.z, &ct)) {          // otherwise no tile under the circle (tile.c:693) and no ring
        const int nt = (int)ceilf(f.radius / 4);
        r0 = ct.chunk_r * 64 + ct.tile_r - nt - 3; c0 = ct.chunk_c * 64 + ct.tile_c - nt - 3;
        rows[w][lane] = 0;
        __syncwarp();
        circle_rows(g, H64, W64, v2f{f.x, f.z}, f.radius, nt, r0, c0, rows[w], lane);
        const unsigned inmap = window_inmap(H64, W64, r0, c0, 2 * nt + 7, lane);
        u = rows[w][lane];
        for (int k = 0; k < f.rings; k++) u |= contour_rows(u, inmap, lane);     // each ring around all tiles so far
    }
    if (lane == 0) org[j] = make_int2(r0, c0);
    rows_out[(size_t)j * 32 + lane] = u;
}

// field f: items[item_off[f] ..) name k_footprint_rows outputs, hitems[hitem_off[f] ..) host tile lists
__global__ void __launch_bounds__(256) k_entity_seed_bits(const pfnav_region_req *__restrict__ reqs, int dim,
                                                          const uint32_t *__restrict__ item_off, const int32_t *__restrict__ items,
                                                          const int2 *__restrict__ org, const uint32_t *__restrict__ rows,
                                                          const uint32_t *__restrict__ hitem_off, const int32_t *__restrict__ hitems,
                                                          const uint32_t *__restrict__ htile_off, const int32_t *__restrict__ htiles,
                                                          uint32_t *__restrict__ bits_out)
{
    __shared__ uint32_t bm[PFNAV_REGION_DIM_MAX * PFNAV_REGION_DIM_MAX / 32];
    const int f = blockIdx.x, tid = threadIdx.x;
    const int wpr = dim >> 5, nw = dim * wpr;           // dim is 64 or 128: whole words per row
    for (int i = tid; i < nw; i += blockDim.x) bm[i] = 0;
    __syncthreads();
    const pfnav_region_req rq = reqs[f];
    const int base_r = (rq.center_r > 0 && dim > 64) ? rq.center_r * 64 - 32 : rq.center_r * 64;
    const int base_c = (rq.center_c > 0 && dim > 64) ? rq.center_c * 64 - 32 : rq.center_c * 64;
    // one thread per (footprint, window row): the row's 32 columns land in at most two bitmap words
    for (uint32_t t = item_off[f] * 32 + tid; t < item_off[f + 1] * 32; t += blockDim.x) {
        const int32_t it = items[t >> 5];
        const int row = t & 31;
        const uint32_t v = rows[(size_t)it * 32 + row];
        if (!v) continue;
        const int2 o = org[it];
        const int dr = o.x + row - base_r, off = o.y - base_c;      // off: the field column of bit 0
        if (dr < 0 || dr >= dim || off <= -32 || off >= dim) continue;
        const uint64_t x = off >= 0 ? (uint64_t)v << (off & 31) : (uint64_t)(v >> -off);
        const int wc = off >= 0 ? off >> 5 : 0;
        if ((uint32_t)x) atomicOr(&bm[dr * wpr + wc], (uint32_t)x);
        if (wc + 1 < wpr && (uint32_t)(x >> 32)) atomicOr(&bm[dr * wpr + wc + 1], (uint32_t)(x >> 32));
    }
    for (uint32_t k = hitem_off[f]; k < hitem_off[f + 1]; k++) {
        const int32_t h = hitems[k];
        for (uint32_t t = htile_off[h] + tid; t < htile_off[h + 1]; t += blockDim.x) {
            const int dr = htiles[2 * t] - base_r, dc = htiles[2 * t + 1] - base_c;
            if (dr >= 0 && dr < dim && dc >= 0 && dc < dim) atomicOr(&bm[dr * wpr + (dc >> 5)], 1u << (dc & 31));
        }
    }
    __syncthreads();
    for (int i = tid; i < nw; i += blockDim.x) bits_out[(size_t)f * nw + i] = bm[i];
}

}   // namespace

// k_footprint_rows rasterises a circle when its tiles and rings fit the 32 x 32 window and can not reach the 512-tile cap
// of pfnav_footprint_tiles: then they are the same set, whatever their order
static bool footprint_on_device(const pfnav_footprint &e, int rings)
{
    if (e.is_building || !std::isfinite(e.x) || !std::isfinite(e.z) || !(e.sel_radius >= 0.0f && e.sel_radius <= 64.0f))
        return false;
    const int side = 2 * (int)ceil(e.sel_radius / 4) + 1 + 2 * rings;
    return side * side <= 512;
}

static bool building_corners_ok(const pfnav_ctx *ctx, const pfnav_footprint &e)
{
    if (!e.is_building) return true;
    const geom g = {ctx->map_x, ctx->map_z, ctx->chunk_w, ctx->chunk_h};
    td t;
    for (int i = 0; i < 4; i++)
        if (!desc_for_point(g, e.corners_xz[2 * i], e.corners_xz[2 * i + 1], &t)) return false;
    return true;
}

// TARGET_ENEMIES footprints of one range, binned by the chunks whose search rectangle holds their position
struct enemy_bins {
    std::vector<uint32_t> off;           // [chunks + 1]
    std::vector<uint32_t> ent;           // absolute footprint indices
    std::vector<uint8_t> bad;            // [chunks]: a building in the bin has a corner outside the map
};

static void bin_enemies(const pfnav_ctx *ctx, const pfnav_footprint *ents, uint32_t off, uint32_t n, enemy_bins &B)
{
    const int cw = ctx->chunk_w, chh = ctx->chunk_h, nch = cw * chh;
    std::vector<search_rect> rx(cw), rz(chh);
    for (int c = 0; c < cw; c++) rx[c] = enemies_search_rect(ctx, 0, c);
    for (int r = 0; r < chh; r++) rz[r] = enemies_search_rect(ctx, r, 0);
    // the chunks whose rectangle holds a position form a contiguous block (the rectangles are translates)
    std::vector<int32_t> span((size_t)n * 4);
    B.off.assign(nch + 1, 0);
    for (uint32_t k = 0; k < n; k++) {
        const int32_t ix = bg_scale_f(ents[off + k].x), iz = bg_scale_f(ents[off + k].z);
        int c0 = cw, c1 = -1, r0 = chh, r1 = -1;
        for (int c = 0; c < cw; c++) if (ix >= rx[c].mnx && ix <= rx[c].mxx) { c0 = std::min(c0, c); c1 = c; }
        for (int r = 0; r < chh; r++) if (iz >= rz[r].mnz && iz <= rz[r].mxz) { r0 = std::min(r0, r); r1 = r; }
        int32_t *s = &span[(size_t)k * 4];
        s[0] = r0; s[1] = r1; s[2] = c0; s[3] = c1;
        for (int r = r0; r <= r1; r++)
            for (int c = c0; c <= c1; c++) B.off[r * cw + c + 1]++;
    }
    for (int i = 0; i < nch; i++) B.off[i + 1] += B.off[i];
    B.ent.resize(B.off[nch]);
    B.bad.assign(nch, 0);
    std::vector<uint32_t> cur(B.off.begin(), B.off.end() - 1);
    for (uint32_t k = 0; k < n; k++) {
        const int32_t *s = &span[(size_t)k * 4];
        const bool bad = !building_corners_ok(ctx, ents[off + k]);
        for (int r = s[0]; r <= s[1]; r++)
            for (int c = s[2]; c <= s[3]; c++) { B.ent[cur[r * cw + c]++] = off + k; B.bad[r * cw + c] |= bad; }
    }
}

// The stages of an entity-field batch, shared by pfnav_pool_request_entity_fields_batch and the job form
// (pf_aux_job_*). entity_validate checks the whole batch before anything changes and bins the TARGET_ENEMIES footprints,
// one bin per distinct footprint range (req_bin[i]: request i's).
struct entity_batch { int dim = 0; std::vector<enemy_bins> bins; std::vector<int32_t> req_bin; };

static int entity_validate(const pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m, const pfnav_footprint *ents,
                           size_t nents, const int32_t *chunks_rc, size_t nchunks, entity_batch &E)
{
    PF_ARG(ctx->d_cost && ctx->pool.d_slot, "map / pool not created");
    PF_ARG(m == 0 || reqs, "reqs");
    PF_ARG((nents == 0 || ents) && (nchunks == 0 || chunks_rc), "ents / chunks_rc");
    PF_ARG(m < (1u << 24) && nents < (1u << 24) && nchunks < (1u << 24), "m / nents / nchunks");
    const int cw = ctx->chunk_w;
    bool any_fields = false;
    for (size_t i = 0; i < m; i++) {
        const pfnav_entity_field_req &q = reqs[i];
        PF_ARG(q.dest >= 0 && q.dest < ctx->pool.ndests, "dest");
        PF_ARG(q.layer >= 0 && q.layer < ctx->nlayers, "layer");
        PF_ARG((uint64_t)q.ent_off + q.ent_n <= nents, "footprint range");
        PF_ARG((uint64_t)q.chunk_off + q.chunk_n <= nchunks, "chunk range");
        int rc = entity_args_ok(ctx, q.ref_layer, q.target_kind, ents + q.ent_off, q.ent_n);
        if (rc) return rc;
        for (uint32_t k = 0; k < q.chunk_n; k++) {
            const int32_t *c = chunks_rc + 2 * ((size_t)q.chunk_off + k);
            PF_ARG(c[0] >= 0 && c[0] < ctx->chunk_h && c[1] >= 0 && c[1] < cw, "entity field: chunk");
        }
        any_fields |= q.chunk_n > 0;
    }
    E.dim = 0;
    if (any_fields) {
        int rc = zone_dim(ctx, &E.dim);
        if (rc) return rc;
    }
    // TARGET_ENEMIES bins, one per distinct footprint range; building corners of every footprint a field will use
    std::map<std::pair<uint32_t, uint32_t>, int> bin_of;
    E.bins.clear();
    E.req_bin.assign(m, -1);
    for (size_t i = 0; i < m; i++) {
        const pfnav_entity_field_req &q = reqs[i];
        if (q.chunk_n == 0) continue;
        if (q.target_kind == PFNAV_TARGET_ENTITY) {
            PF_ARG(building_corners_ok(ctx, ents[q.ent_off]), "entity field: a building corner lies outside the map");
            continue;
        }
        auto it = bin_of.find({q.ent_off, q.ent_n});
        if (it == bin_of.end()) {
            it = bin_of.emplace(std::make_pair(q.ent_off, q.ent_n), (int)E.bins.size()).first;
            E.bins.emplace_back();
            bin_enemies(ctx, ents, q.ent_off, q.ent_n, E.bins.back());
        }
        E.req_bin[i] = it->second;
        for (uint32_t k = 0; k < q.chunk_n; k++) {
            const int32_t *c = chunks_rc + 2 * ((size_t)q.chunk_off + k);
            PF_ARG(!E.bins[it->second].bad[c[0] * cw + c[1]], "enemies field: a building corner lies outside the map");
        }
    }
    return PFNAV_OK;
}

// Slots request by request, in order: the serial calls' reservations and evictions, and the footprints each destination
// remembers. On an error, *out_done is the request that failed.
static int entity_reserve(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m, const pfnav_footprint *ents,
                          const int32_t *chunks_rc, std::vector<aux_field> &fields, size_t *out_done)
{
    const int cw = ctx->chunk_w, nch = cw * ctx->chunk_h;
    if (ctx->aux.size() < (size_t)ctx->pool.ndests) ctx->aux.resize(ctx->pool.ndests);
    std::vector<size_t> keys;
    std::vector<int32_t> slots;
    int rc = PFNAV_OK;
    size_t done = 0;
    for (; done < m; done++) {
        const pfnav_entity_field_req &q = reqs[done];
        const int32_t *crc = chunks_rc + 2 * (size_t)q.chunk_off;
        if (q.chunk_n) {
            keys.resize(q.chunk_n); slots.resize(q.chunk_n);
            for (uint32_t k = 0; k < q.chunk_n; k++) keys[k] = (size_t)q.dest * nch + crc[2 * k] * cw + crc[2 * k + 1];
            bool evicted = false;
            if ((rc = pf_pool_reserve(ctx, keys.data(), q.chunk_n, slots.data(), &evicted))) break;
        }
        // the footprints stay with the destination: the in-place repairs of its fields start from them (field.c:2334-2360)
        pfnav_ctx::aux_target &A = ctx->aux[q.dest];
        A.kind = q.target_kind; A.layer = q.layer; A.ref_layer = q.ref_layer; A.ents.assign(ents + q.ent_off, ents + q.ent_off + q.ent_n);
        for (uint32_t k = 0; k < q.chunk_n; k++) {
            pfnav_field_req fr;
            memset(&fr, 0, sizeof(fr));
            fr.chunk_r = crc[2 * k]; fr.chunk_c = crc[2 * k + 1]; fr.layer = q.layer; fr.faction_id = PFNAV_FACTION_ID_NONE;
            fr.target_type = 2 + q.target_kind;      // beyond the chunk-local kinds: the frontier comes from ctx->aux[dest]
            fr._pad = q.dest;
            ctx->pool.built_flow(slots[k], fr);
            fields.push_back({(uint32_t)done, crc[2 * k], crc[2 * k + 1], slots[k]});
        }
    }
    *out_done = done;
    return rc;
}

// The fields F (each into block F[k].slot of d_out: the pool's flow fields, or a job's staging): their footprints,
// rasters, seed bitmaps and integrations. upload_pool: the slot table and the `has` bytes travel in the same pinned
// staging buffer and go to the device first.
static int entity_build(pfnav_ctx *ctx, cudaStream_t st, const pfnav_entity_field_req *reqs, const pfnav_footprint *ents,
                        size_t nents, const entity_batch &E, const std::vector<aux_field> &F, bool upload_pool, uint8_t *d_out)
{
    const int cw = ctx->chunk_w, dim = E.dim;
    std::vector<pfnav_region_req> kreq;
    std::vector<int32_t> kslot, items, hitems, htiles;
    std::vector<uint32_t> item_off(1, 0), hitem_off(1, 0), htile_off(1, 0);
    std::vector<fp_job> jobs;
    std::vector<int32_t> raster((size_t)4 * nents, -1);      // (rings, footprint) -> job, or -2 - host list
    auto use = [&](uint32_t e, int rings) {
        int32_t &id = raster[(size_t)rings * nents + e];
        if (id == -1) {
            const pfnav_footprint &P = ents[e];
            if (footprint_on_device(P, rings)) {
                id = (int32_t)jobs.size();
                jobs.push_back({P.x, P.z, P.sel_radius, rings});
            } else {
                int32_t tiles[512 * 2];
                const int n = std::max(pfnav_footprint_tiles(ctx, &P, rings, tiles), 0);    // corners checked above
                id = -2 - (int32_t)(htile_off.size() - 1);
                htiles.insert(htiles.end(), tiles, tiles + 2 * n);
                htile_off.push_back((uint32_t)(htiles.size() / 2));
            }
        }
        if (id >= 0) items.push_back(id);
        else hitems.push_back(-2 - id);
    };
    for (const aux_field &f : F) {
        const pfnav_entity_field_req &q = reqs[f.req];
        const int rings = entity_rings(q.target_kind, q.ref_layer);
        if (q.target_kind == PFNAV_TARGET_ENTITY) use(q.ent_off, rings);
        else {
            const enemy_bins &B = E.bins[E.req_bin[f.req]];
            const int c = f.cr * cw + f.cc;
            for (uint32_t k = B.off[c]; k < B.off[c + 1]; k++) use(B.ent[k], rings);
        }
        pfnav_region_req rq = {};
        rq.layer = q.layer; rq.center_r = f.cr; rq.center_c = f.cc; rq.flags = PFNAV_REGION_CREATE;
        kreq.push_back(rq); kslot.push_back(f.slot);
        item_off.push_back((uint32_t)items.size()); hitem_off.push_back((uint32_t)hitems.size());
    }
    const size_t nk = kreq.size(), nj = jobs.size();
    // ---- the inputs, staged (then the slot table and `has` bytes); footprint rows and seed bitmaps follow them on the device
    size_t b_in = 0;
    auto sec = [&](size_t bytes) { const size_t o = b_in; b_in = (b_in + bytes + 15) & ~(size_t)15; return o; };
    const size_t o_req = sec(nk * sizeof(pfnav_region_req)), o_slot = sec(nk * 4);
    const size_t o_ioff = sec(item_off.size() * 4), o_items = sec(items.size() * 4);
    const size_t o_hoff = sec(hitem_off.size() * 4), o_hitems = sec(hitems.size() * 4);
    const size_t o_jobs = sec(nj * sizeof(fp_job)), o_toff = sec(htile_off.size() * 4), o_tiles = sec(htiles.size() * 4);
    const size_t o_org = b_in + 0, o_rows = o_org + ((nj * 8 + 15) & ~(size_t)15), o_bits = o_rows + nj * 128;
    const size_t need = o_bits + nk * ((size_t)dim * dim / 8);
    pf_stage S;
    int rc = pf_stage_begin(ctx, st, b_in, need, upload_pool, &S);
    if (rc) return rc;
    uint8_t *host = S.host, *dev = S.dev;
    memcpy(host + o_req, kreq.data(), nk * sizeof(pfnav_region_req));
    memcpy(host + o_slot, kslot.data(), nk * 4);
    memcpy(host + o_ioff, item_off.data(), item_off.size() * 4);
    memcpy(host + o_items, items.data(), items.size() * 4);
    memcpy(host + o_hoff, hitem_off.data(), hitem_off.size() * 4);
    memcpy(host + o_hitems, hitems.data(), hitems.size() * 4);
    memcpy(host + o_jobs, jobs.data(), nj * sizeof(fp_job));
    memcpy(host + o_toff, htile_off.data(), htile_off.size() * 4);
    memcpy(host + o_tiles, htiles.data(), htiles.size() * 4);
    if ((rc = pf_stage_upload(ctx, st, S, b_in))) return rc;
    const pfnav_region_req *d_req = (const pfnav_region_req *)(dev + o_req);
    int2 *d_org = (int2 *)(dev + o_org);
    uint32_t *d_rows = (uint32_t *)(dev + o_rows), *d_bits = (uint32_t *)(dev + o_bits);
    if (nj) {
        const geom g = {ctx->map_x, ctx->map_z, cw, ctx->chunk_h};
        k_footprint_rows<<<(unsigned)((nj + 3) / 4), 128, 0, st>>>((const fp_job *)(dev + o_jobs), (int)nj, g, ctx->H64, ctx->W64,
                                                                 d_org, d_rows);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    k_entity_seed_bits<<<(unsigned)nk, 256, 0, st>>>(d_req, dim, (const uint32_t *)(dev + o_ioff), (const int32_t *)(dev + o_items),
                                                     d_org, d_rows, (const uint32_t *)(dev + o_hoff), (const int32_t *)(dev + o_hitems),
                                                     (const uint32_t *)(dev + o_toff), (const int32_t *)(dev + o_tiles), d_bits);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    if ((rc = region_launch(ctx, dim, d_req, nk, (const int32_t *)dev, (const int32_t *)dev, d_out, st, 1, d_bits,
                            (const int32_t *)(dev + o_slot))))
        return rc;
    return pf_stage_done(ctx, st);
}

extern "C" int pfnav_pool_request_entity_fields_batch(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m,
                                                      const pfnav_footprint *ents, size_t nents, const int32_t *chunks_rc,
                                                      size_t nchunks, void *stream, int *out_ndone)
{
    if (out_ndone) *out_ndone = 0;
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    entity_batch E;
    int rc = entity_validate(ctx, reqs, m, ents, nents, chunks_rc, nchunks, E);
    if (rc) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    PF_CUDA(pf_fields_join(ctx, st));
    PF_CUDA(pf_pool_refresh(ctx, st));
    std::vector<aux_field> fields;
    size_t done = 0;
    rc = entity_reserve(ctx, reqs, m, ents, chunks_rc, fields, &done);
    if (out_ndone) *out_ndone = (int)done;
    if (fields.empty()) return rc;
    // ---- the last field written to each slot
    std::vector<int32_t> last(ctx->pool.max, -1);
    for (size_t f = 0; f < fields.size(); f++) last[fields[f].slot] = (int32_t)f;
    std::vector<aux_field> build;
    for (size_t f = 0; f < fields.size(); f++)
        if (last[fields[f].slot] == (int32_t)f) build.push_back(fields[f]);
    const int lrc = entity_build(ctx, st, reqs, ents, nents, E, build, true, ctx->pool.d_flow);
    return lrc ? lrc : rc;
}

// ------------------------------------------------------------------------------------------
// Entity-field batches named by uid (pfnav_pool_request_entity_fields_resident and its job forms): the footprints and
// the seekers' chunks come from the resident records, then the batch runs on them as given.
// ------------------------------------------------------------------------------------------
namespace {

// one thread per named uid: the first nfp name footprints ({x, z, radius} of the record), the rest seekers (the chunk
// index under the record's position, M_Tile_DescForPoint2D as the tick takes it; -1 when no tile lies under it)
__global__ void __launch_bounds__(256) k_resident_footprints(const pf_record *__restrict__ rec, const uint32_t *__restrict__ uids,
                                                             int nfp, int n, MapView m, float *__restrict__ fp_out,
                                                             int32_t *__restrict__ chunk_out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const pf_record r = rec[uids[i]];
    if (i < nfp) {
        fp_out[3 * i] = r.px; fp_out[3 * i + 1] = r.pz; fp_out[3 * i + 2] = r.radius;
        return;
    }
    tile_desc t;
    chunk_out[i - nfp] = desc_for_point(m, r.px, r.pz, t) ? t.chunk_r * m.chunk_w + t.chunk_c : -1;
}

// one thread per named entry: the x, z of uid[i]'s record into buf at entry[i] * stride + off, where off is off0 for the
// first n0 entries and off1 for the rest
__global__ void __launch_bounds__(256) k_resident_xz(const pf_record *__restrict__ rec, const uint32_t *__restrict__ entry,
                                                     const uint32_t *__restrict__ uid, int n, int n0, int stride, int off0,
                                                     int off1, float *__restrict__ buf)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const pf_record &r = rec[uid[i]];
    float *p = buf + entry[i] * stride + (i < n0 ? off0 : off1);
    p[0] = r.px; p[1] = r.pz;
}

}   // namespace

int pf_resident_fresh(pfnav_ctx *ctx, const char *what)
{
    if (!ctx->index_stale) return PFNAV_OK;
    pfnav_set_error("%s by uid: records were written after the last index build (pfnav_agents_rebuild_index or a gather "
                    "first)", what);
    return PFNAV_ERR_STATE;
}

int pf_resident_points_begin(pfnav_ctx *ctx, const char *what, size_t n, const uint32_t *uids_a, bool given_a,
                             const uint32_t *uids_b, bool given_b, pf_resident_points &P)
{
    const char *err = nullptr;
    if (pf_resident_points_check(n, uids_a, given_a, uids_b, given_b, ctx->n_agents, P, &err)) PF_ARG(false, err);
    return n ? pf_resident_fresh(ctx, what) : PFNAV_OK;
}

int pf_resident_xz_launch(pfnav_ctx *ctx, cudaStream_t st, const uint8_t *d_pairs, const pf_resident_points &P, int stride,
                          int off0, int off1, float *buf)
{
    const size_t np = P.entry.size();
    if (!np) return PFNAV_OK;
    const uint32_t *d_entry = (const uint32_t *)d_pairs;
    k_resident_xz<<<(unsigned)((np + 255) / 256), 256, 0, st>>>(ctx->d_records, d_entry, d_entry + np, (int)np, (int)P.n0,
                                                                stride, off0, off1, buf);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}

int pf_resident_resolve(pfnav_ctx *ctx, cudaStream_t st, const pfnav_entity_field_req *reqs, size_t m,
                        const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents, const uint32_t *seeker_uids,
                        size_t nseekers, pf_resident_batch &B)
{
    PF_ARG(ctx->d_cost && ctx->pool.d_slot, "map / pool not created");
    pf_resident_names N;
    const char *err = nullptr;
    if (pf_resident_check(reqs, m, ents, ent_uids, nents, seeker_uids, nseekers, ctx->n_agents, N, &err)) PF_ARG(false, err);
    if (m == 0) return PFNAV_OK;
    if (int rc = pf_resident_fresh(ctx, "entity fields")) return rc;
    const size_t n = N.uids.size(), nfp = N.fp_index.size();
    std::vector<float> fp_xzr(3 * nfp);
    std::vector<int32_t> seek_chunk(nseekers);
    if (n) {
        // the uids in, the resolved values out, through the request staging; the one host wait
        const auto up16 = [](size_t b) { return (b + 15) & ~(size_t)15; };
        const size_t o_fp = up16(n * 4), o_ch = o_fp + up16(nfp * 12), need = o_ch + nseekers * 4;
        PF_CUDA(cudaSetDevice(ctx->device));
        pf_stage S;
        if (int rc = pf_stage_begin(ctx, st, std::max(n * 4, need - o_fp), need, false, &S)) return rc;
        memcpy(S.host, N.uids.data(), n * 4);
        if (int rc = pf_stage_upload(ctx, st, S, n * 4)) return rc;
        MapView mv = {};
        mv.W64 = ctx->W64; mv.H64 = ctx->H64; mv.chunk_w = ctx->chunk_w; mv.chunk_h = ctx->chunk_h;
        mv.map_x = ctx->map_x; mv.map_z = ctx->map_z;
        k_resident_footprints<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ctx->d_records, (const uint32_t *)S.dev, (int)nfp,
                                                                          (int)n, mv, (float *)(S.dev + o_fp),
                                                                          (int32_t *)(S.dev + o_ch));
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
        PF_CUDA(cudaMemcpyAsync(S.host, S.dev + o_fp, need - o_fp, cudaMemcpyDeviceToHost, st));
        if (int rc = pf_stage_done(ctx, st)) return rc;
        PF_CUDA(cudaStreamSynchronize(st));
        memcpy(fp_xzr.data(), S.host, nfp * 12);
        memcpy(seek_chunk.data(), S.host + (o_ch - o_fp), nseekers * 4);
    }
    if (pf_resident_merge(reqs, m, ents, nents, N, fp_xzr.data(), seek_chunk.data(), nseekers, ctx->chunk_w, ctx->chunk_h, B, &err))
        PF_ARG(false, err);
    return PFNAV_OK;
}

extern "C" int pfnav_pool_request_entity_fields_resident(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m,
                                                         const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents,
                                                         const uint32_t *seeker_uids, size_t nseekers, void *stream,
                                                         int *out_ndone)
{
    if (out_ndone) *out_ndone = 0;
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    pf_resident_batch B;
    if (int rc = pf_resident_resolve(ctx, pf_stream(ctx, stream), reqs, m, ents, ent_uids, nents, seeker_uids, nseekers, B))
        return rc;
    if (m == 0) return PFNAV_OK;
    return pfnav_pool_request_entity_fields_batch(ctx, B.reqs.data(), m, B.ents.data(), nents, B.chunks_rc.data(),
                                                  B.chunks_rc.size() / 2, stream, out_ndone);
}

// ------------------------------------------------------------------------------------------
// Zone and entity-field batches of a multi-GPU job (pfnav_mgpu_request_zones / pfnav_group_request_zones,
// pfnav_mgpu_request_entity_fields_batch / pfnav_group_request_entity_fields_batch; the exchanges are in pfnav_mgpu.cu,
// the owners and the staging layout in pfnav_plan.cu). A field of either batch depends on its request and the replicated
// map only -- no LOS chains, no parents, no pool field read -- and neither batch skips a field the pool holds, so every
// member writes the same keys with the same bytes, and the last request that names a key decides them. Each member
// reserves exactly as its solo call does (zone_reserve / entity_reserve), so its slots, evictions, `has` bits, remembered
// footprints and counts are the solo call's; the owner of a key builds it into staging with the solo call's build
// (zone_build / entity_build, blocks as slots), and every member copies every key it holds at the end into its slot.
// ------------------------------------------------------------------------------------------
struct aux_job_batch { std::vector<int32_t> ctile; std::vector<uint8_t> on_map; entity_batch E; int dim = 0; };

int pf_aux_job_plan(pfnav_ctx *ctx, pf_job &J)
{
    J.fits = true; J.nf = J.nl = 0;
    J.lack.clear();
    auto S = std::make_shared<aux_job_batch>();
    const bool zones = J.kind == PF_JOB_ZONES;
    int rc = zones ? zone_validate(ctx, J.zreqs, J.m, S->ctile, S->on_map, &S->dim)
                   : entity_validate(ctx, J.ereqs, J.m, J.ents, J.nents, J.chunks_rc, J.nchunks, S->E);
    if (rc) return rc;
    if ((rc = pf_job_check_state(ctx))) return rc;
    J.aux = S;
    const int cw = ctx->chunk_w, nch = cw * ctx->chunk_h;
    std::vector<size_t> keys;
    if (zones) {        // every key the batch names, by the zone rule's verdict
        for (size_t i = 0; i < J.m; i++) {
            if (!S->on_map[i]) continue;
            int ch[4];
            zone_chunks(ctx, J.zreqs[i], &S->ctile[2 * i], ch);
            for (int cr = ch[0]; cr <= ch[1]; cr++)
                for (int cc = ch[2]; cc <= ch[3]; cc++) keys.push_back((size_t)J.zreqs[i].dest * nch + cr * cw + cc);
        }
        J.fits = pf_pool_zone_fits(ctx->pool, keys.data(), keys.size());
        return PFNAV_OK;
    }
    // entity fields: the serial reservations all succeed exactly when each request's does on the pool as it is now
    for (size_t i = 0; i < J.m && J.fits; i++) {
        const pfnav_entity_field_req &q = J.ereqs[i];
        keys.clear();
        for (uint32_t k = 0; k < q.chunk_n; k++) {
            const int32_t *c = J.chunks_rc + 2 * ((size_t)q.chunk_off + k);
            keys.push_back((size_t)q.dest * nch + c[0] * cw + c[1]);
        }
        J.fits = pf_pool_fits(ctx->pool, keys.data(), keys.size());
    }
    return PFNAV_OK;
}

int pf_aux_job_launch(pfnav_ctx *ctx, pf_job &J, int world, int rank, cudaStream_t st)
{
    const aux_job_batch &S = *(const aux_job_batch *)J.aux.get();
    const bool zones = J.kind == PF_JOB_ZONES;
    const int cw = ctx->chunk_w, nch = cw * ctx->chunk_h;
    ctx->job_built[0] = ctx->job_built[1] = 0;
    J.nitems = 0; J.d_items = nullptr;
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(pf_fields_join(ctx, st));
    PF_CUDA(pf_pool_refresh(ctx, st));
    // ---- this member's own slots, exactly as its solo call reserves them (the verdict said they fit)
    std::vector<aux_field> fields;
    std::vector<int32_t> fresh;
    size_t done = 0;
    J.nfields.assign(J.m, 0);
    int rc = zones ? zone_reserve(ctx, J.zreqs, J.m, S.ctile, S.on_map, fields, fresh, J.nfields.data(), &done)
                   : entity_reserve(ctx, J.ereqs, J.m, J.ents, J.chunks_rc, fields, &done);
    if (rc) return rc;
    // ---- owners and staging blocks: `fields` lists what the serial calls write, the same on every member
    const size_t n = fields.size();
    std::vector<int32_t> freq(n), blk;
    std::vector<size_t> fkey(n);
    std::vector<int64_t> fcost(n, 1);
    for (size_t f = 0; f < n; f++) {
        const aux_field &F = fields[f];
        freq[f] = (int32_t)F.req;
        fkey[f] = (size_t)(zones ? J.zreqs[F.req].dest : J.ereqs[F.req].dest) * nch + F.cr * cw + F.cc;
        zone_job j;
        if (zones) fcost[f] = (int64_t)zone_flood(J.zreqs[F.req], &S.ctile[2 * F.req], S.dim, F.cr, F.cc, &j);
    }
    pf_job_layout(ctx, J, freq, fkey, fcost, world, blk);
    if (!J.seg[world]) return PFNAV_OK;
    // ---- the member's copies (every written key it still holds) and the owner's builds (blocks in place of slots)
    std::vector<pf_field_copy> items;
    std::vector<aux_field> own;
    for (size_t f = 0; f < n; f++) {
        if (blk[f] < 0) continue;
        const int32_t s = ctx->pool.slot_of(fkey[f]);
        if (s >= 0) items.push_back({blk[f], s, 0});
        if (ctx->job_owner[freq[f]] == rank) own.push_back({fields[f].req, fields[f].cr, fields[f].cc, blk[f]});
    }
    if ((rc = pf_job_stage(ctx, J, items, world, st))) return rc;
    if (!own.empty()) {
        rc = zones ? zone_build(ctx, st, J.zreqs, S.ctile, S.dim, own, std::vector<int32_t>(), false, ctx->d_job_stage)
                   : entity_build(ctx, st, J.ereqs, J.ents, J.nents, S.E, own, false, ctx->d_job_stage);
        if (rc) return rc;
    }
    ctx->job_built[0] = (int)own.size();
    return PFNAV_OK;
}

extern "C" int pfnav_pool_request_entity_fields(pfnav_ctx *ctx, int dest, int layer, int ref_layer, int target_kind,
                                                const pfnav_footprint *ents, size_t nents, const int32_t *chunks_rc, size_t n,
                                                void *stream)
{
    PF_ARG(ctx && ctx->pool.d_slot, "pool not created");
    PF_ARG(nents < (1u << 24) && n < (1u << 24), "nents / n");
    const pfnav_entity_field_req q = {dest, layer, ref_layer, target_kind, 0, (uint32_t)nents, 0, (uint32_t)n};
    int rc = pfnav_pool_request_entity_fields_batch(ctx, &q, 1, ents, nents, chunks_rc, n, stream, nullptr);
    if (rc) return rc;
    PF_CUDA(cudaStreamSynchronize(pf_stream(ctx, stream)));      // returns once the fields are in the pool
    return PFNAV_OK;
}

// the chunk-local frontier of a TARGET_ENEMIES / TARGET_ENTITY pool destination (field_enemies_initial_frontier /
// field_entity_initial_frontier with the chunk itself as the region, field.c:2334-2360): tile indices r * 64 + c
int pfnav_aux_chunk_seeds(pfnav_ctx *ctx, int dest, int chunk_r, int chunk_c, std::vector<int> &out)
{
    PF_ARG(dest >= 0 && (size_t)dest < ctx->aux.size() && ctx->aux[dest].kind >= 0, "no entity fields were requested for this destination");
    const pfnav_ctx::aux_target &A = ctx->aux[dest];
    std::vector<int32_t> seeds;
    int rc = entity_seeds(ctx, A.ref_layer, A.kind, A.ents.data(), A.ents.size(), 64, chunk_r, chunk_c, seeds);
    if (rc) return rc;
    for (size_t i = 0; i + 1 < seeds.size(); i += 2) out.push_back((seeds[i] - chunk_r * 64) * 64 + (seeds[i + 1] - chunk_c * 64));
    return PFNAV_OK;
}
