// pfnav_ents_query_kernel.cuh -- the position index walk of G_Pos_EntsInCircleFrom (bg_ent_inrange_circle + filter_garrisoned)
// and the kernels of pfnav_ents_in_circles, kept in a header of its own so that tests/emu can run the SAME source on CPU
// threads (tests/emu/ents_query_emu.cpp defines the CUDA keywords and warp collectives as plain C++). pfnav_agents.cu
// includes it: the index build (k_cell_*), the neighbour kernels (k_agent_velocity, k_cohesion*, k_entity_update) and the
// batched queries share this one walk.
// Needs: <stdint.h>, min / max / abs, __float2int_rn, __ballot_sync / __popc / __shfl_sync / __syncwarp, include/pfnav.h,
// pf_record (pfnav_internal.cuh).
#pragma once

#ifndef FULL
#define FULL 0xffffffffu
#endif
// which way a walk went (tests/emu records it; no code on the device): 0 centre off the grid, 1 wide, 2 small, 3 large
#ifndef PF_WALK_TRACE
#define PF_WALK_TRACE(kind, lane)
#endif

struct GridView {
    const uint32_t *cell_start, *cell_count;
    const int32_t *ix, *iy; const uint32_t *id;
    int grid_w, grid_h; int32_t origin_x, origin_y;
};

// scaled integer coordinates + cell of the position index (bitmap_grid.h: 16-wu cells)
__device__ __forceinline__ int32_t bg_scale(float x) { return __float2int_rn(x * 256.0f); }   // BG_SCALE_F
__device__ __forceinline__ int cell_of(int32_t i, int32_t origin, int n)
{
    int c = (i - origin) >> 12;
    return min(max(c, 0), n - 1);
}

// bg_ent_inrange_circle (bitmap_grid.h:1376): visit hits in the reference's order and hand them,
// 32 candidates at a time, to `emit(hit, id)` (called convergently by all lanes; returns a
// warp-uniform "stop").
template <class F>
__device__ __forceinline__ void grid_query(const GridView &g, float x, float z, float range, uint32_t lane,
                                           F &&emit)
{
    const int32_t icx = bg_scale(x), icy = bg_scale(z), ir = bg_scale(range);
    const long long ir2 = (long long)ir * ir;
    const int32_t imnx = icx - ir, imxx = icx + ir, imny = icy - ir, imxy = icy + ir;
    // _bg_cell_extent (bitmap_grid.h:1236)
    if (imxx < g.origin_x || imxy < g.origin_y || imnx >= g.origin_x + (g.grid_w << 12) || imny >= g.origin_y + (g.grid_h << 12)) {
        PF_WALK_TRACE(0, lane);
        return;
    }
    const int cx_lo = max((imnx - g.origin_x) >> 12, 0), cx_hi = min((imxx - g.origin_x) >> 12, g.grid_w - 1);
    const int cy_lo = max((imny - g.origin_y) >> 12, 0), cy_hi = min((imxy - g.origin_y) >> 12, g.grid_h - 1);
    // wide-query fast path: whole pool in pool order == cells in row-major order
    const bool wide = (long long)(cx_hi - cx_lo + 1) * (cy_hi - cy_lo + 1) * 4 >= (long long)g.grid_w * g.grid_h * 3;
    const int ax_lo = wide ? 0 : cx_lo, ax_hi = wide ? g.grid_w - 1 : cx_hi;
    const int ay_lo = wide ? 0 : cy_lo, ay_hi = wide ? g.grid_h - 1 : cy_hi;
    const int cstep = wide ? (1 << 30) : 8;                    // one "coarse block" spans everything when wide
    const bool small = !wide && ir >= 0 && ir <= 12000;         // <= 46 wu
    PF_WALK_TRACE(wide ? 1 : small ? 2 : 3, lane);
    const int cyc_lo = wide ? 0 : ay_lo >> 3, cyc_hi = wide ? 0 : ay_hi >> 3;
    const int cxc_lo = wide ? 0 : ax_lo >> 3, cxc_hi = wide ? 0 : ax_hi >> 3;
    for (int cyc = cyc_lo; cyc <= cyc_hi; cyc++) {
        for (int cxc = cxc_lo; cxc <= cxc_hi; cxc++) {
            const int fy0 = wide ? ay_lo : max(cyc * cstep, ay_lo), fy1 = wide ? ay_hi + 1 : min(cyc * cstep + cstep, ay_hi + 1);
            const int fx0 = wide ? ax_lo : max(cxc * cstep, ax_lo), fx1 = wide ? ax_hi + 1 : min(cxc * cstep + cstep, ax_hi + 1);
            for (int fy = fy0; fy < fy1; fy++) {
                // the cells fx0..fx1-1 of one fine row are adjacent in the cell-major index: one contiguous run of entries,
                // visited in ascending cell x, in-cell order -- the reference's order
                const uint32_t b = g.cell_start[fy * g.grid_w + fx0], e = g.cell_start[fy * g.grid_w + fx1];
                for (uint32_t k0 = b; k0 < e; k0 += 32) {
                    const uint32_t k = k0 + lane;
                    bool hit = false;
                    uint32_t id = 0;
                    if (k < e) {
                        if (small) {        // |d| <= range + one cell on either side: the squares fit 32 bits
                            const int32_t dx = g.ix[k] - icx, dy = g.iy[k] - icy;
                            hit = abs(dx) <= ir && abs(dy) <= ir && dx * dx + dy * dy <= (int32_t)ir2;
                        } else {
                            const long long dx = (long long)g.ix[k] - icx, dy = (long long)g.iy[k] - icy;
                            hit = dx * dx + dy * dy <= ir2;
                        }
                        id = g.id[k];
                    }
                    if (emit(hit, id)) return;
                }
            }
        }
    }
}

// filter_garrisoned (position.c:100-119): swap-remove from the back, applied by G_Pos_EntsInCircleFrom
// (position.c:379) AFTER the raw query was cut at maxout; it reorders the survivors. Serial on lane 0
// (only runs when the population holds garrisoned entities at all); returns the new count to all lanes.
__device__ __forceinline__ int filter_garrisoned(uint32_t *ids, int count, const pf_record *__restrict__ rec, uint32_t lane)
{
    int ret = count;
    if (lane == 0) {
        for (int i = count - 1; i >= 0; i--) {
            if (rec[ids[i]].state_flags & PFNAV_FLAG_GARRISONED) { ids[i] = ids[ret - 1]; ret--; }
        }
    }
    ret = __shfl_sync(FULL, ret, 0);
    __syncwarp();
    return ret;
}

// ------------------------------------------------------------------------------------------
// pfnav_ents_in_circles: one warp per query, a count pass and a write pass over the same walk
// ------------------------------------------------------------------------------------------
// A query with maxout == 0 or range < 0 has no hits. (NaN passes the test, as it did in pfnav_ents_in_circle; the batch
// call rejects it before anything runs.)
__device__ __forceinline__ bool eq_active(const pfnav_ents_query &a) { return a.maxout > 0 && !(a.range < 0.0f); }

// the centre: the point, or the resident position of entity `uid` -- the record the index was built from
__device__ __forceinline__ void eq_centre(const pfnav_ents_query &a, const pf_record *__restrict__ rec, float &x, float &z)
{
    if (a.uid != PFNAV_NULL_UID) { x = rec[a.uid].px; z = rec[a.uid].pz; }
    else { x = a.x; z = a.z; }
}

// Count pass of one query on the calling warp: the raw hits cut at maxout (*raw) and how many of them filter_garrisoned
// keeps (*surv; filter_garr == 0: all of them). Materialises nothing.
__device__ __forceinline__ void eq_count(const GridView &g, const pf_record *__restrict__ rec, const pfnav_ents_query &a,
                                         int filter_garr, uint32_t lane, uint32_t *raw, uint32_t *surv)
{
    int n = 0, garr = 0;
    if (eq_active(a)) {
        const int maxout = a.maxout;
        float x, z;
        eq_centre(a, rec, x, z);
        grid_query(g, x, z, a.range, lane, [&](bool hit, uint32_t id) -> bool {
            const uint32_t m = __ballot_sync(FULL, hit);
            if (filter_garr) {
                const int rank = __popc(m & ((1u << lane) - 1));
                const bool gh = hit && n + rank < maxout && (rec[id].state_flags & PFNAV_FLAG_GARRISONED);
                garr += __popc(__ballot_sync(FULL, gh));
            }
            n += __popc(m);
            return n >= maxout;
        });
        n = min(n, maxout);
    }
    *raw = (uint32_t)n;
    *surv = (uint32_t)(n - garr);
}

// Write pass of one query on the calling warp: its answer at out. Without a garrisoned entity inside the cut the hits go
// straight to out in ballot-rank order; with one (scratch != nullptr, room for the raw cut) the raw cut is built there,
// filter_garrisoned reorders it in place, and the survivors are copied to out.
__device__ __forceinline__ void eq_write(const GridView &g, const pf_record *__restrict__ rec, const pfnav_ents_query &a,
                                         uint32_t lane, uint32_t *out, uint32_t *scratch)
{
    uint32_t *dst = scratch ? scratch : out;
    int n = 0;
    if (eq_active(a)) {
        const int maxout = a.maxout;
        float x, z;
        eq_centre(a, rec, x, z);
        grid_query(g, x, z, a.range, lane, [&](bool hit, uint32_t id) -> bool {
            const uint32_t m = __ballot_sync(FULL, hit);
            const int rank = __popc(m & ((1u << lane) - 1));
            if (hit && n + rank < maxout) dst[n + rank] = id;
            n += __popc(m);
            return n >= maxout;
        });
        n = min(n, maxout);
    }
    if (scratch) {
        __syncwarp();
        const int cnt = filter_garrisoned(scratch, n, rec, lane);
        for (int k = (int)lane; k < cnt; k += 32) out[k] = scratch[k];
    }
}

#define EQ_WARPS 8                                  // queries per CTA

// surv[i]: query i's answer length; with filter_garr also scr[i]: the raw cut when a garrisoned entity lies inside it
// (the write pass builds it in scratch), else 0
__global__ void __launch_bounds__(EQ_WARPS * 32) k_ents_count(GridView g, const pf_record *__restrict__ rec,
                                                              const pfnav_ents_query *__restrict__ q, int n, int filter_garr,
                                                              uint32_t *__restrict__ surv, uint32_t *__restrict__ scr)
{
    const uint32_t lane = threadIdx.x & 31;
    for (int i = blockIdx.x * EQ_WARPS + (threadIdx.x >> 5); i < n; i += gridDim.x * EQ_WARPS) {
        uint32_t raw, s;
        eq_count(g, rec, q[i], filter_garr, lane, &raw, &s);
        if (lane == 0) {
            surv[i] = s;
            if (filter_garr) scr[i] = raw != s ? raw : 0u;
        }
    }
}

// query i's answer at out[off[i] ..); scr_off (filter_garr only): its scratch at scratch[scr_off[i] .. scr_off[i + 1])
__global__ void __launch_bounds__(EQ_WARPS * 32) k_ents_write(GridView g, const pf_record *__restrict__ rec,
                                                              const pfnav_ents_query *__restrict__ q, int n,
                                                              const uint32_t *__restrict__ off, const uint32_t *__restrict__ scr_off,
                                                              uint32_t *__restrict__ out, uint32_t *__restrict__ scratch)
{
    const uint32_t lane = threadIdx.x & 31;
    for (int i = blockIdx.x * EQ_WARPS + (threadIdx.x >> 5); i < n; i += gridDim.x * EQ_WARPS) {
        uint32_t *s = scr_off && scr_off[i + 1] != scr_off[i] ? scratch + scr_off[i] : nullptr;
        eq_write(g, rec, q[i], lane, out + off[i], s);
    }
}
