// pfnav_agents.cu -- device field pool, device spatial index, and the per-agent velocity update.
//
// Replaces (reference file:line):
//   compute_los_state / compute_desired_velocity         src/game/movement.c:4129-4180
//     N_DesiredPointSeekVelocity, n_interpolated_flow_dir  src/navigation/nav.c:3468, 3407
//     N_HasDestLOS                                          src/navigation/nav.c:4026
//     M_Tile_DescForPoint2D / M_Tile_Bounds / RelativeDesc  src/map/tile.c:547, 356, 391
//   move_velocity_work                                    src/game/movement.c:3395-3466
//     point_seek_vpref :1870, point_seek_total_force :1745, arrive_force_point :1546,
//     cohesion_force :1653, separation_force :1690, nullify_impass_components :1831,
//     vec2_truncate :643, find_neighbours :2768
//   G_ClearPath_NewVelocity                               src/game/clearpath.c:694 (all of :123-418, 552-715)
//     C_InfiniteLineIntersection / C_RayRayIntersection2D   src/phys/collision.c:820, 854
//   G_Pos_EntsInCircleFrom -> bg_ent_inrange_circle       src/game/position.c:379, src/lib/public/bitmap_grid.h:1376
//
// Arithmetic mirrors the reference expression by expression (float storage, the same places
// promoted to double, IEEE sqrt/div, no FMA contraction: the TU is built with -fmad=false), so
// that every epsilon-threshold branch of ClearPath takes the same side as on the CPU.
//
// Kernels:
//   K5  k_cell_count / k_cell_scan / k_cell_scatter / k_cell_sort : counting sort of agents into
//       16-wu cells, in-cell order = descending uid (what insert-all + bg_cleanup leaves behind).
//   K6a k_desired_velocity : one thread per work item, bilinear flow blend + LOS bit from the pool.
//   K6b k_cohesion         : one thread per work item, O(|flock|) weighted centre of mass.
//   K6c k_agent_velocity   : ONE WARP PER AGENT. Lanes scan the hash cells, evaluate separation
//       terms, and split ClearPath's O(R^2) ray pairs / O(R) inside-PCR tests among themselves.
#include "pfnav_internal.cuh"
#include <algorithm>
#include <math.h>
#include <memory>
#include <string.h>
#include "pfnav_map_view.cuh"
#include "pfnav_scan.cuh"

#include "pfnav_clearpath_kernel.cuh"   // v2 helpers, ClearPath: build_vos ... clearpath_retry, clearpath_collect / _finish
#include "pfnav_ents_query_kernel.cuh"  // GridView, the index walk grid_query / filter_garrisoned, pfnav_ents_in_circles

// ------------------------------------------------------------------------------------------
// Map / pool views
// ------------------------------------------------------------------------------------------
struct PoolView {
    const int32_t *slot;     // [ndests][chunks]
    const uint8_t *flow;     // [max][4096]
    const uint8_t *los;      // [max][4096] ; first byte of a never-written LOS slot region is valid 0s
    const uint8_t *has;      // [max] bit0 flow present, bit1 LOS present
    int ndests;
    uint32_t *touch;         // [max] last tick that read the slot (LRU stamp), may be NULL
    uint32_t tick_no;
};
// touch == nullptr: the kernel stamps no slot
static PoolView pool_view(const pf_pool &P, uint32_t *touch, uint32_t tick_no) { return {P.d_slot, P.d_flow, P.d_los, P.d_has, P.ndests, touch, tick_no}; }

// Entity_NavLayerWithRadius (entity.c:554)
__device__ __forceinline__ int nav_layer_for(uint32_t flags, float radius)
{
    const bool water = flags & PFNAV_FLAG_WATER, air = flags & PFNAV_FLAG_AIR;
    const int base = water ? 4 : air ? 8 : 0;
    if (radius >= 15.0f) return base + 3;
    if (radius >= 10.0f) return base + 2;
    if (radius >= 5.0f) return base + 1;
    return base;
}

// N_FlowDir (field.c:2429): 1.0f / sqrt(2.0f) is a double division rounded to float
__device__ __forceinline__ v2 flow_dir_vec(int dir)
{
    const float d = (float)(1.0 / 1.4142135623730951);
    switch (dir) {
    case 1: return {d, -d};
    case 2: return {0.0f, -1.0f};
    case 3: return {-d, -d};
    case 4: return {1.0f, 0.0f};
    case 5: return {-1.0f, 0.0f};
    case 6: return {d, d};
    case 7: return {0.0f, 1.0f};
    case 8: return {-d, d};
    default: return {0.0f, 0.0f};
    }
}

// ------------------------------------------------------------------------------------------
// K6a: desired velocity + LOS from the device field pool
// ------------------------------------------------------------------------------------------
// ent_desired_velocity (movement.c:1466) decides per movement state where the desired velocity comes from:
//   TURNING                      zero
//   SEEK_ENEMIES                 N_DesiredEnemySeekVelocity (nav.c:3603): direction of the own tile in the TARGET_ENEMIES
//                                field of its chunk -- pool destination aux_dest1 - 1 -- NOT interpolated
//   SURROUND_ENTITY              N_DesiredSurroundVelocity (nav.c:3687) out of the TARGET_ENTITY field the same way while
//                                ms->using_surround_field (and the target exists); the point-seek field otherwise
//   ARRIVING_TO_CELL             the caller's cell_arrival_vdes (formation.c owns the cell fields)
//   everything else              N_DesiredPointSeekVelocity (nav.c:3468)
// and compute_los_state (movement.c:4129): N_HasDestLOS at prev_pos for entities in a flock, except surround-field users.
__global__ void k_desired_velocity(MapView m, PoolView pool, const pfnav_agent *__restrict__ agents,
                                   const pfnav_flock *__restrict__ flocks, const uint32_t *__restrict__ work,
                                   int nwork, float2 *__restrict__ vdes_out, uint8_t *__restrict__ los_out,
                                   uint32_t *__restrict__ miss_count, const pfnav_movestate_ext *__restrict__ ext,
                                   const pfnav_formation_in *__restrict__ form)
{
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwork) return;
    const uint32_t uid = work[w];
    const pfnav_agent a = agents[uid];
    v2 vdes = {0.0f, 0.0f};
    uint8_t los = 0;
    int dest = (a.flock >= 0) ? flocks[a.flock].dest : -1;
    bool field_dir_only = false, want_los = a.flock >= 0, want_vdes = true;
    if (a.state == PFNAV_STATE_TURNING) want_vdes = false;
    else if (a.state == PFNAV_STATE_ARRIVING_TO_CELL) {
        want_vdes = false;
        if (form) vdes = {form[uid].cell_arrival_vdes[0], form[uid].cell_arrival_vdes[1]};
    } else if (a.state == PFNAV_STATE_SEEK_ENEMIES) {
        dest = (int)a.aux_dest1 - 1; field_dir_only = true; want_los = false;
    } else if (a.state == PFNAV_STATE_SURROUND_ENTITY && ext && ext[uid].surround_target_uid != 0xffffffffu &&
               ext[uid].using_surround_field) {
        dest = (int)a.aux_dest1 - 1; field_dir_only = true; want_los = false;
    }
    if (field_dir_only) {
        tile_desc t;
        if (dest >= 0 && dest < pool.ndests && desc_for_point(m, a.pos[0], a.pos[1], t)) {
            const int s = pool.slot[(size_t)dest * m.chunk_w * m.chunk_h + t.chunk_r * m.chunk_w + t.chunk_c];
            if (s < 0 || !(pool.has[s] & 1)) atomicAdd(miss_count, 1u);
            else {
                vdes = flow_dir_vec(pool.flow[(size_t)s * 4096 + t.tile_r * 64 + t.tile_c] & 0xF);
                if (pool.touch && pool.touch[s] != pool.tick_no) pool.touch[s] = pool.tick_no;
            }
        }
        vdes_out[w] = make_float2(vdes.x, vdes.z);
        los_out[w] = 0;
        return;
    }
    const int pdest = (a.flock >= 0) ? flocks[a.flock].dest : -1;
    if (want_los && pdest >= 0 && pdest < pool.ndests) {
        tile_desc t;
        if (desc_for_point(m, a.prev_pos[0], a.prev_pos[1], t)) {
            const int s = pool.slot[(size_t)pdest * m.chunk_w * m.chunk_h + t.chunk_r * m.chunk_w + t.chunk_c];
            if (s >= 0 && (pool.has[s] & 2)) {
                los = pool.los[(size_t)s * 4096 + t.tile_r * 64 + t.tile_c] & 1;
                if (pool.touch && pool.touch[s] != pool.tick_no) pool.touch[s] = pool.tick_no;
            }
        }
    }
    if (!want_vdes) {
        vdes_out[w] = make_float2(vdes.x, vdes.z);
        los_out[w] = los;
        return;
    }
    if (dest >= 0 && dest < pool.ndests) {
        const int chunks = m.chunk_w * m.chunk_h;
        const int32_t *slots = pool.slot + (size_t)dest * chunks;
        tile_desc t;
        // (N_HasDestLOS, sampled at prev_pos, was evaluated above: movement.c:4137)
        // ---- N_DesiredPointSeekVelocity at pos ----
        if (desc_for_point(m, a.pos[0], a.pos[1], t)) {
            const int s = slots[t.chunk_r * m.chunk_w + t.chunk_c];
            if (s < 0 || !(pool.has[s] & 1)) {
                atomicAdd(miss_count, 1u);      // the host planner must request this (dest, chunk)
            } else {
                const uint8_t *base_ff = pool.flow + (size_t)s * 4096;
                const int base_dir = base_ff[t.tile_r * 64 + t.tile_c] & 0xF;
                if (pool.touch && pool.touch[s] != pool.tick_no) pool.touch[s] = pool.tick_no;
                // n_interpolated_flow_dir (nav.c:3407)
                const float bx = (m.map_x - (float)(t.chunk_c * 256)) - (float)(t.tile_c * 4);
                const float bz = (m.map_z + (float)(t.chunk_r * 256)) + (float)(t.tile_r * 4);
                const float cx = bx - 4.0f / 2.0f, cz = bz + 4.0f / 2.0f;
                const float dx = a.pos[0] - cx, dz = a.pos[1] - cz;
                const int dc = (dx < 0.0f) ? 1 : -1;
                const int dr = (dz > 0.0f) ? 1 : -1;
                const float wc = (float)fmin(fabs((double)dx) / 4.0, 1.0);
                const float wr = (float)fmin(fabs((double)dz) / 4.0, 1.0);
                const int sdc[4] = {0, dc, 0, dc}, sdr[4] = {0, 0, dr, dr};
                const float sw[4] = {(1.0f - wc) * (1.0f - wr), wc * (1.0f - wr), (1.0f - wc) * wr, wc * wr};
                v2 acc = {0.0f, 0.0f};
                float wsum = 0.0f;
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    if (sw[i] <= 0.0f) continue;
                    const int abs_r = t.chunk_r * 64 + t.tile_r + sdr[i], abs_c = t.chunk_c * 64 + t.tile_c + sdc[i];
                    if (abs_r < 0 || abs_r >= m.H64 || abs_c < 0 || abs_c >= m.W64) continue;
                    const int cr2 = abs_r >> 6, cc2 = abs_c >> 6;
                    const uint8_t *ff = base_ff;
                    if (cr2 != t.chunk_r || cc2 != t.chunk_c) {
                        const int s2 = slots[cr2 * m.chunk_w + cc2];
                        if (s2 < 0 || !(pool.has[s2] & 1)) continue;
                        ff = pool.flow + (size_t)s2 * 4096;
                    }
                    const int dir = ff[(abs_r & 63) * 64 + (abs_c & 63)] & 0xF;
                    if (dir == 0) continue;
                    const v2 fd = flow_dir_vec(dir);
                    acc = v2_add(acc, v2_scale(fd, sw[i]));
                    wsum += sw[i];
                }
                if (wsum < 1e-6f || v2_len(acc) < 1e-6f) vdes = flow_dir_vec(base_dir);
                else vdes = v2_normal(acc);
            }
        }
    }
    vdes_out[w] = make_float2(vdes.x, vdes.z);
    los_out[w] = los;
}

// ------------------------------------------------------------------------------------------
// K6b: cohesion_force (movement.c:1653). One thread per work item; members in ascending uid.
// ------------------------------------------------------------------------------------------
// member positions of every flock, contiguous in member-list order (one coalesced stream for k_cohesion)
__global__ void k_gather_flock_pos(const pf_record *__restrict__ rec, const uint32_t *__restrict__ flock_members, int n,
                                   float2 *__restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const pf_record r = rec[flock_members[i]];
    out[i] = make_float2(r.px, r.pz);
}

// cohesion weight exp(-6 (|d| - 37.5) / 50) = 2^(|d| * (-0.12 log2 e) + 4.5 log2 e) on the SFU (rsqrt + ex2, flush-to-zero
// forms: no denormal fix-up code; a flushed weight is < 1e-38 of a neighbour's)
__device__ __forceinline__ float coh_weight(float dx, float dz)
{
    const float len2 = fmaxf(fmaf(dx, dx, dz * dz), 1e-30f);
    float r, w;
    asm("rsqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(len2));
    const float len = len2 * r;
    asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(w) : "f"(fmaf(len, -0.12f * 1.4426950408889634f, 4.5f * 1.4426950408889634f)));
    return w;
}

// the whole member list of the flock (the definition; used for small flocks and as the fall-back of the windowed pass)
__global__ void k_cohesion(const pf_record *__restrict__ rec, const int32_t *__restrict__ flock_of,
                           const uint32_t *__restrict__ flock_start, const float2 *__restrict__ member_pos,
                           const uint32_t *__restrict__ uids, const uint32_t *__restrict__ nuids_dev, int nuids_host,
                           float scaled_max_force, float2 *__restrict__ out_by_uid)
{
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    const int nu = nuids_dev ? (int)*nuids_dev : nuids_host;
    if (w >= nu) return;
    const uint32_t uid = uids[w];
    const int fl = flock_of[uid];
    v2 ret = {0.0f, 0.0f};
    if (fl >= 0) {
        const pf_record self = rec[uid];
        const uint32_t b = flock_start[fl], e = flock_start[fl + 1];
        v2 com = {0.0f, 0.0f};
        // The reference's sum runs over the flock in khash bucket order (movement.c:1660), i.e. it is not
        // reproducible to the last bit anyway; what must hold is the 1e-4 velocity budget. The weight
        // exp(-6 (|d| - 37.5) / 50) is therefore evaluated with the SFU (rsqrt + ex2, relative error < 1e-6) and
        // the member itself is removed afterwards: its weight is exp(4.5) exactly as evaluated here for |d| = 0.
        const float self_scale = coh_weight(0.0f, 0.0f);
#pragma unroll 4
        for (uint32_t k = b; k < e; k++) {
            const float2 p = member_pos[k];
            const float scale = coh_weight(p.x - self.px, p.y - self.pz);
            com.x = fmaf(p.x, scale, com.x);
            com.z = fmaf(p.y, scale, com.z);
        }
        const uint32_t cnt = e - b - 1;
        if (cnt > 0) {
            com.x -= self.px * self_scale;
            com.z -= self.pz * self_scale;
            com = v2_scale(com, 1.0f / (float)cnt);
            ret = v2_sub(com, v2{self.px, self.pz});
            ret = v2_truncate(ret, scaled_max_force);
        }
    }
    out_by_uid[uid] = make_float2(ret.x, ret.z);
}

// cohesion_force (movement.c:1653) for big flocks. The weight of a member falls off as exp(-0.12 d): beyond COH_R = 230 wu
// a member weighs < 1.1e-12 of one standing next to the entity, so the sum over the members within COH_R equals the full
// sum to float precision WHENEVER the entity has company nearby. The pass walks the position index instead of the member
// list: 128 consecutive entries of the index (spatial neighbours: the index is cell-major) share one window of cell rows,
// the window's entries stream through shared memory in tiles, every thread accumulates its own entity's sum. An entity
// whose window holds too little weight to make the cut-off harmless (sum < N * exp(4.5 - 0.12 * 230) * 1e7, i.e. the
// dropped members could matter at the 1e-7 level) is handed to the full-list kernel instead, so the result never
// depends on the cut-off by more than float rounding. The index picks the cells; the weights and the sum use the
// members' float positions from their records, as the full-list kernel does.
#define COH_R 230.0f
#define COH_THREADS 128
__device__ __forceinline__ void coh_finish(float ax, float az, float wsum, float self_w, float sx, float sz,
                                           uint32_t N, float thresh_unit, float scaled_max_force, uint32_t uid,
                                           float2 *__restrict__ out_by_uid, uint32_t *__restrict__ fallback,
                                           uint32_t *__restrict__ nfallback)
{
    if (N <= 1) out_by_uid[uid] = make_float2(0.0f, 0.0f);
    else if (wsum - self_w >= (float)N * thresh_unit) {
        // the entity's own index entry was summed too: take it out again (weight exp(4.5) at distance 0)
        v2 com = {ax - sx * self_w, az - sz * self_w};
        com = v2_scale(com, 1.0f / (float)(N - 1));
        v2 ret = v2_sub(com, v2{sx, sz});
        ret = v2_truncate(ret, scaled_max_force);
        out_by_uid[uid] = make_float2(ret.x, ret.z);
    } else fallback[atomicAdd(nfallback, 1u)] = uid;
}
__global__ void __launch_bounds__(COH_THREADS)
k_cohesion_window(GridView g, const pf_record *__restrict__ rec, const int32_t *__restrict__ sfl,
                  const uint32_t *__restrict__ flock_start, int n, uint32_t lo, uint32_t hi, float scaled_max_force,
                  float2 *__restrict__ out_by_uid, uint32_t *__restrict__ fallback, uint32_t *__restrict__ nfallback,
                  float4 *__restrict__ part, int nsplit)
{
    __shared__ float4 tile[COH_THREADS];       // {x, z, flock id bits, -}
    __shared__ int bb[4];
    const int tid = threadIdx.x;
    const float thresh_unit = __expf(4.5f - 0.12f * COH_R) * 1e7f;
    for (int base = blockIdx.x * COH_THREADS; base < n; base += gridDim.x * COH_THREADS) {
        const int k = base + tid;
        uint32_t uid = 0; int fl = -1; bool active = false;
        float sx = 0.0f, sz = 0.0f, self_w = 0.0f;
        int mycx = 0, mycy = 0;
        if (k < n) {
            uid = g.id[k]; fl = sfl[k];
            active = uid >= lo && uid < hi && fl >= 0;
            mycx = cell_of(g.ix[k], g.origin_x, g.grid_w); mycy = cell_of(g.iy[k], g.origin_y, g.grid_h);
        }
        if (!__syncthreads_or(active)) continue;
        if (tid == 0) { bb[0] = 0x7fffffff; bb[1] = -1; bb[2] = 0x7fffffff; bb[3] = -1; }
        __syncthreads();
        if (active) {
            const pf_record self = rec[uid];
            sx = self.px; sz = self.pz;
            self_w = coh_weight(0.0f, 0.0f);                   // what the loop below adds for the entity's own entry
            atomicMin(&bb[0], mycx); atomicMax(&bb[1], mycx); atomicMin(&bb[2], mycy); atomicMax(&bb[3], mycy);
        }
        __syncthreads();
        const int cy0 = bb[2], cy1 = bb[3];
        float ax = 0.0f, az = 0.0f, wsum = 0.0f;
        const int RC = (int)(COH_R / 16.0f) + 1;
        // One window per grid row of the block's entities: 128 consecutive index entries lie in one row, or wrap from the
        // end of one into the start of the next (then one window around both would span the whole map width).
        for (int cyv = cy0; cyv <= cy1; cyv++) {
            const bool mine = active && mycy == cyv;
            __syncthreads();
            if (tid == 0) { bb[0] = 0x7fffffff; bb[1] = -1; }
            __syncthreads();
            if (mine) { atomicMin(&bb[0], mycx); atomicMax(&bb[1], mycx); }
            __syncthreads();
            const int cx0 = bb[0], cx1 = bb[1];
            if (cx1 < 0) continue;                                  // nobody in this row (uniform: read from shared memory)
            for (int ry = max(cyv - RC, 0) + (int)blockIdx.y; ry <= min(cyv + RC, g.grid_h - 1); ry += nsplit) {
                const int gap = max(abs(ry - cyv) - 1, 0);
                const float dy = (float)gap * 16.0f;
                if (dy > COH_R) continue;
                const int nx = (int)(sqrtf(COH_R * COH_R - dy * dy) / 16.0f) + 1;
                const int x0 = max(cx0 - nx, 0), x1 = min(cx1 + nx, g.grid_w - 1);
                const uint32_t s0 = g.cell_start[ry * g.grid_w + x0], s1 = g.cell_start[ry * g.grid_w + x1 + 1];
                for (uint32_t t0 = s0; t0 < s1; t0 += COH_THREADS) {
                    const uint32_t e = t0 + tid;
                    // the members' own positions, as cohesion_force sums them: the index's 1/256-wu integers would move
                    // the centre of mass by up to 1/512 wu per member
                    if (e < s1) {
                        const pf_record r = rec[g.id[e]];
                        tile[tid] = make_float4(r.px, r.pz, __int_as_float(sfl[e]), 0.0f);
                    }
                    __syncthreads();
                    const int nt = (int)min((uint32_t)COH_THREADS, s1 - t0);
                    if (mine) {
#pragma unroll 4
                        for (int j = 0; j < nt; j++) {
                            const float4 m = tile[j];
                            const float scale = __float_as_int(m.z) == fl ? coh_weight(m.x - sx, m.y - sz) : 0.0f;
                            ax = fmaf(m.x, scale, ax); az = fmaf(m.y, scale, az); wsum += scale;
                        }
                    }
                    __syncthreads();
                }
            }
        }
        if (nsplit > 1) {                    // a small population split over blockIdx.y: k_cohesion_finish adds the parts up
            if (k < n) part[(size_t)blockIdx.y * n + k] = make_float4(ax, az, wsum, 0.0f);
        } else if (active) {
            coh_finish(ax, az, wsum, self_w, sx, sz, flock_start[fl + 1] - flock_start[fl], thresh_unit,
                       scaled_max_force, uid, out_by_uid, fallback, nfallback);
        }
    }
}

// the window rows of one 128-entry run were split over `nsplit` blocks (populations too small to fill the chip with one
// block per run): add the partial sums in split order and finish as the fused path does
__global__ void k_cohesion_finish(GridView g, const pf_record *__restrict__ rec, const int32_t *__restrict__ sfl,
                                  const uint32_t *__restrict__ flock_start, int n, uint32_t lo, uint32_t hi, float scaled_max_force,
                                  float2 *__restrict__ out_by_uid, uint32_t *__restrict__ fallback, uint32_t *__restrict__ nfallback,
                                  const float4 *__restrict__ part, int nsplit)
{
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= n) return;
    const uint32_t uid = g.id[k];
    const int fl = sfl[k];
    if (!(uid >= lo && uid < hi && fl >= 0)) return;
    float ax = 0.0f, az = 0.0f, wsum = 0.0f;
    for (int sp = 0; sp < nsplit; sp++) { const float4 p = part[(size_t)sp * n + k]; ax += p.x; az += p.y; wsum += p.z; }
    const pf_record self = rec[uid];
    coh_finish(ax, az, wsum, coh_weight(0.0f, 0.0f), self.px, self.pz, flock_start[fl + 1] - flock_start[fl],
               __expf(4.5f - 0.12f * COH_R) * 1e7f, scaled_max_force, uid, out_by_uid, fallback, nfallback);
}

// ------------------------------------------------------------------------------------------
// K5: spatial index build (bitmap_grid.h: 16-wu cells, scaled int32 coordinates)
// ------------------------------------------------------------------------------------------

__global__ void k_cell_count(const pf_record *__restrict__ rec, int n, GridView g, uint32_t *__restrict__ count)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int cx = cell_of(bg_scale(rec[i].px), g.origin_x, g.grid_w);
    const int cy = cell_of(bg_scale(rec[i].pz), g.origin_y, g.grid_h);
    atomicAdd(&count[cy * g.grid_w + cx], 1u);
}

// single-CTA exclusive scan (cells <= 1M): a serial run per thread, the runs' sums scanned over the CTA
__global__ void k_cell_scan(const uint32_t *__restrict__ count, uint32_t *__restrict__ start, int ncells)
{
    __shared__ uint32_t warp_tot[32];
    const int tid = threadIdx.x, per = (ncells + 1023) / 1024;
    const int b = tid * per, e = min(b + per, ncells);
    uint32_t s = 0;
    for (int i = b; i < e; i++) s += count[i];
    uint32_t total;
    uint32_t run = pf_block_excl_scan(s, warp_tot, total);
    for (int i = b; i < e; i++) { start[i] = run; run += count[i]; }
    if (tid == 0) start[ncells] = total;
}

// the same scan for big grids, three launches: 4096 cells per block (4 per thread) -> block sums, their scan, apply
__global__ void __launch_bounds__(1024) k_cell_scan_sum(const uint32_t *__restrict__ count, uint32_t *__restrict__ part, int ncells)
{
    __shared__ uint32_t wt[32];
    const int i0 = (blockIdx.x * 1024 + threadIdx.x) * 4;
    uint32_t v = 0;
    for (int j = 0; j < 4; j++) if (i0 + j < ncells) v += count[i0 + j];
    uint32_t total;
    pf_block_excl_scan(v, wt, total);
    if (threadIdx.x == 0) part[blockIdx.x] = total;
}

__global__ void __launch_bounds__(1024) k_cell_scan_parts(uint32_t *__restrict__ part, int nb, uint32_t *__restrict__ start, int ncells)
{
    __shared__ uint32_t wt[32];
    const uint32_t v = (int)threadIdx.x < nb ? part[threadIdx.x] : 0u;
    uint32_t total;
    const uint32_t ex = pf_block_excl_scan(v, wt, total);
    if ((int)threadIdx.x < nb) part[threadIdx.x] = ex;
    if (threadIdx.x == 0) start[ncells] = total;
}

__global__ void __launch_bounds__(1024) k_cell_scan_apply(const uint32_t *__restrict__ count, const uint32_t *__restrict__ part,
                                                          uint32_t *__restrict__ start, int ncells)
{
    __shared__ uint32_t wt[32];
    const int i0 = (blockIdx.x * 1024 + threadIdx.x) * 4;
    uint32_t c[4], v = 0;
    for (int j = 0; j < 4; j++) { c[j] = i0 + j < ncells ? count[i0 + j] : 0u; v += c[j]; }
    uint32_t total;
    uint32_t run = part[blockIdx.x] + pf_block_excl_scan(v, wt, total);
    for (int j = 0; j < 4; j++) if (i0 + j < ncells) { start[i0 + j] = run; run += c[j]; }
}

__global__ void k_cell_scatter(const pf_record *__restrict__ rec, int n, GridView g,
                               const uint32_t *__restrict__ start, uint32_t *__restrict__ fill,
                               uint32_t *__restrict__ sid)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int cx = cell_of(bg_scale(rec[i].px), g.origin_x, g.grid_w);
    const int cy = cell_of(bg_scale(rec[i].pz), g.origin_y, g.grid_h);
    const int c = cy * g.grid_w + cx;
    const uint32_t slot = start[c] + atomicAdd(&fill[c], 1u);
    sid[slot] = (uint32_t)i;
}

// per-cell: order ids DESCENDING (LIFO overflow chain drained by bg_cleanup, bitmap_grid.h:1110,
// 1477), then materialise the scaled coordinates next to them.
__global__ void k_cell_sort(const pf_record *__restrict__ rec, GridView g, const uint32_t *__restrict__ start,
                            uint32_t *__restrict__ sid, int32_t *__restrict__ six, int32_t *__restrict__ siy,
                            int ncells, const int32_t *__restrict__ flock_of, int32_t *__restrict__ sfl)
{
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncells) return;
    const uint32_t b = start[c], e = start[c + 1];
    for (uint32_t i = b + 1; i < e; i++) {      // insertion sort, descending
        const uint32_t v = sid[i];
        uint32_t j = i;
        while (j > b && sid[j - 1] < v) { sid[j] = sid[j - 1]; j--; }
        sid[j] = v;
    }
    for (uint32_t i = b; i < e; i++) {
        const pf_record r = rec[sid[i]];
        six[i] = bg_scale(r.px);
        siy[i] = bg_scale(r.pz);
        sfl[i] = flock_of[sid[i]];
    }
}

#define VEL_WARPS_PER_CTA 4
#ifndef VEL_MIN_CTAS_SINGLE
#define VEL_MIN_CTAS_SINGLE 6
#endif
#ifndef VEL_MIN_CTAS
#define VEL_MIN_CTAS 6          // 24 warps / SM: <= 80 registers (sm_90a, CUDA 12.9: 44 B of spill stores in <0>, 16 B in <2>, none in <1>), 6 x 32 KB of shared memory
#endif

struct TickParams {
    int hz;
    float scaled_max_force;       // (float)SCALED_MAX_FORCE, as passed to vec2_truncate
    double scaled_max_force_d;    // SCALED_MAX_FORCE as the double it is in comparisons (movement.c:1895)
    unsigned long long *stats;    // ClearPath event counters (pfnav_agents_clearpath_stats), never read by the kernels
    unsigned int *queue;          // next work item of the velocity kernels, one counter per MODE; zeroed every tick
};

// ------------------------------------------------------------------------------------------
// K6c: one warp per agent
// ------------------------------------------------------------------------------------------
// MODE 0: the whole update in one pass. MODE 1 / 2: phase A / phase B of the two-phase scheme above.
template <int MODE>
__global__ void __launch_bounds__(VEL_WARPS_PER_CTA * 32, MODE == 0 ? VEL_MIN_CTAS_SINGLE : VEL_MIN_CTAS)
k_agent_velocity(MapView m, GridView g, TickParams tp, const pfnav_agent *__restrict__ agents,
                 const pf_record *__restrict__ rec, const pfnav_flock *__restrict__ flocks,
                 const uint32_t *__restrict__ work, int nwork, const float2 *__restrict__ vdes_in,
                 const uint8_t *__restrict__ los_in, const float2 *__restrict__ cohesion_in,
                 float2 *__restrict__ vel_out, float2 *__restrict__ vpref_out, int filter_garr,
                 uint32_t *__restrict__ nb_scratch, pf_prep *__restrict__ prep,
                 const pfnav_formation_in *__restrict__ form)
{
    extern __shared__ __align__(16) uint8_t vel_smem_raw[];      // VEL_WARPS_PER_CTA x VelSmem (> 48 KB: opt-in, pfnav_agents_init)
    const uint32_t lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    VelSmem &s = reinterpret_cast<VelSmem *>(vel_smem_raw)[warp];
    // work items are taken from a queue, not strided: an entity whose ClearPath solve runs long (no admissible velocity, a
    // sixth of a moving crowd) would otherwise hold its CTA's three other warps idle at the end of their own strides
    for (;;) {
        int w = 0;
        if (lane == 0) w = (int)atomicAdd(tp.queue + MODE, 1u);
        w = __shfl_sync(FULL, w, 0);
        if (w >= nwork) break;
        const uint32_t uid = work[w];
        const pfnav_agent a = agents[uid];
        const uint32_t ent_flags = a.flags & 0xFFFFFFu;
        // COMBAT_HELD (movement.c:3405)
        if (ent_flags & PFNAV_FLAG_COMBAT_HELD) {
            if (MODE != 1 && lane == 0) { vel_out[w] = make_float2(0.f, 0.f); vpref_out[w] = make_float2(0.f, 0.f); }
            continue;
        }
        const v2 pos = {a.pos[0], a.pos[1]};
        const v2 velocity = {a.velocity[0], a.velocity[1]};
        const float2 vd = MODE == 1 ? make_float2(0.f, 0.f) : vdes_in[w];      // phase A runs before the fields exist
        const v2 vdes = {vd.x, vd.y};
        const bool has_los = MODE == 1 ? false : los_in[w] != 0;
        const float hzf = (float)tp.hz;

        v2 vpref = {0.0f, 0.0f};
        if (a.state == PFNAV_STATE_TURNING) {
            vpref = {0.0f, 0.0f};
        } else {
            // ================= point_seek_vpref (movement.c:1870) =================
            // ---- separation_force (movement.c:1690): 30-wu query, first 128 hits in index order ----
            v2 separation = {0.0f, 0.0f};
            if (MODE == 2) {
                separation = {prep[w].sepx, prep[w].sepz};
            } else {
            int num_near = 0;
            grid_query(g, pos.x, pos.z, 30.0f, lane, [&](bool hit, uint32_t id) -> bool {
                const uint32_t mk = __ballot_sync(FULL, hit);
                if (!mk) return false;
                const int rank = __popc(mk & ((1u << lane) - 1));
                if (hit && num_near + rank < 128) s.near_id[num_near + rank] = id;
                num_near += __popc(mk);
                return num_near >= 128;
            });
            num_near = min(num_near, 128);
            __syncwarp();
            if (filter_garr) num_near = filter_garrisoned(s.near_id, num_near, rec, lane);
            for (int k = lane; k < num_near; k += 32) {
                const uint32_t cu = s.near_id[k];
                float2 term = make_float2(0.f, 0.f);
                if (cu != uid) {
                    const pf_record r = rec[cu];
                    const uint32_t fl = r.state_flags & 0xFFFFFFu;
                    if ((fl & PFNAV_FLAG_MOVABLE) && ((ent_flags & PFNAV_FLAG_AIR) == (fl & PFNAV_FLAG_AIR))) {
                        v2 diff = {r.px - pos.x, r.pz - pos.z};
                        const float radius = a.radius + r.radius + 0.0f;
                        const float len = v2_len(diff);
                        if (!(len < EPS_F)) {
                            const float t = (len - radius * 0.85f) / len;
                            const float scale = (float)exp((double)fminf(-20.0f * t, 40.0f));
                            diff = v2_scale(diff, scale);
                            term = make_float2(diff.x, diff.z);
                        }
                    }
                }
                s.term[k] = term;
            }
            __syncwarp();
            separation = {0.0f, 0.0f};
            for (int k = 0; k < num_near; k++) {         // the reference's summation order
                const float2 t = s.term[k];
                separation.x += t.x;
                separation.z += t.y;
            }
            if (num_near == 0) separation = {0.0f, 0.0f};
            else {
                separation = v2_scale(separation, -1.0f);
                separation = v2_truncate(separation, tp.scaled_max_force);
            }
                if (MODE == 1 && lane == 0) { prep[w].sepx = separation.x; prep[w].sepz = separation.z; }
            }
            if (MODE == 1) { /* the rest of point_seek_vpref needs the desired velocity: phase B */ } else {
            // the state picks the steering variant (move_velocity_work, movement.c:3414-3448)
            const uint32_t st_ = a.state;
            pfnav_formation_in fin;
            const bool has_form = form != nullptr && (st_ == PFNAV_STATE_ARRIVING_TO_CELL || st_ == PFNAV_STATE_MOVING_IN_FORMATION);
            if (has_form) fin = form[uid];
            const bool cell_mode = st_ == PFNAV_STATE_ARRIVING_TO_CELL, form_mode = st_ == PFNAV_STATE_MOVING_IN_FORMATION;
            const bool enemy_mode = st_ == PFNAV_STATE_SEEK_ENEMIES;
            const bool ready = has_form && (fin.flags & PFNAV_FORM_ASSIGNMENT_READY);
            v2 arrive;
            if (cell_mode) {
                // ---- arrive_force_cell (movement.c:1571): NOT relative to the current velocity, not truncated ----
                const v2 cell = has_form ? v2{fin.cell_pos[0], fin.cell_pos[1]} : pos;
                v2 desired = v2_sub(cell, pos);
                const float distance = v2_len(desired);
                if (distance < 10.0f) desired = v2_scale(desired, distance / 10.0f);
                else desired = v2_scale(vdes, a.max_speed / hzf);
                arrive = desired;
            } else if (enemy_mode) {
                // ---- arrive_force_enemies (movement.c:1593) ----
                const v2 desired = v2_scale(vdes, a.max_speed / hzf);
                arrive = v2_truncate(v2_sub(desired, velocity), tp.scaled_max_force);
            } else {
            // ---- arrive_force_point (movement.c:1546) ----
            const v2 target = a.flock >= 0 ? v2{flocks[a.flock].target[0], flocks[a.flock].target[1]} : pos;
            v2 desired;
            if (has_los) {
                desired = v2_sub(target, pos);
                const float distance = v2_len(desired);
                desired = v2_normal(desired);
                desired = v2_scale(desired, a.max_speed / hzf);
                if (distance < 10.0f) desired = v2_scale(desired, distance / 10.0f);
            } else {
                desired = v2_scale(vdes, a.max_speed / hzf);
            }
            arrive = v2_truncate(v2_sub(desired, velocity), tp.scaled_max_force);
            }
            // ---- cohesion: the flock-wide pre-pass, or the formation's own forces (fstate, movement.c:215-225) ----
            const float2 ch = cohesion_in[uid];
            const v2 cohesion = (cell_mode || form_mode) ? (has_form ? v2{fin.cohesion[0], fin.cohesion[1]} : v2{0.0f, 0.0f}) : v2{ch.x, ch.y};
            const v2 alignment = has_form ? v2{fin.align[0], fin.align[1]} : v2{0.0f, 0.0f};

            const int layer = nav_layer_for(ent_flags, a.radius);
            bool on_blocked, dummy, lp, lb, rp, rb, tpth, tb, bp, bb;
            probe_tile(m, layer, pos.x, pos.z, dummy, on_blocked);
            probe_tile(m, layer, pos.x + 4.0f, pos.z, lp, lb);      // left  = x + nt_dims.x
            probe_tile(m, layer, pos.x - 4.0f, pos.z, rp, rb);      // right
            probe_tile(m, layer, pos.x, pos.z + 4.0f, tpth, tb);    // top   = z + nt_dims.z
            probe_tile(m, layer, pos.x, pos.z - 4.0f, bp, bb);      // bot

            v2 steer = {0.0f, 0.0f};
            for (int prio = 0; prio < (enemy_mode ? 1 : 3); prio++) {
                if (prio == 0) {
                    // point_seek_total_force / formation_point_seek_total_force / cell_seek_total_force /
                    // enemy_seek_total_force (movement.c:1745, 1960, 1769, 1801)
                    const v2 A = v2_scale(arrive, 0.5f), C = v2_scale(cohesion, 0.15f), S = v2_scale(separation, 0.6f);
                    const v2 AL = v2_scale(alignment, 0.15f);
                    v2 ret = {0.0f, 0.0f};
                    ret = v2_add(ret, A);
                    ret = v2_add(ret, S);
                    if (cell_mode) {
                        const v2 cell = has_form ? v2{fin.cell_pos[0], fin.cell_pos[1]} : pos;
                        if (v2_len(v2_sub(cell, pos)) > 30.0f) { ret = v2_add(ret, C); ret = v2_add(ret, AL); }     // CELL_ARRIVAL_RADIUS
                    } else if (!enemy_mode) ret = v2_add(ret, C);
                    steer = v2_truncate(ret, tp.scaled_max_force);
                } else if (prio == 1) steer = separation;
                else steer = arrive;
                if (enemy_mode) break;              // enemy_seek_vpref (movement.c:1946): no nullify pass, no fall-backs
                // nullify_impass_components (movement.c:1831)
                if (steer.x > 0 && (!lp || (!on_blocked && lb))) steer.x = 0.0f;
                if (steer.x < 0 && (!rp || (!on_blocked && rb))) steer.x = 0.0f;
                if (steer.z > 0 && (!tpth || (!on_blocked && tb))) steer.z = 0.0f;
                if (steer.z < 0 && (!bp || (!on_blocked && bb))) steer.z = 0.0f;
                if ((double)v2_len(steer) > tp.scaled_max_force_d * 0.01) break;
            }
            const v2 accel = v2_scale(steer, 1.0f / 1.0f);
            vpref = v2_truncate(v2_add(velocity, accel), a.speed / hzf);
            if ((cell_mode || form_mode) && has_form) {
                // formation drag caps the speed at 75 % (movement.c:1940, 2017); unassigned members stand still (:3426, :3438)
                if (v2_len(v2{fin.drag[0], fin.drag[1]}) > EPS_F) vpref = v2_truncate(vpref, (float)(((double)a.speed * 0.75) / (double)hzf));
                if (!ready) vpref = {0.0f, 0.0f};
            } else if (cell_mode || form_mode) vpref = {0.0f, 0.0f};
            }
        }

        // ================= find_neighbours (movement.c:2768) =================
        int ndyn = 0, nstat = 0, raw = 0;
        if (MODE == 2) {
            // phase A stored the neighbour lists (ids, in the reference's order); rebuild the cp_ents
            ndyn = (int)prep[w].ndyn; nstat = (int)prep[w].nstat;
            for (int k = lane; k < ndyn + nstat; k += 32) {
                const bool isst = k >= ndyn;
                const pf_record r = rec[isst ? prep[w].stat_id[k - ndyn] : prep[w].dyn_id[k]];
                cp_ent nd;
                nd.pos = {r.px, r.pz}; nd.radius = r.radius;
                nd.vel = isst ? v2{0.0f, 0.0f} : v2{r.vx, r.vz};
                if (isst) s.stat[k - ndyn] = nd; else s.dyn[k] = nd;
            }
        }
        auto classify = [&](bool hit, uint32_t id) -> bool {
            const uint32_t mk = __ballot_sync(FULL, hit);
            if (!mk) return false;
            const int rrank = __popc(mk & ((1u << lane) - 1));
            bool isdyn = false, isstat = false;
            cp_ent nd;
            if (hit && raw + rrank < 512 && id != uid) {
                const pf_record r = rec[id];
                const uint32_t fl = r.state_flags & 0xFFFFFFu;
                const uint32_t st = r.state_flags >> 24;
                if ((fl & PFNAV_FLAG_MOVABLE) && r.radius != 0.0f &&
                    ((ent_flags & PFNAV_FLAG_AIR) == (fl & PFNAV_FLAG_AIR))) {
                    nd.pos = {r.px, r.pz}; nd.vel = {r.vx, r.vz}; nd.radius = r.radius;
                    const bool still = (st == PFNAV_STATE_ARRIVED || st == PFNAV_STATE_WAITING);
                    if (still || v2_len(nd.vel) < 0.3f) { nd.vel = {0.0f, 0.0f}; isstat = true; }
                    else isdyn = true;
                }
            }
            const uint32_t md = __ballot_sync(FULL, isdyn), ms = __ballot_sync(FULL, isstat);
            if (isdyn) { const int k = ndyn + __popc(md & ((1u << lane) - 1)); if (k < PFNAV_MAX_NEIGHBOURS) { s.dyn[k] = nd; if (MODE == 1) prep[w].dyn_id[k] = id; } }
            if (isstat) { const int k = nstat + __popc(ms & ((1u << lane) - 1)); if (k < PFNAV_MAX_NEIGHBOURS) { s.stat[k] = nd; if (MODE == 1) prep[w].stat_id[k] = id; } }
            ndyn = min(ndyn + __popc(md), PFNAV_MAX_NEIGHBOURS);
            nstat = min(nstat + __popc(ms), PFNAV_MAX_NEIGHBOURS);
            raw += __popc(mk);
            return raw >= 512;
        };
        if (MODE == 2) {
            // nothing to gather
        } else if (!filter_garr) {
            grid_query(g, pos.x, pos.z, 10.0f, lane, classify);
        } else {
            // garrisoned entities exist: G_Pos_EntsInCircleFrom (position.c:379) first takes the raw hits (<= 512),
            // then filter_garrisoned swap-removes them, which reorders the survivors -> materialise the list
            uint32_t *lst = nb_scratch + (size_t)(blockIdx.x * VEL_WARPS_PER_CTA + warp) * 512;
            int cnt = 0;
            grid_query(g, pos.x, pos.z, 10.0f, lane, [&](bool hit, uint32_t id) -> bool {
                const uint32_t mk = __ballot_sync(FULL, hit);
                const int rank = __popc(mk & ((1u << lane) - 1));
                if (hit && cnt + rank < 512) lst[cnt + rank] = id;
                cnt += __popc(mk);
                return cnt >= 512;
            });
            cnt = min(cnt, 512);
            __syncwarp();
            cnt = filter_garrisoned(lst, cnt, rec, lane);
            for (int k0 = 0; k0 < cnt; k0 += 32) {
                const int k = k0 + (int)lane;
                if (classify(k < cnt, k < cnt ? lst[k] : 0u)) break;
            }
        }
        __syncwarp();

        // ================= G_ClearPath_NewVelocity (clearpath.c:694) =================
        const cp_ent self = {{a.prev_pos[0], a.prev_pos[1]}, velocity, a.radius};
        if (MODE == 1) {
            const int nx = clearpath_collect(s, self, ndyn, nstat, lane, prep[w].xp);
            if (lane == 0) {
                prep[w].ndyn = (uint32_t)ndyn; prep[w].nstat = (uint32_t)nstat;
                prep[w].nx = nx > PF_PREP_XP_CAP ? PF_PREP_OVERFLOW : (uint32_t)nx;
            }
            __syncwarp();
            continue;
        }
        v2 new_vel = {0.0f, 0.0f};
        {
            // first solve; when it finds no admissible velocity the drop-furthest retry loop (clearpath.c:702-713) is
            // resolved in one pass over the same ray table (clearpath_retry). tests/emu/clearpath_emu.cpp restates this block
            // (kept inline here: as a function in pfnav_clearpath_kernel.cuh it reorders the <2> schedule)
            v2 r;
            int n_rays = 0;
            bool found, exact = true;
            if (MODE == 2 && prep[w].nx != PF_PREP_OVERFLOW)
                found = clearpath_finish(s, self, vpref, ndyn, nstat, lane, prep[w].xp, (int)prep[w].nx, r, n_rays);
            else
                found = clearpath_new_velocity(s, self, vpref, ndyn, nstat, lane, r, n_rays);
            if (found) new_vel = r;
            else {
                if (lane == 0) { atomicAdd(tp.stats + 0, 1ull); if (ndyn > 0 && nstat > 0) atomicAdd(tp.stats + 1, 1ull); }
                new_vel = clearpath_retry(s, self, vpref, ndyn, nstat, n_rays, lane, exact);
                if (!exact) {
                    // replay the reference's loop literally (clearpath.c:702-713)
                    new_vel = {0.0f, 0.0f};
                    unsigned long long solves = 0;
                    while (true) {
                        remove_furthest(s, self.pos, ndyn, nstat, lane);
                        if (!(ndyn > 0 && nstat > 0)) break;
                        int nr2;
                        solves++;
                        if (clearpath_new_velocity(s, self, vpref, ndyn, nstat, lane, r, nr2)) { new_vel = r; break; }
                    }
                    if (lane == 0) { atomicAdd(tp.stats + 2, 1ull); atomicAdd(tp.stats + 3, solves); }
                }
            }
        }
        new_vel = v2_truncate(new_vel, a.max_speed / hzf);      // movement.c:3464
        if (lane == 0) {
            vel_out[w] = make_float2(new_vel.x, new_vel.z);
            vpref_out[w] = make_float2(vpref.x, vpref.z);
        }
        __syncwarp();
    }
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
#define VEL_SMEM_BYTES ((int)(VEL_WARPS_PER_CTA * sizeof(VelSmem)))
int pfnav_agents_init(pfnav_ctx *ctx)
{
    (void)ctx;
    PF_CUDA(cudaFuncSetAttribute(k_agent_velocity<0>, cudaFuncAttributeMaxDynamicSharedMemorySize, VEL_SMEM_BYTES));
    PF_CUDA(cudaFuncSetAttribute(k_agent_velocity<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, VEL_SMEM_BYTES));
    PF_CUDA(cudaFuncSetAttribute(k_agent_velocity<2>, cudaFuncAttributeMaxDynamicSharedMemorySize, VEL_SMEM_BYTES));
    return 0;
}

void pfnav_agents_free(pfnav_ctx *ctx)
{
    if (ctx->update_done) cudaEventDestroy(ctx->update_done);
}

// ---- agents ----
int pf_flocks_reserve(pfnav_ctx *ctx, size_t nflocks)
{
    int rc = ctx->d_flocks.reserve(nflocks + 1);
    if (!rc) rc = ctx->d_flock_start.reserve(nflocks + 2);
    if (rc) { ctx->d_flocks.release(); ctx->d_flock_start.release(); }
    return rc;
}

int pf_work_reserve(pfnav_ctx *ctx, size_t nwork)
{
    int rc = pf_dbuf_reserve_all(nwork, ctx->d_work, ctx->d_vel_out, ctx->d_vpref_out, ctx->d_vdes_out, ctx->d_los_out);
    if (!rc) rc = ctx->d_work_count.reserve(4);
    if (rc) ctx->n_work = 0;
    return rc;
}

static GridView grid_of(const pfnav_ctx *ctx)
{
    GridView g;
    g.cell_start = ctx->d_cell_start; g.cell_count = ctx->d_cell_count;
    g.ix = ctx->d_sorted_ix; g.iy = ctx->d_sorted_iy; g.id = ctx->d_sorted_id;
    g.grid_w = ctx->grid_w; g.grid_h = ctx->grid_h; g.origin_x = ctx->origin_x; g.origin_y = ctx->origin_y;
    return g;
}

// The exclusive scan of count[0 .. n) into start[0 .. n], start[n] = the total, on `st`: the three k_cell_scan_* launches over
// block sums in part (1024 words) when n spans 2 .. 1024 blocks of 4096 (scan_uses_part), else the single-CTA k_cell_scan.
static bool scan_uses_part(int n) { const int nsb = (n + 4095) / 4096; return nsb > 1 && nsb <= 1024; }
static void excl_scan(pfnav_ctx *ctx, const uint32_t *count, uint32_t *part, uint32_t *start, int n, cudaStream_t st)
{
    if (scan_uses_part(n)) {
        const int nsb = (n + 4095) / 4096;
        k_cell_scan_sum<<<nsb, 1024, 0, st>>>(count, part, n);
        k_cell_scan_parts<<<1, 1024, 0, st>>>(part, nsb, start, n);
        k_cell_scan_apply<<<nsb, 1024, 0, st>>>(count, part, start, n);
        ctx->launches += 3;
    } else {
        k_cell_scan<<<1, 1024, 0, st>>>(count, start, n);
        ctx->launches++;
    }
}

int build_index(pfnav_ctx *ctx, cudaStream_t st)
{
    const int n = (int)ctx->n_agents;
    const int ncells = ctx->grid_w * ctx->grid_h;
    pf_prof_scope prof(ctx, st, PF_PROF_INDEX);
    PF_CUDA(cudaMemsetAsync(ctx->d_cell_count, 0, (size_t)ncells * 4, st));
    PF_CUDA(cudaMemsetAsync(ctx->d_cell_fill, 0, (size_t)ncells * 4, st));
    if (n > 0) {
        const GridView g = grid_of(ctx);
        k_cell_count<<<(n + 255) / 256, 256, 0, st>>>(ctx->d_records, n, g, ctx->d_cell_count);
        if (scan_uses_part(ncells))
            if (int rc = ctx->d_scan_part.reserve(1024)) return rc;
        excl_scan(ctx, ctx->d_cell_count, ctx->d_scan_part, ctx->d_cell_start, ncells, st);
        k_cell_scatter<<<(n + 255) / 256, 256, 0, st>>>(ctx->d_records, n, g, ctx->d_cell_start, ctx->d_cell_fill,
                                                       ctx->d_sorted_id);
        k_cell_sort<<<(ncells + 127) / 128, 128, 0, st>>>(ctx->d_records, g, ctx->d_cell_start, ctx->d_sorted_id,
                                                         ctx->d_sorted_ix, ctx->d_sorted_iy, ncells, ctx->d_flock_of, ctx->d_sorted_flock);
        ctx->launches += 3;
    } else {
        PF_CUDA(cudaMemsetAsync(ctx->d_cell_start, 0, (size_t)(ncells + 1) * 4, st));
    }
    PF_CUDA(cudaGetLastError());
    ctx->index_stale = false;
    return 0;
}

// records of the uploaded range + the flock id column (neighbour kernels read other agents' flock through it)
__global__ void k_make_records(const pfnav_agent *__restrict__ agents, pf_record *__restrict__ rec, int32_t *__restrict__ flock_of,
                               int lo, int hi)
{
    const int i = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= hi) return;
    const pfnav_agent a = agents[i];
    pf_record r;
    r.px = a.pos[0]; r.pz = a.pos[1]; r.vx = a.velocity[0]; r.vz = a.velocity[1];
    r.radius = a.radius;
    r.state_flags = (a.state << 24) | (a.flags & 0xFFFFFFu);
    rec[i] = r;
    flock_of[i] = a.flock;
}

// population-wide facts the tick needs from records it did not upload itself (other ranks' shards): the largest
// selection radius (adjacency pre-selection of k_entity_update) and whether any entity is garrisoned
__global__ void k_population_facts(const pf_record *__restrict__ rec, int n, uint32_t *__restrict__ out)
{
    uint32_t mx = 0, garr = 0;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const pf_record r = rec[i];
        mx = max(mx, __float_as_uint(fmaxf(r.radius, 0.0f)));          // non-negative floats order like their bit patterns
        garr |= (r.state_flags & PFNAV_FLAG_GARRISONED) ? 1u : 0u;
    }
    for (int off = 16; off > 0; off >>= 1) { mx = max(mx, __shfl_xor_sync(FULL, mx, off)); garr |= __shfl_xor_sync(FULL, garr, off); }
    if ((threadIdx.x & 31) == 0) { atomicMax(&out[0], mx); if (garr) atomicOr(&out[1], 1u); }
}

int pfnav_mgpu_allgather(pfnav_ctx *ctx, void *d_buf, size_t elem_bytes, cudaStream_t st);      // pfnav_mgpu.cu

// flock member lists (ascending uid: the iteration order our cohesion sum is defined over) from the flock id column
static int rebuild_flock_members(pfnav_ctx *ctx, cudaStream_t st)
{
    const size_t n = ctx->n_agents, nflocks = ctx->n_flocks;
    std::vector<int32_t> fo(n ? n : 1);
    PF_CUDA(cudaMemcpyAsync(fo.data(), ctx->d_flock_of, n * 4, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    std::vector<uint32_t> fstart(nflocks + 1, 0), members(n ? n : 1);
    for (size_t i = 0; i < n; i++) {
        PF_ARG(fo[i] < (int)nflocks, "agent flock index out of range");
        if (fo[i] >= 0) fstart[fo[i] + 1]++;
    }
    for (size_t f = 0; f < nflocks; f++) fstart[f + 1] += fstart[f];
    {
        std::vector<uint32_t> cur(fstart.begin(), fstart.end() - 1);
        for (size_t i = 0; i < n; i++)
            if (fo[i] >= 0) members[cur[fo[i]]++] = (uint32_t)i;
    }
    PF_CUDA(cudaMemcpyAsync(ctx->d_flock_start, fstart.data(), (nflocks + 1) * 4, cudaMemcpyHostToDevice, st));
    if (n) PF_CUDA(cudaMemcpyAsync(ctx->d_flock_members, members.data(), n * 4, cudaMemcpyHostToDevice, st));
    PF_CUDA(cudaStreamSynchronize(st));      // host vectors go out of scope
    ctx->h_flock_start = fstart;
    return 0;
}

// move_copy_gamestate (movement.c:3607) for the index range [lo, hi) of a population of n_total entities
// (uid == index into the whole population). Single GPU: lo = 0, hi = n_total. Multi-GPU: every rank uploads its own
// range (pfnav_mgpu_shard_range) and the 24-byte neighbour records + flock ids of the other ranges arrive through
// the all-gather.
static int agents_upload_impl(pfnav_ctx *ctx, const pfnav_agent *agents, size_t lo, size_t hi, size_t n,
                              const pfnav_flock *flocks, size_t nflocks, int hz, uint32_t flags)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    PF_ARG(lo <= hi && hi <= n, "shard range");
    PF_ARG(hi == lo || agents, "agents");
    PF_ARG(nflocks == 0 || flocks, "flocks");
    PF_ARG(hz == 20 || hz == 10 || hz == 5 || hz == 1, "hz must be 20, 10, 5 or 1 (movement.c:2210)");
    PF_ARG(n < (1u << 31), "n");
    const bool sharded = ctx->mgpu != nullptr;
    PF_ARG(sharded || (lo == 0 && hi == n), "a partial upload needs pfnav_mgpu_init / pfnav_group_create first");
    ctx->events_valid = false;              // the event list's uids name the previous population
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = ctx->tick_stream;
    const bool same = (flags & PFNAV_UPLOAD_SAME_FLOCKS) && ctx->n_agents == n && ctx->n_flocks == nflocks &&
                      ctx->shard_lo == lo && ctx->shard_hi == hi && ctx->hz == hz;
    ctx->hz = hz;
    int rc = pf_dbuf_reserve_all(n, ctx->d_agents, ctx->d_records, ctx->d_flock_members, ctx->d_flock_of, ctx->d_sorted_ix,
                                 ctx->d_sorted_iy, ctx->d_sorted_flock, ctx->d_sorted_id);
    if (!rc) rc = pf_flocks_reserve(ctx, nflocks);
    if (!rc) rc = ctx->d_facts.reserve(2);
    if (rc) return rc;
    ctx->n_agents = n; ctx->n_flocks = nflocks; ctx->shard_lo = lo; ctx->shard_hi = hi;
    if (!same) {
        // what the host needs to know about the entities it will run work items for (its own range)
        ctx->flock_layer_used.assign(nflocks * PFNAV_NAV_LAYER_MAX, 0);
        ctx->has_unsupported_state = false;
        ctx->cmd_mirror.reset(hi - lo, nflocks);      // (flock, layer) per own entity, for pfnav_agents_commands
        for (size_t i = 0; i < hi - lo; i++) {
            // Entity_NavLayerWithRadius (entity.c:554): the layer this agent's tile probes read
            int layer;
            const char *err = pf_agent_check(agents[i], nflocks, ctx->nlayers, &layer);
            PF_ARG(!err, err);
            if (agents[i].flock >= 0) ctx->flock_layer_used[(size_t)agents[i].flock * PFNAV_NAV_LAYER_MAX + layer] = 1;
            ctx->cmd_mirror.set(i, std::max(agents[i].flock, -1), layer);
            const uint32_t stt = agents[i].state;
            if (stt == PFNAV_STATE_MOVING_IN_FORMATION || stt == PFNAV_STATE_SURROUND_ENTITY ||
                stt == PFNAV_STATE_ENTER_ENTITY_RANGE || stt == PFNAV_STATE_TURNING || stt == PFNAV_STATE_ARRIVING_TO_CELL)
                ctx->has_unsupported_state = true;
        }
        ctx->h_flocks.assign(flocks, flocks + nflocks);
        ctx->arrival_valid = false;
        // optional per-entity inputs of the previous population do not carry over
        ctx->d_formation.release();
        ctx->d_ms_ext.release();
    }
    if (hi > lo) PF_CUDA(cudaMemcpyAsync(ctx->d_agents + lo, agents, (hi - lo) * sizeof(pfnav_agent), cudaMemcpyHostToDevice, st));
    if (nflocks && !same) PF_CUDA(cudaMemcpyAsync(ctx->d_flocks, flocks, nflocks * sizeof(pfnav_flock), cudaMemcpyHostToDevice, st));
    // spatial index geometry: G_Pos_Init (position.c:264) + bg_init (bitmap_grid.h:959)
    {
        const float W = (float)(ctx->chunk_w * 256), H = (float)(ctx->chunk_h * 256);
        const float cx = ctx->map_x - W / 2.0f, cz = ctx->map_z + H / 2.0f;
        const float xmin = cx - W / 2.0f, xmax = cx + W / 2.0f, zmin = cz - H / 2.0f, zmax = cz + H / 2.0f;
        ctx->origin_x = (int32_t)lrintf(xmin * 256.0f);
        ctx->origin_y = (int32_t)lrintf(zmin * 256.0f);
        const int32_t span_x = (int32_t)lrintf(xmax * 256.0f) - ctx->origin_x;
        const int32_t span_y = (int32_t)lrintf(zmax * 256.0f) - ctx->origin_y;
        ctx->grid_w = std::max(1, (int)(((uint32_t)span_x + 4095u) >> 12));
        ctx->grid_h = std::max(1, (int)(((uint32_t)span_y + 4095u) >> 12));
        const size_t ncells = (size_t)ctx->grid_w * ctx->grid_h;
        if ((rc = pf_dbuf_reserve_all(ncells + 1, ctx->d_cell_count, ctx->d_cell_start, ctx->d_cell_fill))) return rc;
    }
    if (hi > lo) {
        k_make_records<<<((int)(hi - lo) + 255) / 256, 256, 0, st>>>(ctx->d_agents, ctx->d_records, ctx->d_flock_of, (int)lo, (int)hi);
        ctx->launches++;
    }
    // default work list: none until pfnav_agents_set_work (a same-structure re-upload keeps the current one)
    if (!same) ctx->n_work = 0;
    if (sharded) {
        // the other ranges' records (and, when membership may have changed, flock ids) come from the peers;
        // pfnav_mgpu_gather / pfnav_group_gather follows and finishes the snapshot (index, facts, member lists)
        ctx->members_stale = !same;
        ctx->index_stale = true;
        PF_CUDA(cudaStreamSynchronize(st));
        return PFNAV_OK;
    }
    return pfnav_agents_finish_snapshot(ctx, st, !same);
}

int pfnav_agents_refresh_facts(pfnav_ctx *ctx, cudaStream_t st)
{
    const int n = (int)ctx->n_agents;
    PF_CUDA(cudaMemsetAsync(ctx->d_facts, 0, 8, st));
    if (n) { k_population_facts<<<std::min((n + 255) / 256, 1024), 256, 0, st>>>(ctx->d_records, n, ctx->d_facts); ctx->launches++; }
    uint32_t facts[2] = {0, 0};
    PF_CUDA(cudaMemcpyAsync(facts, ctx->d_facts, 8, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    memcpy(&ctx->max_radius, &facts[0], 4);
    ctx->any_garrisoned = facts[1] != 0;
    return PFNAV_OK;
}

// Everything that needs the WHOLE population's records: member lists, population facts, spatial index.
int pfnav_agents_finish_snapshot(pfnav_ctx *ctx, cudaStream_t st, bool members)
{
    int rc;
    if (members && (rc = rebuild_flock_members(ctx, st))) return rc;
    if (members && (rc = pfnav_agents_refresh_facts(ctx, st))) return rc;
    if ((rc = build_index(ctx, st))) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_upload(pfnav_ctx *ctx, const pfnav_agent *agents, size_t n, const pfnav_flock *flocks,
                                   size_t nflocks, int hz)
{
    PF_ARG(ctx && !ctx->mgpu, "multi-GPU contexts upload their own range: pfnav_agents_upload_shard");
    return agents_upload_impl(ctx, agents, 0, n, n, flocks, nflocks, hz, 0);
}

extern "C" int pfnav_agents_upload_shard(pfnav_ctx *ctx, const pfnav_agent *shard, size_t lo, size_t hi, size_t n_total,
                                         const pfnav_flock *flocks, size_t nflocks, int hz, uint32_t flags)
{
    PF_ARG(ctx, "ctx");
    return agents_upload_impl(ctx, shard, lo, hi, n_total, flocks, nflocks, hz, flags);
}

extern "C" int pfnav_agents_rebuild_index(pfnav_ctx *ctx, void *stream)
{
    PF_ARG(ctx && ctx->d_records, "agents not uploaded");
    PF_CUDA(cudaSetDevice(ctx->device));
    return build_index(ctx, pf_stream(ctx, stream));
}

extern "C" int pfnav_agents_device_ptrs(pfnav_ctx *ctx, void **d_records, void **d_velocities, size_t *n)
{
    PF_ARG(ctx, "ctx");
    if (d_records) *d_records = ctx->d_records;
    if (d_velocities) *d_velocities = ctx->d_vel_out;
    if (n) *n = ctx->n_agents;
    return PFNAV_OK;
}

extern "C" int pfnav_agents_set_work(pfnav_ctx *ctx, const uint32_t *uids, size_t nwork)
{
    PF_ARG(ctx && ctx->d_agents, "agents not uploaded");
    PF_CUDA(cudaSetDevice(ctx->device));
    std::vector<uint32_t> all;
    if (!uids) {
        // every agent that is not still (ent_still, movement.c:652) -- needs the host copy of state
        const size_t lo = ctx->shard_lo, cnt = ctx->shard_hi - ctx->shard_lo;
        std::vector<pfnav_agent> h(cnt);
        PF_CUDA(cudaDeviceSynchronize());
        if (cnt) PF_CUDA(cudaMemcpy(h.data(), ctx->d_agents + lo, cnt * sizeof(pfnav_agent), cudaMemcpyDeviceToHost));
        for (size_t i = 0; i < cnt; i++)
            if (h[i].state != PFNAV_STATE_ARRIVED && h[i].state != PFNAV_STATE_WAITING) all.push_back((uint32_t)(lo + i));
        uids = all.data();
        nwork = all.size();
    }
    for (size_t i = 0; i < nwork; i++)
        PF_ARG(uids[i] >= ctx->shard_lo && uids[i] < ctx->shard_hi, "work uid outside this context's own entity range");
    if (int rc = pf_work_reserve(ctx, nwork)) return rc;
    if (nwork) PF_CUDA(cudaMemcpy(ctx->d_work, uids, nwork * 4, cudaMemcpyHostToDevice));
    ctx->n_work = nwork;
    return PFNAV_OK;
}

__global__ void k_copy_vdes(const pfnav_agent *__restrict__ agents, const uint32_t *__restrict__ work, int nwork,
                            float2 *__restrict__ vdes, uint8_t *__restrict__ los)
{
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwork) return;
    const pfnav_agent &a = agents[work[w]];
    vdes[w] = make_float2(a.vdes[0], a.vdes[1]);
    los[w] = a.has_dest_los ? 1 : 0;
}

extern "C" int pfnav_agents_tick(pfnav_ctx *ctx, uint32_t flags, void *stream)
{
    PF_ARG(ctx && ctx->d_agents, "agents not uploaded");
    if (ctx->n_work == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    const int nwork = (int)ctx->n_work;
    ctx->tick_no++;
    MapView m;
    m.cost = ctx->d_cost; m.blk = ctx->d_blk; m.W64 = ctx->W64; m.H64 = ctx->H64;
    m.chunk_w = ctx->chunk_w; m.chunk_h = ctx->chunk_h; m.map_x = ctx->map_x; m.map_z = ctx->map_z;
    // SCALED_MAX_FORCE = (MAX_FORCE / hz_count(hz) * 20.0): float division, double product (movement.c:93)
    TickParams tp;
    tp.hz = ctx->hz;
    tp.scaled_max_force_d = (double)(0.75f / (float)ctx->hz) * 20.0;
    tp.scaled_max_force = (float)tp.scaled_max_force_d;
    bool grew;
    if (int rc = ctx->d_cp_stats.reserve(16, &grew)) return rc;
    if (grew) PF_CUDA(cudaMemsetAsync(ctx->d_cp_stats, 0, 16 * sizeof(unsigned long long), st));
    tp.stats = ctx->d_cp_stats;
    tp.queue = (unsigned int *)(tp.stats + 8);
    PF_CUDA(cudaMemsetAsync(tp.queue, 0, 4 * sizeof(unsigned int), st));
    PF_CUDA(cudaMemsetAsync(ctx->d_work_count, 0, 4, st));
    {
    pf_prof_scope prof(ctx, st, PF_PROF_COHESION);
    const size_t n1 = std::max<size_t>(ctx->n_agents, 1);
    if (int rc = ctx->d_member_pos.reserve(n1)) return rc;
    if (int rc = ctx->d_cohesion.reserve(n1)) return rc;
    if (int rc = ctx->d_coh_fallback.reserve(n1 + 4)) return rc;
    k_gather_flock_pos<<<((int)ctx->n_agents + 255) / 256, 256, 0, st>>>(ctx->d_records, ctx->d_flock_members, (int)ctx->n_agents,
                                                                        ctx->d_member_pos);
    // big flocks: windowed pass over the position index + full-list fall-back for entities without company; small
    // populations: the full member list directly (the window would cover the whole flock anyway)
    size_t biggest = 0;
    for (size_t f = 0; f + 1 < ctx->h_flock_start.size(); f++) biggest = std::max<size_t>(biggest, ctx->h_flock_start[f + 1] - ctx->h_flock_start[f]);
    const bool windowed = ctx->cohesion_mode == 1 || (ctx->cohesion_mode == 0 && biggest >= 20000);
    if (windowed) {
        uint32_t *d_nfb = ctx->d_coh_fallback + ctx->n_agents;
        PF_CUDA(cudaMemsetAsync(d_nfb, 0, 4, st));
        const int nblk = ((int)ctx->n_agents + COH_THREADS - 1) / COH_THREADS;     // one 128-entry run each: the hardware scheduler balances them
        // fewer runs than ~8 blocks per SM: split every run's window rows over blockIdx.y
        const int nsplit = std::max(1, std::min(8, (ctx->sm_count * 8 + nblk - 1) / nblk));
        if (nsplit > 1)
            if (int rc = ctx->d_coh_part.reserve((size_t)nsplit * ctx->n_agents)) return rc;
        k_cohesion_window<<<dim3(nblk, nsplit), COH_THREADS, 0, st>>>(grid_of(ctx), ctx->d_records, ctx->d_sorted_flock, ctx->d_flock_start,
                                                        (int)ctx->n_agents, (uint32_t)ctx->shard_lo, (uint32_t)ctx->shard_hi,
                                                        tp.scaled_max_force, ctx->d_cohesion, ctx->d_coh_fallback, d_nfb,
                                                        ctx->d_coh_part, nsplit);
        if (nsplit > 1) {
            k_cohesion_finish<<<((int)ctx->n_agents + 127) / 128, 128, 0, st>>>(grid_of(ctx), ctx->d_records, ctx->d_sorted_flock,
                ctx->d_flock_start, (int)ctx->n_agents, (uint32_t)ctx->shard_lo, (uint32_t)ctx->shard_hi, tp.scaled_max_force,
                ctx->d_cohesion, ctx->d_coh_fallback, d_nfb, ctx->d_coh_part, nsplit);
            ctx->launches++;
        }
        // fall-back entities: the grid is sized for the worst case, the kernel reads the count on the device
        const int nown = (int)(ctx->shard_hi - ctx->shard_lo);
        k_cohesion<<<(nown + 127) / 128, 128, 0, st>>>(ctx->d_records, ctx->d_flock_of, ctx->d_flock_start, ctx->d_member_pos,
                                                      ctx->d_coh_fallback, d_nfb, 0, tp.scaled_max_force, ctx->d_cohesion);
        ctx->launches += 2;
    } else {
        k_cohesion<<<(nwork + 127) / 128, 128, 0, st>>>(ctx->d_records, ctx->d_flock_of, ctx->d_flock_start, ctx->d_member_pos,
                                                       ctx->d_work, nullptr, nwork, tp.scaled_max_force, ctx->d_cohesion);
        ctx->launches++;
    }
    }
    const int ctas = std::min((nwork + VEL_WARPS_PER_CTA - 1) / VEL_WARPS_PER_CTA, ctx->sm_count * 8 * 4);
    // per-warp raw neighbour lists for the garrisoned-filter path (find_neighbours, 512 ids each)
    if (ctx->any_garrisoned)
        if (int rc = ctx->d_nb_scratch.reserve((size_t)ctas * VEL_WARPS_PER_CTA * 512)) return rc;
    // Two-phase velocity update while LOS chains are still in flight on the field stream: the part of
    // ClearPath that does not depend on the preferred velocity (neighbours, velocity obstacles, admissible
    // ray intersections) runs now, next to them; only the choice waits for the fields.
    // Policy: splitting costs ~5-30 % extra work (phase B rebuilds the obstacles), so it pays only while the LOS
    // chains outlast a good part of phase A. Both durations are measured on the previous tick. With the level-parallel
    // LOS kernel the C2 cold chain (~1.7 ms) is about half the velocity time, and splitting there still saves ~0.9 ms
    // of a 6 ms step (H100 SXM, 400 W): a quarter of phase A is the bar, not a half.
    if (ctx->vel_timed && cudaEventQuery(ctx->ev_vel1) == cudaSuccess) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, ctx->ev_vel0, ctx->ev_vel1) == cudaSuccess) ctx->last_vel_ms = ms;
    }
    bool worth = true;
    if (ctx->last_los_ms > 0.0f && ctx->last_vel_ms > 0.0f) worth = ctx->last_los_ms > 0.25f * ctx->last_vel_ms;
    bool two_phase = ctx->two_phase && (ctx->two_phase_force ||
                                        (worth && ctx->los_inflight && cudaEventQuery(ctx->ev_los) == cudaErrorNotReady));
    cudaGetLastError();
    PF_CUDA(cudaEventRecord(ctx->ev_vel0, st));
    if (two_phase && ctx->d_prep.reserve((size_t)nwork)) two_phase = false;       // no room: fall back to the single pass
    if (two_phase) {
        pf_prof_scope prof(ctx, st, PF_PROF_VELOCITY);
        // phase A has the whole LOS phase to hide in: a smaller persistent grid leaves the schedulers to the
        // latency-bound LOS threads it shares the SMs with
        const int ctas_a = ctx->phase_a_ctas_per_sm > 0 ? std::min(ctas, ctx->sm_count * ctx->phase_a_ctas_per_sm) : ctas;
        k_agent_velocity<1><<<ctas_a, VEL_WARPS_PER_CTA * 32, VEL_SMEM_BYTES, st>>>(m, grid_of(ctx), tp, ctx->d_agents, ctx->d_records, ctx->d_flocks,
                                                                    ctx->d_work, nwork, ctx->d_vdes_out, ctx->d_los_out,
                                                                    ctx->d_cohesion, ctx->d_vel_out, ctx->d_vpref_out,
                                                                    ctx->any_garrisoned ? 1 : 0, ctx->d_nb_scratch, ctx->d_prep, ctx->d_formation);
        ctx->launches++;
    }
    // everything above is independent of the flow/LOS fields; the LOS chains forked by
    // pfnav_pool_request_goals have been running alongside it
    PF_CUDA(pf_fields_join(ctx, st));
    {
    pf_prof_scope prof(ctx, st, PF_PROF_VDES);
    if (flags & PFNAV_TICK_VDES_FROM_POOL) {
        PF_ARG(ctx->pool.d_slot, "PFNAV_TICK_VDES_FROM_POOL needs a field pool");
        PF_CUDA(pf_pool_refresh(ctx, st));
        const PoolView pv = pool_view(ctx->pool, ctx->pool.d_touch, ctx->tick_no);
        k_desired_velocity<<<(nwork + 127) / 128, 128, 0, st>>>(m, pv, ctx->d_agents, ctx->d_flocks, ctx->d_work, nwork,
                                                               ctx->d_vdes_out, ctx->d_los_out, ctx->d_work_count,
                                                               ctx->d_ms_ext, ctx->d_formation);
    } else {
        k_copy_vdes<<<(nwork + 255) / 256, 256, 0, st>>>(ctx->d_agents, ctx->d_work, nwork, ctx->d_vdes_out, ctx->d_los_out);
    }
    }
    pf_prof_scope prof(ctx, st, PF_PROF_VELOCITY);
    if (two_phase)
        k_agent_velocity<2><<<ctas, VEL_WARPS_PER_CTA * 32, VEL_SMEM_BYTES, st>>>(m, grid_of(ctx), tp, ctx->d_agents, ctx->d_records, ctx->d_flocks,
                                                                    ctx->d_work, nwork, ctx->d_vdes_out, ctx->d_los_out,
                                                                    ctx->d_cohesion, ctx->d_vel_out, ctx->d_vpref_out,
                                                                    ctx->any_garrisoned ? 1 : 0, ctx->d_nb_scratch, ctx->d_prep, ctx->d_formation);
    else
        k_agent_velocity<0><<<ctas, VEL_WARPS_PER_CTA * 32, VEL_SMEM_BYTES, st>>>(m, grid_of(ctx), tp, ctx->d_agents, ctx->d_records, ctx->d_flocks,
                                                                    ctx->d_work, nwork, ctx->d_vdes_out, ctx->d_los_out,
                                                                    ctx->d_cohesion, ctx->d_vel_out, ctx->d_vpref_out,
                                                                    ctx->any_garrisoned ? 1 : 0, ctx->d_nb_scratch, nullptr, ctx->d_formation);
    ctx->launches += 3;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaEventRecord(ctx->ev_vel1, st));
    ctx->vel_timed = true;
    prof.~pf_prof_scope(); prof.a = nullptr;
    PF_CUDA(cudaEventRecord(ctx->tick_done, st));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_read_velocities(pfnav_ctx *ctx, float *out_xz, size_t maxout)
{
    PF_ARG(ctx && out_xz, "null");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaEventSynchronize(ctx->tick_done));
    const size_t n = std::min(maxout, ctx->n_work);
    if (n) PF_CUDA(cudaMemcpy(out_xz, ctx->d_vel_out, n * 8, cudaMemcpyDeviceToHost));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_read_debug(pfnav_ctx *ctx, float *out_vpref_xz, float *out_vdes_xz, uint8_t *out_has_los,
                                       size_t maxout)
{
    PF_ARG(ctx, "null");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaEventSynchronize(ctx->tick_done));
    const size_t n = std::min(maxout, ctx->n_work);
    if (n && out_vpref_xz) PF_CUDA(cudaMemcpy(out_vpref_xz, ctx->d_vpref_out, n * 8, cudaMemcpyDeviceToHost));
    if (n && out_vdes_xz) PF_CUDA(cudaMemcpy(out_vdes_xz, ctx->d_vdes_out, n * 8, cudaMemcpyDeviceToHost));
    if (n && out_has_los) PF_CUDA(cudaMemcpy(out_has_los, ctx->d_los_out, n, cudaMemcpyDeviceToHost));
    return PFNAV_OK;
}

// The queries q[0 .. n) on `st` (validated; n > 0): the count pass, the scan of the answer lengths (and of the garrison
// scratch), one host wait for the offsets and totals, then the write pass into d_eq_ids and the copy of the hits. The
// queries, counts and offsets live in the request staging; the answers in d_eq_ids, whose size the count pass decides.
static int ents_query_run(pfnav_ctx *ctx, cudaStream_t st, const pfnav_ents_query *q, size_t n, uint32_t *out_offsets,
                          uint32_t *out_ids, size_t cap, size_t *out_total)
{
    const int garr = ctx->any_garrisoned ? 1 : 0;
    const auto up16 = [](size_t b) { return (b + 15) & ~(size_t)15; };
    const size_t o_cnt = up16(n * sizeof(pfnav_ents_query)), o_off = o_cnt + up16(n * 4), o_scr = o_off + up16((n + 1) * 4);
    const size_t o_soff = o_scr + (garr ? up16(n * 4) : 0), o_part = o_soff + (garr ? up16((n + 1) * 4) : 0);
    pf_stage S;
    if (int rc = pf_stage_begin(ctx, st, std::max(n * sizeof(pfnav_ents_query), (n + 2) * 4), o_part + 1024 * 4, false, &S))
        return rc;
    memcpy(S.host, q, n * sizeof(pfnav_ents_query));
    if (int rc = pf_stage_upload(ctx, st, S, n * sizeof(pfnav_ents_query))) return rc;
    const pfnav_ents_query *d_q = (const pfnav_ents_query *)S.dev;
    uint32_t *d_cnt = (uint32_t *)(S.dev + o_cnt), *d_off = (uint32_t *)(S.dev + o_off), *d_part = (uint32_t *)(S.dev + o_part);
    uint32_t *d_scr = garr ? (uint32_t *)(S.dev + o_scr) : nullptr, *d_soff = garr ? (uint32_t *)(S.dev + o_soff) : nullptr;
    const GridView g = grid_of(ctx);
    const unsigned grid = (unsigned)((n + EQ_WARPS - 1) / EQ_WARPS);
    k_ents_count<<<grid, EQ_WARPS * 32, 0, st>>>(g, ctx->d_records, d_q, (int)n, garr, d_cnt, d_scr);
    ctx->launches++;
    excl_scan(ctx, d_cnt, d_part, d_off, (int)n, st);
    if (garr) excl_scan(ctx, d_scr, d_part, d_soff, (int)n, st);
    PF_CUDA(cudaGetLastError());
    // the offsets and the scratch total come back through the pinned buffer: the one host wait
    uint32_t *h = (uint32_t *)S.host;
    PF_CUDA(cudaMemcpyAsync(h, d_off, (n + 1) * 4, cudaMemcpyDeviceToHost, st));
    if (garr) PF_CUDA(cudaMemcpyAsync(h + n + 1, d_soff + n, 4, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    const size_t total = h[n], scr_total = garr ? h[n + 1] : 0;
    memcpy(out_offsets, h, (n + 1) * 4);
    *out_total = total;
    if (total > cap) {
        if (int rc = pf_stage_done(ctx, st)) return rc;
        pfnav_set_error("pfnav_ents_in_circles: the answers hold %zu uids, out_ids %zu", total, cap);
        return PFNAV_ERR_NOMEM;
    }
    if (total > 0) {
        if (int rc = ctx->d_eq_ids.reserve(total + scr_total)) return rc;
        k_ents_write<<<grid, EQ_WARPS * 32, 0, st>>>(g, ctx->d_records, d_q, (int)n, d_off, d_soff, ctx->d_eq_ids,
                                                     ctx->d_eq_ids + total);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
        PF_CUDA(cudaMemcpyAsync(out_ids, ctx->d_eq_ids, total * 4, cudaMemcpyDeviceToHost, st));
    }
    if (int rc = pf_stage_done(ctx, st)) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

extern "C" int pfnav_ents_in_circle(pfnav_ctx *ctx, float x, float z, float range, uint32_t *out, int maxout, int *out_n)
{
    PF_ARG(ctx && ctx->d_records && out && out_n && maxout > 0, "args");
    PF_CUDA(cudaSetDevice(ctx->device));
    if (range < 0.0f) { *out_n = 0; return PFNAV_OK; }
    const pfnav_ents_query q = {x, z, range, PFNAV_NULL_UID, maxout, 0u};
    uint32_t off[2];
    size_t total = 0;
    if (int rc = ents_query_run(ctx, ctx->tick_stream, &q, 1, off, out, (size_t)maxout, &total)) return rc;
    *out_n = (int)total;
    return PFNAV_OK;
}

extern "C" int pfnav_ents_in_circles(pfnav_ctx *ctx, const pfnav_ents_query *q, size_t n, uint32_t *out_offsets,
                                     uint32_t *out_ids, size_t cap, size_t *out_total, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_records, "agents not uploaded");
    PF_ARG(n == 0 || (q && out_offsets && out_total), "null argument");
    PF_ARG(cap == 0 || out_ids, "out_ids == NULL with cap > 0");
    PF_ARG(n <= 0x7fffffff, "n");
    uint64_t bound = 0;
    for (size_t i = 0; i < n; i++) {
        const pfnav_ents_query &a = q[i];
        PF_ARG(isfinite(a.x) && isfinite(a.z) && isfinite(a.range), "query x, z and range must be finite");
        PF_ARG(a.maxout >= 0, "query maxout < 0");
        PF_ARG(a.uid == PFNAV_NULL_UID || a.uid < ctx->n_agents, "query uid outside the population");
        if (a.range >= 0.0f) bound += std::min<uint64_t>((uint64_t)a.maxout, ctx->n_agents);
    }
    PF_ARG(bound <= 0xffffffffull, "the answers could exceed 2^32 uids");
    if (ctx->index_stale) {
        pfnav_set_error("pfnav_ents_in_circles: records were written after the last index build (pfnav_agents_rebuild_index "
                        "or a gather first)");
        return PFNAV_ERR_STATE;
    }
    if (n == 0) {
        if (out_offsets) out_offsets[0] = 0;
        if (out_total) *out_total = 0;
        return PFNAV_OK;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    return ents_query_run(ctx, pf_stream(ctx, stream), q, n, out_offsets, out_ids, cap, out_total);
}


// ------------------------------------------------------------------------------------------
// State update: entity_compute_update (movement.c:2303-2650) + the movestate part of
// entity_apply_update (movement.c:2693-2757). One thread per work item.
// The quaternion helpers keep the reference's mix of float and double arithmetic (pf_math.c).
// ------------------------------------------------------------------------------------------
struct quat { float x, y, z, w; };

#define PF_PI_D 3.14159265358979323846

// first column of PFM_Mat4x4_RotFromQuat (pf_math.c:324) applied to (1,0,0,1) by PFM_Quat_PitchDiff (:677)
__device__ __forceinline__ void quat_front(const quat &q, float &dx, float &dz)
{
    dx = (float)(1 - 2 * ((double)q.y * (double)q.y) - 2 * ((double)q.z * (double)q.z));   // pow(y,2) is exact y*y in double
    dz = 2 * q.x * q.z + 2 * q.w * q.y;
    // dir_homo.w == 1; the zero products of PFM_Mat4x4_Mult4x1 add nothing for finite inputs
}

// PFM_Quat_PitchDiff (pf_math.c:677-704)
__device__ __forceinline__ float quat_pitch_diff(const quat &a, const quat &b)
{
    float ax, az, bx, bz;
    quat_front(a, ax, az);
    quat_front(b, bx, bz);
    const float dot = ax * bx + az * bz;
    const float det = ax * bz - az * bx;
    return (float)atan2((double)det, (double)dot);
}

// dir_quat_from_velocity (movement.c:1411)
__device__ __forceinline__ quat dir_quat_from_velocity(v2 v)
{
    const float angle_rad = (float)(atan2((double)v.z, (double)v.x) - PF_PI_D / 2.0f);
    quat q;
    q.x = 0.0f; q.z = 0.0f;
    q.y = (float)(1.0f * sin((double)(angle_rad / 2.0f)));
    q.w = (float)cos((double)(angle_rad / 2.0f));
    return q;
}

// turn_toward (movement.c:2249): PFM_Mat4x4_MakeRotY -> PFM_Quat_FromRotMat -> MultQuat -> Normal
__device__ quat turn_toward(const quat &cur, const quat &target, float max_deg)
{
    float angle_deg = (float)((double)quat_pitch_diff(cur, target) * (180.0f / PF_PI_D));
    if (180.0f - fabs((double)angle_deg) < 1.0f) angle_deg = 180.0f;
    const double mn = ((double)max_deg < fabs((double)angle_deg)) ? (double)max_deg : fabs((double)angle_deg);
    const int sg = (angle_deg > 0) - (angle_deg < 0);
    const float turn_deg = (float)(mn * -sg);
    const float radians = (float)((double)turn_deg * (PF_PI_D / 180.0f));
    const float c = (float)cos((double)radians), sn = (float)sin((double)radians);
    // rotation matrix about Y: cols[0][0] = c, cols[0][2] = -s, cols[2][0] = s, cols[2][2] = c, cols[1][1] = 1
    const float m00 = c, m02 = -sn, m20 = sn, m22 = c, m11 = 1.0f;
    quat rot;
    const float tr = m00 + m11 + m22;
    if (tr > 0) {
        const float S = (float)(sqrt((double)tr + 1.0) * 2);
        rot.w = (float)(0.25 * (double)S);
        rot.x = (0.0f - 0.0f) / S;
        rot.y = (m02 - m20) / S;
        rot.z = (0.0f - 0.0f) / S;
    } else if ((m00 > m11) && (m00 > m22)) {
        const float S = (float)(sqrt(1.0 + (double)m00 - (double)m11 - (double)m22) * 2);
        rot.w = (0.0f - 0.0f) / S; rot.x = (float)(0.25 * (double)S); rot.y = (0.0f + 0.0f) / S; rot.z = (m02 + m20) / S;
    } else if (m11 > m22) {
        const float S = (float)(sqrt(1.0 + (double)m11 - (double)m00 - (double)m22) * 2);
        rot.w = (m02 - m20) / S; rot.x = (0.0f + 0.0f) / S; rot.y = (float)(0.25 * (double)S); rot.z = (0.0f + 0.0f) / S;
    } else {
        const float S = (float)(sqrt(1.0 + (double)m22 - (double)m00 - (double)m11) * 2);
        rot.w = (0.0f - 0.0f) / S; rot.x = (m02 + m20) / S; rot.y = (0.0f + 0.0f) / S; rot.z = (float)(0.25 * (double)S);
    }
    // PFM_Quat_MultQuat(&rot, &cur) (pf_math.c:639)
    quat f;
    f.x = ( rot.x * cur.w) + (rot.y * cur.z) - (rot.z * cur.y) + (rot.w * cur.x);
    f.y = (-rot.x * cur.z) + (rot.y * cur.w) + (rot.z * cur.x) + (rot.w * cur.y);
    f.z = ( rot.x * cur.y) - (rot.y * cur.x) + (rot.z * cur.w) + (rot.w * cur.z);
    f.w = (-rot.x * cur.x) - (rot.y * cur.y) - (rot.z * cur.z) + (rot.w * cur.w);
    const float len = (float)sqrt((double)(f.x * f.x + f.y * f.y + f.z * f.z + f.w * f.w));
    f.x = f.x / len; f.y = f.y / len; f.z = f.z / len; f.w = f.w / len;
    return f;
}

struct UpdateParams { int hz; float turn_rate; float adj_query_r; };

__global__ void __launch_bounds__(128)
k_entity_update(MapView m, GridView g, UpdateParams up, const pfnav_agent *__restrict__ agents,
                const pf_record *__restrict__ rec, const pfnav_movestate *__restrict__ mss,
                const pfnav_flock *__restrict__ flocks, const pf_arrival_dev *__restrict__ arr,
                const float2 *__restrict__ mc_tiles, int nlayers, const uint32_t *__restrict__ work, int nwork,
                const float2 *__restrict__ vel_in, const float2 *__restrict__ vdes_in, pfnav_patch *__restrict__ out,
                const int32_t *__restrict__ flock_of, const pfnav_movestate_ext *__restrict__ exts,
                const pfnav_formation_in *__restrict__ forms, pf_enter_cand *__restrict__ cands,
                uint32_t *__restrict__ cand_count)
{
    const int wi = blockIdx.x * blockDim.x + threadIdx.x;
    if (wi >= nwork) return;
    const uint32_t uid = work[wi];
    const pfnav_agent a = agents[uid];
    const pfnav_movestate ms = mss[uid];
    const float EPS = 1.0f / 1024;
    pfnav_patch p;
    memset(&p, 0, sizeof(p));
    p.next_state = -1;
    p.wait_ticks_left = exts ? exts[uid].wait_ticks_left : 0;
    const quat ms_rot = {ms.next_rot[0], ms.next_rot[1], ms.next_rot[2], ms.next_rot[3]};
    v2 new_vel = {vel_in[wi].x, vel_in[wi].y};
    const v2 vdes = {vdes_in[wi].x, vdes_in[wi].y};
    const v2 ms_vel = {a.velocity[0], a.velocity[1]};
    const v2 curr_xz = {a.pos[0], a.pos[1]};
    const uint32_t state = a.state;

    // flush an unfinished interpolation (movement.c:2311)
    if (ms.left > 0) {
        p.flags |= PFNAV_UPDATE_SET_POSITION | PFNAV_UPDATE_SET_ROTATION | PFNAV_UPDATE_SET_LEFT;
        p.next_pos[0] = ms.next_pos[0]; p.next_pos[1] = ms.next_pos[1]; p.next_pos[2] = ms.next_pos[2];
        p.next_rot[0] = ms_rot.x; p.next_rot[1] = ms_rot.y; p.next_rot[2] = ms_rot.z; p.next_rot[3] = ms_rot.w;
        p.next_left = 0;
    }
    // heading gate (movement.c:2323-2335)
    bool turn_to_move = false;
    quat travel_dir = ms_rot;
    const bool gated = state == PFNAV_STATE_MOVING || state == PFNAV_STATE_SEEK_ENEMIES ||
                       state == PFNAV_STATE_SURROUND_ENTITY || state == PFNAV_STATE_ENTER_ENTITY_RANGE;
    if (v2_len(new_vel) > EPS && gated) {
        travel_dir = dir_quat_from_velocity(v2_len(vdes) > EPS ? vdes : new_vel);
        const float heading_err = (float)fabs((double)quat_pitch_diff(ms_rot, travel_dir) * (180.0f / PF_PI_D));
        const float tolerance = (v2_len(ms_vel) > EPS) ? 90.0f : 10.0f;
        if (heading_err > tolerance) { turn_to_move = true; new_vel = {0.0f, 0.0f}; }
    }
    v2 new_pos_xz = v2_add(curr_xz, new_vel);
    const int layer = nav_layer_for(a.flags, a.radius);
    const bool still = state == PFNAV_STATE_ARRIVED || state == PFNAV_STATE_WAITING;
    if (a.flags & PFNAV_FLAG_GARRISONED) {
        if (!still) { p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_ARRIVED; p.next_block = 0; }
        out[wi] = p;
        return;
    }
    bool dummy, on_blocked, np_path, np_blocked;
    probe_tile(m, layer, curr_xz.x, curr_xz.z, dummy, on_blocked);
    probe_tile(m, layer, new_pos_xz.x, new_pos_xz.z, np_path, np_blocked);
    const float turn_rate = up.turn_rate;
    if (v2_len(new_vel) > 0 && np_path && (on_blocked || !np_blocked)) {
        // unit_height (movement.c:2198) with M_HeightAtPoint == 0: terrain height is render state
        const float y = (a.flags & PFNAV_FLAG_WATER) ? 0.0f : (a.flags & PFNAV_FLAG_AIR) ? 20.0f : 0.0f  /* AIR_UNIT_HEIGHT, game.h:50 */;
        p.flags |= PFNAV_UPDATE_SET_PREV_POS | PFNAV_UPDATE_SET_NEXT_POS | PFNAV_UPDATE_SET_STEP | PFNAV_UPDATE_SET_LEFT;
        p.next_ppos[0] = ms.next_pos[0]; p.next_ppos[1] = ms.next_pos[1]; p.next_ppos[2] = ms.next_pos[2];
        p.next_npos[0] = new_pos_xz.x; p.next_npos[1] = y; p.next_npos[2] = new_pos_xz.z;
        p.next_step = 1.0f / (20 / up.hz);
        p.next_left = (float)((20 / up.hz) - 1);
        p.flags |= PFNAV_UPDATE_SET_POSITION;
        if ((20 / up.hz) - 1 == 0) {
            p.next_pos[0] = new_pos_xz.x; p.next_pos[1] = y; p.next_pos[2] = new_pos_xz.z;
        } else {
            // interpolate_positions(next_ppos, next_npos, ms->step) (movement.c:2221)
            float ix, iy, iz;
            if (fabs(1.0 - (double)ms.step) < EPS) { ix = p.next_npos[0]; iy = p.next_npos[1]; iz = p.next_npos[2]; }
            else {
                ix = p.next_ppos[0] + (p.next_npos[0] - p.next_ppos[0]) * ms.step;
                iy = p.next_ppos[1] + (p.next_npos[1] - p.next_ppos[1]) * ms.step;
                iz = p.next_ppos[2] + (p.next_npos[2] - p.next_ppos[2]) * ms.step;
            }
            new_pos_xz = {ix, iz};
            p.next_pos[0] = ix; p.next_pos[1] = iy; p.next_pos[2] = iz;
        }
        p.flags |= PFNAV_UPDATE_SET_VELOCITY;
        p.next_velocity[0] = new_vel.x; p.next_velocity[1] = new_vel.z;
        p.flags |= PFNAV_UPDATE_SET_PREV_ROT | PFNAV_UPDATE_SET_NEXT_ROT | PFNAV_UPDATE_SET_ROTATION;
        p.next_prot[0] = ms_rot.x; p.next_prot[1] = ms_rot.y; p.next_prot[2] = ms_rot.z; p.next_prot[3] = ms_rot.w;
        // orient_to_velocity_history (movement.c:2291) over vel_wma (movement.c:2067)
        v2 wma = {0.0f, 0.0f};
        float denom = 0.0f;
        for (int i = 0; i < PFNAV_VEL_HIST_LEN; i++) {
            const int k = (ms.vel_hist_idx + i) % PFNAV_VEL_HIST_LEN;
            const float wgt = (float)(PFNAV_VEL_HIST_LEN - i);
            wma.x = wma.x + ms.vel_hist[k][0] * wgt;
            wma.z = wma.z + ms.vel_hist[k][1] * wgt;
            denom += wgt;
        }
        if (denom > EPS) { const float inv = 1.0f / denom; wma.x = wma.x * inv; wma.z = wma.z * inv; }
        quat nrot = ms_rot;
        if (v2_len(wma) > EPS) nrot = turn_toward(ms_rot, dir_quat_from_velocity(wma), turn_rate);
        p.next_nrot[0] = nrot.x; p.next_nrot[1] = nrot.y; p.next_nrot[2] = nrot.z; p.next_nrot[3] = nrot.w;
        p.next_rot[0] = ms_rot.x; p.next_rot[1] = ms_rot.y; p.next_rot[2] = ms_rot.z; p.next_rot[3] = ms_rot.w;
    } else {
        p.flags |= PFNAV_UPDATE_SET_VELOCITY;
        p.next_velocity[0] = 0.0f; p.next_velocity[1] = 0.0f;
        const bool held = a.flags & PFNAV_FLAG_COMBAT_HELD;
        if (held || turn_to_move) {
            p.flags |= PFNAV_UPDATE_SET_PREV_ROT | PFNAV_UPDATE_SET_NEXT_ROT | PFNAV_UPDATE_SET_ROTATION |
                       PFNAV_UPDATE_TURNING_IN_PLACE;
            const quat tgt = held ? quat{ms.combat_facing[0], ms.combat_facing[1], ms.combat_facing[2], ms.combat_facing[3]}
                                  : travel_dir;
            const quat nrot = turn_toward(ms_rot, tgt, turn_rate);
            p.next_prot[0] = ms_rot.x; p.next_prot[1] = ms_rot.y; p.next_prot[2] = ms_rot.z; p.next_prot[3] = ms_rot.w;
            p.next_nrot[0] = nrot.x; p.next_nrot[1] = nrot.y; p.next_nrot[2] = nrot.z; p.next_nrot[3] = nrot.w;
            p.next_rot[0] = ms_rot.x; p.next_rot[1] = ms_rot.y; p.next_rot[2] = ms_rot.z; p.next_rot[3] = ms_rot.w;
        }
    }
    // stuck on non-pathable terrain: keep the state (movement.c:2417)
    bool cur_path, cur_blk;
    probe_tile(m, layer, new_pos_xz.x, new_pos_xz.z, cur_path, cur_blk);
    if (!cur_path) { out[wi] = p; return; }
    pfnav_movestate_ext ex;
    if (exts) ex = exts[uid];
    else { memset(&ex, 0, sizeof(ex)); ex.surround_target_uid = PFNAV_NULL_UID; ex.rot[3] = 1.0f; }
    p.wait_ticks_left = ex.wait_ticks_left;
    uint32_t fflags = 0;
    pfnav_formation_in fin;
    if (forms) { fin = forms[uid]; fflags = fin.flags; }
    const bool has_fid = fflags & PFNAV_FORM_HAS_FORMATION;

    switch (state) {
    case PFNAV_STATE_MOVING:
    case PFNAV_STATE_MOVING_IN_FORMATION: {
        // movement.c:2424-2500 (no arrival group: G_ArrivalGroup_ForLayer is the f-1 consumer, inactive here)
        if (has_fid && !(fflags & PFNAV_FORM_ASSIGNMENT_READY)) break;
        if (has_fid && (fflags & PFNAV_FORM_ASSIGNED_TO_CELL) && (fflags & PFNAV_FORM_IN_RANGE_OF_CELL)) {
            p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_ARRIVING_TO_CELL;
            break;
        }
        if (a.flock < 0) break;
        const pfnav_flock fl = flocks[a.flock];
        const pf_arrival_dev ac = arr[(size_t)a.flock * nlayers + layer];
        bool arrived = false;
        {   // arrived() (movement.c:2170)
            const v2 tgt = {fl.target[0], fl.target[1]};
            const float thresh = a.radius * 1.5f;
            if (v2_len(v2_sub(tgt, new_pos_xz)) < thresh) arrived = true;
            if (!arrived) {
                // N_IsAdjacentToImpassable (nav.c:4745) && N_IsMaximallyClose (nav.c:4707)
                tile_desc td;
                bool adj = false;
                if (desc_for_point(m, new_pos_xz.x, new_pos_xz.z, td)) {
                    const int ar = td.chunk_r * 64 + td.tile_r, acol = td.chunk_c * 64 + td.tile_c;
                    const int dr[4] = {-1, 0, 0, 1}, dc[4] = {0, -1, 1, 0};
                    for (int e = 0; e < 4 && !adj; e++) {
                        const int nr = ar + dr[e], nc = acol + dc[e];
                        if (nr < 0 || nr >= m.H64 || nc < 0 || nc >= m.W64) continue;
                        adj = tile_blocked_abs(m, layer, nr, nc);
                    }
                }
                if (adj) {
                    for (int i = 0; i < ac.mc_n && !arrived; i++) {
                        const float2 tc = mc_tiles[ac.mc_off + i];
                        const v2 d = {tc.x - new_pos_xz.x, tc.y - new_pos_xz.z};
                        if (v2_len(d) <= thresh) arrived = true;
                    }
                }
            }
            if (!arrived && ac.nearest_ok) {
                const v2 d = {ac.nearest[0] - new_pos_xz.x, ac.nearest[1] - new_pos_xz.z};
                if (v2_len(d) < thresh) arrived = true;
            }
        }
        if (!arrived) {
            // adjacent_flock_members (movement.c:953): any flock member within r + r' + ADJACENCY_SEP_DIST that has
            // ARRIVED. The spatial index pre-selects (radius r + max radius + 5 plus slack); the test itself is
            // the reference's float comparison, so the outcome does not depend on the pre-selection.
            const int32_t icx = bg_scale(curr_xz.x), icy = bg_scale(curr_xz.z), ir = bg_scale(a.radius + up.adj_query_r);
            const int cx_lo = max((icx - ir - g.origin_x) >> 12, 0), cx_hi = min((icx + ir - g.origin_x) >> 12, g.grid_w - 1);
            const int cy_lo = max((icy - ir - g.origin_y) >> 12, 0), cy_hi = min((icy + ir - g.origin_y) >> 12, g.grid_h - 1);
            for (int cy = cy_lo; cy <= cy_hi && !arrived; cy++)
                for (int cx = cx_lo; cx <= cx_hi && !arrived; cx++) {
                    const int c = cy * g.grid_w + cx;
                    const uint32_t b = g.cell_start[c], cnt = g.cell_count[c];
                    for (uint32_t k = 0; k < cnt; k++) {
                        const uint32_t o = g.id[b + k];
                        if (o == uid) continue;
                        const pf_record r = rec[o];
                        if ((r.state_flags >> 24) != PFNAV_STATE_ARRIVED) continue;
                        if (flock_of[o] != a.flock) continue;
                        const v2 d = {curr_xz.x - r.px, curr_xz.z - r.pz};
                        if (v2_len(d) <= a.radius + r.radius + 5.0f) { arrived = true; break; }
                    }
                }
        }
        if (arrived) {
            p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_ARRIVED; p.next_block = 1;
        } else if (v2_len(vdes) < EPS) {
            p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_WAITING; p.next_block = 1;
        }
        break;
    }
    case PFNAV_STATE_SEEK_ENEMIES:
        break;                              // stays a soft obstacle and retries next tick (movement.c:2501)
    case PFNAV_STATE_SURROUND_ENTITY:
        if (ex.surround_target_uid == PFNAV_NULL_UID) {
            p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_ARRIVED; p.next_block = 1;
        } else p.engine_todo |= PFNAV_TODO_SURROUND_QUERY;
        break;
    case PFNAV_STATE_ENTER_ENTITY_RANGE: {
        // movement.c:2569-2603
        if (ex.surround_target_uid == PFNAV_NULL_UID) {
            p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_ARRIVED; p.next_block = 1;
            break;
        }
        const pf_record tr = rec[ex.surround_target_uid];
        const v2 xz_target = {tr.px, tr.pz};
        const v2 delta = v2_sub(new_pos_xz, xz_target);
        const bool stop = v2_len(delta) <= ex.target_range;
        if (!stop) {
            // M_NavIsAdjacentToImpassable(new_pos) && M_NavIsMaximallyClose(new_pos, target, 0): the list of the target's
            // tiles is searched after this kernel (pf_enter_range_search), which also ends the update of such an item
            tile_desc td;
            bool adj = false;
            if (desc_for_point(m, new_pos_xz.x, new_pos_xz.z, td)) {
                const int ar = td.chunk_r * 64 + td.tile_r, acol = td.chunk_c * 64 + td.tile_c;
                const int dr[4] = {-1, 0, 0, 1}, dc[4] = {0, -1, 1, 0};
                for (int e = 0; e < 4 && !adj; e++) {
                    const int nr = ar + dr[e], nc = acol + dc[e];
                    if (nr < 0 || nr >= m.H64 || nc < 0 || nc >= m.W64) continue;
                    adj = tile_blocked_abs(m, layer, nr, nc);
                }
            }
            if (adj) {
                // warp-aggregated append: one atomic per warp
                const unsigned act = __activemask();
                const int lane = threadIdx.x & 31, leader = __ffs(act) - 1;
                uint32_t k = 0;
                if (lane == leader) k = atomicAdd(cand_count, (uint32_t)__popc(act));
                k = __shfl_sync(act, k, leader) + __popc(act & ((1u << lane) - 1u));
                cands[k] = {(uint32_t)wi, layer, new_pos_xz.x, new_pos_xz.z, xz_target.x, xz_target.z,
                            ex.target_prev_pos[0], ex.target_prev_pos[1]};
                break;
            }
        }
        pf_enter_range_tail(p, stop, xz_target.x, xz_target.z, ex.target_prev_pos[0], ex.target_prev_pos[1]);
        break;
    }
    case PFNAV_STATE_TURNING: {
        // movement.c:2605-2627
        const quat ent_rot = {ex.rot[0], ex.rot[1], ex.rot[2], ex.rot[3]};
        const quat tdir = {ex.target_dir[0], ex.target_dir[1], ex.target_dir[2], ex.target_dir[3]};
        const float degrees = (float)((double)quat_pitch_diff(ent_rot, tdir) * (180.0f / PF_PI_D));
        if (fabs((double)degrees) <= 5.0f) {
            p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_ARRIVED; p.next_block = 1;
            break;
        }
        const quat fin_rot = turn_toward(ent_rot, tdir, turn_rate);
        p.flags |= PFNAV_UPDATE_SET_ROTATION | PFNAV_UPDATE_SET_PREV_ROT;
        p.next_rot[0] = fin_rot.x; p.next_rot[1] = fin_rot.y; p.next_rot[2] = fin_rot.z; p.next_rot[3] = fin_rot.w;
        p.next_prot[0] = fin_rot.x; p.next_prot[1] = fin_rot.y; p.next_prot[2] = fin_rot.z; p.next_prot[3] = fin_rot.w;
        break;
    }
    case PFNAV_STATE_WAITING:
        // movement.c:2630-2645: the countdown lives in the movestate itself
        p.wait_ticks_left = ex.wait_ticks_left - 1;
        if (p.wait_ticks_left == 0) { p.flags |= PFNAV_UPDATE_SET_MOVING; p.next_state = ex.wait_prev; }
        break;
    case PFNAV_STATE_ARRIVED:
        break;
    case PFNAV_STATE_ARRIVING_TO_CELL:
        // movement.c:2648-2670
        if (!has_fid) { p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_MOVING; break; }
        if (!(fflags & PFNAV_FORM_ASSIGNMENT_READY)) break;
        if (!(fflags & PFNAV_FORM_IN_RANGE_OF_CELL)) { p.flags |= PFNAV_UPDATE_SET_STATE; p.next_state = PFNAV_STATE_MOVING_IN_FORMATION; break; }
        if (fflags & PFNAV_FORM_ARRIVED_AT_CELL) {
            p.flags |= PFNAV_UPDATE_SET_STATE | PFNAV_UPDATE_SET_TARGET_DIR; p.next_state = PFNAV_STATE_TURNING;
            for (int i = 0; i < 4; i++) p.next_target_dir[i] = fin.target_orientation[i];
        }
        break;
    default:
        break;
    }
    {   // ent_update_using_surround_field (movement.c:2672-2691) runs at the end of the apply on the tick's snapshot
        // positions; it is evaluated here, where the snapshot is still intact, and carried in the patch
        const uint32_t after = (p.flags & (PFNAV_UPDATE_SET_STATE | PFNAV_UPDATE_SET_MOVING)) ? (uint32_t)p.next_state : state;
        if (after == PFNAV_STATE_SURROUND_ENTITY && ex.surround_target_uid != PFNAV_NULL_UID) {
            const pf_record tr = rec[ex.surround_target_uid];
            const float dx = (float)fabs((double)(tr.px - curr_xz.x)), dz = (float)fabs((double)(tr.pz - curr_xz.z));
            const float low = (float)(256.0 / 3.0f), high = (float)(256.0 / 2.0f);       // CHUNK_WIDTH / 3, / 2 (movement.c:440-443)
            if (!ex.using_surround_field) { if (dx < low && dz < low) p.engine_todo |= PFNAV_TODO_USE_SURROUND_FIELD; }
            else if (dx >= high || dz >= high) p.engine_todo |= PFNAV_TODO_DROP_SURROUND_FIELD;
        }
    }
    out[wi] = p;
}

// entity_apply_update (movement.c:2693-2757), movestate fields only
__global__ void k_entity_apply(pfnav_agent *__restrict__ agents, pfnav_movestate *__restrict__ mss,
                               pf_record *__restrict__ rec, const uint32_t *__restrict__ work, int nwork,
                               const pfnav_patch *__restrict__ patches, pfnav_movestate_ext *__restrict__ exts)
{
    const int wi = blockIdx.x * blockDim.x + threadIdx.x;
    if (wi >= nwork) return;
    const uint32_t uid = work[wi];
    const pfnav_patch p = patches[wi];
    pfnav_agent a = agents[uid];
    pfnav_movestate ms = mss[uid];
    const float EPS = 1.0f / 1024;
    if (a.flags & PFNAV_FLAG_GARRISONED) return;
    pfnav_movestate_ext ex;
    if (exts) { ex = exts[uid]; ex.wait_ticks_left = p.wait_ticks_left; }      // the countdown of STATE_WAITING (movement.c:2633)
    if (p.flags & PFNAV_UPDATE_SET_STATE) {
        if (p.next_state == PFNAV_STATE_ARRIVED || p.next_state == PFNAV_STATE_WAITING) {
            // entity_finish_moving (movement.c:685): blockers / events / combat stance stay with the engine
            if (exts && p.next_state == PFNAV_STATE_WAITING) { ex.wait_prev = (int32_t)a.state; ex.wait_ticks_left = 60; }     // WAIT_TICKS
            a.velocity[0] = 0.0f; a.velocity[1] = 0.0f;
        }
        a.state = (uint32_t)p.next_state;
    }
    if (p.flags & PFNAV_UPDATE_SET_VELOCITY) {
        a.velocity[0] = p.next_velocity[0]; a.velocity[1] = p.next_velocity[1];
        if (p.flags & PFNAV_UPDATE_TURNING_IN_PLACE) {
            for (int i = 0; i < PFNAV_VEL_HIST_LEN; i++) { ms.vel_hist[i][0] = 0.0f; ms.vel_hist[i][1] = 0.0f; }
        } else {
            bool empty = true;
            for (int i = 0; i < PFNAV_VEL_HIST_LEN; i++)
                if (sqrtf(ms.vel_hist[i][0] * ms.vel_hist[i][0] + ms.vel_hist[i][1] * ms.vel_hist[i][1]) > EPS) empty = false;
            const float vl = sqrtf(a.velocity[0] * a.velocity[0] + a.velocity[1] * a.velocity[1]);
            if (empty && vl > EPS) {
                // seed_vel_hist_facing (movement.c:2046) / facing_dir (:2040)
                const float theta = (float)(2.0 * atan2((double)ms.next_rot[1], (double)ms.next_rot[3]));
                const float dx = (float)(-sin((double)theta)), dz = (float)cos((double)theta);
                for (int i = 0; i < PFNAV_VEL_HIST_LEN; i++) { ms.vel_hist[i][0] = dx * vl; ms.vel_hist[i][1] = dz * vl; }
            }
            ms.vel_hist[ms.vel_hist_idx][0] = a.velocity[0]; ms.vel_hist[ms.vel_hist_idx][1] = a.velocity[1];
            ms.vel_hist_idx = (ms.vel_hist_idx + 1) % PFNAV_VEL_HIST_LEN;
        }
    }
    if (p.flags & PFNAV_UPDATE_SET_POSITION) { a.pos[0] = p.next_pos[0]; a.pos[1] = p.next_pos[2]; }
    if (p.flags & PFNAV_UPDATE_SET_PREV_POS) { a.prev_pos[0] = p.next_ppos[0]; a.prev_pos[1] = p.next_ppos[2]; }
    if (p.flags & PFNAV_UPDATE_SET_NEXT_POS) { ms.next_pos[0] = p.next_npos[0]; ms.next_pos[1] = p.next_npos[1]; ms.next_pos[2] = p.next_npos[2]; }
    if (p.flags & PFNAV_UPDATE_SET_STEP) ms.step = p.next_step;
    if (p.flags & PFNAV_UPDATE_SET_LEFT) ms.left = (int)p.next_left;
    if (p.flags & PFNAV_UPDATE_SET_NEXT_ROT) { ms.next_rot[0] = p.next_nrot[0]; ms.next_rot[1] = p.next_nrot[1]; ms.next_rot[2] = p.next_nrot[2]; ms.next_rot[3] = p.next_nrot[3]; }
    if (exts) {
        if (p.flags & PFNAV_UPDATE_SET_ROTATION) { ex.rot[0] = p.next_rot[0]; ex.rot[1] = p.next_rot[1]; ex.rot[2] = p.next_rot[2]; ex.rot[3] = p.next_rot[3]; }   // Entity_SetRot
        if (p.flags & PFNAV_UPDATE_SET_TARGET_PREV) { ex.target_prev_pos[0] = p.next_target_prev[0]; ex.target_prev_pos[1] = p.next_target_prev[1]; }
        if (p.flags & PFNAV_UPDATE_SET_TARGET_DIR) { ex.target_dir[0] = p.next_target_dir[0]; ex.target_dir[1] = p.next_target_dir[1]; ex.target_dir[2] = p.next_target_dir[2]; ex.target_dir[3] = p.next_target_dir[3]; }
    }
    if (p.flags & PFNAV_UPDATE_SET_MOVING) {
        // movement.c:2750-2755: entity_unblock is the engine's; move_notify_motion_start wipes the velocity history
        if (!(a.flags & PFNAV_FLAG_COMBAT_HELD))
            for (int i = 0; i < PFNAV_VEL_HIST_LEN; i++) { ms.vel_hist[i][0] = 0.0f; ms.vel_hist[i][1] = 0.0f; }
        a.state = (uint32_t)p.next_state;
    }
    if (exts && a.state == PFNAV_STATE_SURROUND_ENTITY) {
        // ent_update_using_surround_field (movement.c:2672), decided by the update pass on the tick's snapshot positions
        if (p.engine_todo & PFNAV_TODO_USE_SURROUND_FIELD) ex.using_surround_field = 1;
        if (p.engine_todo & PFNAV_TODO_DROP_SURROUND_FIELD) ex.using_surround_field = 0;
    }
    if (exts) exts[uid] = ex;
    agents[uid] = a;
    mss[uid] = ms;
    pf_record r;
    r.px = a.pos[0]; r.pz = a.pos[1]; r.vx = a.velocity[0]; r.vz = a.velocity[1];
    r.radius = a.radius;
    r.state_flags = (a.state << 24) | (a.flags & 0xFFFFFFu);
    rec[uid] = r;
}

// the block's narrow | wide << 32 op count of a producer of pf_blocker_ops_append, written by thread 0 to s.bsum
__device__ __forceinline__ void ops_block_sum(unsigned desc, unsigned nops, const pf_op_stage &s)
{
    __shared__ unsigned long long part[PF_OPS_BLOCK / 32];
    const unsigned nwide = ((desc >> 2) & 1u) + ((desc >> 3) & 1u);
    unsigned long long v = (unsigned long long)(nops - nwide) | (unsigned long long)nwide << 32;
    for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xFFFFFFFFu, v, o);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int w = 0; w < PF_OPS_BLOCK / 32; w++) t += part[w];
        s.bsum[blockIdx.x] = t;
    }
}

// entity_block / entity_unblock (movement.c:560-600) per item, staged for pf_blocker_ops_append: ops[2i..2i+1], desc[i],
// per-block narrow | wide << 32 counts. patches != nullptr: the apply's rules (block on SET_STATE with next_block, unblock
// on SET_MOVING, in that order); it runs BEFORE k_entity_apply, so a.pos is still the tick's snapshot position.
// patches == nullptr: pfnav_agents_set_blocking, block (mode 1) or unblock (mode 0) every listed uid.
__global__ void __launch_bounds__(PF_OPS_BLOCK) k_blocking_decide(const pfnav_agent *__restrict__ agents, pfnav_blocking *__restrict__ blk,
                                                                  const uint32_t *__restrict__ uids, int n,
                                                                  const pfnav_patch *__restrict__ patches, int mode, pf_op_stage s)
{
    const int i = blockIdx.x * PF_OPS_BLOCK + threadIdx.x;
    unsigned nops = 0, desc = 0;
    if (i < n) {
        const uint32_t uid = uids[i];
        const pfnav_agent a = agents[uid];
        pfnav_blocking b = blk[uid];
        bool want_block, want_unblock;
        if (patches) {
            const uint32_t pf = patches[i].flags;
            want_block = (pf & PFNAV_UPDATE_SET_STATE) && patches[i].next_block != 0;
            want_unblock = (pf & PFNAV_UPDATE_SET_MOVING) != 0;
        } else {
            want_block = mode != 0; want_unblock = mode == 0;
        }
        if (want_block && !(a.flags & PFNAV_FLAG_GARRISONED) && !b.blocking) {
            b.blocking = 1; b.stop_x = a.pos[0]; b.stop_z = a.pos[1]; b.stop_radius = a.radius;
            s.ops[2 * i + nops] = {b.stop_x, b.stop_z, b.stop_radius, b.faction_id, a.flags, +1};
            desc |= (pf_op_wide(b.stop_radius) ? 4u : 0u) << nops;
            nops++;
        }
        if (want_unblock && b.blocking) {
            b.blocking = 0;
            s.ops[2 * i + nops] = {b.stop_x, b.stop_z, b.stop_radius, b.faction_id, a.flags, -1};
            desc |= (pf_op_wide(b.stop_radius) ? 4u : 0u) << nops;
            nops++;
        }
        if (nops) blk[uid] = b;
        s.desc[i] = (uint8_t)(desc | nops);
    }
    ops_block_sum(desc, nops, s);
}

// pfnav_agents_restore: row i of the restored range [lo, lo + n) queues the incref of its recorded block
// (pf_ckpt_restore_op), staged like k_blocking_decide's ops; the blocking table itself is already the restored one
__global__ void __launch_bounds__(PF_OPS_BLOCK) k_blocking_restore_decide(const pfnav_agent *__restrict__ agents,
                                                                          const pfnav_blocking *__restrict__ blk, uint32_t lo,
                                                                          int n, pf_op_stage s)
{
    const int i = blockIdx.x * PF_OPS_BLOCK + threadIdx.x;
    unsigned nops = 0, desc = 0;
    if (i < n) {
        pfnav_blocker_op op;
        if (pf_ckpt_restore_op(agents[lo + i], blk[lo + i], &op)) {
            s.ops[2 * i] = op;
            desc = pf_op_wide(op.range) ? 4u : 0u;
            nops = 1;
        }
        s.desc[i] = (uint8_t)(desc | nops);
    }
    ops_block_sum(desc, nops, s);
}

// the checks every entry point of the blocking table makes; need_records: the table must describe this population.
// A member of a multi-GPU job takes part only when the job shares blockers (its ops then reach every member's map
// through the exchange); its table covers its own range [shard_lo, shard_hi), at the same index as on one context.
static int blocking_check(pfnav_ctx *ctx, bool need_records)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_agents, "agents not uploaded");
    if (!pf_mgpu_shares_blockers(ctx) && (ctx->mgpu || ctx->shard_lo > 0 || ctx->shard_hi < ctx->n_agents)) {
        pfnav_set_error("device blocking: the context is part of a multi-GPU job that does not share blockers (its ops "
                        "would reach only its own copy of the map)");
        return PFNAV_ERR_STATE;
    }
    PF_ARG(!need_records || (ctx->d_blocking && ctx->blocking_n == ctx->n_agents), "no blocking records uploaded for this population");
    return PFNAV_OK;
}

int blocking_emit(pfnav_ctx *ctx, cudaStream_t st, const uint32_t *d_uids, int n, const pfnav_patch *d_patches, int mode)
{
    pf_op_stage s;
    int rc = pf_blocker_ops_stage(ctx, (size_t)n, &s);
    if (rc) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    k_blocking_decide<<<(n + PF_OPS_BLOCK - 1) / PF_OPS_BLOCK, PF_OPS_BLOCK, 0, st>>>(ctx->d_agents, ctx->d_blocking, d_uids, n,
                                                                                     d_patches, mode, s);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return pf_blocker_ops_append(ctx, st, (size_t)n, ctx->blocking_any_fac);
}

int blocking_restore_emit(pfnav_ctx *ctx, cudaStream_t st, size_t lo, int n)
{
    if (n == 0) return PFNAV_OK;
    pf_op_stage s;
    int rc = pf_blocker_ops_stage(ctx, (size_t)n, &s);
    if (rc) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    k_blocking_restore_decide<<<(n + PF_OPS_BLOCK - 1) / PF_OPS_BLOCK, PF_OPS_BLOCK, 0, st>>>(ctx->d_agents, ctx->d_blocking,
                                                                                             (uint32_t)lo, n, s);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return pf_blocker_ops_append(ctx, st, (size_t)n, ctx->blocking_any_fac);
}

extern "C" int pfnav_agents_upload_blocking(pfnav_ctx *ctx, const pfnav_blocking *b, size_t n)
{
    int rc = blocking_check(ctx, false);
    if (rc) return rc;
    PF_ARG(b || n == 0, "null records");
    PF_ARG(n == ctx->shard_hi - ctx->shard_lo, "one blocking record per uploaded agent (of this context's own range)");
    bool any_fac = false;
    for (size_t i = 0; i < n; i++) {
        const char *err = pf_blocking_check(b[i]);
        PF_ARG(!err, err);
        any_fac |= b[i].faction_id < 15;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    const size_t all = ctx->n_agents;        // uid-indexed; only the own range is held
    if ((rc = ctx->d_blocking.reserve(std::max<size_t>(all, 1)))) { ctx->blocking_n = 0; return rc; }
    if (n) PF_CUDA(cudaMemcpy(ctx->d_blocking + ctx->shard_lo, b, n * sizeof(pfnav_blocking), cudaMemcpyHostToDevice));
    ctx->blocking_n = all; ctx->blocking_any_fac = any_fac;
    return PFNAV_OK;
}

extern "C" int pfnav_agents_read_blocking(pfnav_ctx *ctx, pfnav_blocking *out, size_t maxout)
{
    int rc = blocking_check(ctx, true);
    if (rc) return rc;
    PF_ARG(out || maxout == 0, "out == NULL");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());
    const size_t n = std::min(maxout, ctx->shard_hi - ctx->shard_lo);       // this context's own entity range
    if (n) PF_CUDA(cudaMemcpy(out, ctx->d_blocking + ctx->shard_lo, n * sizeof(pfnav_blocking), cudaMemcpyDeviceToHost));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_set_blocking(pfnav_ctx *ctx, const uint32_t *uids, size_t n, int block, void *stream)
{
    int rc = blocking_check(ctx, true);
    if (rc) return rc;
    PF_ARG(uids || n == 0, "uids == NULL");
    // a repeated uid changes nothing after its first occurrence: keep the first, so that one thread owns each entity
    std::vector<uint32_t> list;
    list.reserve(n);
    std::vector<uint8_t> seen(ctx->n_agents, 0);
    for (size_t i = 0; i < n; i++) {
        PF_ARG(uids[i] >= ctx->shard_lo && uids[i] < ctx->shard_hi, "uid outside this context's own entity range");
        if (!seen[uids[i]]) { seen[uids[i]] = 1; list.push_back(uids[i]); }
    }
    if (list.empty()) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    if ((rc = ctx->d_block_uids.reserve(list.size()))) return rc;
    PF_CUDA(cudaMemcpyAsync(ctx->d_block_uids, list.data(), list.size() * sizeof(uint32_t), cudaMemcpyHostToDevice, st));
    return blocking_emit(ctx, st, ctx->d_block_uids, (int)list.size(), nullptr, block ? 1 : 0);
}

extern "C" int pfnav_agents_upload_movestate(pfnav_ctx *ctx, const pfnav_movestate *ms, size_t n)
{
    PF_ARG(ctx && ctx->d_agents && ms, "agents not uploaded / ms == NULL");
    PF_ARG(n == ctx->shard_hi - ctx->shard_lo, "one movestate record per uploaded agent (of this context's own range)");
    PF_CUDA(cudaSetDevice(ctx->device));
    if (int rc = ctx->d_movestate.reserve(ctx->n_agents)) return rc;
    PF_CUDA(cudaMemcpy(ctx->d_movestate + ctx->shard_lo, ms, n * sizeof(pfnav_movestate), cudaMemcpyHostToDevice));
    ctx->movestate_set = true;
    return PFNAV_OK;
}

extern "C" int pfnav_agents_upload_formation(pfnav_ctx *ctx, const pfnav_formation_in *f, size_t n)
{
    PF_ARG(ctx && ctx->d_agents && f, "agents not uploaded / null");
    PF_ARG(n == ctx->shard_hi - ctx->shard_lo, "one record per uploaded agent (of this context's own range)");
    PF_CUDA(cudaSetDevice(ctx->device));
    bool grew;
    if (int rc = ctx->d_formation.reserve(ctx->n_agents, &grew)) return rc;
    if (grew) PF_CUDA(cudaMemset(ctx->d_formation, 0, ctx->n_agents * sizeof(pfnav_formation_in)));
    PF_CUDA(cudaMemcpy(ctx->d_formation + ctx->shard_lo, f, n * sizeof(pfnav_formation_in), cudaMemcpyHostToDevice));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_upload_movestate_ext(pfnav_ctx *ctx, const pfnav_movestate_ext *ms, size_t n)
{
    PF_ARG(ctx && ctx->d_agents && ms, "agents not uploaded / null");
    PF_ARG(n == ctx->shard_hi - ctx->shard_lo, "one record per uploaded agent (of this context's own range)");
    PF_CUDA(cudaSetDevice(ctx->device));
    if (int rc = ctx->d_ms_ext.reserve(ctx->n_agents)) return rc;
    PF_CUDA(cudaMemcpy(ctx->d_ms_ext + ctx->shard_lo, ms, n * sizeof(pfnav_movestate_ext), cudaMemcpyHostToDevice));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_read_movestate_ext(pfnav_ctx *ctx, pfnav_movestate_ext *out, size_t maxout)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_agents && ctx->d_ms_ext, "no movestate_ext table uploaded");
    PF_ARG(out || maxout == 0, "out == NULL");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());
    const size_t n = std::min(maxout, ctx->shard_hi - ctx->shard_lo);       // this context's own entity range
    if (n) PF_CUDA(cudaMemcpy(out, ctx->d_ms_ext + ctx->shard_lo, n * sizeof(pfnav_movestate_ext), cudaMemcpyDeviceToHost));
    return PFNAV_OK;
}

// The lowest layer of `unrouted` (a bit per layer) on which a work item in STATE_ENTER_ENTITY_RANGE with a target stands,
// into *out (INT_MAX: none). N_IsMaximallyClose needs the layer's global islands for such an item (nav.c:1731).
__global__ void k_enter_unrouted(const pfnav_agent *__restrict__ agents, const pfnav_movestate_ext *__restrict__ exts,
                                 const uint32_t *__restrict__ work, int nwork, uint32_t unrouted, int *__restrict__ out)
{
    const int wi = blockIdx.x * blockDim.x + threadIdx.x;
    if (wi >= nwork) return;
    const uint32_t uid = work[wi];
    const pfnav_agent a = agents[uid];
    if (a.state != PFNAV_STATE_ENTER_ENTITY_RANGE || exts[uid].surround_target_uid == PFNAV_NULL_UID) return;
    const int layer = nav_layer_for(a.flags, a.radius);
    if ((unrouted >> layer) & 1u) atomicMin(out, layer);
}

// ENTER_ENTITY_RANGE items on a layer without pfnav_route_build make compute_updates fail. The host mirror of the own
// entities' layers tells whether any could: only then are the items checked, which waits for the stream.
static int enter_range_route_check(pfnav_ctx *ctx, cudaStream_t st, int nwork)
{
    uint32_t unrouted = 0;
    for (int l = 0; l < ctx->nlayers; l++)
        if (!pfnav_route_dev_islands(ctx, l)) unrouted |= 1u << l;
    bool any = false;
    if (unrouted)
        for (uint8_t l : ctx->cmd_mirror.layer)
            if ((unrouted >> l) & 1u) { any = true; break; }
    if (!any) return 0;
    if (int rc = ctx->d_enter.reserve(sizeof(int))) return rc;
    int *d_layer = (int *)ctx->d_enter.p;
    PF_CUDA(cudaMemsetAsync(d_layer, 0x7f, sizeof(int), st));
    k_enter_unrouted<<<(nwork + 127) / 128, 128, 0, st>>>(ctx->d_agents, ctx->d_ms_ext, ctx->d_work, nwork, unrouted, d_layer);
    ctx->launches++;
    int layer = 0;
    PF_CUDA(cudaMemcpyAsync(&layer, d_layer, sizeof(int), cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    if (layer != 0x7f7f7f7f) {
        pfnav_set_error("pfnav_agents_compute_updates: pfnav_route_build(layer %d) is needed (global islands, nav.c:1731)", layer);
        return PFNAV_ERR_ARG;
    }
    return 0;
}

// The (flock, layer) table k_entity_update reads, rebuilt on the device when the used pairs, the flocks or the committed
// map changed: the host packs the used pairs through the request staging, and the searches run on `st` with no host wait
// (only a growing buffer waits, under the pf_dbuf rule).
static int refresh_arrival_consts(pfnav_ctx *ctx, cudaStream_t st)
{
    if (ctx->arrival_valid && ctx->arrival_epoch == ctx->map_epoch) return 0;
    const size_t nf = ctx->n_flocks, nl = (size_t)ctx->nlayers;
    std::vector<pf_arrival_pair> pairs;
    for (size_t f = 0; f < nf; f++)
        for (size_t l = 0; l < nl; l++) {
            if (!ctx->flock_layer_used[f * PFNAV_NAV_LAYER_MAX + l]) continue;
            if (!pfnav_route_dev_islands(ctx, (int)l)) {
                pfnav_set_error("pfnav_agents_compute_updates: pfnav_route_build(layer %d) is needed (global islands, nav.c:1731)", (int)l);
                return PFNAV_ERR_ARG;
            }
            pairs.push_back({(int32_t)f, (int32_t)l, ctx->h_flocks[f].target[0], ctx->h_flocks[f].target[1]});
        }
    // from here on the old table is overwritten: it stays invalid until the new one is queued
    ctx->arrival_valid = false;
    ctx->arrival_pairs.swap(pairs);
    const size_t np = ctx->arrival_pairs.size();
    const size_t b0 = nf * nl * sizeof(pf_arrival_dev), b1 = np * PF_ARRIVAL_MC_MAX * sizeof(float2);
    if (int rc = ctx->d_arrival.reserve(b0 + b1 + 2 * np + 1)) return rc;
    if (b0) PF_CUDA(cudaMemsetAsync(ctx->d_arrival, 0, b0, st));
    if (np) {
        const size_t bytes = np * sizeof(pf_arrival_pair);
        pf_stage S;
        if (int rc = pf_stage_begin(ctx, st, bytes, bytes, false, &S)) return rc;
        memcpy(S.host, ctx->arrival_pairs.data(), bytes);
        int rc = pf_stage_upload(ctx, st, S, bytes);
        if (!rc) rc = pf_arrival_search(ctx, st, (const pf_arrival_pair *)S.dev, (int)np, (pf_arrival_dev *)ctx->d_arrival.p,
                                        (float2 *)(ctx->d_arrival + b0), ctx->d_arrival + b0 + b1);
        const int rc_done = pf_stage_done(ctx, st);       // whatever was queued may read S.dev
        if (rc) return rc;
        if (rc_done) return rc_done;
    }
    ctx->arrival_valid = true; ctx->arrival_epoch = ctx->map_epoch;
    return 0;
}

extern "C" int pfnav_agents_read_arrival_consts(pfnav_ctx *ctx, pfnav_arrival_record *out, size_t maxout, size_t *out_n)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(out || maxout == 0, "out == NULL");
    PF_ARG(ctx->arrival_valid && ctx->arrival_epoch == ctx->map_epoch,
           "no current arrival constants (pfnav_agents_compute_updates has not run since they or the committed map changed)");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());
    const std::vector<pf_arrival_pair> &pairs = ctx->arrival_pairs;
    const size_t np = pairs.size(), n = std::min(maxout, np), nl = (size_t)ctx->nlayers;
    if (out_n) *out_n = np;
    if (n == 0) return PFNAV_OK;
    std::vector<pf_arrival_dev> table(ctx->n_flocks * nl);
    std::vector<float2> tiles(np * PF_ARRIVAL_MC_MAX);
    const size_t b0 = table.size() * sizeof(pf_arrival_dev);
    PF_CUDA(cudaMemcpy(table.data(), ctx->d_arrival, b0, cudaMemcpyDeviceToHost));
    PF_CUDA(cudaMemcpy(tiles.data(), ctx->d_arrival + b0, tiles.size() * sizeof(float2), cudaMemcpyDeviceToHost));
    for (size_t s = 0; s < n; s++) {
        const pf_arrival_dev &d = table[(size_t)pairs[s].flock * nl + pairs[s].layer];
        pfnav_arrival_record &o = out[s];
        memset(&o, 0, sizeof(o));
        o.flock = pairs[s].flock; o.layer = pairs[s].layer;
        o.nearest_ok = d.nearest_ok; o.nearest[0] = d.nearest[0]; o.nearest[1] = d.nearest[1];
        o.mc_n = d.mc_n;
        for (int i = 0; i < d.mc_n; i++) { o.mc[i][0] = tiles[(size_t)d.mc_off + i].x; o.mc[i][1] = tiles[(size_t)d.mc_off + i].y; }
    }
    return PFNAV_OK;
}

extern "C" int pfnav_agents_compute_updates(pfnav_ctx *ctx, void *stream)
{
    PF_ARG(ctx && ctx->d_agents, "agents not uploaded");
    PF_ARG(ctx->movestate_set, "pfnav_agents_upload_movestate not called");
    ctx->updates_unapplied = true;
    if (ctx->n_work == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    int rc;
    if ((rc = ctx->d_patches.reserve(ctx->n_work))) return rc;
    if ((rc = refresh_arrival_consts(ctx, st))) return rc;
    if (!ctx->update_done) PF_CUDA(cudaEventCreateWithFlags(&ctx->update_done, cudaEventDisableTiming));
    MapView m;
    m.cost = ctx->d_cost; m.blk = ctx->d_blk; m.W64 = ctx->W64; m.H64 = ctx->H64;
    m.chunk_w = ctx->chunk_w; m.chunk_h = ctx->chunk_h; m.map_x = ctx->map_x; m.map_z = ctx->map_z;
    UpdateParams up;
    up.hz = ctx->hz;
    up.turn_rate = (float)((double)(15.0f / (float)ctx->hz) * 20.0);      // SCALED_MAX_TURN_RATE (movement.c:434)
    up.adj_query_r = ctx->max_radius + 5.0f + 0.0625f;
    const int nwork = (int)ctx->n_work;
    const size_t b0 = ctx->n_flocks * (size_t)ctx->nlayers * sizeof(pf_arrival_dev);
    // STATE_ENTER_ENTITY_RANGE: the tiles N_IsMaximallyClose (nav.c:4707) compares with depend on where the TARGET entity
    // stands. k_entity_update appends the items that need them; pf_enter_range_search searches and finishes those items.
    // d_enter: the two counts (16 bytes), nwork candidate records, nwork flagged indices.
    pf_enter_cand *d_cand = nullptr;
    uint32_t *d_cnt = nullptr;
    if (ctx->d_ms_ext) {
        if ((rc = enter_range_route_check(ctx, st, nwork))) return rc;
        if ((rc = ctx->d_enter.reserve(16 + (size_t)nwork * (sizeof(pf_enter_cand) + sizeof(uint32_t))))) return rc;
        d_cnt = (uint32_t *)ctx->d_enter.p;
        d_cand = (pf_enter_cand *)(ctx->d_enter + 16);
        PF_CUDA(cudaMemsetAsync(d_cnt, 0, 2 * sizeof(uint32_t), st));
    }
    pf_prof_scope prof(ctx, st, PF_PROF_UPDATE);
    k_entity_update<<<(nwork + 127) / 128, 128, 0, st>>>(m, grid_of(ctx), up, ctx->d_agents, ctx->d_records, ctx->d_movestate,
        ctx->d_flocks, (const pf_arrival_dev *)ctx->d_arrival.p, (const float2 *)(ctx->d_arrival + b0),
        ctx->nlayers, ctx->d_work, nwork, ctx->d_vel_out, ctx->d_vdes_out, ctx->d_patches, ctx->d_flock_of,
        ctx->d_ms_ext, ctx->d_formation, d_cand, d_cnt);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    if (d_cand && (rc = pf_enter_range_search(ctx, st, d_cand, d_cnt, (uint32_t *)(d_cand + nwork), nwork, ctx->d_patches)))
        return rc;
    PF_CUDA(cudaEventRecord(ctx->update_done, st));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_read_patches(pfnav_ctx *ctx, pfnav_patch *out, size_t maxout)
{
    PF_ARG(ctx && out && ctx->d_patches && ctx->update_done, "no update pass has run");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaEventSynchronize(ctx->update_done));
    const size_t n = std::min(maxout, ctx->n_work);
    PF_CUDA(cudaMemcpy(out, ctx->d_patches, n * sizeof(pfnav_patch), cudaMemcpyDeviceToHost));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_apply_updates(pfnav_ctx *ctx, void *stream)
{
    return pfnav_agents_apply_updates_ex(ctx, 0, stream);
}

extern "C" int pfnav_agents_apply_updates_ex(pfnav_ctx *ctx, uint32_t flags, void *stream)
{
    PF_ARG(ctx, "ctx");
    if (flags) {
        PF_ARG((flags & ~PFNAV_APPLY_BLOCKERS) == 0, "unknown apply flag");
        int rc = blocking_check(ctx, true);
        if (rc) return rc;
    }
    PF_ARG(ctx->d_patches && ctx->update_done, "no update pass has run");
    ctx->updates_unapplied = false;
    if (ctx->n_work == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    const int nwork = (int)ctx->n_work;
    if (flags & PFNAV_APPLY_BLOCKERS) {     // before the apply: it reads the snapshot positions the apply overwrites
        int rc = blocking_emit(ctx, st, ctx->d_work, nwork, ctx->d_patches, 0);
        if (rc) return rc;
    }
    pf_prof_scope prof(ctx, st, PF_PROF_APPLY);
    ctx->index_stale = true;
    k_entity_apply<<<(nwork + 127) / 128, 128, 0, st>>>(ctx->d_agents, ctx->d_movestate, ctx->d_records, ctx->d_work, nwork,
                                                       ctx->d_patches, ctx->d_ms_ext);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaEventRecord(ctx->update_done, st));
    return PFNAV_OK;
}

extern "C" int pfnav_agents_read_state(pfnav_ctx *ctx, pfnav_agent *agents_out, pfnav_movestate *ms_out, size_t maxout)
{
    PF_ARG(ctx && ctx->d_agents, "agents not uploaded");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());
    const size_t n = std::min(maxout, ctx->shard_hi - ctx->shard_lo);       // this context's own entity range
    if (agents_out && n) PF_CUDA(cudaMemcpy(agents_out, ctx->d_agents + ctx->shard_lo, n * sizeof(pfnav_agent), cudaMemcpyDeviceToHost));
    if (ms_out) {
        PF_ARG(ctx->movestate_set, "no movestate uploaded");
        if (n) PF_CUDA(cudaMemcpy(ms_out, ctx->d_movestate + ctx->shard_lo, n * sizeof(pfnav_movestate), cudaMemcpyDeviceToHost));
    }
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// On-miss chain of N_DesiredPointSeekVelocity (nav.c:3484-3554) against the device field pool.
// ------------------------------------------------------------------------------------------
struct pf_miss { uint32_t wi, uid; int32_t dest, chunk, tile, liid; float px, pz; };

// work agents that would take one of the on-miss branches of the navigation tick:
//   kind 0  compute_los_state -> N_HasDestLOS (nav.c:4026): no LOS field for (dest, chunk of prev_pos)
//   kind 1  compute_desired_velocity -> N_DesiredPointSeekVelocity (nav.c:3468): no flow field for (dest, chunk of
//           pos), or the agent's own tile has no direction (dir_idx == FD_NONE)
__global__ void k_collect_misses(MapView m, PoolView pool, const uint16_t *__restrict__ liid_img,
                                 const pfnav_agent *__restrict__ agents, const pfnav_flock *__restrict__ flocks,
                                 const uint32_t *__restrict__ work, int nwork, int kind, pf_miss *__restrict__ out,
                                 uint32_t *__restrict__ count, uint32_t cap, const pfnav_movestate_ext *__restrict__ exts, int nlayers_)
{
    const int w = blockIdx.x * blockDim.x + threadIdx.x;
    if (w >= nwork) return;
    const uint32_t uid = work[w];
    const pfnav_agent a = agents[uid];
    if (kind == 2) {
        // kind 2: N_DesiredEnemySeekVelocity / N_DesiredSurroundVelocity (nav.c:3603, 3687): the entity's TARGET_ENEMIES /
        // TARGET_ENTITY field exists but its own tile has no direction
        const bool seek = a.state == PFNAV_STATE_SEEK_ENEMIES;
        const bool surr = a.state == PFNAV_STATE_SURROUND_ENTITY && exts && exts[uid].surround_target_uid != PFNAV_NULL_UID &&
                          exts[uid].using_surround_field;
        const int dest = (int)a.aux_dest1 - 1;
        if (!(seek || surr) || dest < 0 || dest >= pool.ndests) return;
        tile_desc t;
        if (!desc_for_point(m, a.pos[0], a.pos[1], t)) return;
        const int chunks = m.chunk_w * m.chunk_h, chunk = t.chunk_r * m.chunk_w + t.chunk_c;
        const int sl = pool.slot[(size_t)dest * chunks + chunk];
        if (sl < 0 || !(pool.has[sl] & 1)) return;                      // building it needs the engine's entity list
        const int layer = nav_layer_for(a.flags, a.radius);
        const uint16_t li = layer < nlayers_ ? liid_img[((size_t)layer * m.H64 + t.chunk_r * 64 + t.tile_r) * m.W64 + t.chunk_c * 64 + t.tile_c] : 0xFFFF;
        // the surround variant repairs a blocked tile whether or not it already has a direction (nav.c:3729)
        if ((pool.flow[(size_t)sl * 4096 + t.tile_r * 64 + t.tile_c] & 0xF) != 0 && !(surr && li == 0xFFFF)) return;
        const uint32_t k = atomicAdd(count, 1u);
        if (k >= cap) return;
        pf_miss r;
        r.wi = (uint32_t)w; r.uid = uid; r.dest = dest; r.chunk = chunk; r.tile = t.tile_r * 64 + t.tile_c; r.liid = li;
        r.px = a.pos[0]; r.pz = a.pos[1];
        out[k] = r;
        return;
    }
    if (a.flock < 0) return;
    const pfnav_flock fl = flocks[a.flock];
    if (fl.dest < 0 || fl.dest >= pool.ndests) return;
    const float px = kind == 0 ? a.prev_pos[0] : a.pos[0], pz = kind == 0 ? a.prev_pos[1] : a.pos[1];
    tile_desc t;
    if (!desc_for_point(m, px, pz, t)) return;
    const int chunks = m.chunk_w * m.chunk_h, chunk = t.chunk_r * m.chunk_w + t.chunk_c;
    const int s = pool.slot[(size_t)fl.dest * chunks + chunk];
    bool miss;
    if (kind == 0) miss = (s < 0) || !(pool.has[s] & 2);
    else {
        miss = (s < 0) || !(pool.has[s] & 1);
        if (!miss) miss = (pool.flow[(size_t)s * 4096 + t.tile_r * 64 + t.tile_c] & 0xF) == 0;
    }
    if (!miss) return;
    const uint32_t k = atomicAdd(count, 1u);
    if (k >= cap) return;
    pf_miss r;
    r.wi = (uint32_t)w; r.uid = uid; r.dest = fl.dest; r.chunk = chunk; r.tile = t.tile_r * 64 + t.tile_c;
    r.liid = liid_img[((size_t)fl.layer * m.H64 + t.chunk_r * 64 + t.tile_r) * m.W64 + t.chunk_c * 64 + t.tile_c];
    r.px = px; r.pz = pz;
    out[k] = r;
}

// The in-place repair of the field in pool slot `slot` for miss r: to the nearest pathable tile from a blocked tile,
// else to the nearest tile of the entity's local island. pf_chain_item_seeds sets its mask.
static pf_chain_item chain_item_of(const pfnav_ctx *ctx, const pf_miss &r, int slot, int always)
{
    pf_chain_item it;
    it.q = ctx->pool.req[slot]; it.slot = slot; it.tile = r.tile; it.always = always;
    if (r.liid == 0xFFFF) { it.kind = PFNAV_REPAIR_NEAREST_PATHABLE; it.arg = ((r.tile >> 6) << 8) | (r.tile & 63); }
    else                  { it.kind = PFNAV_REPAIR_ISLAND_TO_NEAREST; it.arg = r.liid; }
    return it;
}

// The on-miss branches of one navigation tick against the device pool, in the reference's order: first every
// work item's LOS state (compute_los_state, movement.c:4129: a (dest, chunk) without LOS field requests the path
// from the entity's previous position), then every work item's desired velocity (compute_desired_velocity, :4163:
// request from the entity's position, then the in-place field repair if its tile still has no direction). The
// reference walks the entities serially and every request changes what the next entity finds; here the candidates
// are collected on the device, reduced to one representative per (dest, chunk[, local island | blocked tile]) in work
// order, and each representative is RE-CHECKED against the pool as the requests before it left it -- an entity the
// reference would have found served by an earlier entity's request does not request again.
extern "C" int pfnav_pool_repair(pfnav_ctx *ctx, int *out_nrequests, int *out_nrepairs)
{
    PF_ARG(ctx && ctx->d_agents && ctx->pool.d_slot, "agents / pool missing");
    if (out_nrequests) *out_nrequests = 0;
    if (out_nrepairs) *out_nrepairs = 0;
    if (ctx->n_work == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(pf_fields_sync(ctx));
    cudaStream_t st = ctx->tick_stream;
    PF_CUDA(pf_pool_refresh(ctx, st));
    PF_CUDA(cudaDeviceSynchronize());
    const int nwork = (int)ctx->n_work;
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    // the misses and their counter in the scratch of pfnav_pool_repair_batch: the path requests and repairs between the
    // collections restage their own inputs
    const size_t b_m = (size_t)nwork * sizeof(pf_miss);
    if (int rc = ctx->d_rep_buf.reserve(b_m + 4)) return rc;
    pf_miss *d_miss = (pf_miss *)ctx->d_rep_buf.p;
    uint32_t *d_cnt = (uint32_t *)(ctx->d_rep_buf + b_m);
    MapView m;
    m.cost = ctx->d_cost; m.blk = ctx->d_blk; m.W64 = ctx->W64; m.H64 = ctx->H64;
    m.chunk_w = ctx->chunk_w; m.chunk_h = ctx->chunk_h; m.map_x = ctx->map_x; m.map_z = ctx->map_z;
    std::vector<int> flock_of_dest(ctx->pool.ndests, -1);
    for (size_t f = 0; f < ctx->h_flocks.size(); f++)
        if (ctx->h_flocks[f].dest >= 0 && ctx->h_flocks[f].dest < ctx->pool.ndests) flock_of_dest[ctx->h_flocks[f].dest] = (int)f;
    int nreq = 0, nrep = 0, rc = 0;
    auto collect = [&](int kind, std::vector<pf_miss> &reps) -> int {
        const PoolView pv = pool_view(ctx->pool, nullptr, 0);
        PF_CUDA(cudaMemsetAsync(d_cnt, 0, 4, st));
        k_collect_misses<<<(nwork + 127) / 128, 128, 0, st>>>(m, pv, ctx->d_liid, ctx->d_agents, ctx->d_flocks, ctx->d_work, nwork,
                                                             kind, d_miss, d_cnt, (uint32_t)nwork, ctx->d_ms_ext, ctx->nlayers);
        ctx->launches++;
        uint32_t cnt = 0;
        PF_CUDA(cudaMemcpyAsync(&cnt, d_cnt, 4, cudaMemcpyDeviceToHost, st));
        PF_CUDA(cudaStreamSynchronize(st));
        std::vector<pf_miss> miss(std::min<uint32_t>(cnt, (uint32_t)nwork));
        if (!miss.empty()) PF_CUDA(cudaMemcpy(miss.data(), d_miss, miss.size() * sizeof(pf_miss), cudaMemcpyDeviceToHost));
        std::sort(miss.begin(), miss.end(), [](const pf_miss &a, const pf_miss &b) { return a.wi < b.wi; });
        std::vector<uint64_t> seen;
        reps.clear();
        for (const pf_miss &r : miss) {
            uint64_t key = ((uint64_t)r.dest << 40) | ((uint64_t)r.chunk << 20);
            if (kind >= 1) key |= (r.liid == 0xFFFF ? (0x10000u | (uint32_t)r.tile) : (uint32_t)r.liid);
            if (std::find(seen.begin(), seen.end(), key) != seen.end()) continue;
            seen.push_back(key);
            reps.push_back(r);
        }
        return 0;
    };
    auto request_from = [&](const pf_miss &r, int *ok) -> int {
        const int f = flock_of_dest[r.dest];
        *ok = 0;
        if (f < 0) return 0;
        const pfnav_flock &fl = ctx->h_flocks[f];
        int nf = 0, nl = 0; uint32_t did = 0;
        int rc2 = pfnav_pool_request_path(ctx, r.dest, fl.layer, r.px, r.pz, fl.target[0], fl.target[1], nullptr, &did, ok, &nf, &nl);
        if (rc2) return rc2;
        if (nf + nl > 0) nreq++;
        return 0;
    };
    auto repair = [&](const pf_miss &r, int slot) -> int {        // blocking, as the read-back that follows expects
        pf_chain_item it = chain_item_of(ctx, r, slot, 1);
        std::vector<uint64_t> masks;
        int rc2 = pf_chain_item_seeds(ctx, it, masks);
        if (!rc2) rc2 = pfnav_repair_chain_launch(ctx, st, {it}, masks, ctx->pool.d_flow, 0, nullptr);
        if (!rc2) PF_CUDA(cudaStreamSynchronize(st));
        return rc2;
    };
    std::vector<pf_miss> reps;
    // ---- LOS state (N_HasDestLOS, nav.c:4038-4045) ----
    if (!(rc = collect(0, reps))) {
        for (const pf_miss &r : reps) {
            if (ctx->pool.has_of((size_t)r.dest * chunks + r.chunk) & 2) continue;          // an earlier entity's request built it
            int ok;
            if ((rc = request_from(r, &ok))) break;
        }
    }
    // ---- desired velocity (N_DesiredPointSeekVelocity, nav.c:3483-3554) ----
    if (!rc && !(rc = collect(1, reps))) {
        for (const pf_miss &r : reps) {
            auto dir_now = [&](int *dir) -> int {          // the tile's direction as the pool holds it right now, -1 = no field
                const int slot = ctx->pool.slot[(size_t)r.dest * chunks + r.chunk];
                *dir = -1;
                if (slot < 0 || !(ctx->pool.has[slot] & 1)) return 0;
                uint8_t d = 0;
                PF_CUDA(cudaDeviceSynchronize());
                PF_CUDA(cudaMemcpy(&d, ctx->pool.d_flow + (size_t)slot * 4096 + r.tile, 1, cudaMemcpyDeviceToHost));
                *dir = d & 0xF;
                return 0;
            };
            int dir;
            if ((rc = dir_now(&dir))) break;
            if (dir > 0) continue;                                        // served by an earlier entity's request / repair
            int ok;
            if ((rc = request_from(r, &ok))) break;
            if (!ok) continue;                                            // no path from here: zero vector, nothing repaired (nav.c:3501)
            if ((rc = dir_now(&dir))) break;
            if (dir != 0) continue;                                       // case 1: the path query fixed it (or no field: no path)
            if ((rc = repair(r, ctx->pool.slot[(size_t)r.dest * chunks + r.chunk]))) break;
            nrep++;
        }
    }
    // ---- enemy-seek / surround fields: in-place repairs only (nav.c:3647-3675, 3729-3757) ----
    if (!rc && !(rc = collect(2, reps))) {
        for (const pf_miss &r : reps) {
            const int slot = ctx->pool.slot[(size_t)r.dest * chunks + r.chunk];
            if (slot < 0 || !(ctx->pool.has[slot] & 1)) continue;
            uint8_t d = 0;
            if (cudaDeviceSynchronize() != cudaSuccess ||
                cudaMemcpy(&d, ctx->pool.d_flow + (size_t)slot * 4096 + r.tile, 1, cudaMemcpyDeviceToHost) != cudaSuccess) {
                pfnav_set_error("pfnav_pool_repair: read-back failed"); rc = PFNAV_ERR_CUDA; break;
            }
            const pfnav_field_req tg = ctx->pool.req[slot];
            if ((tg.target_type & 0xFF) < 2) continue;
            const bool surround = (tg.target_type & 0xFF) == 2 + PFNAV_TARGET_ENTITY;
            if (r.liid == 0xFFFF) {
                if ((d & 0xF) != 0 && !surround) continue;
            } else {
                if ((d & 0xF) != 0) continue;
            }
            if ((rc = repair(r, slot))) break;
            nrep++;
        }
    }
    if (rc) return rc;
    if (nrep) ctx->goal_batch.valid = false;      // pool bytes changed under a resident plan
    if (out_nrequests) *out_nrequests = nreq;
    if (out_nrepairs) *out_nrepairs = nrep;
    return PFNAV_OK;
}

// ---- pfnav_pool_repair_batch: representative selection and the round gather ----
__device__ __forceinline__ uint64_t rep_key(const pf_miss &r, int kind)
{
    uint64_t key = ((uint64_t)r.dest << 40) | ((uint64_t)r.chunk << 20);
    if (kind >= 1) key |= (r.liid == 0xFFFF ? (0x10000u | (uint32_t)r.tile) : (uint32_t)r.liid);
    return key;
}
__device__ __forceinline__ uint32_t rep_hash(uint64_t key, uint32_t mask)
{
    key ^= key >> 33; key *= 0xff51afd7ed558ccdull; key ^= key >> 33;
    return (uint32_t)key & mask;
}

// the first work index of every key among the misses (open addressing; keys are never ~0)
__global__ void k_rep_mark(const pf_miss *__restrict__ miss, const uint32_t *__restrict__ cnt, uint32_t cap, int kind,
                           unsigned long long *__restrict__ hkey, uint32_t *__restrict__ hwi, uint32_t hmask)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(cnt[0], cap)) return;
    const pf_miss r = miss[i];
    const unsigned long long key = rep_key(r, kind);
    for (uint32_t h = rep_hash(key, hmask);; h = (h + 1) & hmask) {
        const unsigned long long prev = atomicCAS(&hkey[h], ~0ull, key);
        if (prev == ~0ull || prev == key) { atomicMin(&hwi[h], r.wi); return; }
    }
}

// a miss that holds its key's first work index is the representative: place it at its work index
__global__ void k_rep_flag(const pf_miss *__restrict__ miss, const uint32_t *__restrict__ cnt, uint32_t cap, int kind,
                           const unsigned long long *__restrict__ hkey, const uint32_t *__restrict__ hwi, uint32_t hmask,
                           pf_miss *__restrict__ by_wi, uint32_t *__restrict__ flag)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= min(cnt[0], cap)) return;
    const pf_miss r = miss[i];
    const unsigned long long key = rep_key(r, kind);
    uint32_t h = rep_hash(key, hmask);
    while (hkey[h] != key) h = (h + 1) & hmask;
    if (hwi[h] != r.wi) return;
    by_wi[r.wi] = r;
    flag[r.wi] = 1;
}

// ordered compaction of the flagged work indices (one CTA): out = the representatives in work order, cnt[1] = their number
#define REP_COMPACT_THREADS 1024
__global__ void __launch_bounds__(REP_COMPACT_THREADS)
k_rep_compact(const pf_miss *__restrict__ by_wi, const uint32_t *__restrict__ flag, int nwork, pf_miss *__restrict__ out,
              uint32_t *__restrict__ cnt)
{
    __shared__ uint32_t warp_tot[REP_COMPACT_THREADS / 32];
    const int tid = threadIdx.x, per = (nwork + REP_COMPACT_THREADS - 1) / REP_COMPACT_THREADS;
    const int lo = min(tid * per, nwork), hi = min(lo + per, nwork);
    uint32_t n = 0;
    for (int w = lo; w < hi; w++) n += flag[w];
    uint32_t total;
    uint32_t o = pf_block_excl_scan(n, warp_tot, total);
    for (int w = lo; w < hi; w++)
        if (flag[w]) out[o++] = by_wi[w];
    if (tid == 0) cnt[1] = total;
}

// the direction byte of the tiles the remaining representatives stand on, at a round boundary
__global__ void k_repair_gather(const int2 *__restrict__ slot_tile, int n, const uint8_t *__restrict__ flow, uint8_t *__restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const int2 st = slot_tile[i];
    out[i] = st.x < 0 ? 0xFF : (flow[(size_t)st.x * 4096 + st.y] & 0xF);
}

// The on-miss chain of pfnav_pool_repair in device rounds (pfnav.h, DESIGN.md §3 a-4). Same phases, same representatives,
// same decisions; the serial loop's per-representative read-backs become predicates the device evaluates (k_repair_chain)
// or answers the host already holds, and a round ends only where neither is enough.
extern "C" int pfnav_pool_repair_batch(pfnav_ctx *ctx, void *stream, int *out_nrequests, int *out_nrepairs, int *out_nrounds)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_agents && ctx->pool.d_slot, "agents / pool missing");
    int *stats = ctx->repair_stats;           // pfnav_pool_repair_batch_stats
    for (int k = 0; k < 6; k++) stats[k] = 0;
    if (out_nrequests) *out_nrequests = 0;
    if (out_nrepairs) *out_nrepairs = 0;
    if (out_nrounds) *out_nrounds = 0;
    if (ctx->n_work == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    PF_CUDA(pf_fields_join(ctx, st));
    PF_CUDA(pf_pool_refresh(ctx, st));
    const int nwork = (int)ctx->n_work;
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    uint32_t cap = 1;
    while (cap < 2u * (uint32_t)nwork) cap <<= 1;
    // scratch: misses, misses by work index, representatives, flags, hash keys, hash minima, counters, gather in / out
    const size_t b_m = (size_t)nwork * sizeof(pf_miss);
    const size_t o_bywi = b_m, o_reps = 2 * b_m, o_flag = 3 * b_m, o_hkey = (o_flag + (size_t)nwork * 4 + 7) & ~(size_t)7;
    const size_t o_hwi = o_hkey + (size_t)cap * 8, o_cnt = o_hwi + (size_t)cap * 4, o_gin = (o_cnt + 16 + 7) & ~(size_t)7;
    const size_t o_gout = o_gin + (size_t)nwork * 8, total = o_gout + (size_t)nwork;
    if (int rc = ctx->d_rep_buf.reserve(total)) return rc;
    uint8_t *buf = ctx->d_rep_buf;
    pf_miss *d_miss = (pf_miss *)buf, *d_bywi = (pf_miss *)(buf + o_bywi), *d_reps = (pf_miss *)(buf + o_reps);
    uint32_t *d_flag = (uint32_t *)(buf + o_flag), *d_hwi = (uint32_t *)(buf + o_hwi), *d_cnt = (uint32_t *)(buf + o_cnt);
    unsigned long long *d_hkey = (unsigned long long *)(buf + o_hkey);
    int2 *d_gin = (int2 *)(buf + o_gin);
    uint8_t *d_gout = buf + o_gout;
    PF_CUDA(cudaMemsetAsync(d_cnt + 2, 0, 4, st));           // repairs applied by k_repair_chain
    MapView m;
    m.cost = ctx->d_cost; m.blk = ctx->d_blk; m.W64 = ctx->W64; m.H64 = ctx->H64;
    m.chunk_w = ctx->chunk_w; m.chunk_h = ctx->chunk_h; m.map_x = ctx->map_x; m.map_z = ctx->map_z;
    std::vector<int> flock_of_dest(ctx->pool.ndests, -1);
    for (size_t f = 0; f < ctx->h_flocks.size(); f++)
        if (ctx->h_flocks[f].dest >= 0 && ctx->h_flocks[f].dest < ctx->pool.ndests) flock_of_dest[ctx->h_flocks[f].dest] = (int)f;
    int nreq = 0, nrounds = 0;
    // the misses of one phase, one per key, first in work order, read back in work order
    auto collect = [&](int kind, std::vector<pf_miss> &reps) -> int {
        const PoolView pv = pool_view(ctx->pool, nullptr, 0);
        PF_CUDA(cudaMemsetAsync(d_cnt, 0, 8, st));
        PF_CUDA(cudaMemsetAsync(d_flag, 0, (size_t)nwork * 4, st));
        PF_CUDA(cudaMemsetAsync(d_hkey, 0xFF, (size_t)cap * 8, st));
        PF_CUDA(cudaMemsetAsync(d_hwi, 0xFF, (size_t)cap * 4, st));
        const unsigned nb = (nwork + 127) / 128;
        k_collect_misses<<<nb, 128, 0, st>>>(m, pv, ctx->d_liid, ctx->d_agents, ctx->d_flocks, ctx->d_work, nwork, kind, d_miss,
                                             d_cnt, (uint32_t)nwork, ctx->d_ms_ext, ctx->nlayers);
        k_rep_mark<<<nb, 128, 0, st>>>(d_miss, d_cnt, (uint32_t)nwork, kind, d_hkey, d_hwi, cap - 1);
        k_rep_flag<<<nb, 128, 0, st>>>(d_miss, d_cnt, (uint32_t)nwork, kind, d_hkey, d_hwi, cap - 1, d_bywi, d_flag);
        k_rep_compact<<<1, REP_COMPACT_THREADS, 0, st>>>(d_bywi, d_flag, nwork, d_reps, d_cnt);
        ctx->launches += 4;
        PF_CUDA(cudaGetLastError());
        uint32_t nrep = 0;
        PF_CUDA(cudaMemcpyAsync(&nrep, d_cnt + 1, 4, cudaMemcpyDeviceToHost, st));
        PF_CUDA(cudaStreamSynchronize(st));
        reps.resize(std::min<uint32_t>(nrep, (uint32_t)nwork));
        if (!reps.empty()) {
            PF_CUDA(cudaMemcpyAsync(reps.data(), d_reps, reps.size() * sizeof(pf_miss), cudaMemcpyDeviceToHost, st));
            PF_CUDA(cudaStreamSynchronize(st));
        }
        stats[kind] = (int)reps.size();
        return 0;
    };
    auto key_of = [&](const pf_miss &r) { return (size_t)r.dest * chunks + r.chunk; };
    auto has_flow = [&](int slot) { return slot >= 0 && (ctx->pool.has[slot] & 1); };
    // the path requests of a phase's representatives, planned up front (flock target, flock layer)
    auto plan = [&](const std::vector<pf_miss> &reps, pf_path_batch **out) -> int {
        const size_t n = reps.size();
        std::vector<int32_t> dests(n), layers(n);
        std::vector<float> src(2 * n), dst(2 * n);
        for (size_t i = 0; i < n; i++) {
            const int f = flock_of_dest[reps[i].dest];
            const pfnav_flock &fl = ctx->h_flocks[f < 0 ? 0 : f];
            dests[i] = reps[i].dest; layers[i] = f < 0 ? -1 : fl.layer;
            src[2 * i] = reps[i].px; src[2 * i + 1] = reps[i].pz;
            dst[2 * i] = f < 0 ? 0.0f : fl.target[0]; dst[2 * i + 1] = f < 0 ? 0.0f : fl.target[1];
        }
        return pf_path_batch_begin(ctx, (int)n, dests.data(), layers.data(), src.data(), dst.data(), st, out);
    };
    using batch_ptr = std::unique_ptr<pf_path_batch, void (*)(pf_path_batch *)>;
    std::vector<pf_miss> reps;
    int rc = 0;
    pf_path_probe pr;
    // ---- LOS state (N_HasDestLOS, nav.c:4038-4045): one request batch, skipping a (dest, chunk) whose LOS field an
    //      earlier representative's request built ----
    if ((rc = collect(0, reps))) return rc;
    if (!reps.empty()) {
        pf_path_batch *pb = nullptr;
        if ((rc = plan(reps, &pb))) return rc;
        batch_ptr B(pb, pf_path_batch_end);
        bool any = false;
        for (size_t i = 0; i < reps.size() && !rc; i++) {
            if (ctx->pool.has_of(key_of(reps[i])) & 2) continue;
            if (flock_of_dest[reps[i].dest] < 0) continue;
            if ((rc = pf_path_batch_probe(pb, (int)i, &pr))) break;    // PFNAV_ERR_ARG, as pfnav_pool_request_path's
            if (pr.nf + pr.nl == 0) continue;
            if ((rc = pf_path_batch_commit(pb, nullptr))) break;
            nreq++; any = true;
        }
        int frc = pf_path_batch_flush(pb);
        if (frc) return frc;
        nrounds += any;
        if (rc) return rc;
    }
    // ---- desired velocity (N_DesiredPointSeekVelocity, nav.c:3483-3554): requests and predicated repairs in rounds ----
    if ((rc = collect(1, reps))) return rc;
    if (!reps.empty()) {
        const size_t n = reps.size();
        pf_path_batch *pb = nullptr;
        if ((rc = plan(reps, &pb))) return rc;
        batch_ptr B(pb, pf_path_batch_end);
        // what each representative's tile holds at the start of the round: its slot then, and the direction byte
        std::vector<int32_t> slot0(n);
        std::vector<uint8_t> dir0(n, 0);
        std::vector<uint8_t> written(ctx->pool.max, 0), chained(ctx->pool.max, 0);
        std::vector<int32_t> touched;                     // slots marked in written / chained this round
        std::vector<pf_chain_item> items;
        std::vector<uint64_t> masks;
        bool pending = false;
        std::vector<int2> gin;
        std::vector<uint8_t> gout;
        // read the bytes representatives from.. stand on, as the pool holds them once the work queued so far is done
        auto gather = [&](size_t from) -> int {
            gin.clear();
            for (size_t k = from; k < n; k++) {
                const int s = ctx->pool.slot[key_of(reps[k])];
                slot0[k] = has_flow(s) ? s : -1;
                gin.push_back(make_int2(slot0[k], reps[k].tile));
            }
            if (gin.empty()) return 0;
            gout.resize(gin.size());
            PF_CUDA(cudaMemcpyAsync(d_gin, gin.data(), gin.size() * sizeof(int2), cudaMemcpyHostToDevice, st));
            k_repair_gather<<<((unsigned)gin.size() + 127) / 128, 128, 0, st>>>(d_gin, (int)gin.size(), ctx->pool.d_flow, d_gout);
            ctx->launches++;
            PF_CUDA(cudaGetLastError());
            PF_CUDA(cudaMemcpyAsync(gout.data(), d_gout, gout.size(), cudaMemcpyDeviceToHost, st));
            PF_CUDA(cudaStreamSynchronize(st));
            for (size_t k = from; k < n; k++) dir0[k] = gout[k - from];
            return 0;
        };
        // end the round: launch its requests and chain items, then gather for the representatives still to come
        auto boundary = [&](size_t from) -> int {
            int r2 = pf_path_batch_flush(pb);
            if (r2) return r2;
            if ((r2 = pfnav_repair_chain_launch(ctx, st, items, masks, ctx->pool.d_flow, 0, d_cnt + 2))) return r2;
            nrounds += pending;
            items.clear(); masks.clear();
            for (int32_t s : touched) written[s] = chained[s] = 0;
            touched.clear();
            pending = false;
            return gather(from);
        };
        if ((rc = gather(0))) return rc;
        auto mark = [&](std::vector<uint8_t> &v, int32_t s) { if (!written[s] && !chained[s]) touched.push_back(s); v[s] = 1; };
        std::vector<int32_t> wslots;
        for (size_t i = 0; i < n;) {
            const pf_miss &r = reps[i];
            const size_t key = key_of(r);
            if (flock_of_dest[r.dest] < 0) { i++; continue; }       // no request, no repair (nav.c:3501)
            // step a of the serial loop: the tile's direction before the request, if the host knows it
            const int s = ctx->pool.slot[key];
            int dir = -1;                                            // -1: no flow field
            bool known = true;
            if (has_flow(s)) {
                if (written[s] || chained[s] || s != slot0[i]) known = false;
                else dir = dir0[i];
            }
            if (!pf_path_batch_planned(pb, (int)i)) {
                // the serial request fails (PFNAV_ERR_ARG) unless an earlier representative served this tile
                if (!known) { stats[3]++; if ((rc = boundary(i))) break; continue; }
                if (dir > 0) { i++; continue; }
                rc = pf_path_batch_probe(pb, (int)i, &pr);
                break;
            }
            if ((rc = pf_path_batch_probe(pb, (int)i, &pr))) break;
            if (pr.nf + pr.nl > 0) {
                if (!known) { stats[3]++; if ((rc = boundary(i))) break; continue; }         // rule (i)
                if (dir > 0) { i++; continue; }                                                // served: no request
                bool hit = false;
                for (int32_t ws : pr.write_slots) hit |= chained[ws] != 0;
                if (hit || (pr.would_evict && pending)) {                                     // rules (ii), (iii)
                    stats[hit ? 4 : 5]++;
                    if ((rc = boundary(i))) break;
                    continue;
                }
                if ((rc = pf_path_batch_commit(pb, &wslots))) break;
                nreq++; pending = true;
                for (int32_t ws : wslots) mark(written, ws);
            } else if (known && dir > 0) { i++; continue; }
            if (!pr.ok) { i++; continue; }                           // no path from here: zero vector, nothing repaired
            const int sl = ctx->pool.slot[key];
            if (!has_flow(sl)) { i++; continue; }                    // no field: nothing to repair
            pf_chain_item it = chain_item_of(ctx, r, sl, 0);
            if (const int src = pf_chain_item_seeds(ctx, it, masks)) {
                // the serial loop fails here only if the repair runs: decide on the byte as the round leaves it. With
                // nothing pending, nothing ran since the last gather and the byte read there is still the pool's.
                const int keep = src;
                if (pending && (rc = boundary(i))) break;
                if (dir0[i] == 0) { rc = keep; break; }
                i++;
                continue;
            }
            items.push_back(it);
            mark(chained, sl);
            pending = true;
            i++;
        }
        if (pending || !items.empty()) {
            const int rc2 = boundary(n);
            if (!rc) rc = rc2;
        } else {
            const int rc2 = pf_path_batch_flush(pb);
            if (!rc) rc = rc2;
        }
        if (rc) return rc;
    }
    // ---- enemy-seek / surround fields: in-place repairs only (nav.c:3647-3675, 3729-3757), one launch ----
    if ((rc = collect(2, reps))) return rc;
    {
        std::vector<pf_chain_item> items;
        std::vector<uint64_t> masks;
        for (size_t i = 0; i < reps.size(); i++) {
            const pf_miss &r = reps[i];
            const int slot = ctx->pool.slot[key_of(r)];
            if (!has_flow(slot)) continue;
            const pfnav_field_req tg = ctx->pool.req[slot];
            if ((tg.target_type & 0xFF) < 2) continue;
            const bool surround = (tg.target_type & 0xFF) == 2 + PFNAV_TARGET_ENTITY;
            pf_chain_item it = chain_item_of(ctx, r, slot, r.liid == 0xFFFF && surround);
            if (const int src = pf_chain_item_seeds(ctx, it, masks)) {
                // fails only if the repair runs: apply what comes before it, then read the byte
                if ((rc = pfnav_repair_chain_launch(ctx, st, items, masks, ctx->pool.d_flow, 0, d_cnt + 2))) return rc;
                if (!items.empty()) nrounds++;
                items.clear(); masks.clear();
                uint8_t d = 0;
                PF_CUDA(cudaMemcpyAsync(&d, ctx->pool.d_flow + (size_t)slot * 4096 + r.tile, 1, cudaMemcpyDeviceToHost, st));
                PF_CUDA(cudaStreamSynchronize(st));
                if (it.always || (d & 0xF) == 0) { rc = src; break; }
                continue;
            }
            items.push_back(it);
        }
        if (!items.empty()) {
            const int rc2 = pfnav_repair_chain_launch(ctx, st, items, masks, ctx->pool.d_flow, 0, d_cnt + 2);
            if (!rc) rc = rc2;
            nrounds++;
        }
    }
    if (rc) return rc;
    uint32_t nrep = 0;
    PF_CUDA(cudaMemcpyAsync(&nrep, d_cnt + 2, 4, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    if (nrep) ctx->goal_batch.valid = false;      // pool bytes changed under a resident plan
    if (out_nrequests) *out_nrequests = nreq;
    if (out_nrepairs) *out_nrepairs = (int)nrep;
    if (out_nrounds) *out_nrounds = nrounds;
    return PFNAV_OK;
}

// Test / measurement hook: what the last pfnav_pool_repair_batch call did (pfnav.h).
extern "C" int pfnav_pool_repair_batch_stats(pfnav_ctx *ctx, int *out6)
{
    PF_ARG(ctx && out6, "args");
    for (int k = 0; k < 6; k++) out6[k] = ctx->repair_stats[k];
    return PFNAV_OK;
}

// Test / tuning hook: 0 = always the single-pass velocity kernel, 1 (default) = split it around the field join
// whenever LOS chains are still in flight, 2 = always split (exercises the two-phase path without fields).
// Test / tuning hook: cohesion pass, 0 = automatic (windowed for flocks of >= 20 000), 1 = always windowed, 2 = always the
// full member list. Results agree to float rounding (the windowed pass falls back per entity where they would not).
extern "C" int pfnav_set_cohesion_mode(pfnav_ctx *ctx, int mode)
{
    PF_ARG(ctx && mode >= 0 && mode <= 2, "mode");
    ctx->cohesion_mode = mode;
    return PFNAV_OK;
}

// Test / tuning hook: how often G_ClearPath_NewVelocity's retry loop (clearpath.c:702-713) was entered since the last reset.
// out[0] = first solves without an admissible velocity, out[1] = of those with both neighbour lists non-empty (the loop
// can run), out[2] = entities that replayed the loop literally (order-dependent tie), out[3] = solves inside those replays.
extern "C" int pfnav_agents_clearpath_stats(pfnav_ctx *ctx, uint64_t *out4, int reset)
{
    PF_ARG(ctx && out4, "args");
    PF_NEED_DEVICE(ctx);
    memset(out4, 0, 4 * sizeof(uint64_t));
    if (!ctx->d_cp_stats) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());
    PF_CUDA(cudaMemcpy(out4, ctx->d_cp_stats, 4 * sizeof(uint64_t), cudaMemcpyDeviceToHost));
    if (reset) PF_CUDA(cudaMemset(ctx->d_cp_stats, 0, 8 * sizeof(unsigned long long)));
    return PFNAV_OK;
}

extern "C" int pfnav_set_two_phase(pfnav_ctx *ctx, int mode)
{
    PF_ARG(ctx && mode >= 0 && (mode & 3) <= 2, "mode");
    ctx->two_phase = (mode & 3) != 0;
    ctx->two_phase_force = (mode & 3) == 2;
    ctx->phase_a_ctas_per_sm = mode >> 4;          // tuning: bits 4.. = resident CTAs per SM of phase A (0 = default)
    return PFNAV_OK;
}
