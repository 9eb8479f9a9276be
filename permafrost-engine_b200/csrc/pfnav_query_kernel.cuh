// pfnav_query_kernel.cuh -- the device code of pfnav_map_query, kept in a header of its own so that tests/emu can run
// the SAME source on CPU threads (tests/emu/query_emu.cpp defines the CUDA keywords and __syncwarp as plain C++);
// pfnav_query.cu includes it.
// Needs: <stdint.h>, <stddef.h>, sqrtf / fabs / min / max, include/pfnav.h, pfnav_map_view.cuh.
#pragma once

// n_dest_id (nav.c:839), as plan_init packs it (pfnav_route.cu)
__device__ __forceinline__ uint32_t mq_dest_id(const tile_desc &d, int layer, int faction_id)
{
    return (((uint32_t)d.chunk_r & 0x3f) << 26) | (((uint32_t)d.chunk_c & 0x3f) << 20) | (((uint32_t)d.tile_r & 0x3f) << 14) |
           (((uint32_t)d.tile_c & 0x3f) << 8) | (((uint32_t)layer & 0xf) << 4) | ((uint32_t)faction_id & 0xfu);
}

// The probe kinds and DEST_ID, one thread per query. The search kinds get ok = 0 here; k_map_search overwrites them.
__global__ void __launch_bounds__(256) k_map_probe(MapView m, const pfnav_map_query_req *__restrict__ q, int n,
                                                   pfnav_map_query_result *__restrict__ out)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const pfnav_map_query_req a = q[i];
    pfnav_map_query_result r = {0, 0u, 0.0f, 0.0f};
    tile_desc td;
    if (desc_for_point(m, a.x, a.z, td)) {
        bool pathable, blocked;
        switch (a.kind) {
        case PFNAV_QUERY_PATHABLE: probe_tile(m, a.layer, a.x, a.z, pathable, blocked); r.ok = pathable; break;
        case PFNAV_QUERY_BLOCKED: probe_tile(m, a.layer, a.x, a.z, pathable, blocked); r.ok = blocked; break;
        case PFNAV_QUERY_ADJACENT_IMPASSABLE: r.ok = adjacent_impassable(m, a.layer, td); break;
        case PFNAV_QUERY_DEST_ID: r.ok = 1; r.dest_id = mq_dest_id(td, a.layer, a.faction_id); break;
        default: break;
        }
    }
    out[i] = r;
}

// ---- the two searches, one warp per query ----
// The lanes stage a dim x dim window of the layer around the start tile into a bitmap, lane 0 replays the reference's
// FIFO search inside it, and the lanes evaluate the tolerance test. A replay that would have to look outside the
// window is not trusted: the 32 x 32 window is tried first, then the 128 x 128 one, then the host (the fallback flag).
#define MQ_DIM_MAX 128
#define MQ_WORDS_MAX (MQ_DIM_MAX * MQ_DIM_MAX / 32)
#define MQ_LIST_MAX 256                  /* PF_ARRIVAL_MC_MAX: FIELD_RES_R*2 + FIELD_RES_C*2 (nav.c:4721) */

struct mq_shared {
    uint32_t bits[MQ_WORDS_MAX];         // CLOSEST_PATHABLE: 0xFF or blocked; MAXIMALLY_CLOSE: listable (island, no blocker)
    uint32_t vis[MQ_WORDS_MAX];
    uint16_t queue[MQ_DIM_MAX * MQ_DIM_MAX + 1];     // window indices; the unmarked start tile can be queued twice
    uint16_t list[MQ_LIST_MAX];          // MAXIMALLY_CLOSE: the listed tiles, window indices, in the reference's order
    int status;                          // replay result: MQ_FOUND / MQ_NONE / MQ_OUTSIDE (+ count for the list)
    int n, tile, hit;
    int r0, c0, dim;                     // the window of the last replay
};
enum { MQ_NONE = 0, MQ_FOUND = 1, MQ_OUTSIDE = -1 };

__device__ __forceinline__ bool mq_bit(const uint32_t *bm, int i) { return (bm[i >> 5] >> (i & 31)) & 1u; }
__device__ __forceinline__ void mq_set(uint32_t *bm, int i) { bm[i >> 5] |= 1u << (i & 31); }
__device__ __forceinline__ int mq_abs(int v) { return v < 0 ? -v : v; }

// N_ClosestPathable (nav.c:4126) as pfnav_arrival_consts restates it, inside the window, on one lane. S.bits: 1 = cost
// 0xFF or a blocker. The search visits every tile in Manhattan-level order, so the replay is exact when the tile found
// lies on a lower level than every in-map tile the window left out (those are noted as they would be queued).
__device__ __forceinline__ void mq_closest_pathable(mq_shared &S, int H64, int W64, int tr, int tc)
{
    const int dim = S.dim, r0 = S.r0, c0 = S.c0;
    const int dr[4] = {0, 0, -1, 1}, dc[4] = {-1, 1, 0, 0};
    int head = 0, tail = 0, cut = 0x7fffffff;
    S.queue[tail++] = (uint16_t)((tr - r0) * dim + (tc - c0));       // the start tile is not marked visited
    while (head < tail) {
        const int t = S.queue[head++];
        const int ar = r0 + t / dim, ac = c0 + t % dim;
        if (!mq_bit(S.bits, t)) {
            const bool exact = mq_abs(ar - tr) + mq_abs(ac - tc) < cut;
            S.status = exact ? MQ_FOUND : MQ_OUTSIDE; S.tile = t;
            return;
        }
        for (int e = 0; e < 4; e++) {
            const int nr = ar + dr[e], nc = ac + dc[e];
            if (nr < 0 || nr >= H64 || nc < 0 || nc >= W64) continue;
            const int wr = nr - r0, wc = nc - c0;
            if (wr < 0 || wr >= dim || wc < 0 || wc >= dim) { cut = min(cut, mq_abs(nr - tr) + mq_abs(nc - tc)); continue; }
            const int i = wr * dim + wc;
            if (mq_bit(S.vis, i)) continue;
            mq_set(S.vis, i);
            S.queue[tail++] = (uint16_t)i;
        }
    }
    S.status = cut == 0x7fffffff ? MQ_NONE : MQ_OUTSIDE;
}

// n_closest_island_tiles(dst, giid(dst), ignore_blockers = false, maxout = 256) (nav.c:1226) as pfnav_arrival_consts
// restates it, inside the window, on one lane. S.bits: 1 = same global island as the destination tile and no blocker.
// The order in which tiles are met depends on the geometry alone, so the replay is exact as long as it meets no in-map
// tile outside the window -- or the first one it meets ends the search through the Manhattan cut.
__device__ __forceinline__ void mq_closest_island_tiles(mq_shared &S, int H64, int W64, int tr, int tc)
{
    const int dim = S.dim, r0 = S.r0, c0 = S.c0;
    const int dr[9] = {0, 0, 0, -1, 1, -1, -1, 1, 1}, dc[9] = {0, -1, 1, 0, 0, -1, 1, -1, 1};
    int head = 0, tail = 0, first_mh = -1, n = 0;
    const int s = (tr - r0) * dim + (tc - c0);
    mq_set(S.vis, s);
    S.queue[tail++] = (uint16_t)s;
    S.status = MQ_FOUND;
    while (head < tail) {
        const int t = S.queue[head++];
        const int ar = r0 + t / dim, ac = c0 + t % dim;
        for (int e = 0; e < 9; e++) {
            const int nr = ar + dr[e], nc = ac + dc[e];
            if (nr < 0 || nr >= H64 || nc < 0 || nc >= W64) continue;
            const int wr = nr - r0, wc = nc - c0;
            const int mh = mq_abs(tr - nr) + mq_abs(tc - nc);
            if (wr < 0 || wr >= dim || wc < 0 || wc >= dim) {
                // never met before: the reference takes the Manhattan cut here, or goes on with a tile the window lacks
                if (!(first_mh > 0 && mh > first_mh)) S.status = MQ_OUTSIDE;
                S.n = n;
                return;
            }
            const int i = wr * dim + wc;
            if (mq_bit(S.vis, i)) continue;
            if (first_mh > 0 && mh > first_mh) { S.n = n; return; }
            if (mq_bit(S.bits, i)) {
                S.list[n++] = (uint16_t)i;
                if (first_mh == -1) first_mh = mh;
                if (n == MQ_LIST_MAX) { S.n = n; return; }
            }
            mq_set(S.vis, i);
            S.queue[tail++] = (uint16_t)i;
        }
    }
    S.n = n;
}

// Stage the window's bits (one word of 32 columns per lane at a time) and clear `vis`. Window tiles outside the map
// stay 0; the replays test the map bounds before the window's.
__device__ __forceinline__ void mq_stage(mq_shared &S, const MapView &m, const uint16_t *gisl, int layer, int kind,
                                         uint16_t giid, int lane)
{
    const int dim = S.dim, wpr = dim >> 5, nw = dim * wpr;
    const size_t lbase = (size_t)layer * m.H64 * m.W64;
    for (int w = lane; w < nw; w += 32) {
        const int ar = S.r0 + w / wpr, ac0 = S.c0 + (w % wpr) * 32;
        uint32_t word = 0;
        if (ar < m.H64)
            for (int b = 0; b < 32 && ac0 + b < m.W64; b++) {
                const size_t off = lbase + (size_t)ar * m.W64 + ac0 + b;
                const bool set = kind == PFNAV_QUERY_CLOSEST_PATHABLE ? (m.cost[off] == 0xFF || m.blk[off] > 0)
                                                                      : (gisl[off] == giid && m.blk[off] == 0);
                word |= (uint32_t)set << b;
            }
        S.bits[w] = word;
        S.vis[w] = 0;
    }
}

// the window of side dim around (tr, tc), kept inside the map where the map is large enough
__device__ __forceinline__ int mq_origin(int t, int dim, int extent)
{
    return min(max(t - dim / 2, 0), max(extent - dim, 0));
}

// One CLOSEST_PATHABLE or MAXIMALLY_CLOSE query on the calling warp. Writes *out and *fallback (1: finish on the host)
// from lane 0. A MAXIMALLY_CLOSE replay leaves its list in S.list[0 .. S.n) (window S.r0, S.c0, S.dim).
__device__ __forceinline__ void mq_search(mq_shared &S, const MapView &m, const uint16_t *gisl, const pfnav_map_query_req &a,
                                          pfnav_map_query_result *out, uint8_t *fallback, int lane)
{
    const bool cp = a.kind == PFNAV_QUERY_CLOSEST_PATHABLE;
    tile_desc td;
    // the point whose tile starts the search: the target of N_ClosestPathable, the destination of N_IsMaximallyClose
    const bool on_map = cp ? desc_for_point(m, a.x, a.z, td) : desc_for_point(m, a.dst_x, a.dst_z, td);
    pfnav_map_query_result r = {0, 0u, 0.0f, 0.0f};
    uint8_t fb = 0;
    tile_desc pd;
    if (on_map && (cp || desc_for_point(m, a.x, a.z, pd))) {          // MAXIMALLY_CLOSE: the position must lie on the map too
        const int tr = td.chunk_r * 64 + td.tile_r, tc = td.chunk_c * 64 + td.tile_c;
        if (cp && !tile_blocked_abs(m, a.layer, tr, tc)) {
            r.ok = 1; r.x = a.x; r.z = a.z;
        } else {
            const uint16_t giid = cp ? 0 : gisl[((size_t)a.layer * m.H64 + tr) * m.W64 + tc];
            int status = MQ_OUTSIDE;
            for (int dim = 32; dim <= MQ_DIM_MAX && status == MQ_OUTSIDE; dim *= 4) {
                if (lane == 0) { S.dim = dim; S.r0 = mq_origin(tr, dim, m.H64); S.c0 = mq_origin(tc, dim, m.W64); }
                __syncwarp();
                mq_stage(S, m, gisl, a.layer, a.kind, giid, lane);
                __syncwarp();
                if (lane == 0) {
                    if (cp) mq_closest_pathable(S, m.H64, m.W64, tr, tc);
                    else mq_closest_island_tiles(S, m.H64, m.W64, tr, tc);
                    S.hit = 0;
                }
                __syncwarp();
                status = S.status;
                __syncwarp();
            }
            if (status == MQ_OUTSIDE) {
                fb = 1;
            } else if (cp) {
                if (status == MQ_FOUND) {
                    const int ar = S.r0 + S.tile / S.dim, ac = S.c0 + S.tile % S.dim;
                    // M_Tile_Bounds (tile.c:356): x decreases with the column, z increases with the row
                    r.ok = 1;
                    r.x = (m.map_x - (float)((ac >> 6) * 256)) - (float)((ac & 63) * 4);
                    r.z = (m.map_z + (float)((ar >> 6) * 256)) + (float)((ar & 63) * 4);
                }
            } else {
                // N_IsMaximallyClose (nav.c:4729-4737): a listed "centre" (map_pos -/+ abs tile index * 4) within tolerance,
                // in the float arithmetic of k_entity_update (v2_len of the difference)
                for (int i = lane; i < S.n; i += 32) {
                    const int t = S.list[i];
                    const float cx = m.map_x - (float)(S.c0 + t % S.dim) * 4.0f, cz = m.map_z + (float)(S.r0 + t / S.dim) * 4.0f;
                    const float dx = cx - a.x, dz = cz - a.z;
                    if (sqrtf(dx * dx + dz * dz) <= a.tolerance) S.hit = 1;
                }
                __syncwarp();
                r.ok = S.hit;
            }
        }
    }
    if (lane == 0) { *out = r; *fallback = fb; }
    __syncwarp();
}

// idx: the ns query indices of the search kinds; fallback[k] = 1 flags search k for the host
__global__ void __launch_bounds__(32) k_map_search(MapView m, const uint16_t *__restrict__ gisl, const pfnav_map_query_req *__restrict__ q,
                                                   const int32_t *__restrict__ idx, int ns, pfnav_map_query_result *__restrict__ out,
                                                   uint8_t *__restrict__ fallback)
{
    __shared__ mq_shared S;
    const int lane = threadIdx.x & 31;
    for (int k = blockIdx.x; k < ns; k += gridDim.x) {
        const int i = idx[k];
        mq_search(S, m, gisl, q[i], out + i, fallback + k, lane);
    }
}
