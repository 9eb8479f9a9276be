// pfnav_layer_search.cuh -- the whole-layer tier of the map searches (N_ClosestPathable, n_closest_island_tiles): the
// searches the window replays of pfnav_query_kernel.cuh flag are finished here on the device, one CTA per search. Kept in
// a header of its own so that tests/emu/arrival_emu.cpp can run the SAME source on CPU threads; pfnav_query.cu includes it.
// Needs: pfnav_query_kernel.cuh (and what it needs), float2, __syncthreads, atomicOr / atomicMin / atomicAdd, __popc.
#pragma once

// ---- the whole-layer tier: one CTA per search that left the 128 x 128 window ----
// Both searches queue every in-map tile, blocked or not, so the order in which they meet tiles is the geometry's alone.
// Level d is the Manhattan ring (N_ClosestPathable, 4 deltas) or the Chebyshev ring (n_closest_island_tiles, 9 deltas) of
// radius d around the start, clipped to the map. A tile's FIFO rank within its level is the lexicographic order of
// (rank of its first-ranked neighbour on level d-1, index of the delta from that neighbour to it): level d-1 is popped
// in rank order and each pop queues its unvisited neighbours in delta order. The tier keeps the ranks of two levels,
// indexed by ring position, ranks the next level with a bitmap over those keys (K * |level d-1| bits) and reads the answer
// off in rank order. N_ClosestPathable does not mark its start visited, so the start is queued a second time on level 2;
// it is blocked (else the search ends at once) and every neighbour of it is visited by then, so that copy neither
// answers nor queues anything, and it cannot change the answer.
struct mq_layer_shared {
    int nlev;                            // tiles on the last ranked level
    int best;                            // CLOSEST_PATHABLE: the rank found on the level (INT_MAX: none)
    int first_mh, n, done;               // MAXIMALLY_CLOSE: the Manhattan cut, tiles listed, search over
    int j, cut, add;                     // MAXIMALLY_CLOSE: the current chunk's first listed rank, cut rank, listed count
    int tile;                            // CLOSEST_PATHABLE: the tile found (row * W64 + col), -1 for none
    int hit;                             // tolerance test of the listed tiles
    int tsum[256];                       // mq_block_scan: per-thread popcount sums, then the listing flags
};
#define MQ_LAYER_THREADS 256

// ring positions: a Chebyshev ring d > 0 has 8d, a Manhattan ring 4d, ring 0 is the start alone
__host__ __device__ __forceinline__ size_t mq_layer_positions(int W64, int H64) { return 8 * (size_t)(W64 + H64); }
// int32 words of one CTA's scratch: the ranks of two levels and the rank -> position order (positions each), the key
// bitmap and its word prefix (9 keys per position each, in bits)
__host__ __device__ __forceinline__ size_t mq_layer_scratch_words(int W64, int H64)
{
    const size_t P = mq_layer_positions(W64, H64), nb = (9 * P + 31) / 32;
    return 3 * P + 2 * nb;
}

__device__ __forceinline__ void mq_ring_off(bool cheb, int d, int p, int &dr, int &dc)
{
    if (d == 0) { dr = dc = 0; return; }
    if (cheb) {
        const int s = p / (2 * d), k = p - s * 2 * d;
        if (s == 0) { dr = -d; dc = -d + k; }
        else if (s == 1) { dr = -d + k; dc = d; }
        else if (s == 2) { dr = d; dc = d - k; }
        else { dr = d - k; dc = -d; }
    } else {
        const int s = p / d, k = p - s * d;
        if (s == 0) { dr = -d + k; dc = k; }
        else if (s == 1) { dr = k; dc = d - k; }
        else if (s == 2) { dr = d - k; dc = -k; }
        else { dr = -k; dc = -d + k; }
    }
}

__device__ __forceinline__ int mq_ring_pos(bool cheb, int d, int dr, int dc)
{
    if (d == 0) return 0;
    if (cheb) {
        if (dr == -d && dc < d) return d + dc;
        if (dc == d && dr < d) return 3 * d + dr;
        if (dr == d && dc > -d) return 5 * d - dc;
        return 7 * d - dr;
    }
    if (dr < 0 && dc >= 0) return dc;
    if (dr >= 0 && dc > 0) return d + dr;
    if (dr > 0 && dc <= 0) return 2 * d - dc;
    return 3 * d - dr;
}

__device__ __forceinline__ int mq_level(bool cheb, int dr, int dc)
{
    return cheb ? max(mq_abs(dr), mq_abs(dc)) : mq_abs(dr) + mq_abs(dc);
}

// L.tsum[t] = the inclusive sum of v over threads 0 .. t (nt <= 256 threads, all of them call it)
__device__ __forceinline__ void mq_block_scan(mq_layer_shared &L, int v, int tid, int nt)
{
    L.tsum[tid] = v;
    __syncthreads();
    for (int off = 1; off < nt; off <<= 1) {
        const int u = tid >= off ? L.tsum[tid - off] : 0;
        __syncthreads();
        L.tsum[tid] += u;
        __syncthreads();
    }
}

// One whole-layer search on the calling CTA (thread tid of nt <= 256), from the in-map start tile (tr, tc) whose
// CLOSEST_PATHABLE start is blocked. cp: N_ClosestPathable, leaving L.tile; otherwise n_closest_island_tiles of the start's
// global island, leaving L.n tile centres in list[0 .. L.n) in the reference's order (nav.c:4729-4732). scratch:
// mq_layer_scratch_words(W64, H64) words of this CTA's own.
__device__ __forceinline__ void mq_layer_search(mq_layer_shared &L, int32_t *scratch, const MapView &m, const uint16_t *gisl,
                                                int layer, bool cp, int tr, int tc, float2 *list, int tid, int nt)
{
    const int W = m.W64, H = m.H64, K = cp ? 4 : 9;
    const bool cheb = !cp;
    const int dr4[4] = {0, 0, -1, 1}, dc4[4] = {-1, 1, 0, 0};
    const int dr9[9] = {0, 0, 0, -1, 1, -1, -1, 1, 1}, dc9[9] = {0, -1, 1, 0, 0, -1, 1, -1, 1};
    const size_t P = mq_layer_positions(W, H), lbase = (size_t)layer * H * W;
    int32_t *ra = scratch, *rb = scratch + P, *order = scratch + 2 * P;
    uint32_t *bits = (uint32_t *)(scratch + 3 * P);
    int32_t *wpre = scratch + 3 * P + (9 * P + 31) / 32;
    const uint16_t giid = cp ? 0 : gisl[lbase + (size_t)tr * W + tc];
    const int dmax = cheb ? max(max(tr, H - 1 - tr), max(tc, W - 1 - tc)) : max(tr, H - 1 - tr) + max(tc, W - 1 - tc);
    if (tid == 0) {
        ra[0] = 0;
        L.nlev = 1; L.first_mh = -1; L.n = 0; L.done = 0; L.tile = -1;
    }
    __syncthreads();
    for (int d = 1; d <= dmax; d++) {
        const int npos = (cheb ? 8 : 4) * d, nb = (K * L.nlev + 31) / 32;
        for (int w = tid; w < nb; w += nt) bits[w] = 0;
        __syncthreads();
        // each tile's key: (rank of its first-ranked parent on level d-1) * K + the delta from that parent
        for (int p = tid; p < npos; p += nt) {
            int dr, dc;
            mq_ring_off(cheb, d, p, dr, dc);
            const int r = tr + dr, c = tc + dc;
            int key = -1;
            if (r >= 0 && r < H && c >= 0 && c < W) {
                key = 0x7fffffff;
                for (int e = 0; e < K; e++) {
                    const int pdr = dr - (cp ? dr4[e] : dr9[e]), pdc = dc - (cp ? dc4[e] : dc9[e]);
                    const int pr = tr + pdr, pc = tc + pdc;
                    if (pr < 0 || pr >= H || pc < 0 || pc >= W || mq_level(cheb, pdr, pdc) != d - 1) continue;
                    key = min(key, ra[mq_ring_pos(cheb, d - 1, pdr, pdc)] * K + e);
                }
                atomicOr(&bits[key >> 5], 1u << (key & 31));
            }
            rb[p] = key;
        }
        __syncthreads();
        // exclusive prefix of the bitmap's popcounts: a contiguous run of words per thread, then a scan of the runs
        const int per = (nb + nt - 1) / nt, w0 = min(tid * per, nb), w1 = min(w0 + per, nb);
        int s = 0;
        for (int w = w0; w < w1; w++) s += __popc(bits[w]);
        mq_block_scan(L, s, tid, nt);
        s = L.tsum[tid] - s;
        for (int w = w0; w < w1; w++) { wpre[w] = s; s += __popc(bits[w]); }
        __syncthreads();
        if (tid == 0) { L.nlev = L.tsum[nt - 1]; L.best = 0x7fffffff; }
        for (int p = tid; p < npos; p += nt) {
            const int key = rb[p];
            if (key < 0) continue;
            const int rank = wpre[key >> 5] + __popc(bits[key >> 5] & ((1u << (key & 31)) - 1u));
            rb[p] = rank;
            order[rank] = p;
        }
        __syncthreads();
        const int nlev = L.nlev;
        if (cp) {
            // the first tile popped that is neither impassable nor blocked
            for (int i = tid; i < nlev; i += nt) {
                int dr, dc;
                mq_ring_off(cheb, d, order[i], dr, dc);
                const size_t off = lbase + (size_t)(tr + dr) * W + tc + dc;
                if (!(m.cost[off] == 0xFF || m.blk[off] > 0)) atomicMin(&L.best, i);
            }
            __syncthreads();
            if (L.best != 0x7fffffff) {
                if (tid == 0) {
                    int dr, dc;
                    mq_ring_off(cheb, d, order[L.best], dr, dc);
                    L.tile = (tr + dr) * W + tc + dc;
                }
                __syncthreads();
                return;
            }
        } else {
            // the tiles met in rank order: list the island's tiles until the first one past the Manhattan cut, or 256
            for (int base = 0; base < nlev; base += nt) {
                const int i = base + tid;
                int dr = 0, dc = 0, mh = 0;
                bool listable = false;
                if (i < nlev) {
                    mq_ring_off(cheb, d, order[i], dr, dc);
                    const size_t off = lbase + (size_t)(tr + dr) * W + tc + dc;
                    listable = gisl[off] == giid && m.blk[off] == 0;
                    mh = mq_abs(dr) + mq_abs(dc);
                }
                if (tid == 0) { L.j = 0x7fffffff; L.cut = 0x7fffffff; L.add = 0; }
                __syncthreads();
                if (L.first_mh < 0 && listable) atomicMin(&L.j, i);
                __syncthreads();
                if (i == L.j) L.first_mh = mh;           // the first listed tile sets the cut
                __syncthreads();
                const int fm = L.first_mh, j = L.j;
                if (i < nlev && fm > 0 && mh > fm && (j == 0x7fffffff || i > j)) atomicMin(&L.cut, i);
                __syncthreads();
                const bool listed = listable && fm > 0 && i < L.cut;
                if (listed) atomicAdd(&L.add, 1);
                __syncthreads();
                if (L.add) {                             // the listed tiles' slots: an exclusive scan of the flags
                    mq_block_scan(L, listed, tid, nt);
                    const int k = L.n + L.tsum[tid] - listed;
                    if (listed && k < MQ_LIST_MAX)
                        list[k] = make_float2(m.map_x - (float)(tc + dc) * 4.0f, m.map_z + (float)(tr + dr) * 4.0f);
                    __syncthreads();
                }
                if (tid == 0) {
                    L.n = min(L.n + L.add, MQ_LIST_MAX);
                    if (L.n == MQ_LIST_MAX || L.cut != 0x7fffffff) L.done = 1;
                }
                __syncthreads();
                if (L.done) return;
            }
        }
        int32_t *t = ra; ra = rb; rb = t;
    }
}

// The searches k_map_search flagged, finished on the whole layer: writes out[idx[k]] as the host routine would.
// scratch: mq_layer_scratch_words(W64, H64) words plus a 256-entry list per CTA (mq_layer_cta_words).
__host__ __device__ __forceinline__ size_t mq_layer_cta_words(int W64, int H64) { return mq_layer_scratch_words(W64, H64) + 2 * MQ_LIST_MAX; }

__device__ __forceinline__ void mq_finish_one(mq_layer_shared &L, int32_t *scratch, const MapView &m, const uint16_t *gisl,
                                              const pfnav_map_query_req &a, pfnav_map_query_result *out, int tid, int nt)
{
    const bool cp = a.kind == PFNAV_QUERY_CLOSEST_PATHABLE;
    tile_desc td;
    desc_for_point(m, cp ? a.x : a.dst_x, cp ? a.z : a.dst_z, td);
    const int tr = td.chunk_r * 64 + td.tile_r, tc = td.chunk_c * 64 + td.tile_c;
    float2 *list = (float2 *)(scratch + mq_layer_scratch_words(m.W64, m.H64));
    mq_layer_search(L, scratch, m, gisl, a.layer, cp, tr, tc, list, tid, nt);
    pfnav_map_query_result r = {0, 0u, 0.0f, 0.0f};
    if (cp) {
        if (L.tile >= 0) {
            const int ar = L.tile / m.W64, ac = L.tile % m.W64;
            r.ok = 1;
            r.x = (m.map_x - (float)((ac >> 6) * 256)) - (float)((ac & 63) * 4);
            r.z = (m.map_z + (float)((ar >> 6) * 256)) + (float)((ar & 63) * 4);
        }
    } else {
        if (tid == 0) L.hit = 0;
        __syncthreads();
        for (int i = tid; i < L.n; i += nt) {
            const float dx = list[i].x - a.x, dz = list[i].y - a.z;
            if (sqrtf(dx * dx + dz * dz) <= a.tolerance) L.hit = 1;
        }
        __syncthreads();
        r.ok = L.hit;
    }
    if (tid == 0) *out = r;
    __syncthreads();
}

__global__ void __launch_bounds__(MQ_LAYER_THREADS) k_map_search_layer(MapView m, const uint16_t *__restrict__ gisl,
                                                                       const pfnav_map_query_req *__restrict__ q,
                                                                       const int32_t *__restrict__ idx, int ns,
                                                                       pfnav_map_query_result *__restrict__ out,
                                                                       const uint8_t *__restrict__ fallback, int32_t *scratch)
{
    __shared__ mq_layer_shared L;
    int32_t *mine = scratch + blockIdx.x * mq_layer_cta_words(m.W64, m.H64);
    for (int k = blockIdx.x; k < ns; k += gridDim.x) {
        if (!fallback[k]) continue;
        const int i = idx[k];
        mq_finish_one(L, mine, m, gisl, q[i], out + i, threadIdx.x, blockDim.x);
    }
}
