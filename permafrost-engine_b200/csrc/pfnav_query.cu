// pfnav_query.cu -- pfnav_map_query: the engine's map point queries (seam B3, src/navigation/public/nav.h) answered in
// batches from the device's committed map state.
//
// Restates (reference file:line):
//   N_PositionPathable / N_PositionBlocked (M_NavPosition*)   src/navigation/nav.c:4055, 4070; src/map/map.c:817-845
//   N_IsAdjacentToImpassable                                  src/navigation/nav.c:4745
//   N_ClosestPathable                                         src/navigation/nav.c:4126
//   N_IsMaximallyClose -> n_closest_island_tiles              src/navigation/nav.c:4707, 1226
//   N_DestIDForPos / N_DestIDForPosAttacking (n_dest_id)      src/navigation/nav.c:839
//
// Kernels (pfnav_query_kernel.cuh): k_map_probe, one thread per query, answers the probe kinds and DEST_ID; k_map_search,
// one warp per CLOSEST_PATHABLE / MAXIMALLY_CLOSE query, replays the reference's search inside a window of the layer.
// The searches that would leave the window are finished on the device by k_map_search_layer, one CTA per search over
// the whole layer.
// pfnav_map_query_resident takes the positions of resident entities by uid: k_resident_xz (pfnav_region.cu) writes them
// into the uploaded queries before the same kernels run.
#include "pfnav_internal.cuh"
#include <algorithm>
#include <math.h>
#include <string.h>
#include "pfnav_map_view.cuh"
#include "pfnav_query_kernel.cuh"
#include "pfnav_layer_search.cuh"

static_assert(sizeof(pfnav_map_query_req) == 32, "pfnav_map_query_req must be 32 bytes");
static_assert(sizeof(pfnav_map_query_result) == 16, "pfnav_map_query_result must be 16 bytes");

// the searches k_map_search flagged (d_fallback), finished over the whole layer on `st`
static int pf_map_search_layer(pfnav_ctx *ctx, cudaStream_t st, const MapView &m, const pfnav_map_query_req *d_q, const int32_t *d_idx,
                        int ns, pfnav_map_query_result *d_out, const uint8_t *d_fallback)
{
    const unsigned grid = (unsigned)std::min<size_t>((size_t)ns, (size_t)ctx->sm_count);
    if (int rc = ctx->d_layer_scratch.reserve(grid * mq_layer_cta_words(ctx->W64, ctx->H64))) return rc;
    k_map_search_layer<<<grid, MQ_LAYER_THREADS, 0, st>>>(m, ctx->d_gisl, d_q, d_idx, ns, d_out, d_fallback, ctx->d_layer_scratch);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}

// pfnav_map_query, and its resident form when P is not NULL: after the queries are uploaded, k_resident_xz writes P's
// named positions over (x, z) (the first array) and (dst_x, dst_z) (the second) of the device copy
static int map_query(pfnav_ctx *ctx, const pfnav_map_query_req *q, size_t n, pfnav_map_query_result *out, void *stream,
                     const pf_resident_points *P)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_cost, "map not created");
    if (n == 0) return PFNAV_OK;
    PF_ARG(q && out, "null argument");
    PF_ARG(n <= 0x7fffffff, "n");
    std::vector<int32_t> search;
    for (size_t i = 0; i < n; i++) {
        const pfnav_map_query_req &a = q[i];
        PF_ARG(a.kind >= PFNAV_QUERY_PATHABLE && a.kind <= PFNAV_QUERY_DEST_ID, "query kind");
        PF_ARG(a.layer >= 0 && a.layer < ctx->nlayers, "query layer");
        if (a.kind == PFNAV_QUERY_MAXIMALLY_CLOSE) {
            PF_ARG(isfinite(a.tolerance), "MAXIMALLY_CLOSE tolerance must be finite");
            PF_ARG(pfnav_route_dev_islands(ctx, a.layer), "MAXIMALLY_CLOSE needs pfnav_route_build(layer) (global islands, nav.c:1731)");
        }
        if (a.kind == PFNAV_QUERY_DEST_ID) PF_ARG(a.faction_id >= 0 && a.faction_id <= PFNAV_FACTION_ID_NONE, "DEST_ID faction_id");
        if (a.kind == PFNAV_QUERY_CLOSEST_PATHABLE || a.kind == PFNAV_QUERY_MAXIMALLY_CLOSE) search.push_back((int32_t)i);
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    const cudaStream_t st = pf_stream(ctx, stream);
    PF_CUDA(pf_fields_join(ctx, st));
    // one device buffer: queries, results, search indices, fallback flags
    const size_t ns = search.size();
    const size_t o_res = n * sizeof(pfnav_map_query_req), o_idx = o_res + n * sizeof(pfnav_map_query_result);
    const size_t o_fb = o_idx + ns * 4, need = o_fb + ns;
    if (int rc = ctx->d_mq_buf.reserve(need)) return rc;
    uint8_t *dev = ctx->d_mq_buf;
    const pfnav_map_query_req *d_q = (const pfnav_map_query_req *)dev;
    pfnav_map_query_result *d_out = (pfnav_map_query_result *)(dev + o_res);
    PF_CUDA(cudaMemcpyAsync(dev, q, o_res, cudaMemcpyHostToDevice, st));
    if (ns) PF_CUDA(cudaMemcpyAsync(dev + o_idx, search.data(), ns * 4, cudaMemcpyHostToDevice, st));
    const bool named = P && !P->entry.empty();
    if (named) {
        // the pairs through the request staging; x, z are floats 2, 3 and dst_x, dst_z floats 4, 5 of a 32-byte record
        pf_stage S;
        if (int rc = pf_stage_begin(ctx, st, P->bytes(), P->bytes(), false, &S)) return rc;
        P->pack(S.host);
        if (int rc = pf_stage_upload(ctx, st, S, P->bytes())) return rc;
        if (int rc = pf_resident_xz_launch(ctx, st, S.dev, *P, 8, 2, 4, (float *)dev)) return rc;
        if (int rc = pf_stage_done(ctx, st)) return rc;
    }
    MapView m;
    m.cost = ctx->d_cost; m.blk = ctx->d_blk; m.W64 = ctx->W64; m.H64 = ctx->H64;
    m.chunk_w = ctx->chunk_w; m.chunk_h = ctx->chunk_h; m.map_x = ctx->map_x; m.map_z = ctx->map_z;
    k_map_probe<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(m, d_q, (int)n, d_out);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    if (ns) {
        // the global islands of every layer are one image; layers without a route build are never read (validated above)
        const unsigned grid = (unsigned)std::min<size_t>(ns, (size_t)ctx->sm_count * 16);
        k_map_search<<<grid, 32, 0, st>>>(m, ctx->d_gisl, d_q, (const int32_t *)(dev + o_idx), (int)ns, d_out, dev + o_fb);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
        if (int rc = pf_map_search_layer(ctx, st, m, d_q, (const int32_t *)(dev + o_idx), (int)ns, d_out, dev + o_fb)) return rc;
    }
    PF_CUDA(cudaMemcpyAsync(out, d_out, n * sizeof(pfnav_map_query_result), cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

extern "C" int pfnav_map_query(pfnav_ctx *ctx, const pfnav_map_query_req *q, size_t n, pfnav_map_query_result *out, void *stream)
{
    return map_query(ctx, q, n, out, stream, nullptr);
}

extern "C" int pfnav_map_query_resident(pfnav_ctx *ctx, const pfnav_map_query_req *q, const uint32_t *pos_uids,
                                        const uint32_t *dst_uids, size_t n, pfnav_map_query_result *out, void *stream)
{
    PF_ARG(ctx, "ctx");
    pf_resident_points P;
    if (int rc = pf_resident_points_begin(ctx, "map queries", n, pos_uids, q != nullptr, dst_uids, q != nullptr, P)) return rc;
    return map_query(ctx, q, n, out, stream, &P);
}

// ------------------------------------------------------------------------------------------
// The constants of arrived() (movement.c:2170-2196) per used (flock, layer) pair, built on the device: N_ClosestPathable
// and the tile list of n_closest_island_tiles from the flock target, exactly as pfnav_arrival_consts computes them on the
// host. k_arrival_window replays both searches in the 32 x 32 and 128 x 128 windows, one warp per pair, and flags the
// searches that leave them (flags[2 s] N_ClosestPathable, flags[2 s + 1] the list); k_arrival_layer finishes the flagged
// ones over the whole layer. Pair s writes arr[flock * nlayers + layer] and its list at tiles[s * 256].
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32) k_arrival_window(MapView m, const uint16_t *__restrict__ gisl,
                                                       const pf_arrival_pair *__restrict__ pairs, int npairs, int nlayers,
                                                       pf_arrival_dev *__restrict__ arr, float2 *__restrict__ tiles,
                                                       uint8_t *__restrict__ flags)
{
    __shared__ mq_shared S;
    __shared__ pfnav_map_query_result R;
    __shared__ uint8_t fb;
    const int lane = threadIdx.x & 31;
    for (int s = blockIdx.x; s < npairs; s += gridDim.x) {
        const pf_arrival_pair P = pairs[s];
        pf_arrival_dev d = {0, {0.0f, 0.0f}, 0, s * MQ_LIST_MAX, {0, 0, 0}};
        tile_desc td;
        const bool on_map = desc_for_point(m, P.tx, P.tz, td);
        pfnav_map_query_req a = {PFNAV_QUERY_CLOSEST_PATHABLE, P.layer, P.tx, P.tz, P.tx, P.tz, 0.0f, 0};
        mq_search(S, m, gisl, a, &R, &fb, lane);
        d.nearest_ok = R.ok; d.nearest[0] = R.x; d.nearest[1] = R.z;
        const uint8_t fb_cp = fb;
        uint8_t fb_mc = 0;
        if (on_map) {
            a.kind = PFNAV_QUERY_MAXIMALLY_CLOSE;
            mq_search(S, m, gisl, a, &R, &fb, lane);
            fb_mc = fb;
            if (!fb_mc) {
                d.mc_n = S.n;
                for (int i = lane; i < S.n; i += 32) {
                    const int t = S.list[i];
                    tiles[(size_t)s * MQ_LIST_MAX + i] = make_float2(m.map_x - (float)(S.c0 + t % S.dim) * 4.0f,
                                                                     m.map_z + (float)(S.r0 + t / S.dim) * 4.0f);
                }
            }
        }
        if (lane == 0) {
            arr[(size_t)P.flock * nlayers + P.layer] = d;
            flags[2 * s] = fb_cp; flags[2 * s + 1] = fb_mc;
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(MQ_LAYER_THREADS) k_arrival_layer(MapView m, const uint16_t *__restrict__ gisl,
                                                                    const pf_arrival_pair *__restrict__ pairs, int npairs,
                                                                    int nlayers, pf_arrival_dev *__restrict__ arr,
                                                                    float2 *__restrict__ tiles, const uint8_t *__restrict__ flags,
                                                                    int32_t *scratch)
{
    __shared__ mq_layer_shared L;
    int32_t *mine = scratch + blockIdx.x * mq_layer_cta_words(m.W64, m.H64);
    for (int k = blockIdx.x; k < 2 * npairs; k += gridDim.x) {
        if (!flags[k]) continue;
        const int s = k >> 1;
        const bool cp = !(k & 1);
        const pf_arrival_pair P = pairs[s];
        tile_desc td;
        desc_for_point(m, P.tx, P.tz, td);
        const int tr = td.chunk_r * 64 + td.tile_r, tc = td.chunk_c * 64 + td.tile_c;
        mq_layer_search(L, mine, m, gisl, P.layer, cp, tr, tc, tiles + (size_t)s * MQ_LIST_MAX, threadIdx.x, blockDim.x);
        if (threadIdx.x == 0) {
            pf_arrival_dev &d = arr[(size_t)P.flock * nlayers + P.layer];
            if (!cp) d.mc_n = L.n;
            else if (L.tile >= 0) {
                const int ar = L.tile / m.W64, ac = L.tile % m.W64;
                d.nearest_ok = 1;
                d.nearest[0] = (m.map_x - (float)((ac >> 6) * 256)) - (float)((ac & 63) * 4);
                d.nearest[1] = (m.map_z + (float)((ar >> 6) * 256)) + (float)((ar & 63) * 4);
            }
        }
        __syncthreads();
    }
}

int pf_arrival_search(pfnav_ctx *ctx, cudaStream_t st, const pf_arrival_pair *d_pairs, int npairs, pf_arrival_dev *d_arr,
                      float2 *d_tiles, uint8_t *d_flags)
{
    MapView m;
    m.cost = ctx->d_cost; m.blk = ctx->d_blk; m.W64 = ctx->W64; m.H64 = ctx->H64;
    m.chunk_w = ctx->chunk_w; m.chunk_h = ctx->chunk_h; m.map_x = ctx->map_x; m.map_z = ctx->map_z;
    const unsigned grid = (unsigned)std::min<size_t>((size_t)npairs, (size_t)ctx->sm_count * 16);
    k_arrival_window<<<grid, 32, 0, st>>>(m, ctx->d_gisl, d_pairs, npairs, ctx->nlayers, d_arr, d_tiles, d_flags);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    const unsigned lgrid = (unsigned)std::min<size_t>(2 * (size_t)npairs, (size_t)ctx->sm_count);
    if (int rc = ctx->d_arrival_scratch.reserve(lgrid * mq_layer_cta_words(ctx->W64, ctx->H64))) return rc;
    k_arrival_layer<<<lgrid, MQ_LAYER_THREADS, 0, st>>>(m, ctx->d_gisl, d_pairs, npairs, ctx->nlayers, d_arr, d_tiles, d_flags,
                                                        ctx->d_arrival_scratch);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// ENTER_ENTITY_RANGE's N_IsMaximallyClose(new_pos, target, 0) (movement.c:2583-2584) for the candidates k_entity_update
// appended: the same query as pfnav_map_query's MAXIMALLY_CLOSE, so the same list and the same tolerance test as the host
// routine. k_enter_window runs the window tiers, one warp per candidate, and finishes the candidate's patch; the searches
// that leave the 128 x 128 window are appended to `flagged` and k_enter_layer finishes them over the whole layer. Both
// read their counts on the device: with no candidates they return at once.
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ void enter_finish(pfnav_patch *patches, const pf_enter_cand &c, bool hit)
{
    pfnav_patch p = patches[c.wi];
    pf_enter_range_tail(p, hit, c.tx, c.tz, c.prev_x, c.prev_z);
    patches[c.wi] = p;
}

__global__ void __launch_bounds__(32) k_enter_window(MapView m, const uint16_t *__restrict__ gisl,
                                                     const pf_enter_cand *__restrict__ cands, uint32_t *__restrict__ count,
                                                     uint32_t *__restrict__ flagged, pfnav_patch *__restrict__ patches)
{
    __shared__ mq_shared S;
    __shared__ pfnav_map_query_result R;
    __shared__ uint8_t fb;
    const int lane = threadIdx.x & 31;
    const uint32_t n = count[0];
    for (uint32_t k = blockIdx.x; k < n; k += gridDim.x) {
        const pf_enter_cand c = cands[k];
        const pfnav_map_query_req a = {PFNAV_QUERY_MAXIMALLY_CLOSE, c.layer, c.nx, c.nz, c.tx, c.tz, 0.0f, 0};
        mq_search(S, m, gisl, a, &R, &fb, lane);
        if (lane == 0) {
            if (fb) flagged[atomicAdd(&count[1], 1u)] = k;
            else enter_finish(patches, c, R.ok != 0);
        }
        __syncwarp();
    }
}

__global__ void __launch_bounds__(MQ_LAYER_THREADS) k_enter_layer(MapView m, const uint16_t *__restrict__ gisl,
                                                                  const pf_enter_cand *__restrict__ cands,
                                                                  const uint32_t *__restrict__ count,
                                                                  const uint32_t *__restrict__ flagged,
                                                                  pfnav_patch *__restrict__ patches, int32_t *scratch)
{
    __shared__ mq_layer_shared L;
    __shared__ pfnav_map_query_result R;
    int32_t *mine = scratch + blockIdx.x * mq_layer_cta_words(m.W64, m.H64);
    const uint32_t n = count[1];
    for (uint32_t k = blockIdx.x; k < n; k += gridDim.x) {
        const pf_enter_cand c = cands[flagged[k]];
        const pfnav_map_query_req a = {PFNAV_QUERY_MAXIMALLY_CLOSE, c.layer, c.nx, c.nz, c.tx, c.tz, 0.0f, 0};
        mq_finish_one(L, mine, m, gisl, a, &R, threadIdx.x, blockDim.x);
        if (threadIdx.x == 0) enter_finish(patches, c, R.ok != 0);
        __syncthreads();
    }
}

int pf_enter_range_search(pfnav_ctx *ctx, cudaStream_t st, const pf_enter_cand *d_cand, uint32_t *d_count,
                          uint32_t *d_flagged, int nwork, pfnav_patch *d_patches)
{
    MapView m;
    m.cost = ctx->d_cost; m.blk = ctx->d_blk; m.W64 = ctx->W64; m.H64 = ctx->H64;
    m.chunk_w = ctx->chunk_w; m.chunk_h = ctx->chunk_h; m.map_x = ctx->map_x; m.map_z = ctx->map_z;
    // the layer tier shares the arrival tiers' scratch: both run on `st`, after refresh_arrival_consts
    const unsigned lgrid = (unsigned)std::max(ctx->sm_count, 1);
    if (int rc = ctx->d_arrival_scratch.reserve(lgrid * mq_layer_cta_words(ctx->W64, ctx->H64))) return rc;
    // about 37 KB of static shared memory per window CTA: a few resident per SM, the rest follow as they retire
    const unsigned grid = (unsigned)std::min<size_t>((size_t)nwork, (size_t)lgrid * 4);
    k_enter_window<<<grid, 32, 0, st>>>(m, ctx->d_gisl, d_cand, d_count, d_flagged, d_patches);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    k_enter_layer<<<lgrid, MQ_LAYER_THREADS, 0, st>>>(m, ctx->d_gisl, d_cand, d_count, d_flagged, d_patches,
                                                      ctx->d_arrival_scratch);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}
