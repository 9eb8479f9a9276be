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
// The searches that would leave the window are finished here with the host routine pfnav_arrival_consts.
// pfnav_map_query_resident takes the positions of resident entities by uid: k_resident_xz (pfnav_region.cu) writes them
// into the uploaded queries before the same kernels run.
#include "pfnav_internal.cuh"
#include <algorithm>
#include <math.h>
#include <string.h>
#include "pfnav_map_view.cuh"
#include "pfnav_query_kernel.cuh"

static_assert(sizeof(pfnav_map_query_req) == 32, "pfnav_map_query_req must be 32 bytes");
static_assert(sizeof(pfnav_map_query_result) == 16, "pfnav_map_query_result must be 16 bytes");

// pfnav_map_query, and its resident form when P is not NULL: after the queries are uploaded, k_resident_xz writes P's
// named positions over (x, z) (the first array) and (dst_x, dst_z) (the second) of the device copy, and the searches'
// substituted records come back with the results for the host finish
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
    std::vector<uint8_t> fallback(ns);
    if (ns) {
        // the global islands of every layer are one image; layers without a route build are never read (validated above)
        const unsigned grid = (unsigned)std::min<size_t>(ns, (size_t)ctx->sm_count * 16);
        k_map_search<<<grid, 32, 0, st>>>(m, ctx->d_gisl, d_q, (const int32_t *)(dev + o_idx), (int)ns, d_out, dev + o_fb);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
        PF_CUDA(cudaMemcpyAsync(fallback.data(), dev + o_fb, ns, cudaMemcpyDeviceToHost, st));
    }
    PF_CUDA(cudaMemcpyAsync(out, d_out, n * sizeof(pfnav_map_query_result), cudaMemcpyDeviceToHost, st));
    // the resident form: the substituted records from the first search to the last, which the host finish reads
    std::vector<pfnav_map_query_req> sub;
    if (named && ns) {
        sub.resize((size_t)(search.back() - search.front()) + 1);
        PF_CUDA(cudaMemcpyAsync(sub.data(), d_q + search.front(), sub.size() * sizeof(pfnav_map_query_req),
                                cudaMemcpyDeviceToHost, st));
    }
    PF_CUDA(cudaStreamSynchronize(st));
    // the searches that left the window: the host routine on the host mirrors, which the last commit made equal to the
    // device images
    for (size_t k = 0; k < ns; k++) {
        if (!fallback[k]) continue;
        const pfnav_map_query_req &a = sub.empty() ? q[search[k]] : sub[search[k] - search.front()];
        pfnav_map_query_result &r = out[search[k]];
        pf_arrival_consts c;
        r = {0, 0u, 0.0f, 0.0f};
        if (a.kind == PFNAV_QUERY_CLOSEST_PATHABLE) {
            int rc = pfnav_arrival_consts(ctx, a.layer, a.x, a.z, &c, PF_ARRIVAL_NEAREST);
            if (rc) return rc;
            r.ok = c.nearest_ok; r.x = c.nearest[0]; r.z = c.nearest[1];
        } else {
            int rc = pfnav_arrival_consts(ctx, a.layer, a.dst_x, a.dst_z, &c, PF_ARRIVAL_MC);
            if (rc) return rc;
            for (int i = 0; i < c.mc_n && !r.ok; i++) {
                const float dx = c.mc[i][0] - a.x, dz = c.mc[i][1] - a.z;
                r.ok = sqrtf(dx * dx + dz * dz) <= a.tolerance;
            }
        }
    }
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
