// pfnav_checkpoint.cu -- pfnav_agents_save and pfnav_agents_restore: the device-resident population of a context (its own
// range) as one checkpoint segment, and back. pfnav_checkpoint_host.h holds the format and its validation; the group form
// pfnav_group_restore is in pfnav_mgpu.cu.
#include "pfnav_internal.cuh"
#include <string.h>

// word w of the packed rows of [lo, lo + nrows): row w / row.words, word w % row.words of it (pf_ckpt_word_source)
__global__ void k_ckpt_pack(pf_ckpt_src src, pf_ckpt_row row, uint32_t tables, uint32_t lo, uint32_t nrows, uint4 *__restrict__ out)
{
    const size_t nw = (size_t)nrows * row.words;
    for (size_t w = (size_t)blockIdx.x * blockDim.x + threadIdx.x; w < nw; w += (size_t)gridDim.x * blockDim.x) {
        const uint32_t i = (uint32_t)(w / row.words), q = (uint32_t)(w - (size_t)i * row.words);
        int t;
        uint32_t k;
        pf_ckpt_word_source(row, tables, q, &t, &k);
        // selects, not an indexed parameter array: a dynamic index would put src in local memory
        const uint4 *base = t == 0 ? src.p[0] : t == 1 ? src.p[1] : t == 2 ? src.p[2] : t == 3 ? src.p[3] : src.p[4];
        const uint32_t words = t == 0 ? src.words[0] : t == 1 ? src.words[1] : t == 2 ? src.words[2] : t == 3 ? src.words[3] : src.words[4];
        out[w] = base[(size_t)(lo + i) * words + k];
    }
}

pf_ckpt_src pf_ckpt_sources(const pfnav_ctx *ctx)
{
    pf_ckpt_src src;
    const void *p[5] = {ctx->d_agents.p, ctx->d_movestate.p, ctx->d_ms_ext.p, ctx->d_formation.p, ctx->d_blocking.p};
    for (int t = 0; t < 5; t++) { src.p[t] = (const uint4 *)p[t]; src.words[t] = pf_ckpt_sizes[t] / 16; }
    return src;
}

uint32_t pf_ckpt_tables(const pfnav_ctx *ctx)
{
    return (ctx->movestate_set ? PF_CKPT_MS : 0u) | (ctx->d_ms_ext != nullptr ? PF_CKPT_EXT : 0u) |
           (ctx->d_formation != nullptr ? PF_CKPT_FORM : 0u) |
           (ctx->d_blocking != nullptr && ctx->blocking_n == ctx->n_agents ? PF_CKPT_BLK : 0u);
}

extern "C" int pfnav_agents_save(pfnav_ctx *ctx, void *out, size_t cap, size_t *out_size, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(out_size, "out_size == NULL");
    PF_ARG(ctx->d_agents, "agents not uploaded");
    if (ctx->updates_unapplied) {
        pfnav_set_error("pfnav_agents_save: the last update pass is not applied (save after the apply and the commit)");
        return PFNAV_ERR_STATE;
    }
    if (pf_blocker_ops_pending(ctx)) {
        pfnav_set_error("pfnav_agents_save: device blocker ops are not committed%s (save after pfnav_map_commit)",
                        pf_blocker_ops_unexchanged(ctx) ? " or exchanged" : "");
        return PFNAV_ERR_STATE;
    }
    const uint32_t tables = pf_ckpt_tables(ctx);
    const size_t lo = ctx->shard_lo, hi = ctx->shard_hi, nf = ctx->h_flocks.size();
    const size_t size = pf_ckpt_bytes(tables, nf, hi - lo);
    *out_size = size;
    if (!out || cap < size) {
        pfnav_set_error("pfnav_agents_save: the segment needs %zu bytes", size);
        return PFNAV_ERR_NOMEM;
    }
    const pf_ckpt_header h = pf_ckpt_header_make(tables, ctx->n_agents, lo, hi, ctx->hz, nf);
    uint8_t *o = (uint8_t *)out;
    memcpy(o, &h, sizeof(h));
    if (nf) memcpy(o + sizeof(h), ctx->h_flocks.data(), nf * sizeof(pfnav_flock));
    if (hi == lo) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    const pf_ckpt_row row = pf_ckpt_row_of(tables);
    const size_t bytes = (hi - lo) * (size_t)row.words * 16;
    if (int rc = ctx->d_ckpt.reserve(bytes)) return rc;
    const pf_ckpt_src src = pf_ckpt_sources(ctx);
    const size_t nw = bytes / 16;
    const int grid = (int)std::min<size_t>((nw + 255) / 256, (size_t)ctx->sm_count * 16);
    k_ckpt_pack<<<grid, 256, 0, st>>>(src, row, tables, (uint32_t)lo, (uint32_t)(hi - lo), (uint4 *)ctx->d_ckpt.p);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaMemcpyAsync(o + sizeof(h) + nf * sizeof(pfnav_flock), ctx->d_ckpt.p, bytes, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

int pf_ckpt_restore_ready(pfnav_ctx *ctx)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_cost, "map not created");
    return PFNAV_OK;
}

int pf_ckpt_restore_check(pfnav_ctx *ctx, const pf_ckpt_set &S, size_t *lo, size_t *hi)
{
    for (int l = 0; l < ctx->nlayers; l++)
        if (S.layers_used[l] && !pfnav_route_dev_islands(ctx, l)) {
            pfnav_set_error("pfnav_agents_restore: pfnav_route_build(layer %d) is needed: entities of a flock stand on it", l);
            return PFNAV_ERR_STATE;
        }
    if ((S.h.tables & PF_CKPT_BLK) && ctx->mgpu && !pf_mgpu_shares_blockers(ctx)) {
        pfnav_set_error("pfnav_agents_restore: the segments hold blocking records and the context is part of a multi-GPU job "
                        "that does not share blockers");
        return PFNAV_ERR_STATE;
    }
    int rank, world;
    pf_mgpu_rank_world(ctx, &rank, &world);
    return pfnav_mgpu_shard_range(S.h.n_total, rank, world, lo, hi);
}

int pf_ckpt_restore_apply(pfnav_ctx *ctx, const pf_ckpt_set &S, size_t lo, size_t hi, cudaStream_t st)
{
    const size_t n = hi - lo, nf = S.h.nflocks, m = std::max<size_t>(n, 1);     // an empty range still passes non-NULL tables
    const uint32_t T = S.h.tables;
    std::vector<pfnav_agent> a(m);
    std::vector<pfnav_movestate> ms((T & PF_CKPT_MS) ? m : 0);
    std::vector<pfnav_movestate_ext> ext((T & PF_CKPT_EXT) ? m : 0);
    std::vector<pfnav_formation_in> form((T & PF_CKPT_FORM) ? m : 0);
    std::vector<pfnav_blocking> blk((T & PF_CKPT_BLK) ? m : 0);
    pf_ckpt_gather(S, lo, hi, a.data(), ms.data(), ext.data(), form.data(), blk.data());
    std::vector<pfnav_flock> fl(nf);
    if (nf) memcpy(fl.data(), S.flocks, nf * sizeof(pfnav_flock));
    // the uploads of the same records: an upload drops the movestate_ext and formation tables of the previous population
    int rc = pfnav_agents_upload_shard(ctx, a.data(), lo, hi, S.h.n_total, fl.data(), nf, S.h.hz, 0);
    if (!rc && (T & PF_CKPT_MS)) rc = pfnav_agents_upload_movestate(ctx, ms.data(), n);
    if (!rc && (T & PF_CKPT_EXT)) rc = pfnav_agents_upload_movestate_ext(ctx, ext.data(), n);
    if (!rc && (T & PF_CKPT_FORM)) rc = pfnav_agents_upload_formation(ctx, form.data(), n);
    if (!rc && (T & PF_CKPT_BLK)) rc = pfnav_agents_upload_blocking(ctx, blk.data(), n);
    if (rc) return rc;
    if (!(T & PF_CKPT_MS)) ctx->movestate_set = false;
    if (!(T & PF_CKPT_BLK)) ctx->blocking_n = 0;
    ctx->updates_unapplied = false;
    // what an upload does not do: take the recorded blocks again, as device ops the next commit applies
    if (T & PF_CKPT_BLK) return blocking_restore_emit(ctx, st, lo, (int)n);
    return PFNAV_OK;
}

extern "C" int pfnav_agents_restore(pfnav_ctx *ctx, const void *const *segs, const size_t *sizes, size_t nseg, void *stream)
{
    if (int rc = pf_ckpt_restore_ready(ctx)) return rc;
    pf_ckpt_set S;
    const char *e = pf_ckpt_check(segs, sizes, nseg, ctx->nlayers, S);
    PF_ARG(!e, e);
    size_t lo = 0, hi = 0;
    if (int rc = pf_ckpt_restore_check(ctx, S, &lo, &hi)) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    return pf_ckpt_restore_apply(ctx, S, lo, hi, pf_stream(ctx, stream));
}
