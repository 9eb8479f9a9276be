// pfnav_pool.cu -- the field pool: its device copies, the entry points that manage it, and the context-level forms of
// the slot policies of pfnav_pool_host.h. No kernels.
#include <string.h>
#include "pfnav_internal.cuh"

cudaError_t pf_pool_refresh(pfnav_ctx *ctx, cudaStream_t st)
{
    pf_pool &P = ctx->pool;
    if (!P.dev_stale) return cudaSuccess;
    cudaError_t e = pf_fields_join(ctx, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(P.d_slot, 0xFF, P.slot.size() * sizeof(int32_t), st);
    if (e == cudaSuccess) e = cudaMemsetAsync(P.d_has, 0, P.max, st);
    if (e == cudaSuccess) e = cudaMemsetAsync(P.d_touch, 0, (size_t)P.max * 4, st);
    if (e == cudaSuccess) P.dev_stale = false;
    return e;
}

// pf_pool_refresh for entry points that go on with blocking copies (legacy default stream): wait for the reset
static cudaError_t pf_pool_refresh_sync(pfnav_ctx *ctx)
{
    if (!ctx->pool.dev_stale) return cudaSuccess;
    cudaError_t e = pf_pool_refresh(ctx, ctx->tick_stream);
    return e == cudaSuccess ? cudaStreamSynchronize(ctx->tick_stream) : e;
}

int pf_pool_free(pfnav_ctx *ctx)
{
    pf_pool &P = ctx->pool;
    if (ctx->device >= 0 && P.d_slot) {
        PF_CUDA(cudaSetDevice(ctx->device));
        PF_CUDA(cudaDeviceSynchronize());
        cudaFree(P.d_slot); cudaFree(P.d_flow); cudaFree(P.d_los); cudaFree(P.d_touch);
    }
    P = pf_pool();
    ctx->goal_batch.valid = false;
    return PFNAV_OK;
}

int pf_pool_reserve(pfnav_ctx *ctx, const size_t *keys, size_t n, int32_t *slots_out, bool *out_evicted)
{
    pf_pool &P = ctx->pool;
    const int rc = pf_pool_reserve(P, keys, n, ctx->tick_no, slots_out, out_evicted, [&](std::vector<uint32_t> &stamp) -> int {
        if (ctx->device < 0 || !P.d_touch || P.dev_stale) return PFNAV_OK;    // stale: cleared, no tick read a slot since
        PF_CUDA(cudaSetDevice(ctx->device));
        PF_CUDA(cudaDeviceSynchronize());         // ticks on any stream may still be stamping slots (eviction is rare)
        std::vector<uint32_t> dev(P.max);
        PF_CUDA(cudaMemcpy(dev.data(), P.d_touch, (size_t)P.max * 4, cudaMemcpyDeviceToHost));
        for (int s = 0; s < P.max; s++) stamp[s] = std::max(stamp[s], dev[s]);
        return PFNAV_OK;
    });
    if (rc == PFNAV_OK) ctx->goal_batch.valid = false;
    return rc;
}

int32_t pf_pool_zone_take(pfnav_ctx *ctx, size_t key)
{
    const int32_t s = pf_pool_zone_take(ctx->pool, key);
    if (s >= 0) ctx->goal_batch.valid = false;
    return s;
}

void pf_pool_drop(pfnav_ctx *ctx, int dest, int chunk)
{
    pf_pool_drop(ctx->pool, (size_t)dest * ctx->chunk_w * ctx->chunk_h + chunk);
    ctx->goal_batch.valid = false;
}

int pf_pool_stage_table(pfnav_ctx *ctx, uint8_t *host, cudaStream_t st)
{
    const pf_pool &P = ctx->pool;
    const size_t b_slot = P.slot.size() * 4;
    memcpy(host, P.slot.data(), b_slot);
    memcpy(host + b_slot, P.has.data(), P.max);
    PF_CUDA(cudaMemcpyAsync(P.d_slot, host, b_slot, cudaMemcpyHostToDevice, st));
    PF_CUDA(cudaMemcpyAsync(P.d_has, host + b_slot, P.max, cudaMemcpyHostToDevice, st));
    return PFNAV_OK;
}

extern "C" int pfnav_pool_create(pfnav_ctx *ctx, int ndests, int max_fields)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ndests > 0 && max_fields > 0, "ndests/max_fields");
    PF_CUDA(cudaSetDevice(ctx->device));
    if (int rc = pf_pool_free(ctx)) return rc;
    ctx->los_inflight = false;
    pf_pool &P = ctx->pool;
    const size_t nslots = (size_t)ndests * ctx->chunk_w * ctx->chunk_h;
    PF_CUDA(cudaMalloc(&P.d_slot, nslots * sizeof(int32_t)));
    PF_CUDA(cudaMalloc(&P.d_flow, (size_t)max_fields * 4096));
    PF_CUDA(cudaMalloc(&P.d_los, (size_t)max_fields * 4096 + max_fields));
    P.d_has = P.d_los + (size_t)max_fields * 4096;
    PF_CUDA(cudaMemset(P.d_slot, 0xFF, nslots * sizeof(int32_t)));
    PF_CUDA(cudaMemset(P.d_has, 0, max_fields));
    PF_CUDA(cudaMalloc(&P.d_touch, (size_t)max_fields * 4));
    PF_CUDA(cudaMemset(P.d_touch, 0, (size_t)max_fields * 4));
    P.slot.assign(nslots, -1); P.ffid.assign(nslots, 0);
    P.has.assign(max_fields, 0); P.req.assign(max_fields, pfnav_field_req{}); P.touch.assign(max_fields, 0); P.owner.assign(max_fields, -1);
    P.ndests = ndests; P.max = max_fields;
    return PFNAV_OK;
}

extern "C" int pfnav_pool_clear(pfnav_ctx *ctx)
{
    PF_ARG(ctx && ctx->pool.d_slot, "pool not created");
    // host mirrors only: the device copies are reset by the next entry point that uses the pool, on its stream
    // (pf_pool_refresh), so the clear neither waits for the GPU nor races a tick still reading the slot table
    pf_host_timer ht(ctx);
    pf_pool_reset(ctx->pool);
    ctx->goal_batch.valid = false;
    ctx->pool.dev_stale = true;
    ht.lap(PF_HPROF_CLEAR);
    return PFNAV_OK;
}

extern "C" int pfnav_pool_put(pfnav_ctx *ctx, int dest, int chunk_r, int chunk_c, const uint8_t *flow_field,
                              const uint8_t *los_field)
{
    PF_ARG(ctx && ctx->pool.d_slot, "pool not created");
    pf_pool &P = ctx->pool;
    PF_ARG(dest >= 0 && dest < P.ndests, "dest");
    PF_ARG(chunk_r >= 0 && chunk_r < ctx->chunk_h && chunk_c >= 0 && chunk_c < ctx->chunk_w, "chunk");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(pf_fields_sync(ctx));
    PF_CUDA(pf_pool_refresh_sync(ctx));
    const size_t si = (size_t)dest * ctx->chunk_w * ctx->chunk_h + chunk_r * ctx->chunk_w + chunk_c;
    int32_t slot = P.slot_of(si);
    if (slot < 0) {
        bool evicted = false;
        int rc = pf_pool_reserve(ctx, &si, 1, &slot, &evicted);
        if (rc) return rc;
        if (evicted) {
            PF_CUDA(cudaMemcpy(P.d_slot, P.slot.data(), P.slot.size() * 4, cudaMemcpyHostToDevice));
            PF_CUDA(cudaMemcpy(P.d_has, P.has.data(), P.max, cudaMemcpyHostToDevice));
        } else {
            PF_CUDA(cudaMemcpy(P.d_slot + si, &slot, sizeof(int32_t), cudaMemcpyHostToDevice));
        }
    }
    if (flow_field) { PF_CUDA(cudaMemcpy(P.d_flow + (size_t)slot * 4096, flow_field, 4096, cudaMemcpyHostToDevice)); P.built(slot, 1); }
    if (los_field) { PF_CUDA(cudaMemcpy(P.d_los + (size_t)slot * 4096, los_field, 4096, cudaMemcpyHostToDevice)); P.built(slot, 2); }
    PF_CUDA(cudaMemcpy(P.d_has + slot, &P.has[slot], 1, cudaMemcpyHostToDevice));
    ctx->goal_batch.valid = false;
    return PFNAV_OK;
}

// Read one pool entry back to the host (4096 B each; either pointer may be NULL). *out_has: bit0 flow, bit1 LOS.
extern "C" int pfnav_pool_get(pfnav_ctx *ctx, int dest, int chunk_r, int chunk_c, uint8_t *flow_out, uint8_t *los_out,
                              int *out_has, uint64_t *out_ffid)
{
    PF_ARG(ctx && ctx->pool.d_slot && out_has, "args");
    PF_NEED_DEVICE(ctx);
    const pf_pool &P = ctx->pool;
    PF_ARG(dest >= 0 && dest < P.ndests && chunk_r >= 0 && chunk_r < ctx->chunk_h && chunk_c >= 0 && chunk_c < ctx->chunk_w, "dest/chunk");
    const size_t si = (size_t)dest * ctx->chunk_w * ctx->chunk_h + chunk_r * ctx->chunk_w + chunk_c;
    const int slot = P.slot_of(si);
    *out_has = P.has_of(si);
    if (out_ffid) *out_ffid = P.ffid[si];
    if (slot < 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(pf_pool_refresh(ctx, ctx->tick_stream));
    PF_CUDA(cudaDeviceSynchronize());
    if (flow_out && (*out_has & 1)) PF_CUDA(cudaMemcpy(flow_out, P.d_flow + (size_t)slot * 4096, 4096, cudaMemcpyDeviceToHost));
    if (los_out && (*out_has & 2)) PF_CUDA(cudaMemcpy(los_out, P.d_los + (size_t)slot * 4096, 4096, cudaMemcpyDeviceToHost));
    return PFNAV_OK;
}
