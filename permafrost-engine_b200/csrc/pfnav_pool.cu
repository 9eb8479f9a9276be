// pfnav_pool.cu -- the field pool: its device copies, the entry points that manage it, the context-level forms of the
// slot policies of pfnav_pool_host.h, and the save and restore of the whole pool (pfnav_pool_save / pfnav_pool_restore)
// with their kernels: the map digest, and the pack and unpack of the stored fields.
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

// ---- save and restore ----

// One CTA per (layer, chunk) block of the row-major device images: the wrapping sum of pf_digest_tile over the block's
// 4096 tiles, then pf_digest_block added to *out. Every sum is a wrapping integer sum, so the bits do not depend on the
// launch configuration or the order in which blocks finish.
__global__ void __launch_bounds__(256) k_map_digest(const uint8_t *__restrict__ cost, const uint16_t *__restrict__ blk,
                                                    const uint16_t *__restrict__ liid, const uint16_t *__restrict__ fmask,
                                                    int chunk_w, int W64, int chunks, unsigned long long *__restrict__ out)
{
    const int layer = blockIdx.x / chunks, chunk = blockIdx.x - layer * chunks;
    const int cr = chunk / chunk_w, cc = chunk - cr * chunk_w;
    const size_t lbase = (size_t)layer * chunks * 4096;
    uint64_t sum = 0;
    for (uint32_t t = threadIdx.x; t < 4096; t += blockDim.x) {
        const size_t i = lbase + (size_t)(cr * 64 + (t >> 6)) * W64 + cc * 64 + (t & 63);
        sum += pf_digest_tile(t, cost[i], blk[i], liid[i], fmask[i]);
    }
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xFFFFFFFFu, sum, o);
    __shared__ uint64_t warp_sum[8];
    if (pf_lane() == 0) warp_sum[threadIdx.x >> 5] = sum;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint64_t b = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); w++) b += warp_sum[w];
        atomicAdd(out, (unsigned long long)pf_digest_block(b, layer, chunk));
    }
}

// k_pool_pack: the device touch stamps into out_touch, zeros up to the section's padded length ntouch, and the flow then
// LOS field of slot slots[b] into 16-byte words [b * 512, b * 512 + 512) of out_fields (one CTA per stored slot).
// k_pool_unpack: the reverse, without the padding.
__global__ void __launch_bounds__(256) k_pool_pack(const int32_t *__restrict__ slots, int nstored, const uint4 *__restrict__ flow,
                                                   const uint4 *__restrict__ los, const uint32_t *__restrict__ touch, int max,
                                                   int ntouch, uint32_t *__restrict__ out_touch, uint4 *__restrict__ out_fields)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < ntouch; i += gridDim.x * blockDim.x)
        out_touch[i] = i < max ? touch[i] : 0u;
    for (int b = blockIdx.x; b < nstored; b += gridDim.x) {
        const size_t s = (size_t)slots[b] * 256;
        for (int w = threadIdx.x; w < 512; w += blockDim.x)
            out_fields[(size_t)b * 512 + w] = w < 256 ? flow[s + w] : los[s + w - 256];
    }
}

__global__ void __launch_bounds__(256) k_pool_unpack(const int32_t *__restrict__ slots, int nstored, uint4 *__restrict__ flow,
                                                     uint4 *__restrict__ los, uint32_t *__restrict__ touch, int max,
                                                     const uint32_t *__restrict__ in_touch, const uint4 *__restrict__ in_fields)
{
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < max; i += gridDim.x * blockDim.x) touch[i] = in_touch[i];
    for (int b = blockIdx.x; b < nstored; b += gridDim.x) {
        const size_t s = (size_t)slots[b] * 256;
        for (int w = threadIdx.x; w < 512; w += blockDim.x) {
            const uint4 v = in_fields[(size_t)b * 512 + w];
            if (w < 256) flow[s + w] = v;
            else los[s + w - 256] = v;
        }
    }
}

int pf_map_digest_launch(pfnav_ctx *ctx, cudaStream_t st, unsigned long long *d_sum)
{
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    k_map_digest<<<(unsigned)(ctx->nlayers * chunks), 256, 0, st>>>(ctx->d_cost, ctx->d_blk, ctx->d_liid, ctx->d_fmask,
                                                                     ctx->chunk_w, ctx->W64, chunks, d_sum);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}

// The context's map digest (pfnav_digest_host.h) on `st`; d_ckpt holds at least 16 bytes. Waits for `st`.
static int map_digest(pfnav_ctx *ctx, cudaStream_t st, uint64_t *out)
{
    unsigned long long *d = (unsigned long long *)ctx->d_ckpt.p;
    PF_CUDA(cudaMemsetAsync(d, 0, 8, st));
    if (int rc = pf_map_digest_launch(ctx, st, d)) return rc;
    uint64_t sum = 0;
    PF_CUDA(cudaMemcpyAsync(&sum, d, 8, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    *out = pf_digest_fold(sum, ctx->nlayers, ctx->chunk_w, ctx->chunk_h, ctx->map_x, ctx->map_z, ctx->enemies);
    return PFNAV_OK;
}

static pf_pool_target target_of(const pfnav_ctx *ctx, uint64_t digest)
{
    return {ctx->chunk_w, ctx->chunk_h, ctx->nlayers, ctx->pool.ndests, ctx->pool.max, digest};
}

// the staging of a save or restore in d_ckpt: the digest word, the stored slots' indices, then the device touch stamps
// and the fields exactly as they lie in the segment from L.dtouch on
static const size_t STAGE_SLOTS = 16;
static size_t stage_dev_at(size_t nstored) { return STAGE_SLOTS + ((nstored * 4 + 15) & ~(size_t)15); }

extern "C" int pfnav_pool_save(pfnav_ctx *ctx, void *out, size_t cap, size_t *out_size, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(out_size, "out_size == NULL");
    PF_ARG(ctx->pool.d_slot, "pool not created");
    if (pf_map_uncommitted(ctx)) {
        pfnav_set_error("pfnav_pool_save: blocker ops are not committed (the next pfnav_map_commit drops fields; save after it)");
        return PFNAV_ERR_STATE;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    PF_CUDA(pf_fields_join(ctx, st));
    PF_CUDA(pf_pool_refresh(ctx, st));
    const pf_pool &P = ctx->pool;
    // the stored slots come from the host `has` mirror: every writer of d_has copies it from P.has (pf_pool_stage_table,
    // pfnav_pool_put, pfnav_map_commit, k_pool_scatter of the zone batches)
    std::vector<int32_t> stored;
    const pf_pool_layout L = pf_pool_seg_plan(P, ctx->aux, stored);
    *out_size = L.size;
    if (!out || cap < L.size) {
        pfnav_set_error("pfnav_pool_save: the segment needs %zu bytes", L.size);
        return PFNAV_ERR_NOMEM;
    }
    const size_t o_dev = stage_dev_at(stored.size()), dev_bytes = L.size - L.dtouch;
    if (int rc = ctx->d_ckpt.reserve(o_dev + dev_bytes)) return rc;
    uint64_t digest = 0;
    if (int rc = map_digest(ctx, st, &digest)) return rc;
    uint8_t *o = (uint8_t *)out;
    pf_pool_seg_write(P, ctx->aux, target_of(ctx, digest), ctx->tick_no, stored, L, o);
    uint8_t *stage = ctx->d_ckpt.p;
    if (!stored.empty())
        PF_CUDA(cudaMemcpyAsync(stage + STAGE_SLOTS, stored.data(), stored.size() * 4, cudaMemcpyHostToDevice, st));
    const int grid = std::max<int>(1, (int)stored.size());
    k_pool_pack<<<grid, 256, 0, st>>>((const int32_t *)(stage + STAGE_SLOTS), (int)stored.size(), (const uint4 *)P.d_flow,
                                      (const uint4 *)P.d_los, P.d_touch, P.max, (int)((L.fields - L.dtouch) / 4),
                                      (uint32_t *)(stage + o_dev),
                                      (uint4 *)(stage + o_dev + (L.fields - L.dtouch)));
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    PF_CUDA(cudaMemcpyAsync(o + L.dtouch, stage + o_dev, dev_bytes, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}

extern "C" int pfnav_pool_restore(pfnav_ctx *ctx, const void *seg, size_t size, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->pool.d_slot, "pool not created");
    if (pf_map_uncommitted(ctx)) {
        pfnav_set_error("pfnav_pool_restore: blocker ops are not committed (the next pfnav_map_commit drops fields; restore "
                        "after it)");
        return PFNAV_ERR_STATE;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    if (int rc = ctx->d_ckpt.reserve(16)) return rc;
    uint64_t digest = 0;
    if (int rc = map_digest(ctx, st, &digest)) return rc;
    pf_pool_image I;
    const char *e = pf_pool_check(seg, size, target_of(ctx, digest), I);
    if (e) {
        pfnav_set_error("pfnav_pool_restore: %s", e);
        return PFNAV_ERR_ARG;
    }
    // nothing may still read or write the pool: the forked field work, and ticks on any stream
    PF_CUDA(pf_fields_sync(ctx));
    PF_CUDA(cudaDeviceSynchronize());
    const size_t nstored = I.stored.size(), o_dev = stage_dev_at(nstored), dev_bytes = I.L.size - I.L.dtouch;
    if (int rc = ctx->d_ckpt.reserve(o_dev + dev_bytes)) return rc;
    uint8_t *stage = ctx->d_ckpt.p;
    if (nstored) PF_CUDA(cudaMemcpyAsync(stage + STAGE_SLOTS, I.stored.data(), nstored * 4, cudaMemcpyHostToDevice, st));
    PF_CUDA(cudaMemcpyAsync(stage + o_dev, I.base + I.L.dtouch, dev_bytes, cudaMemcpyHostToDevice, st));
    pf_pool &P = ctx->pool;
    k_pool_unpack<<<std::max<int>(1, (int)nstored), 256, 0, st>>>((const int32_t *)(stage + STAGE_SLOTS), (int)nstored,
                                                                  (uint4 *)P.d_flow, (uint4 *)P.d_los, P.d_touch, P.max,
                                                                  (const uint32_t *)(stage + o_dev),
                                                                  (const uint4 *)(stage + o_dev + (I.L.fields - I.L.dtouch)));
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    pf_pool_load(I, P, ctx->aux, &ctx->tick_no);
    P.dev_stale = false;                      // every device copy is written here: slot table, `has`, touch stamps
    ctx->goal_batch.valid = false;
    pf_stage S;
    if (int rc = pf_stage_begin(ctx, st, 0, 0, true, &S)) return rc;
    if (int rc = pf_stage_upload(ctx, st, S, 0)) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    return PFNAV_OK;
}
