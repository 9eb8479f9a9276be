// pfnav_events.cu -- the tick's decisions for the engine as a compact event list built on the device (sm_90a).
//
// pfnav_agents_collect_events decides and compacts in work order with the count / scan / compact shape of k_work_*:
// block b owns the work items [b * per, (b + 1) * per), per a multiple of 1024 and at most 1024 blocks. k_events_count
// keeps every warp's ballot of the items that give an event (pf_event_wanted, pfnav_events_kernel.cuh) and the block's
// total; k_events_scan turns the block totals into offsets and writes the count; k_events_compact writes the events
// (pf_event_make) of the set ballot bits behind their block's offset. Only the items that give an event are read twice.
#include "pfnav_internal.cuh"
#include "pfnav_events_kernel.cuh"

#define FULL 0xFFFFFFFFu
#define EV_THREADS 1024

// ctx->d_event_aux: the block offsets, the count, then one ballot word per 32 work items
#define EV_AUX_COUNT 1024
#define EV_AUX_BAL 1025

__global__ void __launch_bounds__(EV_THREADS) k_events_count(const pfnav_patch *__restrict__ patches,
                                                             const pfnav_agent *__restrict__ agents,
                                                             const uint32_t *__restrict__ work, int n, int per,
                                                             uint32_t *__restrict__ bal, uint32_t *__restrict__ part)
{
    __shared__ uint32_t wsum[EV_THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int b0 = blockIdx.x * per, b1 = min(b0 + per, n);
    uint32_t c = 0;
    for (int base = b0; base < b1; base += EV_THREADS) {
        const int i = base + threadIdx.x;
        const bool want = i < b1 && pf_event_wanted(patches, agents, work, i);
        const unsigned m = __ballot_sync(FULL, want);
        if (lane == 0 && i < b1) bal[i >> 5] = m;
        c += __popc(m);
    }
    if (lane == 0) wsum[wid] = c;
    __syncthreads();
    if (wid == 0) {
        uint32_t s = wsum[lane];
        for (int o = 16; o; o >>= 1) s += __shfl_down_sync(FULL, s, o);
        if (lane == 0) part[blockIdx.x] = s;
    }
}

// one block: part[0 .. nb) (nb <= 1024) become offsets, *count the number of events
__global__ void __launch_bounds__(EV_THREADS) k_events_scan(uint32_t *__restrict__ part, int nb, uint32_t *__restrict__ count)
{
    __shared__ uint32_t wsum[EV_THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const uint32_t v = (int)threadIdx.x < nb ? part[threadIdx.x] : 0;
    uint32_t x = v;
    for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULL, x, o); if (lane >= o) x += y; }
    if (lane == 31) wsum[wid] = x;
    __syncthreads();
    if (wid == 0) {
        uint32_t s = wsum[lane];
        for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULL, s, o); if (lane >= o) s += y; }
        wsum[lane] = s;
    }
    __syncthreads();
    if ((int)threadIdx.x < nb) part[threadIdx.x] = (wid ? wsum[wid - 1] : 0) + x - v;
    if (threadIdx.x == 0) *count = wsum[31];
}

__global__ void __launch_bounds__(EV_THREADS) k_events_compact(const pfnav_patch *__restrict__ patches,
                                                               const pfnav_agent *__restrict__ agents,
                                                               const uint32_t *__restrict__ work, int n, int per,
                                                               const uint32_t *__restrict__ bal,
                                                               const uint32_t *__restrict__ part, pfnav_event *__restrict__ out)
{
    __shared__ uint32_t wsum[EV_THREADS / 32];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int b0 = blockIdx.x * per, b1 = min(b0 + per, n);
    uint32_t o0 = part[blockIdx.x];
    for (int base = b0; base < b1; base += EV_THREADS) {
        const int i = base + threadIdx.x;
        const unsigned m = base + (wid << 5) < b1 ? bal[(base >> 5) + wid] : 0u;
        if (lane == 0) wsum[wid] = __popc(m);
        __syncthreads();
        if (wid == 0) {
            uint32_t s = wsum[lane];
            for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(FULL, s, o); if (lane >= o) s += y; }
            wsum[lane] = s;
        }
        __syncthreads();
        if ((m >> lane) & 1u) {
            const pfnav_event e = pf_event_make(patches, agents, work, i);
            // 48-byte records from a cudaMalloc base: every record starts on 16 bytes
            uint4 *d = reinterpret_cast<uint4 *>(out + o0 + (wid ? wsum[wid - 1] : 0) + __popc(m & ((1u << lane) - 1)));
            d[0] = make_uint4(e.uid, e.flags, e.todo, (uint32_t)e.attack);
            d[1] = make_uint4(e.state_before, e.state_after, __float_as_uint(e.dest[0]), __float_as_uint(e.dest[1]));
            d[2] = make_uint4(__float_as_uint(e.pos[0]), __float_as_uint(e.pos[1]), 0u, 0u);
        }
        o0 += wsum[31];
        __syncthreads();
    }
}

void pf_events_free(pfnav_ctx *ctx)
{
    if (ctx->events_done) cudaEventDestroy(ctx->events_done);
    if (ctx->h_event_count) cudaFreeHost(ctx->h_event_count);
    if (ctx->h_events) cudaFreeHost(ctx->h_events);
    ctx->events_done = nullptr; ctx->h_event_count = nullptr; ctx->h_events = nullptr; ctx->h_events_cap = 0;
}

extern "C" int pfnav_agents_collect_events(pfnav_ctx *ctx, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_patches && ctx->update_done, "no update pass has run");
    if (!ctx->updates_unapplied) {
        pfnav_set_error("pfnav_agents_collect_events: the last update pass has been applied (collect before the apply)");
        return PFNAV_ERR_STATE;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    const int n = (int)ctx->n_work;
    const int nb = std::min(1024, (n + EV_THREADS - 1) / EV_THREADS);
    const int per = nb ? ((n + nb - 1) / nb + EV_THREADS - 1) / EV_THREADS * EV_THREADS : 0;
    ctx->events_valid = false;              // a failed reservation may have dropped the previous list
    int rc;
    if ((rc = ctx->d_events.reserve(std::max(n, 1)))) return rc;
    if ((rc = ctx->d_event_aux.reserve(EV_AUX_BAL + ((size_t)n + 31) / 32))) return rc;
    if (!ctx->events_done) PF_CUDA(cudaEventCreateWithFlags(&ctx->events_done, cudaEventDisableTiming));
    if (!ctx->h_event_count) PF_CUDA(cudaMallocHost(&ctx->h_event_count, 4));
    uint32_t *part = ctx->d_event_aux, *d_count = part + EV_AUX_COUNT, *bal = part + EV_AUX_BAL;
    if (n) {
        k_events_count<<<nb, EV_THREADS, 0, st>>>(ctx->d_patches, ctx->d_agents, ctx->d_work, n, per, bal, part);
        k_events_scan<<<1, EV_THREADS, 0, st>>>(part, nb, d_count);
        k_events_compact<<<nb, EV_THREADS, 0, st>>>(ctx->d_patches, ctx->d_agents, ctx->d_work, n, per, bal, part, ctx->d_events);
        ctx->launches += 3;
        PF_CUDA(cudaGetLastError());
    } else {
        PF_CUDA(cudaMemsetAsync(d_count, 0, 4, st));
    }
    // the count lands in pinned memory behind the list; pfnav_agents_read_events waits for the event, not for the stream
    PF_CUDA(cudaMemcpyAsync(ctx->h_event_count, d_count, 4, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaEventRecord(ctx->events_done, st));
    ctx->events_valid = true;
    return PFNAV_OK;
}

extern "C" int pfnav_agents_read_events(pfnav_ctx *ctx, pfnav_event *out, size_t maxout, size_t *out_n)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(out_n, "out_n == NULL");
    PF_ARG(out || maxout == 0, "out == NULL with maxout > 0");
    if (!ctx->events_valid) {
        pfnav_set_error("pfnav_agents_read_events: no event list (no collect has run, or the population was renumbered "
                        "since)");
        return PFNAV_ERR_STATE;
    }
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaEventSynchronize(ctx->events_done));
    const size_t n = *ctx->h_event_count;
    *out_n = n;
    if (n > maxout) {
        pfnav_set_error("pfnav_agents_read_events: the list holds %zu events, out %zu", n, maxout);
        return PFNAV_ERR_NOMEM;
    }
    if (n == 0) return PFNAV_OK;
    if (ctx->h_events_cap < n) {
        const size_t want = std::max(n, 2 * ctx->h_events_cap);
        if (ctx->h_events) PF_CUDA(cudaFreeHost(ctx->h_events));
        ctx->h_events = nullptr; ctx->h_events_cap = 0;
        PF_CUDA(cudaMallocHost(&ctx->h_events, want * sizeof(pfnav_event)));
        ctx->h_events_cap = want;
    }
    // the legacy stream waits for none of the context's streams: the event above is the only wait
    PF_CUDA(cudaMemcpy(ctx->h_events, ctx->d_events, n * sizeof(pfnav_event), cudaMemcpyDeviceToHost));
    memcpy(out, ctx->h_events, n * sizeof(pfnav_event));
    return PFNAV_OK;
}
