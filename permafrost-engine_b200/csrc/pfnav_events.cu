// pfnav_events.cu -- the tick's decisions for the engine as a compact event list built on the device (sm_90a).
//
// pfnav_agents_collect_events decides and compacts in work order with the ordered compaction of pfnav_scan.cuh, as
// pfnav_agents_set_work_dev builds the work list: one launch keeps every warp's ballot of the work items that give an
// event (pf_event_wanted, pfnav_events_kernel.cuh) and the block's count, one CTA turns the counts into offsets and
// writes the number of events, and the last launch writes the events (pf_event_make) of the set ballot bits behind
// their block's offset. Only the items that give an event are read twice.
#include "pfnav_internal.cuh"
#include "pfnav_events_kernel.cuh"
#include "pfnav_scan.cuh"

// ctx->d_event_aux: the block offsets, the count, then one ballot word per 32 work items
#define EV_AUX_COUNT 1024
#define EV_AUX_BAL 1025

// the event list's compaction (pfnav_scan.cuh) over the work items
struct events_compact {
    const pfnav_patch *patches; const pfnav_agent *agents; const uint32_t *work; pfnav_event *out;
    __device__ bool keep(int i) const { return pf_event_wanted(patches, agents, work, i); }
    __device__ void emit(int i, uint32_t slot) const
    {
        const pfnav_event e = pf_event_make(patches, agents, work, i);
        // 48-byte records from a cudaMalloc base: every record starts on 16 bytes
        uint4 *d = reinterpret_cast<uint4 *>(out + slot);
        d[0] = make_uint4(e.uid, e.flags, e.todo, (uint32_t)e.attack);
        d[1] = make_uint4(e.state_before, e.state_after, __float_as_uint(e.dest[0]), __float_as_uint(e.dest[1]));
        d[2] = make_uint4(__float_as_uint(e.pos[0]), __float_as_uint(e.pos[1]), 0u, 0u);
    }
};

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
    const pf_compact_grid g = pf_compact_grid_of(n);
    ctx->events_valid = false;              // a failed reservation may have dropped the previous list
    int rc;
    if ((rc = ctx->d_events.reserve(std::max(n, 1)))) return rc;
    if ((rc = ctx->d_event_aux.reserve(EV_AUX_BAL + ((size_t)n + 31) / 32))) return rc;
    if (!ctx->events_done) PF_CUDA(cudaEventCreateWithFlags(&ctx->events_done, cudaEventDisableTiming));
    if (!ctx->h_event_count) PF_CUDA(cudaMallocHost(&ctx->h_event_count, 4));
    uint32_t *part = ctx->d_event_aux, *d_count = part + EV_AUX_COUNT, *bal = part + EV_AUX_BAL;
    if (n) {
        const events_compact f = {ctx->d_patches, ctx->d_agents, ctx->d_work, ctx->d_events};
        k_compact_count<<<g.nb, PF_COMPACT_THREADS, 0, st>>>(f, 0, n, g.per, bal, part);
        k_compact_offsets<events_compact><<<1, PF_COMPACT_THREADS, 0, st>>>(part, g.nb, d_count);
        k_compact_write<<<g.nb, PF_COMPACT_THREADS, 0, st>>>(f, 0, n, g.per, bal, part);
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
