// pfnav_mgpu.cu -- multi-GPU: entities (and with them their flocks' destinations) are partitioned by contiguous
// index range, the reference's own fork-join split (src/game/movement.c:3751-3762: equal ranges of the work
// array, one per task); every GPU updates its own range and needs every potential neighbour's 24-byte record
// {pos, vel, radius, state|flags} (SURVEY.md 8e) -> ONE all-gather of those records per tick, nothing else.
//
// Two transports behind the same per-tick call:
//   * NCCL, one process per GPU (pfnav_mgpu_init): libnccl.so.2 is resolved at run time with dlopen (the copy the
//     host program already loaded, e.g. torch's, else the system one); ncclAllGather in place on the record array,
//     stream-ordered on the caller's stream, NVLink / NVSwitch underneath.
//   * in-process group (pfnav_group_create): one engine process driving several contexts (on one or several
//     devices) from one thread, which is how the engine itself would use 8 GPUs; the ranges are pulled with
//     cudaMemcpyPeerAsync (NVLink peer copies between devices), ordered by events.
// The map, the field pool of the rank's own destinations and the spatial index are per rank; the index is rebuilt
// from the gathered records on every rank (identical order on all of them).
#include "pfnav_internal.cuh"
#include <dlfcn.h>
#include <string.h>
#include <algorithm>

// ---- minimal NCCL surface (nccl.h:  ncclUniqueId 128 bytes, ncclResult_t, ncclDataType_t ncclInt8 = 0) ----
typedef struct { char internal[128]; } pf_nccl_id;
typedef void *pf_nccl_comm;
typedef int (*fn_ncclGetUniqueId)(pf_nccl_id *);
typedef int (*fn_ncclCommInitRank)(pf_nccl_comm *, int, pf_nccl_id, int);
typedef int (*fn_ncclAllGather)(const void *, void *, size_t, int, pf_nccl_comm, cudaStream_t);
typedef int (*fn_ncclBroadcast)(const void *, void *, size_t, int, int, pf_nccl_comm, cudaStream_t);
typedef int (*fn_ncclGroup)(void);
typedef int (*fn_ncclCommDestroy)(pf_nccl_comm);
typedef const char *(*fn_ncclGetErrorString)(int);

struct pf_nccl_api {
    void *lib = nullptr;
    fn_ncclGetUniqueId GetUniqueId = nullptr; fn_ncclCommInitRank CommInitRank = nullptr;
    fn_ncclAllGather AllGather = nullptr; fn_ncclBroadcast Broadcast = nullptr;
    fn_ncclGroup GroupStart = nullptr, GroupEnd = nullptr;
    fn_ncclCommDestroy CommDestroy = nullptr; fn_ncclGetErrorString GetErrorString = nullptr;
};

static int nccl_load(pf_nccl_api &api)
{
    if (api.lib) return 0;
    const char *names[] = {"libnccl.so.2", "libnccl.so"};
    for (const char *nm : names) { api.lib = dlopen(nm, RTLD_NOW | RTLD_NOLOAD); if (api.lib) break; }     // already in the process?
    for (const char *nm : names) { if (api.lib) break; api.lib = dlopen(nm, RTLD_NOW | RTLD_GLOBAL); }
    if (!api.lib) { pfnav_set_error("pfnav_mgpu: libnccl.so.2 not found (%s)", dlerror()); return PFNAV_ERR_STATE; }
#define PF_SYM(name) api.name = (fn_nccl##name)dlsym(api.lib, "nccl" #name)
    PF_SYM(GetUniqueId); PF_SYM(CommInitRank); PF_SYM(AllGather); PF_SYM(Broadcast); PF_SYM(CommDestroy); PF_SYM(GetErrorString);
#undef PF_SYM
    api.GroupStart = (fn_ncclGroup)dlsym(api.lib, "ncclGroupStart");
    api.GroupEnd = (fn_ncclGroup)dlsym(api.lib, "ncclGroupEnd");
    if (!api.GetUniqueId || !api.CommInitRank || !api.AllGather || !api.Broadcast || !api.GroupStart || !api.GroupEnd || !api.CommDestroy) {
        pfnav_set_error("pfnav_mgpu: libnccl.so.2 lacks a required symbol");
        return PFNAV_ERR_STATE;
    }
    return 0;
}
static pf_nccl_api g_nccl;        // resolved symbols only (immutable after the first load)

struct pfnav_group {
    std::vector<pfnav_ctx *> ctxs;
    std::vector<cudaEvent_t> ready, pulled;      // per member: own range final / every peer range copied
};

struct pf_mgpu {
    int rank = 0, world = 1;
    pf_nccl_comm comm = nullptr;                 // NCCL transport
    pfnav_group *group = nullptr;                // in-process transport
    bool share_blockers = false;                 // pfnav_mgpu_share_blockers / pfnav_group_share_blockers
    pf_dbuf<uint32_t> d_xcnt;                    // NCCL: all-gathered records of PF_XCNT words per rank: the blocker
                                                 // exchange's counts, a command batch's verdicts; read before the call returns
    pf_dbuf<uint8_t> d_xgoal;                    // NCCL: the goal batch's all-gathered member records
};
#define PF_XCNT 8                                // {narrow, wide, sent narrow, sent wide, faction flag, 0, 0, 0}
                                                 // or {status, n_agents, n_flocks, tables present, 0, 0, 0, 0}

bool pf_mgpu_shares_blockers(const pfnav_ctx *ctx)
{
    const pf_mgpu *m = (const pf_mgpu *)ctx->mgpu;
    return m && m->share_blockers;
}

void pf_mgpu_rank_world(const pfnav_ctx *ctx, int *rank, int *world)
{
    const pf_mgpu *m = (const pf_mgpu *)ctx->mgpu;
    *rank = m ? m->rank : 0;
    *world = m ? m->world : 1;
}

#define PF_NCCL(call)                                                                                  \
    do {                                                                                               \
        int _r = (call);                                                                               \
        if (_r != 0) {                                                                                 \
            pfnav_set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #call,                              \
                            g_nccl.GetErrorString ? g_nccl.GetErrorString(_r) : "nccl error");         \
            return PFNAV_ERR_CUDA;                                                                     \
        }                                                                                              \
    } while (0)

// balanced contiguous ranges (movement.c:3751-3762 splits the work array the same way)
extern "C" int pfnav_mgpu_shard_range(size_t n_total, int rank, int world, size_t *lo, size_t *hi)
{
    PF_ARG(world > 0 && rank >= 0 && rank < world && lo && hi, "rank / world");
    const size_t base = n_total / world, rem = n_total % world;
    *lo = (size_t)rank * base + std::min<size_t>(rank, rem);
    *hi = *lo + base + ((size_t)rank < rem ? 1 : 0);
    return PFNAV_OK;
}

extern "C" int pfnav_mgpu_unique_id(void *out_id)
{
    PF_ARG(out_id, "out_id");
    int rc = nccl_load(g_nccl);
    if (rc) return rc;
    pf_nccl_id id;
    PF_NCCL(g_nccl.GetUniqueId(&id));
    memcpy(out_id, &id, sizeof(id));
    return PFNAV_OK;
}

extern "C" int pfnav_mgpu_init(pfnav_ctx *ctx, int rank, int world, const void *id)
{
    PF_ARG(ctx && id && world >= 1 && rank >= 0 && rank < world, "args");
    PF_NEED_DEVICE(ctx);
    PF_ARG(!ctx->mgpu, "context already belongs to a multi-GPU job");
    int rc = nccl_load(g_nccl);
    if (rc) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    pf_mgpu *m = new pf_mgpu();
    m->rank = rank; m->world = world;
    pf_nccl_id nid;
    memcpy(&nid, id, sizeof(nid));
    int r = g_nccl.CommInitRank(&m->comm, world, nid, rank);
    if (r != 0) {
        pfnav_set_error("pfnav_mgpu_init: ncclCommInitRank -> %s", g_nccl.GetErrorString ? g_nccl.GetErrorString(r) : "error");
        delete m;
        return PFNAV_ERR_CUDA;
    }
    ctx->mgpu = m;
    return PFNAV_OK;
}

extern "C" int pfnav_mgpu_finalize(pfnav_ctx *ctx)
{
    PF_ARG(ctx, "ctx");
    pf_mgpu *m = (pf_mgpu *)ctx->mgpu;
    if (!m) return PFNAV_OK;
    PF_ARG(!m->group, "member of an in-process group: pfnav_group_destroy");
    if (ctx->device >= 0) { cudaSetDevice(ctx->device); cudaDeviceSynchronize(); }
    if (m->comm) g_nccl.CommDestroy(m->comm);
    delete m;
    ctx->mgpu = nullptr;
    return PFNAV_OK;
}

// all-gather of one per-entity column (elem_bytes per entity, uid order) in place: every rank holds its own range
// and receives the others'. Ranges are the balanced split, so they differ by at most one entity: equal ranges use
// ncclAllGather, unequal ones a group of ncclBroadcast (the all-gather-v idiom).
static int nccl_allgather(pfnav_ctx *ctx, pf_mgpu *m, void *d_buf, size_t elem_bytes, cudaStream_t st)
{
    const size_t n = ctx->n_agents;
    if (n % m->world == 0) {
        const size_t cnt = n / m->world * elem_bytes;
        PF_NCCL(g_nccl.AllGather((const uint8_t *)d_buf + (size_t)m->rank * cnt, d_buf, cnt, /*ncclInt8*/ 0, m->comm, st));
        return 0;
    }
    PF_NCCL(g_nccl.GroupStart());
    for (int r = 0; r < m->world; r++) {
        size_t lo, hi;
        pfnav_mgpu_shard_range(n, r, m->world, &lo, &hi);
        uint8_t *p = (uint8_t *)d_buf + lo * elem_bytes;
        PF_NCCL(g_nccl.Broadcast(p, p, (hi - lo) * elem_bytes, 0, r, m->comm, st));
    }
    PF_NCCL(g_nccl.GroupEnd());
    return 0;
}

int pfnav_mgpu_allgather(pfnav_ctx *ctx, void *d_buf, size_t elem_bytes, cudaStream_t st)
{
    pf_mgpu *m = (pf_mgpu *)ctx->mgpu;
    if (!m || m->world == 1) return 0;
    PF_ARG(m->comm, "in-process groups gather through pfnav_group_gather");
    return nccl_allgather(ctx, m, d_buf, elem_bytes, st);
}

static int check_shard(pfnav_ctx *ctx, const pf_mgpu *m)
{
    size_t lo, hi;
    pfnav_mgpu_shard_range(ctx->n_agents, m->rank, m->world, &lo, &hi);
    PF_ARG(ctx->d_records && lo == ctx->shard_lo && hi == ctx->shard_hi,
           "upload this rank's own range first (pfnav_agents_upload_shard with the range of pfnav_mgpu_shard_range)");
    return 0;
}

// The per-tick collective (NCCL transport): all-gather of the 24-byte records -- and of the flock id column when
// membership may have changed since the last gather -- then the whole-population part of the snapshot on this rank
// (member lists if stale, spatial index). Asynchronous on `stream` unless member lists are rebuilt.
extern "C" int pfnav_mgpu_gather(pfnav_ctx *ctx, void *stream)
{
    PF_ARG(ctx && ctx->mgpu, "pfnav_mgpu_init not called");
    PF_NEED_DEVICE(ctx);
    pf_mgpu *m = (pf_mgpu *)ctx->mgpu;
    PF_ARG(!m->group, "member of an in-process group: pfnav_group_gather");
    int rc = check_shard(ctx, m);
    if (rc) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    if ((rc = nccl_allgather(ctx, m, ctx->d_records, sizeof(pf_record), st))) return rc;
    const bool members = ctx->members_stale;
    if (members && (rc = nccl_allgather(ctx, m, ctx->d_flock_of, sizeof(int32_t), st))) return rc;
    ctx->members_stale = false;
    if (members) return pfnav_agents_finish_snapshot(ctx, st, true);
    return pfnav_agents_rebuild_index(ctx, st);
}

// ------------------------------------------------------------------------------------------
// Shared device blockers. The map is replicated, so the ops a member decides on the device (PFNAV_APPLY_BLOCKERS,
// pfnav_agents_set_blocking) must reach every member before any of them commits. Blocker counts are additive and a
// commit's result does not depend on the order of its ops, so every member only needs the union of the members' ops:
// the exchange appends the peers' new ops (those after their `sent` prefix) behind the member's own, in rank order.
// ------------------------------------------------------------------------------------------
static int not_shared(const char *fn)
{
    pfnav_set_error("%s: the context is not in a multi-GPU job that shares blockers (pfnav_mgpu_share_blockers / "
                    "pfnav_group_share_blockers)", fn);
    return PFNAV_ERR_STATE;
}

extern "C" int pfnav_mgpu_share_blockers(pfnav_ctx *ctx)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    pf_mgpu *m = (pf_mgpu *)ctx->mgpu;
    if (!m) {
        pfnav_set_error("pfnav_mgpu_share_blockers: pfnav_mgpu_init not called");
        return PFNAV_ERR_STATE;
    }
    PF_ARG(!m->group, "member of an in-process group: pfnav_group_share_blockers");
    m->share_blockers = true;
    return PFNAV_OK;
}

// NCCL: all-gather of every rank's count record, one read of them, then a group of broadcasts (the all-gather-v
// idiom) that puts each rank's new narrow and wide ops behind the receiver's own. Every rank makes the same calls in
// the same order, from the gathered counts.
extern "C" int pfnav_mgpu_exchange_blocker_ops(pfnav_ctx *ctx, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    pf_mgpu *m = (pf_mgpu *)ctx->mgpu;
    if (!m) return not_shared(__func__);
    PF_ARG(!m->group, "member of an in-process group: pfnav_group_exchange_blocker_ops");
    if (!m->share_blockers) return not_shared(__func__);
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    pf_ops_view v;
    int rc = pf_blocker_ops_view(ctx, &v);
    if (rc) return rc;
    const int world = m->world, rank = m->rank;
    if ((rc = m->d_xcnt.reserve((size_t)world * PF_XCNT))) return rc;
    uint32_t *mine = m->d_xcnt + (size_t)rank * PF_XCNT;
    const uint32_t tail[PF_XCNT - 2] = {v.sent[0], v.sent[1], v.fac ? 1u : 0u, 0, 0, 0};
    PF_CUDA(cudaMemcpyAsync(mine, v.d_cnt, 2 * sizeof(uint32_t), cudaMemcpyDeviceToDevice, st));
    PF_CUDA(cudaMemcpyAsync(mine + 2, tail, sizeof(tail), cudaMemcpyHostToDevice, st));
    PF_NCCL(g_nccl.AllGather(mine, m->d_xcnt, PF_XCNT * sizeof(uint32_t), /*ncclInt8*/ 0, m->comm, st));
    std::vector<uint32_t> all((size_t)world * PF_XCNT);
    PF_CUDA(cudaMemcpyAsync(all.data(), m->d_xcnt, all.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    uint32_t cnt[2] = {all[(size_t)rank * PF_XCNT], all[(size_t)rank * PF_XCNT + 1]};
    bool fac = false;
    for (int r = 0; r < world; r++) {
        const uint32_t *x = &all[(size_t)r * PF_XCNT];
        fac |= x[4] != 0;
        if (r != rank) { cnt[0] += x[0] - x[2]; cnt[1] += x[1] - x[3]; }
    }
    if ((rc = pf_blocker_ops_reserve(ctx, std::max(cnt[0], cnt[1]), &v))) return rc;
    pfnav_blocker_op *buf[2] = {v.narrow, v.wide};
    size_t off[2] = {all[(size_t)rank * PF_XCNT], all[(size_t)rank * PF_XCNT + 1]};
    PF_NCCL(g_nccl.GroupStart());
    for (int r = 0; r < world; r++) {
        const uint32_t *x = &all[(size_t)r * PF_XCNT];
        for (int k = 0; k < 2; k++) {
            const size_t seg = x[k] - x[2 + k];
            if (!seg) continue;
            pfnav_blocker_op *send = buf[k] + x[2 + k];               // read on the root only
            pfnav_blocker_op *recv = r == rank ? send : buf[k] + off[k];
            if (r != rank) off[k] += seg;
            PF_NCCL(g_nccl.Broadcast(send, recv, seg * sizeof(pfnav_blocker_op), /*ncclInt8*/ 0, r, m->comm, st));
        }
    }
    PF_NCCL(g_nccl.GroupEnd());
    return pf_blocker_ops_exchanged(ctx, cnt, fac);
}

// ------------------------------------------------------------------------------------------
// In-process group: several contexts of ONE process (one per GPU, or several on one GPU for tests), driven from
// one thread. Member i is rank i of world = n.
// ------------------------------------------------------------------------------------------
extern "C" int pfnav_group_create(pfnav_ctx **ctxs, int world, pfnav_group **out)
{
    PF_ARG(ctxs && out && world >= 1, "args");
    for (int i = 0; i < world; i++) {
        PF_ARG(ctxs[i] && !ctxs[i]->mgpu, "context missing or already in a multi-GPU job");
        PF_NEED_DEVICE(ctxs[i]);
    }
    pfnav_group *g = new pfnav_group();
    g->ctxs.assign(ctxs, ctxs + world);
    g->ready.resize(world); g->pulled.resize(world);
    for (int i = 0; i < world; i++) {
        PF_CUDA(cudaSetDevice(ctxs[i]->device));
        PF_CUDA(cudaEventCreateWithFlags(&g->ready[i], cudaEventDisableTiming));
        PF_CUDA(cudaEventCreateWithFlags(&g->pulled[i], cudaEventDisableTiming));
        for (int j = 0; j < world; j++) {                 // NVLink peer copies between the members' devices
            if (ctxs[j]->device == ctxs[i]->device) continue;
            int can = 0;
            cudaDeviceCanAccessPeer(&can, ctxs[i]->device, ctxs[j]->device);
            if (can && cudaDeviceEnablePeerAccess(ctxs[j]->device, 0) != cudaSuccess) cudaGetLastError();   // already enabled
        }
        pf_mgpu *m = new pf_mgpu();
        m->rank = i; m->world = world; m->group = g;
        ctxs[i]->mgpu = m;
    }
    *out = g;
    return PFNAV_OK;
}

extern "C" void pfnav_group_destroy(pfnav_group *g)
{
    if (!g) return;
    for (size_t i = 0; i < g->ctxs.size(); i++) {
        pfnav_ctx *c = g->ctxs[i];
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();
        cudaEventDestroy(g->ready[i]); cudaEventDestroy(g->pulled[i]);
        delete (pf_mgpu *)c->mgpu;
        c->mgpu = nullptr;
    }
    delete g;
}

// The per-tick collective of the group: every member pulls the other members' ranges of the record array (and of
// the flock id column when membership may have changed) and finishes its snapshot. All on the members' own streams.
extern "C" int pfnav_group_gather(pfnav_group *g)
{
    PF_ARG(g, "group");
    const int world = (int)g->ctxs.size();
    int rc;
    bool members = false;
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_ARG(c->n_agents == g->ctxs[0]->n_agents, "members hold populations of different sizes");
        if ((rc = check_shard(c, (pf_mgpu *)c->mgpu))) return rc;
        members |= c->members_stale;
        PF_CUDA(cudaSetDevice(c->device));
        PF_CUDA(cudaEventRecord(g->ready[i], c->tick_stream));       // my range is final once my stream gets here
    }
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        for (int p = 0; p < world; p++) {
            if (p == i) continue;
            pfnav_ctx *src = g->ctxs[p];
            PF_CUDA(cudaStreamWaitEvent(c->tick_stream, g->ready[p], 0));
            const size_t lo = src->shard_lo, cnt = src->shard_hi - src->shard_lo;
            if (!cnt) continue;
            PF_CUDA(cudaMemcpyPeerAsync(c->d_records + lo, c->device, src->d_records + lo, src->device, cnt * sizeof(pf_record), c->tick_stream));
            if (members)
                PF_CUDA(cudaMemcpyPeerAsync(c->d_flock_of + lo, c->device, src->d_flock_of + lo, src->device, cnt * 4, c->tick_stream));
        }
        PF_CUDA(cudaEventRecord(g->pulled[i], c->tick_stream));
    }
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        // whatever member i does next to its own range (the state apply of the next tick) must wait until every
        // peer has copied the current version
        for (int p = 0; p < world; p++)
            if (p != i) PF_CUDA(cudaStreamWaitEvent(c->tick_stream, g->pulled[p], 0));
        c->members_stale = false;
        rc = members ? pfnav_agents_finish_snapshot(c, c->tick_stream, true) : pfnav_agents_rebuild_index(c, c->tick_stream);
        if (rc) return rc;
    }
    return PFNAV_OK;
}

// an exchange copies between every pair of member devices: refuse up front rather than fail halfway through one
static int peer_check(const pfnav_group *g, const char *fn)
{
    const int world = (int)g->ctxs.size();
    for (int i = 0; i < world; i++)
        for (int j = 0; j < world; j++) {
            const int di = g->ctxs[i]->device, dj = g->ctxs[j]->device;
            if (di == dj) continue;
            int can = 0;
            PF_CUDA(cudaDeviceCanAccessPeer(&can, di, dj));
            if (!can) {
                pfnav_set_error("%s: device %d cannot access the memory of device %d", fn, di, dj);
                return PFNAV_ERR_STATE;
            }
        }
    return 0;
}

extern "C" int pfnav_group_share_blockers(pfnav_group *g)
{
    PF_ARG(g, "group");
    const int world = (int)g->ctxs.size();
    for (int i = 0; i < world; i++)
        PF_ARG(g->ctxs[i]->n_agents == g->ctxs[0]->n_agents, "members hold populations of different sizes");
    if (int rc = peer_check(g, __func__)) return rc;
    for (int i = 0; i < world; i++) ((pf_mgpu *)g->ctxs[i]->mgpu)->share_blockers = true;
    return PFNAV_OK;
}

// In-process group: every member's counts are read once, its buffers grown, and its stream pulls the peers' new ops
// behind its own with cudaMemcpyPeerAsync. Every member's stream then waits until every peer has finished pulling, so
// that nothing a member does next (an emit, a commit's reset, a buffer growth) reaches ops a peer is still copying.
extern "C" int pfnav_group_exchange_blocker_ops(pfnav_group *g)
{
    PF_ARG(g, "group");
    const int world = (int)g->ctxs.size();
    if (!((pf_mgpu *)g->ctxs[0]->mgpu)->share_blockers) return not_shared(__func__);
    int rc;
    std::vector<pf_ops_view> v(world);
    std::vector<uint32_t> cnt(2 * (size_t)world), seg(2 * (size_t)world);
    uint32_t tot[2] = {0, 0};
    bool fac = false;
    for (int i = 0; i < world; i++)
        PF_ARG(g->ctxs[i]->n_agents == g->ctxs[0]->n_agents, "members hold populations of different sizes");
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        if ((rc = pf_blocker_ops_view(c, &v[i]))) return rc;        // waits for the member's device
        PF_CUDA(cudaMemcpy(&cnt[2 * i], v[i].d_cnt, 2 * sizeof(uint32_t), cudaMemcpyDeviceToHost));
        for (int k = 0; k < 2; k++) { seg[2 * i + k] = cnt[2 * i + k] - v[i].sent[k]; tot[k] += seg[2 * i + k]; }
        fac |= v[i].fac;
    }
    std::vector<uint32_t> after(2 * (size_t)world);
    for (int i = 0; i < world; i++) {
        for (int k = 0; k < 2; k++) after[2 * i + k] = cnt[2 * i + k] + tot[k] - seg[2 * i + k];
        if ((rc = pf_blocker_ops_reserve(g->ctxs[i], std::max(after[2 * i], after[2 * i + 1]), &v[i]))) return rc;
    }
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        pfnav_blocker_op *dst[2] = {v[i].narrow, v[i].wide};
        size_t off[2] = {cnt[2 * i], cnt[2 * i + 1]};
        for (int p = 0; p < world; p++) {
            if (p == i) continue;
            const pfnav_blocker_op *src[2] = {v[p].narrow, v[p].wide};
            for (int k = 0; k < 2; k++) {
                const size_t n = seg[2 * p + k];
                if (!n) continue;
                PF_CUDA(cudaMemcpyPeerAsync(dst[k] + off[k], c->device, src[k] + v[p].sent[k], g->ctxs[p]->device,
                                            n * sizeof(pfnav_blocker_op), c->tick_stream));
                off[k] += n;
            }
        }
        PF_CUDA(cudaEventRecord(g->pulled[i], c->tick_stream));
    }
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        for (int p = 0; p < world; p++)
            if (p != i) PF_CUDA(cudaStreamWaitEvent(c->tick_stream, g->pulled[p], 0));
        if ((rc = pf_blocker_ops_exchanged(c, &after[2 * i], fac))) return rc;
    }
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// Batches of a job (pfnav_plan.cu: pf_job_*; zone and entity-field batches: pfnav_region.cu). Every member plans the
// whole batch and describes itself in one record -- its verdict on the arguments, whether its pool can hold its fields,
// and for a goal batch the (goal, chunk) fields it lacks -- and every member reads every record before anything changes.
// Then each goal's or request's owner builds its fields into its staging segment, the segments are exchanged (segment
// r is rank r's), and every member copies the fields it needs into its own slots. The owners and the segment sizes
// follow from the plan (and a goal batch's union of lacks), which every member computes alike, so no count is exchanged.
// ------------------------------------------------------------------------------------------
static void job_init(pf_job &J, int ngoals, const int32_t *dests, int layer, const int32_t *targets, uint32_t flags)
{
    J.ngoals = ngoals; J.dests = dests; J.layer = layer; J.targets = targets; J.flags = flags;
}

static void job_init_zones(pf_job &J, const pfnav_zone_req *reqs, size_t m)
{
    J.kind = PF_JOB_ZONES; J.zreqs = reqs; J.m = m;
}

static void job_init_entity(pf_job &J, const pfnav_entity_field_req *reqs, size_t m, const pfnav_footprint *ents, size_t nents,
                            const int32_t *chunks_rc, size_t nchunks)
{
    J.kind = PF_JOB_ENTITY; J.ereqs = reqs; J.m = m; J.ents = ents; J.nents = nents; J.chunks_rc = chunks_rc; J.nchunks = nchunks;
}

// the NCCL form's rank: a context of a job, not of an in-process group
static int nccl_rank(pfnav_ctx *ctx, const char *fn, const char *group_fn, pf_mgpu **out)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    pf_mgpu *m = (pf_mgpu *)ctx->mgpu;
    if (!m) {
        pfnav_set_error("%s: pfnav_mgpu_init not called", fn);
        return PFNAV_ERR_STATE;
    }
    if (m->group) {
        pfnav_set_error("%s: member of an in-process group: %s", fn, group_fn);
        return PFNAV_ERR_STATE;
    }
    *out = m;
    return PFNAV_OK;
}

// ... of a field batch: with a pool
static int nccl_member(pfnav_ctx *ctx, const char *fn, const char *group_fn, pf_mgpu **out)
{
    if (int rc = nccl_rank(ctx, fn, group_fn, out)) return rc;
    PF_ARG(ctx->pool.d_slot, "pool not created");
    return PFNAV_OK;
}

// NCCL: one all-gather of the member records on `stream` (and a host wait for it), the owners' builds, a group of
// broadcasts (one per owner with a non-empty segment) on `stream`, the copies into the pool on `stream`.
static int nccl_job(pfnav_ctx *ctx, pf_mgpu *m, pf_job &J, cudaStream_t st, const char *fn)
{
    const int local = J.refused ? J.refused : pf_job_plan(ctx, J);
    const std::string local_err = local ? pfnav_last_error() : "";
    // record: {verdict, fits, 0, 0} then, for a goal batch, one lack byte per (goal, chunk); every rank has the same
    // arguments and map
    const int world = m->world, rank = m->rank;
    const size_t nlack = J.kind == PF_JOB_GOALS ? (size_t)J.ngoals * ctx->chunk_w * ctx->chunk_h : 0;
    const size_t rec = 16 + ((nlack + 15) & ~(size_t)15);
    if (int rc = m->d_xgoal.reserve(rec * world)) return rc;
    std::vector<uint8_t> all(rec * world, 0);
    uint8_t *mine = all.data() + rec * rank;
    const int32_t hdr[4] = {local, J.fits ? 1 : 0, 0, 0};
    memcpy(mine, hdr, sizeof(hdr));
    if (!local && nlack) memcpy(mine + 16, J.lack.data(), nlack);
    PF_CUDA(cudaMemcpyAsync(m->d_xgoal + rec * rank, mine, rec, cudaMemcpyHostToDevice, st));
    PF_NCCL(g_nccl.AllGather(m->d_xgoal + rec * rank, m->d_xgoal, rec, /*ncclInt8*/ 0, m->comm, st));
    PF_CUDA(cudaMemcpyAsync(all.data(), m->d_xgoal, all.size(), cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    std::vector<uint8_t> uni(nlack, 0);
    int refused = -1, refused_rc = 0, full = -1;
    for (int r = 0; r < world; r++) {
        int32_t h[4];
        memcpy(h, all.data() + rec * r, sizeof(h));
        if (h[0] && refused < 0) { refused = r; refused_rc = h[0]; }
        if (!h[1] && full < 0) full = r;
        const uint8_t *l = all.data() + rec * r + 16;
        for (size_t k = 0; k < nlack; k++) uni[k] |= l[k];
    }
    if (local) {
        pfnav_set_error("%s", local_err.c_str());
        return local;
    }
    if (refused >= 0) {
        pfnav_set_error("%s: rank %d refused the batch (error %d); no rank changed its pool", fn, refused, refused_rc);
        return refused_rc;
    }
    if (full >= 0) {
        pfnav_set_error("%s: the field pool of rank %d cannot hold its fields; no rank changed its pool", fn, full);
        return PFNAV_ERR_NOMEM;
    }
    int rc = pf_job_launch(ctx, J, uni.data(), world, rank, st);
    if (rc) return rc;
    if (J.seg[world]) {
        PF_NCCL(g_nccl.GroupStart());
        for (int r = 0; r < world; r++) {
            const size_t n = J.seg[r + 1] - J.seg[r];
            if (!n) continue;
            uint8_t *p = ctx->d_job_stage + J.seg[r] * 4096;           // sent from the root, received in place elsewhere
            PF_NCCL(g_nccl.Broadcast(p, p, n * 4096, /*ncclInt8*/ 0, r, m->comm, st));
        }
        PF_NCCL(g_nccl.GroupEnd());
    }
    return pf_job_scatter(ctx, J, st);
}

// the group form's members: pools created, maps and pools of one shape, peer access between their devices
static int group_members(pfnav_group *g, const char *fn)
{
    PF_ARG(g, "group");
    const int world = (int)g->ctxs.size();
    const pfnav_ctx *c0 = g->ctxs[0];
    for (int i = 0; i < world; i++) {
        const pfnav_ctx *c = g->ctxs[i];
        PF_ARG(c->pool.d_slot, "pool not created");
        PF_ARG(c->chunk_w == c0->chunk_w && c->chunk_h == c0->chunk_h && c->pool.ndests == c0->pool.ndests,
               "members hold maps or pools of different shapes");
    }
    return peer_check(g, fn);
}

// In-process group: the records are read on the host; member i pulls every owner's segment into its staging with
// cudaMemcpyPeerAsync on its context stream, copies what it needs into its pool, and then waits until every peer has
// finished pulling its own segment.
static int group_job(pfnav_group *g, std::vector<pf_job> &J, const char *fn)
{
    const int world = (int)g->ctxs.size();
    int rc = 0;
    for (int i = 0; i < world; i++)
        if ((rc = J[i].refused ? J[i].refused : pf_job_plan(g->ctxs[i], J[i]))) return rc;   // no member has changed anything yet
    for (int i = 0; i < world; i++)
        if (!J[i].fits) {
            pfnav_set_error("%s: the field pool of member %d cannot hold its fields; no member changed its pool", fn, i);
            return PFNAV_ERR_NOMEM;
        }
    std::vector<uint8_t> uni(J[0].lack.size(), 0);
    for (int i = 0; i < world; i++)
        for (size_t k = 0; k < uni.size(); k++) uni[k] |= J[i].lack[k];
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        if ((rc = pf_job_launch(c, J[i], uni.data(), world, i, c->tick_stream))) return rc;
    }
    const std::vector<size_t> &seg = J[0].seg;
    if (seg[world]) {
        for (int r = 0; r < world; r++) {
            if (seg[r + 1] == seg[r]) continue;
            PF_CUDA(cudaSetDevice(g->ctxs[r]->device));
            PF_CUDA(cudaEventRecord(g->ready[r], g->ctxs[r]->tick_stream));      // owner r's segment is built
        }
        for (int i = 0; i < world; i++) {
            pfnav_ctx *c = g->ctxs[i];
            PF_CUDA(cudaSetDevice(c->device));
            for (int p = 0; p < world; p++) {
                const size_t n = seg[p + 1] - seg[p];
                if (p == i || !n) continue;
                const pfnav_ctx *src = g->ctxs[p];
                PF_CUDA(cudaStreamWaitEvent(c->tick_stream, g->ready[p], 0));
                PF_CUDA(cudaMemcpyPeerAsync(c->d_job_stage + seg[p] * 4096, c->device, src->d_job_stage + seg[p] * 4096,
                                            src->device, n * 4096, c->tick_stream));
            }
            PF_CUDA(cudaEventRecord(g->pulled[i], c->tick_stream));
        }
        for (int i = 0; i < world; i++) {
            pfnav_ctx *c = g->ctxs[i];
            PF_CUDA(cudaSetDevice(c->device));
            if ((rc = pf_job_scatter(c, J[i], c->tick_stream))) return rc;
            // the member's next batch writes its staging: only after every peer has pulled its segment of this one
            for (int p = 0; p < world; p++)
                if (p != i) PF_CUDA(cudaStreamWaitEvent(c->tick_stream, g->pulled[p], 0));
        }
    }
    return PFNAV_OK;
}

extern "C" int pfnav_mgpu_request_goals_ex(pfnav_ctx *ctx, int ngoals, const int32_t *dests, int layer, const int32_t *targets,
                                           uint32_t flags, void *stream, int *out_n_flow, int *out_n_los)
{
    pf_mgpu *m = nullptr;
    if (int rc = nccl_member(ctx, __func__, "pfnav_group_request_goals_ex", &m)) return rc;
    PF_ARG(ngoals >= 0 && (ngoals == 0 || (dests && targets)), "goals");
    if (out_n_flow) *out_n_flow = 0;
    if (out_n_los) *out_n_los = 0;
    if (ngoals == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    pf_job J;
    job_init(J, ngoals, dests, layer, targets, flags);
    if (int rc = nccl_job(ctx, m, J, pf_stream(ctx, stream), __func__)) return rc;
    if (out_n_flow) *out_n_flow = J.nf;
    if (out_n_los) *out_n_los = J.nl;
    return PFNAV_OK;
}

// out_n_flow / out_n_los: `world` entries, member i's solo counts
extern "C" int pfnav_group_request_goals_ex(pfnav_group *g, int ngoals, const int32_t *dests, int layer, const int32_t *targets,
                                            uint32_t flags, int *out_n_flow, int *out_n_los)
{
    if (int rc = group_members(g, __func__)) return rc;
    const int world = (int)g->ctxs.size();
    PF_ARG(ngoals >= 0 && (ngoals == 0 || (dests && targets)), "goals");
    for (int i = 0; i < world; i++) {
        if (out_n_flow) out_n_flow[i] = 0;
        if (out_n_los) out_n_los[i] = 0;
    }
    if (ngoals == 0) return PFNAV_OK;
    std::vector<pf_job> J(world);
    for (int i = 0; i < world; i++) job_init(J[i], ngoals, dests, layer, targets, flags);
    if (int rc = group_job(g, J, __func__)) return rc;
    for (int i = 0; i < world; i++) {
        if (out_n_flow) out_n_flow[i] = J[i].nf;
        if (out_n_los) out_n_los[i] = J[i].nl;
    }
    return PFNAV_OK;
}

extern "C" int pfnav_mgpu_request_zones(pfnav_ctx *ctx, const pfnav_zone_req *reqs, size_t m, void *stream, int32_t *out_nfields)
{
    pf_mgpu *mg = nullptr;
    if (int rc = nccl_member(ctx, __func__, "pfnav_group_request_zones", &mg)) return rc;
    PF_ARG(m == 0 || reqs, "reqs");
    if (out_nfields) std::fill(out_nfields, out_nfields + m, 0);
    if (m == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    pf_job J;
    job_init_zones(J, reqs, m);
    if (int rc = nccl_job(ctx, mg, J, pf_stream(ctx, stream), __func__)) return rc;
    if (out_nfields) std::copy(J.nfields.begin(), J.nfields.end(), out_nfields);
    return PFNAV_OK;
}

// out_nfields: m entries, the same on every member
extern "C" int pfnav_group_request_zones(pfnav_group *g, const pfnav_zone_req *reqs, size_t m, int32_t *out_nfields)
{
    if (int rc = group_members(g, __func__)) return rc;
    PF_ARG(m == 0 || reqs, "reqs");
    if (out_nfields) std::fill(out_nfields, out_nfields + m, 0);
    if (m == 0) return PFNAV_OK;
    std::vector<pf_job> J(g->ctxs.size());
    for (pf_job &j : J) job_init_zones(j, reqs, m);
    if (int rc = group_job(g, J, __func__)) return rc;
    if (out_nfields) std::copy(J[0].nfields.begin(), J[0].nfields.end(), out_nfields);
    return PFNAV_OK;
}

extern "C" int pfnav_mgpu_request_entity_fields_batch(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m,
                                                      const pfnav_footprint *ents, size_t nents, const int32_t *chunks_rc,
                                                      size_t nchunks, void *stream)
{
    pf_mgpu *mg = nullptr;
    if (int rc = nccl_member(ctx, __func__, "pfnav_group_request_entity_fields_batch", &mg)) return rc;
    PF_ARG(m == 0 || reqs, "reqs");
    if (m == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    pf_job J;
    job_init_entity(J, reqs, m, ents, nents, chunks_rc, nchunks);
    return nccl_job(ctx, mg, J, pf_stream(ctx, stream), __func__);
}

extern "C" int pfnav_group_request_entity_fields_batch(pfnav_group *g, const pfnav_entity_field_req *reqs, size_t m,
                                                       const pfnav_footprint *ents, size_t nents, const int32_t *chunks_rc,
                                                       size_t nchunks)
{
    if (int rc = group_members(g, __func__)) return rc;
    PF_ARG(m == 0 || reqs, "reqs");
    if (m == 0) return PFNAV_OK;
    std::vector<pf_job> J(g->ctxs.size());
    for (pf_job &j : J) job_init_entity(j, reqs, m, ents, nents, chunks_rc, nchunks);
    return group_job(g, J, __func__);
}

// Named by uid: each member resolves the batch from its own record column, which a gather made equal on every member, so
// every member plans the same batch. A member that cannot resolve it (stale records, a seeker off the map) enters the
// error as its verdict, and the verdicts are exchanged as for any batch.
extern "C" int pfnav_mgpu_request_entity_fields_resident(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m,
                                                         const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents,
                                                         const uint32_t *seeker_uids, size_t nseekers, void *stream)
{
    pf_mgpu *mg = nullptr;
    if (int rc = nccl_member(ctx, __func__, "pfnav_group_request_entity_fields_resident", &mg)) return rc;
    PF_CUDA(cudaSetDevice(ctx->device));
    const cudaStream_t st = pf_stream(ctx, stream);
    pf_resident_batch B;
    const int rc = pf_resident_resolve(ctx, st, reqs, m, ents, ent_uids, nents, seeker_uids, nseekers, B);
    if (m == 0) return rc;                  // nothing resolved: every rank has the same arguments and population
    pf_job J;
    job_init_entity(J, B.reqs.data(), m, B.ents.data(), nents, B.chunks_rc.data(), B.chunks_rc.size() / 2);
    J.refused = rc;
    return nccl_job(ctx, mg, J, st, __func__);
}

extern "C" int pfnav_group_request_entity_fields_resident(pfnav_group *g, const pfnav_entity_field_req *reqs, size_t m,
                                                          const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents,
                                                          const uint32_t *seeker_uids, size_t nseekers)
{
    if (int rc = group_members(g, __func__)) return rc;
    const size_t world = g->ctxs.size();
    std::vector<pf_resident_batch> B(world);
    std::vector<pf_job> J(world);
    for (size_t i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        const int rc = pf_resident_resolve(c, c->tick_stream, reqs, m, ents, ent_uids, nents, seeker_uids, nseekers, B[i]);
        if (m == 0 && rc) return rc;
        job_init_entity(J[i], B[i].reqs.data(), m, B[i].ents.data(), nents, B[i].chunks_rc.data(), B[i].chunks_rc.size() / 2);
        J[i].refused = rc;
    }
    if (m == 0) return PFNAV_OK;
    return group_job(g, J, __func__);
}

// ------------------------------------------------------------------------------------------
// Movement commands of a job (pfnav_commands.cu: pf_cmd_job_*). Every member gets the job's whole batch, checks what it
// owns and describes itself in one record {status, n_agents, n_flocks}; every member reads every record before anything
// changes, because a member cannot check another's layers or flock indices, and a flock table taken by some members only
// would split the job's member lists.
// ------------------------------------------------------------------------------------------
extern "C" int pfnav_mgpu_commands(pfnav_ctx *ctx, const pfnav_agent_delta *deltas, size_t n, const pfnav_flock *flocks,
                                   size_t nflocks, void *stream)
{
    pf_mgpu *m = nullptr;
    if (int rc = nccl_rank(ctx, __func__, "pfnav_group_commands", &m)) return rc;
    if (n == 0 && !flocks) return PFNAV_OK;                 // the same arguments on every rank: none of them exchanges
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    pf_cmd_job J;
    int local = check_shard(ctx, m);
    if (!local) local = pf_cmd_job_check(ctx, deltas, n, flocks, nflocks, J);
    const std::string local_err = local ? pfnav_last_error() : "";
    const int world = m->world, rank = m->rank;
    if (int rc = m->d_xcnt.reserve((size_t)world * PF_XCNT)) return rc;
    uint32_t *mine = m->d_xcnt + (size_t)rank * PF_XCNT;
    const uint32_t verdict[PF_XCNT] = {(uint32_t)local, (uint32_t)ctx->n_agents, (uint32_t)ctx->n_flocks, 0, 0, 0, 0, 0};
    PF_CUDA(cudaMemcpyAsync(mine, verdict, sizeof(verdict), cudaMemcpyHostToDevice, st));
    PF_NCCL(g_nccl.AllGather(mine, m->d_xcnt, PF_XCNT * sizeof(uint32_t), /*ncclInt8*/ 0, m->comm, st));
    std::vector<uint32_t> all((size_t)world * PF_XCNT);
    PF_CUDA(cudaMemcpyAsync(all.data(), m->d_xcnt, all.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    for (int r = 0; r < world; r++) {
        const uint32_t *x = &all[(size_t)r * PF_XCNT];
        if (!x[0]) continue;
        if (r == rank) pfnav_set_error("%s: rank %d refused the batch (%s); no rank changed anything", __func__, r, local_err.c_str());
        else pfnav_set_error("%s: rank %d refused the batch (error %d); no rank changed anything", __func__, r, (int)x[0]);
        return (int)x[0];
    }
    for (int r = 0; r < world; r++)
        PF_ARG(all[(size_t)r * PF_XCNT + 1] == all[1] && all[(size_t)r * PF_XCNT + 2] == all[2],
               "ranks hold populations or flock tables of different sizes; no rank changed anything");
    return pf_cmd_job_apply(ctx, J, st);
}

// The segments are validated once, against the fewest layers any member created (a record is refused exactly when some
// member would refuse it), then every member's own state; only then does any member change. Each member then restores
// its range on its context stream.
extern "C" int pfnav_group_restore(pfnav_group *g, const void *const *segs, const size_t *sizes, size_t nseg)
{
    PF_ARG(g, "group");
    const int world = (int)g->ctxs.size();
    int nlayers = PFNAV_NAV_LAYER_MAX;
    for (int i = 0; i < world; i++) {
        if (int rc = pf_ckpt_restore_ready(g->ctxs[i])) return rc;
        nlayers = std::min(nlayers, g->ctxs[i]->nlayers);
    }
    pf_ckpt_set S;
    const char *e = pf_ckpt_check(segs, sizes, nseg, nlayers, S);
    PF_ARG(!e, e);
    std::vector<size_t> lo(world), hi(world);
    for (int i = 0; i < world; i++)
        if (int rc = pf_ckpt_restore_check(g->ctxs[i], S, &lo[i], &hi[i])) {
            const std::string m = pfnav_last_error();
            pfnav_set_error("%s: member %d refused the restore (%s); no member changed anything", __func__, i, m.c_str());
            return rc;
        }
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        if (int rc = pf_ckpt_restore_apply(c, S, lo[i], hi[i], c->tick_stream)) return rc;
    }
    return PFNAV_OK;
}

// In-process group: the members' verdicts are their host state, so nothing is exchanged on the devices; each member then
// applies the batch on its context stream.
extern "C" int pfnav_group_commands(pfnav_group *g, const pfnav_agent_delta *deltas, size_t n, const pfnav_flock *flocks,
                                    size_t nflocks)
{
    PF_ARG(g, "group");
    if (n == 0 && !flocks) return PFNAV_OK;
    const int world = (int)g->ctxs.size();
    std::vector<pf_cmd_job> J(world);
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        int rc = check_shard(c, (pf_mgpu *)c->mgpu);
        if (!rc) rc = pf_cmd_job_check(c, deltas, n, flocks, nflocks, J[i]);
        if (rc) {
            const std::string e = pfnav_last_error();
            pfnav_set_error("%s: member %d refused the batch (%s); no member changed anything", __func__, i, e.c_str());
            return rc;
        }
    }
    for (int i = 0; i < world; i++)
        PF_ARG(g->ctxs[i]->n_agents == g->ctxs[0]->n_agents && g->ctxs[i]->n_flocks == g->ctxs[0]->n_flocks,
               "members hold populations or flock tables of different sizes; no member changed anything");
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        if (int rc = pf_cmd_job_apply(c, J[i], c->tick_stream)) return rc;
    }
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// Input deltas of a job (pfnav_inputs.cu: pf_input_job_*). Every member gets the job's whole batch, checks all of it and
// describes itself in one record {status, n_agents, n_flocks, tables present}, exchanged as for a command batch; then each
// member writes the records of its own uids, and creates the formation table when the batch needs one.
// ------------------------------------------------------------------------------------------
extern "C" int pfnav_mgpu_input_deltas(pfnav_ctx *ctx, const pfnav_input_delta *d, size_t n, void *stream)
{
    pf_mgpu *m = nullptr;
    if (int rc = nccl_rank(ctx, __func__, "pfnav_group_input_deltas", &m)) return rc;
    if (n == 0) return PFNAV_OK;                            // the same arguments on every rank: none of them exchanges
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    pf_input_job J;
    int local = check_shard(ctx, m);
    if (!local) local = pf_input_job_check(ctx, d, n, J);
    const std::string local_err = local ? pfnav_last_error() : "";
    const int world = m->world, rank = m->rank;
    if (int rc = m->d_xcnt.reserve((size_t)world * PF_XCNT)) return rc;
    uint32_t *mine = m->d_xcnt + (size_t)rank * PF_XCNT;
    const uint32_t verdict[PF_XCNT] = {(uint32_t)local, (uint32_t)ctx->n_agents, (uint32_t)ctx->n_flocks, pf_input_tables(ctx),
                                       0, 0, 0, 0};
    PF_CUDA(cudaMemcpyAsync(mine, verdict, sizeof(verdict), cudaMemcpyHostToDevice, st));
    PF_NCCL(g_nccl.AllGather(mine, m->d_xcnt, PF_XCNT * sizeof(uint32_t), /*ncclInt8*/ 0, m->comm, st));
    std::vector<uint32_t> all((size_t)world * PF_XCNT);
    PF_CUDA(cudaMemcpyAsync(all.data(), m->d_xcnt, all.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    for (int r = 0; r < world; r++) {
        const uint32_t *x = &all[(size_t)r * PF_XCNT];
        if (!x[0]) continue;
        if (r == rank) pfnav_set_error("%s: rank %d refused the batch (%s); no rank changed anything", __func__, r, local_err.c_str());
        else pfnav_set_error("%s: rank %d refused the batch (error %d); no rank changed anything", __func__, r, (int)x[0]);
        return (int)x[0];
    }
    for (int r = 0; r < world; r++)
        PF_ARG(all[(size_t)r * PF_XCNT + 1] == all[1] && all[(size_t)r * PF_XCNT + 3] == all[3],
               "ranks hold populations or sets of tables that differ; no rank changed anything");
    return pf_input_job_apply(ctx, J, st);
}

// In-process group: the members' verdicts are their host state; each member then writes on its context stream.
extern "C" int pfnav_group_input_deltas(pfnav_group *g, const pfnav_input_delta *d, size_t n)
{
    PF_ARG(g, "group");
    if (n == 0) return PFNAV_OK;
    const int world = (int)g->ctxs.size();
    std::vector<pf_input_job> J(world);
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        int rc = check_shard(c, (pf_mgpu *)c->mgpu);
        if (!rc) rc = pf_input_job_check(c, d, n, J[i]);
        if (rc) {
            const std::string e = pfnav_last_error();
            pfnav_set_error("%s: member %d refused the batch (%s); no member changed anything", __func__, i, e.c_str());
            return rc;
        }
    }
    for (int i = 0; i < world; i++)
        PF_ARG(g->ctxs[i]->n_agents == g->ctxs[0]->n_agents && pf_input_tables(g->ctxs[i]) == pf_input_tables(g->ctxs[0]),
               "members hold populations or sets of tables that differ; no member changed anything");
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        if (int rc = pf_input_job_apply(c, J[i], c->tick_stream)) return rc;
    }
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// Population change of a job (pfnav_commands.cu: pf_pop_job_*). Every member gets the job's whole batch, checks it and its
// own entities' flock indices, and describes itself in one record {status, n_agents, n_flocks, tables present}; every
// member reads every record before anything changes. Then each member releases its removed entities' blocks, compacts its
// own survivors and the replicated columns into its scratch, the segments of survivors that cross a member boundary move
// (at most R + A rows per boundary), and each member writes its new range and rebuilds its member lists.
// ------------------------------------------------------------------------------------------
static uint32_t pop_tables_bits(const pf_pop_tables &T)
{
    return (T.ms ? 1u : 0u) | (T.ext ? 2u : 0u) | (T.formation ? 4u : 0u) | (T.blocking ? 8u : 0u);
}

// NCCL: per segment (sender s, receiver q) and table one broadcast from s, grouped; every rank receives every segment into
// its receive block for the pair, so every rank makes the same calls from the plan alone
static int nccl_pop_segments(pf_mgpu *m, pf_pop_member &M, cudaStream_t st)
{
    const pf_pop_job &J = M.J;
    const int world = m->world, rank = m->rank;
    PF_NCCL(g_nccl.GroupStart());
    for (int s = 0; s < world; s++)
        for (int q = 0; q < world; q++) {
            const size_t a = J.seg_lo(s, q), n = J.seg_hi(s, q) - a;
            if (s == q || !n) continue;
            const pf_pop_rows &dst = M.pair[(size_t)s * world + q];
            const size_t k = s == rank ? a - M.own.first : 0;      // the sender's rows, read on the root only
            auto bc = [&](const void *src, void *recv, size_t bytes) {
                return g_nccl.Broadcast(s == rank ? src : recv, recv, bytes, /*ncclInt8*/ 0, s, m->comm, st);
            };
            PF_NCCL(bc(M.own.agents + k, dst.agents, n * sizeof(pfnav_agent)));
            PF_NCCL(bc(M.own.rec + k, dst.rec, n * sizeof(pf_record)));
            PF_NCCL(bc(M.own.flock + k, dst.flock, n * 4));
            if (M.T.ms) PF_NCCL(bc(M.own.ms + k, dst.ms, n * sizeof(pfnav_movestate)));
            if (M.T.ext) PF_NCCL(bc(M.own.ext + k, dst.ext, n * sizeof(pfnav_movestate_ext)));
            if (M.T.formation) PF_NCCL(bc(M.own.form + k, dst.form, n * sizeof(pfnav_formation_in)));
            if (M.T.blocking) PF_NCCL(bc(M.own.blk + k, dst.blk, n * sizeof(pfnav_blocking)));
        }
    PF_NCCL(g_nccl.GroupEnd());
    return 0;
}

extern "C" int pfnav_mgpu_change_population(pfnav_ctx *ctx, const uint32_t *remove_uids, size_t nremove, const pfnav_agent *add,
                                            const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext,
                                            const pfnav_formation_in *add_formation, const pfnav_blocking *add_blocking,
                                            size_t nadd, const pfnav_flock *flocks, size_t nflocks, void *stream)
{
    pf_mgpu *m = nullptr;
    if (int rc = nccl_rank(ctx, __func__, "pfnav_group_change_population", &m)) return rc;
    if (nremove == 0 && nadd == 0 && !flocks) return PFNAV_OK;     // the same arguments on every rank: none of them exchanges
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    pf_pop_member M;
    int local = check_shard(ctx, m);
    if (!local) local = pf_pop_job_check(ctx, remove_uids, nremove, add, add_ms, add_ext, add_formation, add_blocking, nadd, flocks,
                                         nflocks, m->world, m->rank, M);
    const std::string local_err = local ? pfnav_last_error() : "";
    const int world = m->world, rank = m->rank;
    if (int rc = m->d_xcnt.reserve((size_t)world * PF_XCNT)) return rc;
    uint32_t *mine = m->d_xcnt + (size_t)rank * PF_XCNT;
    const uint32_t verdict[PF_XCNT] = {(uint32_t)local, (uint32_t)ctx->n_agents, (uint32_t)ctx->n_flocks, local ? 0u : pop_tables_bits(M.T),
                                       0, 0, 0, 0};
    PF_CUDA(cudaMemcpyAsync(mine, verdict, sizeof(verdict), cudaMemcpyHostToDevice, st));
    PF_NCCL(g_nccl.AllGather(mine, m->d_xcnt, PF_XCNT * sizeof(uint32_t), /*ncclInt8*/ 0, m->comm, st));
    std::vector<uint32_t> all((size_t)world * PF_XCNT);
    PF_CUDA(cudaMemcpyAsync(all.data(), m->d_xcnt, all.size() * sizeof(uint32_t), cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    for (int r = 0; r < world; r++) {
        const uint32_t *x = &all[(size_t)r * PF_XCNT];
        if (!x[0]) continue;
        if (r == rank) pfnav_set_error("%s: rank %d refused the batch (%s); no rank changed anything", __func__, r, local_err.c_str());
        else pfnav_set_error("%s: rank %d refused the batch (error %d); no rank changed anything", __func__, r, (int)x[0]);
        return (int)x[0];
    }
    for (int r = 0; r < world; r++)
        PF_ARG(all[(size_t)r * PF_XCNT + 1] == all[1] && all[(size_t)r * PF_XCNT + 2] == all[2] && all[(size_t)r * PF_XCNT + 3] == all[3],
               "ranks hold populations, flock tables or sets of uploaded tables that differ; no rank changed anything");
    int rc;
    if ((rc = pf_pop_job_stage(ctx, M, true, st))) return rc;
    if (world > 1 && (rc = nccl_pop_segments(m, M, st))) return rc;
    if ((rc = pf_pop_job_write(ctx, M, st))) return rc;
    return pf_pop_job_commit(ctx, M, st);
}

// In-process group: the verdicts are the members' host state. Every member stages on its context stream; a receiver
// pulls each segment straight from the sender's scratch with cudaMemcpyPeerAsync once the sender's stream has compacted
// it (ready), and no member reuses its scratch (the member sort of the commit) before every member has pulled (pulled).
extern "C" int pfnav_group_change_population(pfnav_group *g, const uint32_t *remove_uids, size_t nremove, const pfnav_agent *add,
                                             const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext,
                                             const pfnav_formation_in *add_formation, const pfnav_blocking *add_blocking,
                                             size_t nadd, const pfnav_flock *flocks, size_t nflocks)
{
    PF_ARG(g, "group");
    if (int rc = peer_check(g, __func__)) return rc;
    if (nremove == 0 && nadd == 0 && !flocks) return PFNAV_OK;
    const int world = (int)g->ctxs.size();
    std::vector<pf_pop_member> M(world);
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        int rc = check_shard(c, (pf_mgpu *)c->mgpu);
        if (!rc) rc = pf_pop_job_check(c, remove_uids, nremove, add, add_ms, add_ext, add_formation, add_blocking, nadd, flocks,
                                       nflocks, world, i, M[i]);
        if (rc) {
            const std::string e = pfnav_last_error();
            pfnav_set_error("%s: member %d refused the batch (%s); no member changed anything", __func__, i, e.c_str());
            return rc;
        }
    }
    for (int i = 0; i < world; i++)
        PF_ARG(g->ctxs[i]->n_agents == g->ctxs[0]->n_agents && g->ctxs[i]->n_flocks == g->ctxs[0]->n_flocks &&
               pop_tables_bits(M[i].T) == pop_tables_bits(M[0].T),
               "members hold populations, flock tables or sets of uploaded tables that differ; no member changed anything");
    int rc;
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        if ((rc = pf_pop_job_stage(c, M[i], false, c->tick_stream))) return rc;
        PF_CUDA(cudaEventRecord(g->ready[i], c->tick_stream));             // member i's survivors are compacted
    }
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        for (int s = 0; s < world; s++) {
            if (s == i) continue;
            M[i].from[s] = M[s].own;
            if (M[i].J.seg_hi(s, i) > M[i].J.seg_lo(s, i)) PF_CUDA(cudaStreamWaitEvent(c->tick_stream, g->ready[s], 0));
        }
        if ((rc = pf_pop_job_write(c, M[i], c->tick_stream))) return rc;
        PF_CUDA(cudaEventRecord(g->pulled[i], c->tick_stream));
    }
    for (int i = 0; i < world; i++) {
        pfnav_ctx *c = g->ctxs[i];
        PF_CUDA(cudaSetDevice(c->device));
        for (int p = 0; p < world; p++)
            if (p != i) PF_CUDA(cudaStreamWaitEvent(c->tick_stream, g->pulled[p], 0));
        if ((rc = pf_pop_job_commit(c, M[i], c->tick_stream))) return rc;
    }
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// State digests of a job (pfnav_digest.cu). The group form digests every member on its context stream and combines the
// members' records on the host; the NCCL form all-gathers the ranks' fixed-size records on `stream` and leaves the
// combination to pfnav_state_digest_read.
// ------------------------------------------------------------------------------------------
extern "C" int pfnav_group_state_digest(pfnav_group *g, uint32_t what, int block_log2, pfnav_digest *out, uint64_t *blocks,
                                        size_t cap, size_t *nblocks)
{
    PF_ARG(g && out, "group / out");
    PF_ARG(!blocks || nblocks, "nblocks == NULL with a block array");
    const int world = (int)g->ctxs.size();
    for (int i = 0; i < world; i++)
        if (int rc = pf_digest_check(g->ctxs[i], what, block_log2)) {
            const std::string e = pfnav_last_error();
            pfnav_set_error("%s: member %d refused the digest (%s); no member queued one", __func__, i, e.c_str());
            return rc;
        }
    const size_t n_total = g->ctxs[0]->n_agents;
    if (what & (PFNAV_DIGEST_POPULATION | PFNAV_DIGEST_RECORDS))
        for (int i = 0; i < world; i++) PF_ARG(g->ctxs[i]->n_agents == n_total, "members hold populations of different sizes");
    const size_t nb = (what & PFNAV_DIGEST_POPULATION) ? pf_digest_nblocks(n_total, block_log2) : 0;
    if (nblocks) *nblocks = nb;
    if (blocks && cap < nb) {
        pfnav_set_error("%s: the block array holds %zu entries, cap %zu", __func__, nb, cap);
        return PFNAV_ERR_NOMEM;
    }
    for (int i = 0; i < world; i++)
        if (int rc = pfnav_state_digest(g->ctxs[i], what, block_log2, nullptr)) return rc;
    pfnav_digest job;
    memset(&job, 0, sizeof(job));
    std::vector<uint64_t> mine(nb);
    if (blocks) std::fill(blocks, blocks + nb, 0);
    for (int i = 0; i < world; i++) {
        pfnav_digest &d = out[1 + i];
        size_t n = 0;
        if (int rc = pfnav_state_digest_read(g->ctxs[i], &d, mine.data(), nb, &n)) return rc;
        if (i == 0) {
            job = d;
            job.lo = 0; job.hi = n_total; job.population = 0; job.pool = 0;
        }
        const uint64_t bit = 1ull << std::min(i, 63);
        job.population += d.population;
        if (d.flocks != out[1].flocks) job.differ_flocks |= bit;
        if (d.records != out[1].records) job.differ_records |= bit;
        if (d.map != out[1].map) job.differ_map |= bit;
        if (blocks)
            for (size_t b = 0; b < nb; b++) blocks[b] += mine[b];
    }
    out[0] = job;
    return PFNAV_OK;
}

extern "C" int pfnav_mgpu_state_digest(pfnav_ctx *ctx, uint32_t what, int block_log2, void *stream)
{
    pf_mgpu *m = nullptr;
    if (int rc = nccl_rank(ctx, __func__, "pfnav_group_state_digest", &m)) return rc;
    if (int rc = pf_digest_check(ctx, what, block_log2)) return rc;
    cudaStream_t st = pf_stream(ctx, stream);
    if (int rc = pf_digest_launch(ctx, what, block_log2, st, m->world, m->rank)) return rc;
    unsigned long long *rec = ctx->d_digest.p;
    PF_NCCL(g_nccl.AllGather(rec + (size_t)m->rank * PF_DIGEST_REC, rec, PF_DIGEST_REC * sizeof(uint64_t), /*ncclInt8*/ 0,
                             m->comm, st));
    return pf_digest_finish(ctx, st);
}
