// pfnav_commands.cu -- the engine's movement commands on the device-resident population (sm_90a).
//
// pfnav_agents_commands applies per-entity deltas (pfnav_commands_host.h validates and merges them, one record per uid)
// with one thread per entity, replaces the flock table, and rebuilds the flock member lists from the flock id column
// with a stable counting sort: every warp owns a contiguous uid range, counts its entities per flock, the counts are
// scanned (pf_block_excl_scan, pfnav_scan.cuh) per flock across the warps and over the flocks, and every warp writes
// its entities behind the offsets of its range. Members are therefore ascending by uid within a flock, as the host pass
// of an upload leaves them.
// A member of a multi-GPU job takes the job's whole batch (pf_cmd_job_check / pf_cmd_job_apply, for pfnav_mgpu.cu): the
// deltas of its own uids as above, and for the others the flock id, radius and flag bits (k_apply_foreign), so that it
// rebuilds the member lists and population facts from its own complete columns.
// pfnav_agents_set_work_dev compacts the uids that are not still into the work list, in uid order, with the ordered
// compaction of pfnav_scan.cuh: count and scan, one host read of the count to size the list, then the write.
// pfnav_agents_change_population removes and appends entities (pfnav_commands_host.h plans the batch and holds the
// numbering rule): k_pop_gather writes every new row of every table with one thread per row, then the member lists,
// population facts and spatial index are rebuilt for the new population. Its job form (pf_pop_job_*, for pfnav_mgpu.cu)
// compacts each member's own survivors with k_pop_gather over a row window and the replicated record and flock columns
// with k_pop_columns; the segments of survivors that cross a member boundary move between the stages.
#include "pfnav_internal.cuh"
#include "pfnav_scan.cuh"
#include <algorithm>

#define FULL 0xFFFFFFFFu

__global__ void k_apply_deltas(const pfnav_agent_delta *__restrict__ deltas, int n, pfnav_agent *__restrict__ agents,
                               pfnav_movestate *__restrict__ mss, pfnav_movestate_ext *__restrict__ exts,
                               int32_t *__restrict__ flock_of, pf_record *__restrict__ rec)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const pfnav_agent_delta d = deltas[i];
    pfnav_agent a = agents[d.uid];
    // the host refuses the bits that write a table that was not uploaded, so these pointers are valid when used
    pf_delta_apply(&a, mss ? mss + d.uid : nullptr, exts ? exts + d.uid : nullptr, d);
    agents[d.uid] = a;
    flock_of[d.uid] = a.flock;
    pf_record r;                       // as k_make_records / k_entity_apply pack it
    r.px = a.pos[0]; r.pz = a.pos[1]; r.vx = a.velocity[0]; r.vz = a.velocity[1];
    r.radius = a.radius;
    r.state_flags = (a.state << 24) | (a.flags & 0xFFFFFFu);
    rec[d.uid] = r;
}

// a job member's writes for the entities other members own (pf_foreign_apply): flock column, radius, low flag bits
__global__ void k_apply_foreign(const pf_cmd_foreign *__restrict__ f, int n, int32_t *__restrict__ flock_of,
                                pf_record *__restrict__ rec)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const pf_cmd_foreign x = f[i];
    pf_foreign_apply(x, flock_of[x.uid], rec[x.uid].radius, rec[x.uid].state_flags);
}

// ---- flock member lists: stable counting sort of the uids by flock ----
// Warp w owns uids [w * per, (w + 1) * per), per a multiple of 32; hist is [nflocks][W]. Only the warp itself touches
// its column, one leader lane per flock and step, so plain read-modify-writes ordered by __syncwarp are enough.
__global__ void k_flock_hist(const int32_t *__restrict__ flock_of, int n, int per, int W, uint32_t *hist)
{
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= W) return;
    const int lo = w * per, hi = min(lo + per, n);
    for (int base = lo; base < hi; base += 32) {
        const int i = base + lane;
        const int32_t f = i < hi ? flock_of[i] : -1;
        const unsigned m = __match_any_sync(FULL, f);
        if (f >= 0 && lane == __ffs(m) - 1) hist[(size_t)f * W + w] += __popc(m);
        __syncwarp();
    }
}

// block f: the counts of flock f become each warp's offset within the flock; the flock's size goes to start[f + 1]
__global__ void __launch_bounds__(1024) k_flock_scan(uint32_t *hist, int W, uint32_t *__restrict__ start)
{
    __shared__ uint32_t wsum[32];
    uint32_t *row = hist + (size_t)blockIdx.x * W;
    uint32_t carry = 0;
    for (int base = 0; base < W; base += 1024) {
        const int w = base + threadIdx.x;
        const uint32_t v = w < W ? row[w] : 0;
        uint32_t total;
        const uint32_t e = pf_block_excl_scan(v, wsum, total);
        if (w < W) row[w] = carry + e;
        carry += total;
    }
    if (threadIdx.x == 0) start[blockIdx.x + 1] = carry;
}

// one block: start[1 .. nflocks] holds the flock sizes; make start[0 .. nflocks] the offsets
__global__ void __launch_bounds__(1024) k_flock_starts(uint32_t *__restrict__ start, int nflocks)
{
    __shared__ uint32_t wsum[32];
    uint32_t carry = 0;
    for (int base = 0; base < nflocks; base += 1024) {
        const int f = base + threadIdx.x;
        const uint32_t v = f < nflocks ? start[f + 1] : 0;
        uint32_t total;
        const uint32_t e = pf_block_excl_scan(v, wsum, total);
        if (f < nflocks) start[f + 1] = carry + e + v;
        carry += total;
    }
    if (threadIdx.x == 0) start[0] = 0;
}

__global__ void k_flock_scatter(const int32_t *__restrict__ flock_of, int n, int per, int W, uint32_t *hist,
                                const uint32_t *__restrict__ start, uint32_t *__restrict__ members)
{
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= W) return;
    const int lo = w * per, hi = min(lo + per, n);
    for (int base = lo; base < hi; base += 32) {
        const int i = base + lane;
        const int32_t f = i < hi ? flock_of[i] : -1;
        const unsigned m = __match_any_sync(FULL, f);
        const int leader = __ffs(m) - 1;
        uint32_t off = 0;
        if (f >= 0 && lane == leader) { off = hist[(size_t)f * W + w]; hist[(size_t)f * W + w] = off + __popc(m); }
        off = __shfl_sync(FULL, off, leader);
        if (f >= 0) members[start[f] + off + __popc(m & ((1u << lane) - 1))] = (uint32_t)i;
        __syncwarp();
    }
}

// ---- work list: the own range's uids that are not still (ent_still, movement.c:652), ascending ----
// The ordered compaction of pfnav_scan.cuh over the uids [lo, hi). The state is read from the 24-byte neighbour records
// (state << 24 | flags), which every writer of agent.state keeps current (k_make_records, k_entity_apply,
// k_apply_deltas): a seventh of the agent table's stride.
struct work_compact {
    const pf_record *rec; uint32_t *work;
    __device__ bool keep(int i) const
    {
        const uint32_t s = rec[i].state_flags >> 24;
        return s != PFNAV_STATE_ARRIVED && s != PFNAV_STATE_WAITING;
    }
    __device__ void emit(int i, uint32_t slot) const { work[slot] = (uint32_t)i; }
};

// ---- population change: new rows [row0, n_new) of every table, by the numbering rule of pf_pop_source ----
// Rows below n_keep are survivors, gathered from the tables as they were (surround targets renumbered); rows from n_keep
// on are the appended records, or the defaults the tick uses for a missing table. o_ms / o_ext / o_form / o_blk are null
// for a table that does not exist; a_ext / a_form null for defaults.
struct pf_pop_gather {
    const pfnav_agent *agents; const pfnav_movestate *ms; const pfnav_movestate_ext *ext;
    const pfnav_formation_in *form; const pfnav_blocking *blk;
    const pfnav_agent *a_agents; const pfnav_movestate *a_ms; const pfnav_movestate_ext *a_ext;
    const pfnav_formation_in *a_form; const pfnav_blocking *a_blk;
    pfnav_agent *o_agents; pf_record *o_rec; int32_t *o_flock; pfnav_movestate *o_ms; pfnav_movestate_ext *o_ext;
    pfnav_formation_in *o_form; pfnav_blocking *o_blk;
    const uint32_t *removed, *key; uint32_t R, n_old;
    int row0, row1, out0, n_keep, n_new;     // new rows [row0, row1), written at index row - out0 of the o_ tables
    uint32_t *any_fac;           // set when a written blocking record names a faction other than 15
};

__device__ __forceinline__ pf_record pop_record(const pfnav_agent &a)
{
    pf_record r;                       // as k_make_records packs it
    r.px = a.pos[0]; r.pz = a.pos[1]; r.vx = a.velocity[0]; r.vz = a.velocity[1];
    r.radius = a.radius;
    r.state_flags = (a.state << 24) | (a.flags & 0xFFFFFFu);
    return r;
}

__global__ void k_pop_gather(const pf_pop_gather g)
{
    const int i = g.row0 + blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= g.row1) return;
    const int o = i - g.out0;
    pfnav_agent a;
    pfnav_blocking b;
    if (i < g.n_keep) {
        const uint32_t s = pf_pop_source(g.key, g.R, (uint32_t)i);
        a = g.agents[s];
        if (g.o_ms) g.o_ms[o] = g.ms[s];
        if (g.o_ext) {
            pfnav_movestate_ext x = g.ext[s];
            if (x.surround_target_uid != PFNAV_NULL_UID)
                x.surround_target_uid = pf_pop_renumber(g.removed, g.R, g.n_old, x.surround_target_uid);
            g.o_ext[o] = x;
        }
        if (g.o_form) g.o_form[o] = g.form[s];
        if (g.o_blk) b = g.blk[s];
    } else {
        const int k = i - g.n_keep;
        a = g.a_agents[k];
        if (g.o_ms) g.o_ms[o] = g.a_ms[k];
        if (g.o_ext) {
            pfnav_movestate_ext x = {};
            if (g.a_ext) x = g.a_ext[k];
            else { x.surround_target_uid = PFNAV_NULL_UID; x.rot[3] = 1.0f; }
            g.o_ext[o] = x;
        }
        if (g.o_form) {
            pfnav_formation_in f = {};
            if (g.a_form) f = g.a_form[k];
            g.o_form[o] = f;
        }
        if (g.o_blk) b = g.a_blk[k];
    }
    g.o_agents[o] = a;
    g.o_flock[o] = a.flock;
    g.o_rec[o] = pop_record(a);
    if (g.o_blk) {
        g.o_blk[o] = b;
        if (b.faction_id < 15) *g.any_fac = 1u;
    }
}

// A job member's replicated columns over the new population. It holds valid agent rows for its own range only, so the
// survivors' records and flock ids are compacted from the columns themselves (their radius, flag bits and flock id are
// current on every member; position, velocity and state of other members' entities arrive with the next gather) and
// the appended entities' are packed from their agent records.
__global__ void k_pop_columns(const pf_record *__restrict__ rec, const int32_t *__restrict__ flock, const uint32_t *__restrict__ key,
                              uint32_t R, int n_keep, int n_new, const pfnav_agent *__restrict__ a_agents,
                              pf_record *__restrict__ o_rec, int32_t *__restrict__ o_flock)
{
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_new) return;
    if (i < n_keep) {
        const uint32_t s = pf_pop_source(key, R, (uint32_t)i);
        o_rec[i] = rec[s];
        o_flock[i] = flock[s];
    } else {
        const pfnav_agent a = a_agents[i - n_keep];
        o_rec[i] = pop_record(a);
        o_flock[i] = a.flock;
    }
}

// *word = 1 when a blocking record of [lo, hi) names a faction other than 15 (pfnav_agents_upload_blocking's fact)
__global__ void k_pop_any_fac(const pfnav_blocking *__restrict__ b, int lo, int hi, uint32_t *word)
{
    const int i = lo + blockIdx.x * blockDim.x + threadIdx.x;
    if (i < hi && b[i].faction_id < 15) *word = 1u;
}

// ------------------------------------------------------------------------------------------
// Host side
// ------------------------------------------------------------------------------------------
// d_flock_start / d_flock_members from d_flock_of on `st`; hist: nflocks * W words of scratch
static int members_on_device(pfnav_ctx *ctx, cudaStream_t st, uint32_t *hist, int per, int W)
{
    const int n = (int)ctx->n_agents, nflocks = (int)ctx->n_flocks;
    PF_CUDA(cudaMemsetAsync(ctx->d_flock_start, 0, ((size_t)nflocks + 1) * 4, st));
    if (n && nflocks) {
        PF_CUDA(cudaMemsetAsync(hist, 0, (size_t)nflocks * W * 4, st));
        PF_CUDA(cudaMemsetAsync(ctx->d_flock_members, 0, (size_t)n * 4, st));      // the tail behind the last flock, as an upload leaves it
        const int ctas = (W + 7) / 8;
        k_flock_hist<<<ctas, 256, 0, st>>>(ctx->d_flock_of, n, per, W, hist);
        k_flock_scan<<<nflocks, 1024, 0, st>>>(hist, W, ctx->d_flock_start);
        k_flock_starts<<<1, 1024, 0, st>>>(ctx->d_flock_start, nflocks);
        k_flock_scatter<<<ctas, 256, 0, st>>>(ctx->d_flock_of, n, per, W, hist, ctx->d_flock_start, ctx->d_flock_members);
        ctx->launches += 4;
        PF_CUDA(cudaGetLastError());
    }
    // the tick sizes its cohesion pass from the biggest flock
    std::vector<uint32_t> fstart((size_t)nflocks + 1, 0);
    PF_CUDA(cudaMemcpyAsync(fstart.data(), ctx->d_flock_start, fstart.size() * 4, cudaMemcpyDeviceToHost, st));
    PF_CUDA(cudaStreamSynchronize(st));
    ctx->h_flock_start.swap(fstart);
    return 0;
}

// warps of the member sort of n entities over nflocks flocks: at most 4096 ranges of `per` uids (a multiple of 32), and at
// most 16 M histogram words
static void member_sort_shape(size_t n, size_t nflocks, int &per, int &W)
{
    const size_t max_w = std::max<size_t>(1, std::min<size_t>(4096, ((size_t)1 << 24) / std::max<size_t>(nflocks, 1)));
    per = (int)(((n + max_w - 1) / max_w + 31) / 32 * 32);
    W = per ? (int)((n + per - 1) / per) : 0;
}

static int cmd_apply(pfnav_ctx *ctx, cudaStream_t st, const std::vector<pfnav_agent_delta> &merged,
                     const std::vector<pf_cmd_foreign> &foreign, const std::vector<pf_cmd_change> &changes,
                     const pfnav_flock *flocks, size_t nflocks);

extern "C" int pfnav_agents_commands(pfnav_ctx *ctx, const pfnav_agent_delta *deltas, size_t n, const pfnav_flock *flocks,
                                     size_t nflocks, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_agents, "agents not uploaded");
    if (ctx->mgpu || ctx->shard_lo > 0 || ctx->shard_hi < ctx->n_agents) {
        pfnav_set_error("pfnav_agents_commands: the context is part of a multi-GPU job (the other members would keep the old "
                        "flock table and flock column)");
        return PFNAV_ERR_STATE;
    }
    PF_ARG(deltas || n == 0, "deltas == NULL");
    PF_ARG(n < (1u << 31) && nflocks < (1u << 31), "n / nflocks");
    if (!flocks) nflocks = ctx->n_flocks;
    pf_cmd_limits lim = {ctx->shard_lo, ctx->shard_hi, ctx->n_agents, nflocks, ctx->movestate_set && ctx->d_movestate != nullptr,
                         ctx->d_ms_ext != nullptr};
    std::vector<pfnav_agent_delta> merged;
    std::vector<pf_cmd_change> changes;
    const char *err = pf_cmd_merge(deltas, n, lim, merged);
    if (!err) err = pf_cmd_plan(ctx->cmd_mirror, ctx->shard_lo, merged, nflocks, ctx->nlayers, changes);
    PF_ARG(!err, err);
    if (merged.empty() && !flocks) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    return cmd_apply(ctx, pf_stream(ctx, stream), merged, {}, changes, flocks, nflocks);
}

// Everything after validation, on `st`: the flock table, the merged records of the own range (k_apply_deltas), a job
// member's foreign records (k_apply_foreign), the host facts, the member lists and the population facts.
static int cmd_apply(pfnav_ctx *ctx, cudaStream_t st, const std::vector<pfnav_agent_delta> &merged,
                     const std::vector<pf_cmd_foreign> &foreign, const std::vector<pf_cmd_change> &changes,
                     const pfnav_flock *flocks, size_t nflocks)
{
    ctx->index_stale = true;            // the deltas write records: the position index waits for the next rebuild
    uint32_t any = 0;
    for (const pfnav_agent_delta &m : merged) any |= m.mask;
    for (const pf_cmd_foreign &f : foreign) any |= f.mask;
    const bool members = (any & PFNAV_DELTA_FLOCK) || nflocks != ctx->n_flocks;
    int rc, per, W;
    member_sort_shape(ctx->n_agents, nflocks, per, W);
    const size_t b_deltas = merged.size() * sizeof(pfnav_agent_delta), b_foreign = foreign.size() * sizeof(pf_cmd_foreign);
    if ((rc = ctx->d_cmd_buf.reserve(b_deltas + b_foreign + (members ? nflocks * (size_t)W * 4 : 0)))) return rc;
    // keeps no content: the table follows, the offsets are rebuilt (members)
    if ((rc = pf_flocks_reserve(ctx, nflocks))) return rc;
    if (flocks) {
        // from the context's own pageable copy, which is staged before the call returns: the caller's array may be pinned
        ctx->h_flocks.assign(flocks, flocks + nflocks);
        if (nflocks) PF_CUDA(cudaMemcpyAsync(ctx->d_flocks, ctx->h_flocks.data(), nflocks * sizeof(pfnav_flock), cudaMemcpyHostToDevice, st));
        ctx->n_flocks = nflocks;
    }
    if (!merged.empty()) {
        const bool have_ms = ctx->movestate_set && ctx->d_movestate != nullptr;
        PF_CUDA(cudaMemcpyAsync(ctx->d_cmd_buf, merged.data(), b_deltas, cudaMemcpyHostToDevice, st));
        k_apply_deltas<<<((int)merged.size() + 127) / 128, 128, 0, st>>>((const pfnav_agent_delta *)ctx->d_cmd_buf.p, (int)merged.size(),
            ctx->d_agents, have_ms ? ctx->d_movestate.p : nullptr, ctx->d_ms_ext, ctx->d_flock_of, ctx->d_records);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    if (!foreign.empty()) {
        pf_cmd_foreign *d_foreign = (pf_cmd_foreign *)(ctx->d_cmd_buf + b_deltas);
        PF_CUDA(cudaMemcpyAsync(d_foreign, foreign.data(), b_foreign, cudaMemcpyHostToDevice, st));
        k_apply_foreign<<<((int)foreign.size() + 127) / 128, 128, 0, st>>>(d_foreign, (int)foreign.size(), ctx->d_flock_of,
                                                                             ctx->d_records);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    // host facts, as a fresh upload of the resulting population (of the own range, on a job member) would leave them
    pf_cmd_commit(ctx->cmd_mirror, changes, nflocks);
    std::vector<uint8_t> used;
    ctx->cmd_mirror.used(used);
    if (flocks || used != ctx->flock_layer_used) ctx->arrival_valid = false;
    ctx->flock_layer_used.swap(used);
    if (members && (rc = members_on_device(ctx, st, (uint32_t *)(ctx->d_cmd_buf + b_deltas + b_foreign), per, W))) return rc;
    if ((any & (PFNAV_DELTA_RADIUS | PFNAV_DELTA_FLAGS)) && (rc = pfnav_agents_refresh_facts(ctx, st))) return rc;
    return PFNAV_OK;
}

// Everything after validation, on `st`. The tables are gathered by k_pop_gather: in place when nothing is removed and no
// table regrows (only the appended rows are written), otherwise into the command scratch and copied back once the tables
// have regrown, since pf_dbuf::reserve drops the contents of a buffer it grows. Scratch: [gathered tables] [removals, keys,
// appended records, the any-faction word]; the member sort's histogram reuses it from the start afterwards.
static int pop_apply(pfnav_ctx *ctx, cudaStream_t st, const pf_pop_tables &T, const pf_pop_plan &P, const pfnav_agent *add,
                     const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext, const pfnav_formation_in *add_form,
                     const pfnav_blocking *add_blk, size_t nadd, const pfnav_flock *flocks, size_t nflocks)
{
    const size_t R = P.removed.size(), n_new = P.n_new;
    const bool full = R > 0 || std::min({ctx->d_agents.cap, ctx->d_records.cap, ctx->d_flock_of.cap}) < n_new ||
                      (T.ms && ctx->d_movestate.cap < n_new) || (T.ext && ctx->d_ms_ext.cap < n_new) ||
                      (T.formation && ctx->d_formation.cap < n_new) || (T.blocking && ctx->d_blocking.cap < n_new);
    size_t top = 0;
    auto take = [&top](size_t bytes) { const size_t o = top; top += (bytes + 255) & ~(size_t)255; return o; };
    const size_t rows = full ? n_new : 0;
    const size_t g_agents = take(rows * sizeof(pfnav_agent)), g_rec = take(rows * sizeof(pf_record)), g_flock = take(rows * 4);
    const size_t g_ms = take(T.ms ? rows * sizeof(pfnav_movestate) : 0), g_ext = take(T.ext ? rows * sizeof(pfnav_movestate_ext) : 0);
    const size_t g_form = take(T.formation ? rows * sizeof(pfnav_formation_in) : 0);
    const size_t g_blk = take(T.blocking ? rows * sizeof(pfnav_blocking) : 0);
    // the staged inputs, one copy from one host image
    const size_t s0 = top;
    const size_t s_removed = take(R * 4) - s0, s_key = take(R * 4) - s0, s_agents = take(nadd * sizeof(pfnav_agent)) - s0;
    const size_t s_ms = take(add_ms ? nadd * sizeof(pfnav_movestate) : 0) - s0;
    const size_t s_ext = take(add_ext ? nadd * sizeof(pfnav_movestate_ext) : 0) - s0;
    const size_t s_form = take(add_form ? nadd * sizeof(pfnav_formation_in) : 0) - s0;
    const size_t s_blk = take(add_blk ? nadd * sizeof(pfnav_blocking) : 0) - s0;
    const size_t s_fac = take(4) - s0;
    std::vector<uint8_t> h(top - s0, 0);
    auto put = [&h](size_t off, const void *src, size_t bytes) { if (bytes) memcpy(h.data() + off, src, bytes); };
    put(s_removed, P.removed.data(), R * 4); put(s_key, P.key.data(), R * 4);
    put(s_agents, add, nadd * sizeof(pfnav_agent));
    if (add_ms) put(s_ms, add_ms, nadd * sizeof(pfnav_movestate));
    if (add_ext) put(s_ext, add_ext, nadd * sizeof(pfnav_movestate_ext));
    if (add_form) put(s_form, add_form, nadd * sizeof(pfnav_formation_in));
    if (add_blk) put(s_blk, add_blk, nadd * sizeof(pfnav_blocking));
    int per, W;
    member_sort_shape(n_new, nflocks, per, W);
    int rc;
    if ((rc = ctx->d_cmd_buf.reserve(std::max(top, nflocks * (size_t)W * 4)))) return rc;
    if ((rc = pf_flocks_reserve(ctx, nflocks))) return rc;        // keeps no content: the table follows, the offsets are rebuilt
    uint8_t *buf = ctx->d_cmd_buf.p, *stage = buf + s0;
    PF_CUDA(cudaMemcpyAsync(stage, h.data(), h.size(), cudaMemcpyHostToDevice, st));
    const uint32_t *d_removed = (const uint32_t *)(stage + s_removed);
    // the blocks of removed entities are released as pfnav_agents_set_blocking(removed, 0) would, before the compaction
    if (T.blocking && R && (rc = blocking_emit(ctx, st, d_removed, (int)R, nullptr, 0))) return rc;
    if (flocks) {
        // from the context's own pageable copy, which is staged before the call returns: the caller's array may be pinned
        ctx->h_flocks.assign(flocks, flocks + nflocks);
        if (nflocks) PF_CUDA(cudaMemcpyAsync(ctx->d_flocks, ctx->h_flocks.data(), nflocks * sizeof(pfnav_flock), cudaMemcpyHostToDevice, st));
    }
    pf_pop_gather g = {};
    g.agents = ctx->d_agents; g.ms = T.ms ? ctx->d_movestate.p : nullptr; g.ext = ctx->d_ms_ext; g.form = ctx->d_formation;
    g.blk = T.blocking ? ctx->d_blocking.p : nullptr;
    g.a_agents = (const pfnav_agent *)(stage + s_agents);
    g.a_ms = add_ms ? (const pfnav_movestate *)(stage + s_ms) : nullptr;
    g.a_ext = add_ext ? (const pfnav_movestate_ext *)(stage + s_ext) : nullptr;
    g.a_form = add_form ? (const pfnav_formation_in *)(stage + s_form) : nullptr;
    g.a_blk = add_blk ? (const pfnav_blocking *)(stage + s_blk) : nullptr;
    if (full) {
        g.o_agents = (pfnav_agent *)(buf + g_agents); g.o_rec = (pf_record *)(buf + g_rec); g.o_flock = (int32_t *)(buf + g_flock);
        g.o_ms = T.ms ? (pfnav_movestate *)(buf + g_ms) : nullptr;
        g.o_ext = T.ext ? (pfnav_movestate_ext *)(buf + g_ext) : nullptr;
        g.o_form = T.formation ? (pfnav_formation_in *)(buf + g_form) : nullptr;
        g.o_blk = T.blocking ? (pfnav_blocking *)(buf + g_blk) : nullptr;
    } else {
        g.o_agents = ctx->d_agents; g.o_rec = ctx->d_records; g.o_flock = ctx->d_flock_of;
        g.o_ms = T.ms ? ctx->d_movestate.p : nullptr; g.o_ext = ctx->d_ms_ext; g.o_form = ctx->d_formation;
        g.o_blk = T.blocking ? ctx->d_blocking.p : nullptr;
    }
    g.removed = d_removed; g.key = (const uint32_t *)(stage + s_key); g.R = (uint32_t)R; g.n_old = (uint32_t)P.n_old;
    g.row0 = full ? 0 : (int)P.n_keep; g.row1 = (int)n_new; g.out0 = 0; g.n_keep = (int)P.n_keep; g.n_new = (int)n_new;
    uint32_t *d_fac = (uint32_t *)(stage + s_fac);
    g.any_fac = d_fac;
    if (n_new > (size_t)g.row0) {
        k_pop_gather<<<((int)n_new - g.row0 + 127) / 128, 128, 0, st>>>(g);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    // the tables at their new length (a regrowth waits for the device, so the gather has finished), then the copy back
    if ((rc = pf_dbuf_reserve_all(n_new, ctx->d_agents, ctx->d_records, ctx->d_flock_members, ctx->d_flock_of, ctx->d_sorted_ix,
                                  ctx->d_sorted_iy, ctx->d_sorted_flock, ctx->d_sorted_id))) return rc;
    if (T.ms && (rc = ctx->d_movestate.reserve(n_new))) return rc;
    if (T.ext && (rc = ctx->d_ms_ext.reserve(n_new))) return rc;
    if (T.formation && (rc = ctx->d_formation.reserve(n_new))) return rc;
    if (T.blocking && (rc = ctx->d_blocking.reserve(std::max<size_t>(n_new, 1)))) { ctx->blocking_n = 0; return rc; }
    if (full && n_new) {
        auto back = [&](void *dst, size_t off, size_t elem) { return cudaMemcpyAsync(dst, buf + off, n_new * elem, cudaMemcpyDeviceToDevice, st); };
        PF_CUDA(back(ctx->d_agents, g_agents, sizeof(pfnav_agent)));
        PF_CUDA(back(ctx->d_records, g_rec, sizeof(pf_record)));
        PF_CUDA(back(ctx->d_flock_of, g_flock, 4));
        if (T.ms) PF_CUDA(back(ctx->d_movestate, g_ms, sizeof(pfnav_movestate)));
        if (T.ext) PF_CUDA(back(ctx->d_ms_ext, g_ext, sizeof(pfnav_movestate_ext)));
        if (T.formation) PF_CUDA(back(ctx->d_formation, g_form, sizeof(pfnav_formation_in)));
        if (T.blocking) PF_CUDA(back(ctx->d_blocking, g_blk, sizeof(pfnav_blocking)));
    }
    // host facts, as a fresh upload of the resulting population would leave them
    ctx->n_agents = n_new; ctx->shard_lo = 0; ctx->shard_hi = n_new; ctx->n_flocks = nflocks;
    ctx->cmd_mirror.compact_append(P.removed, P.add_flock.data(), P.add_layer.data(), nadd, nflocks);
    std::vector<uint8_t> used;
    ctx->cmd_mirror.used(used);
    if (flocks || used != ctx->flock_layer_used) ctx->arrival_valid = false;
    ctx->flock_layer_used.swap(used);
    ctx->n_work = 0;
    if (T.blocking) {
        ctx->blocking_n = n_new;
        if (ctx->blocking_any_fac && R) {
            // some survivor may have held the only faction other than 15: the gather, which wrote every row, tells
            uint32_t fac = 0;
            PF_CUDA(cudaMemcpyAsync(&fac, d_fac, 4, cudaMemcpyDeviceToHost, st));
            PF_CUDA(cudaStreamSynchronize(st));
            ctx->blocking_any_fac = fac != 0;
        } else {
            ctx->blocking_any_fac = ctx->blocking_any_fac || P.add_any_fac;
        }
    }
    if ((rc = members_on_device(ctx, st, (uint32_t *)buf, per, W))) return rc;
    if ((rc = pfnav_agents_refresh_facts(ctx, st))) return rc;
    return build_index(ctx, st);
}

extern "C" int pfnav_agents_change_population(pfnav_ctx *ctx, const uint32_t *remove_uids, size_t nremove, const pfnav_agent *add,
                                              const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext,
                                              const pfnav_formation_in *add_formation, const pfnav_blocking *add_blocking,
                                              size_t nadd, const pfnav_flock *flocks, size_t nflocks, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_agents, "agents not uploaded");
    if (ctx->mgpu || ctx->shard_lo > 0 || ctx->shard_hi < ctx->n_agents) {
        pfnav_set_error("pfnav_agents_change_population: the context is part of a multi-GPU job (a population change would "
                        "move the other members' entity ranges)");
        return PFNAV_ERR_STATE;
    }
    PF_ARG(nremove < (1u << 31) && nadd < (1u << 31) && nflocks < (1u << 31), "nremove / nadd / nflocks");
    if (!flocks) nflocks = ctx->n_flocks;
    const pf_pop_tables T = {ctx->movestate_set && ctx->d_movestate != nullptr, ctx->d_ms_ext != nullptr,
                             ctx->d_formation != nullptr, ctx->d_blocking != nullptr && ctx->blocking_n == ctx->n_agents};
    pf_pop_plan P;
    const char *err = pf_pop_plan_batch(ctx->cmd_mirror, ctx->nlayers, T, remove_uids, nremove, add, add_ms, add_ext,
                                        add_formation, add_blocking, nadd, nflocks, P);
    PF_ARG(!err, err);
    if (P.removed.empty() && nadd == 0 && !flocks) return PFNAV_OK;
    ctx->events_valid = false;              // the event list's uids name the previous population
    PF_CUDA(cudaSetDevice(ctx->device));
    return pop_apply(ctx, pf_stream(ctx, stream), T, P, add, add_ms, add_ext, add_formation, add_blocking, nadd, flocks, nflocks);
}

// ---- the job form of a population change (pfnav_mgpu.cu runs the verdict exchange and moves the segments) ----
int pf_pop_job_check(pfnav_ctx *ctx, const uint32_t *remove_uids, size_t nremove, const pfnav_agent *add,
                     const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext, const pfnav_formation_in *add_form,
                     const pfnav_blocking *add_blk, size_t nadd, const pfnav_flock *flocks, size_t nflocks, int world, int rank,
                     pf_pop_member &M)
{
    PF_ARG(ctx->d_agents, "agents not uploaded");
    if (ctx->members_stale) {
        pfnav_set_error("the member's flock column is incomplete until the gather that follows pfnav_agents_upload_shard");
        return PFNAV_ERR_STATE;
    }
    PF_ARG(nremove < (1u << 31) && nadd < (1u << 31) && nflocks < (1u << 31), "nremove / nadd / nflocks");
    M.flocks = flocks;
    M.nflocks = flocks ? nflocks : ctx->n_flocks;
    M.T = {ctx->movestate_set && ctx->d_movestate != nullptr, ctx->d_ms_ext != nullptr, ctx->d_formation != nullptr,
           ctx->d_blocking != nullptr && ctx->blocking_n == ctx->n_agents};
    M.add = add; M.add_ms = add_ms; M.add_ext = add_ext; M.add_form = add_form; M.add_blk = add_blk; M.nadd = nadd;
    const char *err = pf_pop_job_plan(ctx->cmd_mirror, ctx->n_agents, world, rank, ctx->nlayers, M.T, remove_uids, nremove, add,
                                      add_ms, add_ext, add_form, add_blk, nadd, M.nflocks, M.J);
    PF_ARG(!err, err);
    return PFNAV_OK;
}

// a block of `rows` rows of every table that exists, taken from the scratch at base + top (base null: sizing only)
static pf_pop_rows pop_rows(uint8_t *base, size_t &top, size_t rows, const pf_pop_tables &T, size_t first, int device)
{
    auto take = [&](size_t bytes) { uint8_t *p = (uint8_t *)((uintptr_t)base + top); top += (bytes + 255) & ~(size_t)255; return p; };
    pf_pop_rows b;
    b.agents = (pfnav_agent *)take(rows * sizeof(pfnav_agent));
    b.rec = (pf_record *)take(rows * sizeof(pf_record));
    b.flock = (int32_t *)take(rows * 4);
    if (T.ms) b.ms = (pfnav_movestate *)take(rows * sizeof(pfnav_movestate));
    if (T.ext) b.ext = (pfnav_movestate_ext *)take(rows * sizeof(pfnav_movestate_ext));
    if (T.formation) b.form = (pfnav_formation_in *)take(rows * sizeof(pfnav_formation_in));
    if (T.blocking) b.blk = (pfnav_blocking *)take(rows * sizeof(pfnav_blocking));
    b.first = first; b.device = device;
    return b;
}

// the rows of every table for the new uids [a, a + n) of this member, from block b (on this or a peer device)
static int pop_copy_rows(pfnav_ctx *ctx, const pf_pop_rows &b, const pf_pop_tables &T, size_t a, size_t n, cudaStream_t st)
{
    const size_t k = a - b.first;
    auto cp = [&](void *dst, const void *src, size_t bytes) { return cudaMemcpyPeerAsync(dst, ctx->device, src, b.device, bytes, st); };
    PF_CUDA(cp(ctx->d_agents + a, b.agents + k, n * sizeof(pfnav_agent)));
    PF_CUDA(cp(ctx->d_records + a, b.rec + k, n * sizeof(pf_record)));
    PF_CUDA(cp(ctx->d_flock_of + a, b.flock + k, n * 4));
    if (T.ms) PF_CUDA(cp(ctx->d_movestate + a, b.ms + k, n * sizeof(pfnav_movestate)));
    if (T.ext) PF_CUDA(cp(ctx->d_ms_ext + a, b.ext + k, n * sizeof(pfnav_movestate_ext)));
    if (T.formation) PF_CUDA(cp(ctx->d_formation + a, b.form + k, n * sizeof(pfnav_formation_in)));
    if (T.blocking) PF_CUDA(cp(ctx->d_blocking + a, b.blk + k, n * sizeof(pfnav_blocking)));
    return 0;
}

// k_pop_gather of the new rows [row0, row1) from the member's tables as they were and the staged appended records
static pf_pop_gather pop_gather_args(pfnav_ctx *ctx, const pf_pop_member &M, size_t row0, size_t row1, size_t out0)
{
    const pf_pop_tables &T = M.T;
    const pf_pop_plan &P = M.J.P;
    uint8_t *st = M.stage;
    pf_pop_gather g = {};
    g.agents = ctx->d_agents; g.ms = T.ms ? ctx->d_movestate.p : nullptr; g.ext = ctx->d_ms_ext; g.form = ctx->d_formation;
    g.blk = T.blocking ? ctx->d_blocking.p : nullptr;
    g.a_agents = (const pfnav_agent *)(st + M.s_agents);
    g.a_ms = M.add_ms ? (const pfnav_movestate *)(st + M.s_ms) : nullptr;
    g.a_ext = M.add_ext ? (const pfnav_movestate_ext *)(st + M.s_ext) : nullptr;
    g.a_form = M.add_form ? (const pfnav_formation_in *)(st + M.s_form) : nullptr;
    g.a_blk = M.add_blk ? (const pfnav_blocking *)(st + M.s_blk) : nullptr;
    g.removed = (const uint32_t *)(st + M.s_removed); g.key = (const uint32_t *)(st + M.s_key);
    g.R = (uint32_t)P.removed.size(); g.n_old = (uint32_t)P.n_old;
    g.row0 = (int)row0; g.row1 = (int)row1; g.out0 = (int)out0; g.n_keep = (int)P.n_keep; g.n_new = (int)P.n_new;
    g.any_fac = (uint32_t *)(st + M.s_fac);              // word 0: the gathers' (unused), word 1: k_pop_any_fac's
    return g;
}

static void pop_launch(pfnav_ctx *ctx, const pf_pop_gather &g, cudaStream_t st)
{
    k_pop_gather<<<(g.row1 - g.row0 + 127) / 128, 128, 0, st>>>(g);
    ctx->launches++;
}

// Scratch: [own survivors' block] [compacted record column] [compacted flock column] [receive blocks] [staged inputs]; the
// member sort's histogram reuses it from the start in pf_pop_job_commit.
int pf_pop_job_stage(pfnav_ctx *ctx, pf_pop_member &M, bool receive_all, cudaStream_t st)
{
    const pf_pop_job &J = M.J;
    const pf_pop_plan &P = J.P;
    const pf_pop_tables &T = M.T;
    const int r = J.rank, world = J.world;
    const size_t R = P.removed.size(), n_new = P.n_new, nadd = M.nadd;
    ctx->events_valid = false;              // the event list's uids name the previous population
    auto layout = [&](uint8_t *base) {
        size_t top = 0;
        auto take = [&](size_t bytes) { const size_t o = top; top += (bytes + 255) & ~(size_t)255; return o; };
        M.own = pop_rows(base, top, J.keep_lo[r + 1] - J.keep_lo[r], T, J.keep_lo[r], ctx->device);
        M.c_rec = (pf_record *)((uintptr_t)base + take(n_new * sizeof(pf_record)));
        M.c_flock = (int32_t *)((uintptr_t)base + take(n_new * 4));
        M.pair.clear();
        if (receive_all)
            for (int s = 0; s < world; s++)
                for (int q = 0; q < world; q++)
                    M.pair.push_back(pop_rows(base, top, s == q ? 0 : J.seg_hi(s, q) - J.seg_lo(s, q), T, J.seg_lo(s, q), ctx->device));
        const size_t s0 = top;
        M.stage = (uint8_t *)((uintptr_t)base + s0);
        M.s_removed = take(R * 4) - s0; M.s_key = take(R * 4) - s0; M.s_agents = take(nadd * sizeof(pfnav_agent)) - s0;
        M.s_ms = take(M.add_ms ? nadd * sizeof(pfnav_movestate) : 0) - s0;
        M.s_ext = take(M.add_ext ? nadd * sizeof(pfnav_movestate_ext) : 0) - s0;
        M.s_form = take(M.add_form ? nadd * sizeof(pfnav_formation_in) : 0) - s0;
        M.s_blk = take(M.add_blk ? nadd * sizeof(pfnav_blocking) : 0) - s0;
        M.s_fac = take(8) - s0;
        return std::make_pair(s0, top);
    };
    int per, W, rc;
    member_sort_shape(n_new, M.nflocks, per, W);
    const size_t top = layout(nullptr).second;
    if ((rc = ctx->d_cmd_buf.reserve(std::max(top, M.nflocks * (size_t)W * 4)))) return rc;
    if ((rc = pf_flocks_reserve(ctx, M.nflocks))) return rc;     // keeps no content: the table follows, the offsets are rebuilt
    const size_t s0 = layout(ctx->d_cmd_buf.p).first;
    M.from.assign(world, pf_pop_rows());
    for (int s = 0; s < world; s++) M.from[s] = s == r ? M.own : receive_all ? M.pair[(size_t)s * world + r] : pf_pop_rows();
    // the staged inputs, one copy from one host image
    std::vector<uint8_t> h(top - s0, 0);
    auto put = [&h](size_t off, const void *src, size_t bytes) { if (bytes) memcpy(h.data() + off, src, bytes); };
    put(M.s_removed, P.removed.data(), R * 4); put(M.s_key, P.key.data(), R * 4);
    put(M.s_agents, M.add, nadd * sizeof(pfnav_agent));
    if (M.add_ms) put(M.s_ms, M.add_ms, nadd * sizeof(pfnav_movestate));
    if (M.add_ext) put(M.s_ext, M.add_ext, nadd * sizeof(pfnav_movestate_ext));
    if (M.add_form) put(M.s_form, M.add_form, nadd * sizeof(pfnav_formation_in));
    if (M.add_blk) put(M.s_blk, M.add_blk, nadd * sizeof(pfnav_blocking));
    PF_CUDA(cudaMemcpyAsync(M.stage, h.data(), h.size(), cudaMemcpyHostToDevice, st));
    // the blocks of the member's removed entities are released as pfnav_agents_set_blocking(removed, 0) would, before
    // anything moves
    const size_t m0 = std::lower_bound(P.removed.begin(), P.removed.end(), (uint32_t)J.old_lo[r]) - P.removed.begin();
    const size_t m1 = std::lower_bound(P.removed.begin(), P.removed.end(), (uint32_t)J.old_lo[r + 1]) - P.removed.begin();
    if (T.blocking && m1 > m0 && (rc = blocking_emit(ctx, st, (const uint32_t *)(M.stage + M.s_removed) + m0, (int)(m1 - m0), nullptr, 0)))
        return rc;
    if (M.flocks) {
        // from the context's own pageable copy, which is staged before the call returns: the caller's array may be pinned
        ctx->h_flocks.assign(M.flocks, M.flocks + M.nflocks);
        if (M.nflocks) PF_CUDA(cudaMemcpyAsync(ctx->d_flocks, ctx->h_flocks.data(), M.nflocks * sizeof(pfnav_flock), cudaMemcpyHostToDevice, st));
    }
    if (J.keep_lo[r + 1] > J.keep_lo[r]) {
        pf_pop_gather g = pop_gather_args(ctx, M, J.keep_lo[r], J.keep_lo[r + 1], J.keep_lo[r]);
        g.o_agents = M.own.agents; g.o_rec = M.own.rec; g.o_flock = M.own.flock; g.o_ms = M.own.ms; g.o_ext = M.own.ext;
        g.o_form = M.own.form; g.o_blk = M.own.blk;
        pop_launch(ctx, g, st);
    }
    if (n_new) {
        k_pop_columns<<<((int)n_new + 127) / 128, 128, 0, st>>>(ctx->d_records, ctx->d_flock_of, (const uint32_t *)(M.stage + M.s_key),
                                                                (uint32_t)R, (int)P.n_keep, (int)n_new,
                                                                (const pfnav_agent *)(M.stage + M.s_agents), M.c_rec, M.c_flock);
        ctx->launches++;
    }
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}

int pf_pop_job_write(pfnav_ctx *ctx, pf_pop_member &M, cudaStream_t st)
{
    ctx->index_stale = true;            // new records until the gather rebuilds the index
    const pf_pop_job &J = M.J;
    const pf_pop_tables &T = M.T;
    const int r = J.rank, world = J.world;
    const size_t n_new = J.P.n_new, lo = J.new_lo[r], hi = J.new_lo[r + 1];
    // the mirror: the received rows' flock ids, radii and flag bits from the member's own compacted columns
    size_t nrecv = 0;
    for (int s = 0; s < world; s++)
        if (s != r) nrecv += J.seg_hi(s, r) - J.seg_lo(s, r);
    std::vector<int32_t> fl(nrecv);
    std::vector<pf_record> rec(nrecv);
    for (int s = 0, k = 0; s < world; s++) {
        const size_t a = J.seg_lo(s, r), n = J.seg_hi(s, r) - a;
        if (s == r || !n) continue;
        PF_CUDA(cudaMemcpyAsync(fl.data() + k, M.c_flock + a, n * 4, cudaMemcpyDeviceToHost, st));
        PF_CUDA(cudaMemcpyAsync(rec.data() + k, M.c_rec + a, n * sizeof(pf_record), cudaMemcpyDeviceToHost, st));
        k += (int)n;
    }
    if (nrecv) PF_CUDA(cudaStreamSynchronize(st));
    std::vector<float> rad(nrecv);
    std::vector<uint32_t> sf(nrecv);
    for (size_t k = 0; k < nrecv; k++) { rad[k] = rec[k].radius; sf[k] = rec[k].state_flags; }
    pf_pop_job_mirror(ctx->cmd_mirror, J, fl.data(), rad.data(), sf.data(), M.mirror);
    // the tables at their new length (a regrowth waits for the device and drops the contents: everything is in the scratch)
    int rc;
    if ((rc = pf_dbuf_reserve_all(n_new, ctx->d_agents, ctx->d_records, ctx->d_flock_members, ctx->d_flock_of, ctx->d_sorted_ix,
                                  ctx->d_sorted_iy, ctx->d_sorted_flock, ctx->d_sorted_id))) return rc;
    if (T.ms && (rc = ctx->d_movestate.reserve(n_new))) return rc;
    if (T.ext && (rc = ctx->d_ms_ext.reserve(n_new))) return rc;
    if (T.formation && (rc = ctx->d_formation.reserve(n_new))) return rc;
    if (T.blocking && (rc = ctx->d_blocking.reserve(std::max<size_t>(n_new, 1)))) { ctx->blocking_n = 0; return rc; }
    if (n_new) {
        PF_CUDA(cudaMemcpyAsync(ctx->d_records, M.c_rec, n_new * sizeof(pf_record), cudaMemcpyDeviceToDevice, st));
        PF_CUDA(cudaMemcpyAsync(ctx->d_flock_of, M.c_flock, n_new * 4, cudaMemcpyDeviceToDevice, st));
    }
    // the new own range: the senders' segments (the member's own survivors that stay among them), then the appended rows
    for (int s = 0; s < world; s++) {
        const size_t a = J.seg_lo(s, r), n = J.seg_hi(s, r) - a;
        if (n && (rc = pop_copy_rows(ctx, M.from[s], T, a, n, st))) return rc;
    }
    if (J.app_hi(r) > J.app_lo(r)) {
        pf_pop_gather g = pop_gather_args(ctx, M, J.app_lo(r), J.app_hi(r), 0);
        g.o_agents = ctx->d_agents; g.o_rec = ctx->d_records; g.o_flock = ctx->d_flock_of;
        g.o_ms = T.ms ? ctx->d_movestate.p : nullptr; g.o_ext = ctx->d_ms_ext; g.o_form = ctx->d_formation;
        g.o_blk = T.blocking ? ctx->d_blocking.p : nullptr;
        pop_launch(ctx, g, st);
    }
    if (T.blocking && hi > lo) {
        uint32_t *word = (uint32_t *)(M.stage + M.s_fac) + 1;
        PF_CUDA(cudaMemsetAsync(word, 0, 4, st));
        k_pop_any_fac<<<(int)(hi - lo + 255) / 256, 256, 0, st>>>(ctx->d_blocking, (int)lo, (int)hi, word);
        ctx->launches++;
    }
    PF_CUDA(cudaGetLastError());
    return PFNAV_OK;
}

// host facts as pfnav_agents_upload_shard of the new range would leave them, then the member lists and population facts
// from the member's complete columns
int pf_pop_job_commit(pfnav_ctx *ctx, pf_pop_member &M, cudaStream_t st)
{
    const pf_pop_job &J = M.J;
    const size_t n_new = J.P.n_new, lo = J.new_lo[J.rank], hi = J.new_lo[J.rank + 1];
    if (M.T.blocking) {
        uint32_t fac = 0;
        if (hi > lo) {
            PF_CUDA(cudaMemcpyAsync(&fac, (uint32_t *)(M.stage + M.s_fac) + 1, 4, cudaMemcpyDeviceToHost, st));
            PF_CUDA(cudaStreamSynchronize(st));
        }
        ctx->blocking_n = n_new;
        ctx->blocking_any_fac = fac != 0;
    }
    ctx->n_agents = n_new; ctx->shard_lo = lo; ctx->shard_hi = hi; ctx->n_flocks = M.nflocks;
    ctx->cmd_mirror = std::move(M.mirror);
    std::vector<uint8_t> used;
    ctx->cmd_mirror.used(used);
    if (M.flocks || used != ctx->flock_layer_used) ctx->arrival_valid = false;
    ctx->flock_layer_used.swap(used);
    ctx->n_work = 0;
    int per, W, rc;
    member_sort_shape(n_new, M.nflocks, per, W);
    if ((rc = members_on_device(ctx, st, (uint32_t *)ctx->d_cmd_buf.p, per, W))) return rc;
    return pfnav_agents_refresh_facts(ctx, st);
}

// A job member: the whole batch is checked against the population, the own records against the member's mirror. Its
// flock column must be complete -- a full pfnav_agents_upload_shard leaves the other ranges' entries to the next
// gather -- because the member lists are rebuilt from it.
int pf_cmd_job_check(pfnav_ctx *ctx, const pfnav_agent_delta *deltas, size_t n, const pfnav_flock *flocks, size_t nflocks,
                     pf_cmd_job &J)
{
    PF_ARG(ctx->d_agents, "agents not uploaded");
    if (ctx->members_stale) {
        pfnav_set_error("the member's flock column is incomplete until the gather that follows pfnav_agents_upload_shard");
        return PFNAV_ERR_STATE;
    }
    PF_ARG(deltas || n == 0, "deltas == NULL");
    PF_ARG(n < (1u << 31) && nflocks < (1u << 31), "n / nflocks");
    J.flocks = flocks;
    J.nflocks = flocks ? nflocks : ctx->n_flocks;
    const pf_cmd_limits lim = {0, ctx->n_agents, ctx->n_agents, J.nflocks, ctx->movestate_set && ctx->d_movestate != nullptr,
                               ctx->d_ms_ext != nullptr};
    const char *err = pf_cmd_job_plan(deltas, n, lim, ctx->shard_lo, ctx->shard_hi, ctx->cmd_mirror, ctx->nlayers, J.own,
                                      J.foreign, J.changes);
    PF_ARG(!err, err);
    return PFNAV_OK;
}

int pf_cmd_job_apply(pfnav_ctx *ctx, const pf_cmd_job &J, cudaStream_t st)
{
    if (J.own.empty() && J.foreign.empty() && !J.flocks) return PFNAV_OK;
    return cmd_apply(ctx, st, J.own, J.foreign, J.changes, J.flocks, J.nflocks);
}

extern "C" int pfnav_agents_set_work_dev(pfnav_ctx *ctx, void *stream, size_t *out_nwork)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->d_agents, "agents not uploaded");
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    const int lo = (int)ctx->shard_lo, hi = (int)ctx->shard_hi, cnt = hi - lo;
    int rc;
    uint32_t nwork = 0;
    const pf_compact_grid g = pf_compact_grid_of(cnt);
    // d_cmd_buf: the block offsets, the count, then one ballot word per 32 uids
    if (cnt) {
        if ((rc = ctx->d_cmd_buf.reserve(((size_t)g.nb + 1 + ((size_t)cnt + 31) / 32) * 4))) return rc;
        uint32_t *part = (uint32_t *)ctx->d_cmd_buf.p;
        k_compact_count<<<g.nb, PF_COMPACT_THREADS, 0, st>>>(work_compact{ctx->d_records, nullptr}, lo, hi, g.per,
                                                             part + g.nb + 1, part);
        k_compact_offsets<work_compact><<<1, PF_COMPACT_THREADS, 0, st>>>(part, g.nb, part + g.nb);
        ctx->launches += 2;
        PF_CUDA(cudaGetLastError());
        PF_CUDA(cudaMemcpyAsync(&nwork, part + g.nb, 4, cudaMemcpyDeviceToHost, st));
        PF_CUDA(cudaStreamSynchronize(st));
    }
    if ((rc = pf_work_reserve(ctx, nwork))) return rc;
    if (nwork) {
        const uint32_t *part = (const uint32_t *)ctx->d_cmd_buf.p;
        k_compact_write<<<g.nb, PF_COMPACT_THREADS, 0, st>>>(work_compact{ctx->d_records, ctx->d_work}, lo, hi, g.per,
                                                             part + g.nb + 1, part);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
    }
    ctx->n_work = nwork;
    if (out_nwork) *out_nwork = nwork;
    return PFNAV_OK;
}

extern "C" int pfnav_agents_read_work(pfnav_ctx *ctx, uint32_t *out, size_t maxout, size_t *out_n)
{
    PF_ARG(ctx && ctx->d_agents, "agents not uploaded");
    PF_ARG(out || maxout == 0, "out == NULL");
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(cudaDeviceSynchronize());
    const size_t n = std::min(maxout, ctx->n_work);
    if (n) PF_CUDA(cudaMemcpy(out, ctx->d_work, n * 4, cudaMemcpyDeviceToHost));
    if (out_n) *out_n = ctx->n_work;
    return PFNAV_OK;
}
