// pfnav_plan.cu -- host-side navigation structure: local islands, portals, and a goal planner
// that emits the flow/LOS field requests the device kernels consume.
//
// Restates (reference file:line):
//   n_update_local_islands / n_visit_island_local     src/navigation/nav.c:967-984, 903-950
//   n_create_portals / n_link_chunks                  src/navigation/nav.c:563-591, 477-561
// and provides a breadth-first goal planner over (chunk, local island) nodes that yields, for
// EVERY chunk connected to the goal, the same kind of TARGET_TILE / TARGET_PORTAL requests
// n_request_path (nav.c:1774-2047) issues along one portal path. It minimises hop count, not the
// reference's portal travel cost, so which portal a chunk steers to may differ from
// AStar_PortalGraphPath's choice (a_star.c:429); each emitted field is still the reference's
// field for that request. The cost-faithful search is listed under "next" in DESIGN.md.
#include "pfnav_internal.cuh"
#include <algorithm>
#include <atomic>
#include <condition_variable>
#include <functional>
#include <mutex>
#include <string.h>
#include <thread>

static inline size_t chunk_off(const pfnav_ctx *ctx, int layer, int cr, int cc)
{
    return ((size_t)layer * ctx->chunk_w * ctx->chunk_h + (size_t)cr * ctx->chunk_w + cc) * 4096;
}

// n_update_local_islands (nav.c:967): ids from 1 in row-major discovery order, 4-connected flood
// inside the chunk over tiles that are passable and not blocked; 0xFFFF elsewhere.
static void local_islands_chunk(const uint8_t *cost, const uint16_t *blk, uint16_t *out)
{
    for (int i = 0; i < 4096; i++) out[i] = 0xFFFF;
    uint16_t next = 0;
    std::vector<int> q;
    q.reserve(4096);
    for (int t = 0; t < 4096; t++) {
        if (out[t] != 0xFFFF || cost[t] == 0xFF || blk[t] > 0) continue;
        const uint16_t id = ++next;
        q.clear();
        q.push_back(t);
        out[t] = id;
        for (size_t h = 0; h < q.size(); h++) {
            const int cur = q[h], r = cur >> 6, c = cur & 63;
            const int nb[4] = {c > 0 ? cur - 1 : -1, c < 63 ? cur + 1 : -1, r > 0 ? cur - 64 : -1, r < 63 ? cur + 64 : -1};
            for (int e = 0; e < 4; e++) {
                const int n = nb[e];
                if (n < 0 || out[n] != 0xFFFF || cost[n] == 0xFF || blk[n] > 0) continue;
                out[n] = id;
                q.push_back(n);
            }
        }
    }
}

// n_link_chunks (nav.c:477): a portal is a maximal run of border tiles passable on both sides
// (cost only, blockers ignored); a run that would start on the last tile of the line is never
// closed and therefore dropped, exactly as the reference's loop does.
static void link_chunks(pfnav_ctx *ctx, int layer, int ar, int ac, int br, int bc, bool vertical_pair)
{
    // vertical_pair: a is above b (a's bottom row vs b's top row); else a is left of b
    auto &pa = ctx->portals[layer][ar * ctx->chunk_w + ac];
    auto &pb = ctx->portals[layer][br * ctx->chunk_w + bc];
    const uint8_t *ca = ctx->h_cost.data() + chunk_off(ctx, layer, ar, ac);
    const uint8_t *cb = ctx->h_cost.data() + chunk_off(ctx, layer, br, bc);
    bool in_portal = false;
    int start = 0;
    for (int i = 0; i < 64; i++) {
        const uint8_t va = vertical_pair ? ca[63 * 64 + i] : ca[i * 64 + 63];
        const uint8_t vb = vertical_pair ? cb[i] : cb[i * 64];
        const bool can_cross = va != 0xFF && vb != 0xFF;
        if (can_cross && !in_portal) {
            in_portal = true;
            start = i;
        } else if (in_portal && (!can_cross || i == 63)) {
            const int end = !can_cross ? i - 1 : i;
            in_portal = false;
            pfnav_ctx::portal_t A, B;
            A.chunk_r = (int16_t)ar; A.chunk_c = (int16_t)ac; B.chunk_r = (int16_t)br; B.chunk_c = (int16_t)bc;
            if (vertical_pair) {
                A.r0 = 63; A.c0 = (int16_t)start; A.r1 = 63; A.c1 = (int16_t)end;
                B.r0 = 0;  B.c0 = (int16_t)start; B.r1 = 0;  B.c1 = (int16_t)end;
            } else {
                A.r0 = (int16_t)start; A.c0 = 63; A.r1 = (int16_t)end; A.c1 = 63;
                B.r0 = (int16_t)start; B.c0 = 0;  B.r1 = (int16_t)end; B.c1 = 0;
            }
            A.conn_chunk = br * ctx->chunk_w + bc; A.conn_idx = (int32_t)pb.size();
            B.conn_chunk = ar * ctx->chunk_w + ac; B.conn_idx = (int32_t)pa.size();
            pa.push_back(A);
            pb.push_back(B);
        }
    }
}

// N_NewCtxForMapData's structural part for one layer (nav.c:2284): local islands (uploaded to the
// device for TARGET_PORTAL seeding) and the portal table. Call after pfnav_map_upload_layer.
extern "C" int pfnav_map_build_nav(pfnav_ctx *ctx, int layer)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    const size_t ltiles = (size_t)chunks * 4096;
    for (int ch = 0; ch < chunks; ch++)
        local_islands_chunk(ctx->h_cost.data() + ltiles * layer + (size_t)ch * 4096,
                            ctx->h_blk.data() + ltiles * layer + (size_t)ch * 4096,
                            ctx->h_liid.data() + ltiles * layer + (size_t)ch * 4096);
    // n_create_portals (nav.c:563): chunks row-major, bottom link before right link
    ctx->portals[layer].assign(chunks, {});
    for (int r = 0; r < ctx->chunk_h; r++)
        for (int c = 0; c < ctx->chunk_w; c++) {
            if (r < ctx->chunk_h - 1) link_chunks(ctx, layer, r, c, r + 1, c, true);
            if (c < ctx->chunk_w - 1) link_chunks(ctx, layer, r, c, r, c + 1, false);
        }
    for (int ch = 0; ch < chunks; ch++)
        if (ctx->portals[layer][ch].size() > 64) {
            pfnav_set_error("pfnav_map_build_nav: chunk %d has %zu portals (MAX_PORTALS_PER_CHUNK is 64, nav_data.h:44)",
                            ch, ctx->portals[layer][ch].size());
            return PFNAV_ERR_STATE;
        }
    // push the islands to the device image (host-only contexts just keep the mirrors)
    return pfnav_map_upload_layer(ctx, layer, ctx->h_cost.data() + ltiles * layer, ctx->h_blk.data() + ltiles * layer,
                                  ctx->h_liid.data() + ltiles * layer);
}

// Recompute the local islands of one chunk after its blockers changed (n_update_dirty_local_islands,
// nav.c:986) and push the chunk to the device.
extern "C" int pfnav_map_refresh_chunk(pfnav_ctx *ctx, int layer, int chunk_r, int chunk_c)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG(chunk_r >= 0 && chunk_r < ctx->chunk_h && chunk_c >= 0 && chunk_c < ctx->chunk_w, "chunk coords");
    const size_t off = chunk_off(ctx, layer, chunk_r, chunk_c);
    local_islands_chunk(ctx->h_cost.data() + off, ctx->h_blk.data() + off, ctx->h_liid.data() + off);
    return pfnav_map_update_chunk(ctx, layer, chunk_r, chunk_c, nullptr, ctx->h_blk.data() + off, ctx->h_liid.data() + off);
}

extern "C" int pfnav_local_islands_get(pfnav_ctx *ctx, int layer, uint16_t *out)
{
    PF_ARG(ctx && out && layer >= 0 && layer < ctx->nlayers, "args");
    const size_t ltiles = (size_t)ctx->chunk_w * ctx->chunk_h * 4096;
    memcpy(out, ctx->h_liid.data() + ltiles * layer, ltiles * 2);
    return PFNAV_OK;
}

// Portal table in the same 10-int row format as the oracle harness (chunk_r, chunk_c, idx, ep0.r,
// ep0.c, ep1.r, ep1.c, conn_chunk_idx, conn_portal_idx, 0). Returns the count via *out_n.
extern "C" int pfnav_portals_get(pfnav_ctx *ctx, int layer, int32_t *out, int maxout, int *out_n)
{
    PF_ARG(ctx && out_n && layer >= 0 && layer < ctx->nlayers, "args");
    PF_ARG((size_t)layer < ctx->portals.size() && !ctx->portals[layer].empty(), "pfnav_map_build_nav not called for this layer");
    int n = 0;
    for (size_t ch = 0; ch < ctx->portals[layer].size(); ch++)
        for (size_t p = 0; p < ctx->portals[layer][ch].size(); p++) {
            const auto &P = ctx->portals[layer][ch][p];
            if (out && n < maxout) {
                int32_t *o = out + (size_t)n * 10;
                o[0] = P.chunk_r; o[1] = P.chunk_c; o[2] = (int32_t)p; o[3] = P.r0; o[4] = P.c0; o[5] = P.r1; o[6] = P.c1;
                o[7] = P.conn_chunk; o[8] = P.conn_idx; o[9] = 0;
            }
            n++;
        }
    *out_n = n;
    return PFNAV_OK;
}

// Goal planner: breadth-first over (chunk, local island) nodes from the goal tile. For every node
// emits one flow request (TARGET_TILE for the goal's own node, TARGET_PORTAL towards the parent
// node otherwise; a chunk's first node has init=1, later nodes of the same chunk merge in place
// like nav.c:1998-2008) and, for a chunk's first node, one LOS request chained to its parent chunk.
// `field_slot[i]` / `los_slot[i]` give the chunk index each request's output belongs to, and
// `flow_wave[i]` the launch wave (requests that update the same chunk are serialised by wave).
extern "C" int pfnav_plan_goal(pfnav_ctx *ctx, int layer, int tgt_chunk_r, int tgt_chunk_c, int tgt_tile_r,
                               int tgt_tile_c, pfnav_field_req *flow_out, int32_t *flow_chunk, int32_t *flow_wave,
                               int max_flow, int *n_flow, pfnav_los_req *los_out, int32_t *los_chunk, int max_los,
                               int *n_los)
{
    PF_ARG(ctx && ctx->d_cost && n_flow && n_los, "args");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG((size_t)layer < ctx->portals.size() && !ctx->portals[layer].empty(), "pfnav_map_build_nav not called for this layer");
    PF_ARG(tgt_chunk_r >= 0 && tgt_chunk_r < ctx->chunk_h && tgt_chunk_c >= 0 && tgt_chunk_c < ctx->chunk_w &&
           tgt_tile_r >= 0 && tgt_tile_r < 64 && tgt_tile_c >= 0 && tgt_tile_c < 64, "target tile");
    const int cw = ctx->chunk_w, chunks = cw * ctx->chunk_h;
    const size_t ltiles = (size_t)chunks * 4096;
    const uint16_t *liid = ctx->h_liid.data() + ltiles * layer;
    *n_flow = 0; *n_los = 0;
    // scratch reused across calls (planner threads are persistent): the BFS queue, and the (chunk, island) nodes
    // already planned as an open-addressing set whose entries carry the call's generation (no clearing per call)
    struct node { int chunk; uint16_t li; };
    struct scratch { std::vector<node> q; std::vector<uint64_t> seen; uint32_t gen = 0; std::vector<int> los_index, nodes_in_chunk; std::vector<uint16_t> first_li; };
    static thread_local scratch tls;
    scratch &S = tls;                       // one TLS lookup, not one per use in the loops below
    size_t tab = 64;
    while (tab < 2 * ((size_t)std::max(max_flow, 0) + 2)) tab *= 2;        // every insert emits a flow request: load <= 1/2
    if (S.seen.size() < tab) { S.seen.assign(tab, 0); S.gen = 0; }
    tab = S.seen.size();
    int shift = 64;
    for (size_t t = tab; t > 1; t >>= 1) shift--;                          // Fibonacci hashing: the top log2(tab) bits
    if (++S.gen == 0) { std::fill(S.seen.begin(), S.seen.end(), 0); S.gen = 1; }
    const uint64_t gen = (uint64_t)S.gen << 32;
    auto first_visit = [&](int chunk, uint16_t li) -> bool {      // insert (chunk, island); false if it was there
        if (S.first_li[chunk] == li) return false;                 // most chunks are reached through one island
        if (S.first_li[chunk] == 0xFFFF) S.first_li[chunk] = li;
        const uint64_t key = gen | ((uint64_t)chunk << 16) | li;
        for (size_t h = (size_t)(((uint64_t)chunk << 16 | li) * 0x9E3779B97F4A7C15ull >> shift);; h = (h + 1) & (tab - 1)) {
            if (S.seen[h] == key) return false;
            if ((S.seen[h] >> 32) != (gen >> 32)) { S.seen[h] = key; return true; }
        }
    };
    S.q.clear();
    S.los_index.assign(chunks, -1); S.nodes_in_chunk.assign(chunks, 0); S.first_li.assign(chunks, 0xFFFF);
    std::vector<int> &los_index = S.los_index, &nodes_in_chunk = S.nodes_in_chunk;
    const int tchunk = tgt_chunk_r * cw + tgt_chunk_c;
    const uint16_t tli = liid[(size_t)tchunk * 4096 + tgt_tile_r * 64 + tgt_tile_c];
    auto emit_flow = [&](const pfnav_field_req &rq, int chunk) -> bool {
        if (*n_flow >= max_flow) return false;
        flow_out[*n_flow] = rq;
        flow_out[*n_flow].init = nodes_in_chunk[chunk] == 0;
        flow_chunk[*n_flow] = chunk;
        flow_wave[*n_flow] = nodes_in_chunk[chunk];
        nodes_in_chunk[chunk]++;
        (*n_flow)++;
        return true;
    };
    pfnav_field_req base;
    memset(&base, 0, sizeof(base));
    base.layer = layer; base.faction_id = PFNAV_FACTION_ID_NONE;
    {   // the goal's own chunk: TARGET_TILE field + destination LOS (nav.c:1819-1847)
        pfnav_field_req rq = base;
        rq.chunk_r = tgt_chunk_r; rq.chunk_c = tgt_chunk_c; rq.target_type = PFNAV_TARGET_TILE;
        rq.tile_r = tgt_tile_r; rq.tile_c = tgt_tile_c;
        if (!emit_flow(rq, tchunk)) { pfnav_set_error("pfnav_plan_goal: flow output too small"); return PFNAV_ERR_NOMEM; }
        if (*n_los >= max_los) { pfnav_set_error("pfnav_plan_goal: los output too small"); return PFNAV_ERR_NOMEM; }
        pfnav_los_req lq;
        memset(&lq, 0, sizeof(lq));
        lq.chunk_r = tgt_chunk_r; lq.chunk_c = tgt_chunk_c; lq.layer = layer; lq.faction_id = PFNAV_FACTION_ID_NONE;
        lq.tgt_chunk_r = tgt_chunk_r; lq.tgt_chunk_c = tgt_chunk_c; lq.tgt_tile_r = tgt_tile_r; lq.tgt_tile_c = tgt_tile_c;
        lq.prev_index = -1;
        los_index[tchunk] = *n_los;
        los_out[*n_los] = lq; los_chunk[*n_los] = tchunk; (*n_los)++;
    }
    if (tli == 0xFFFF) return PFNAV_OK;      // goal tile impassable/blocked: nothing can flow to it
    first_visit(tchunk, tli);
    S.q.push_back({tchunk, tli});
    for (size_t head = 0; head < S.q.size(); head++) {
        const node cur = S.q[head];
        const auto &ports = ctx->portals[layer][cur.chunk];
        for (size_t pi = 0; pi < ports.size(); pi++) {
            const auto &P = ports[pi];                                // portal of the current (parent) chunk
            const auto &Q = ctx->portals[layer][P.conn_chunk][P.conn_idx];   // facing portal in the neighbour chunk
            const int nchunk = P.conn_chunk;
            // every island M of the neighbour that touches island cur.li across this portal
            const int len = (P.r1 - P.r0) + (P.c1 - P.c0) + 1;
            uint16_t lastM = 0xFFFF;                                  // a repeat along the portal was just visited
            for (int k = 0; k < len; k++) {
                const int pr = P.r0 + (P.r1 > P.r0 ? k : 0), pc = P.c0 + (P.c1 > P.c0 ? k : 0);
                const int qr = Q.r0 + (Q.r1 > Q.r0 ? k : 0), qc = Q.c0 + (Q.c1 > Q.c0 ? k : 0);
                if (liid[(size_t)cur.chunk * 4096 + pr * 64 + pc] != cur.li) continue;
                const uint16_t M = liid[(size_t)nchunk * 4096 + qr * 64 + qc];
                if (M == 0xFFFF || M == lastM) continue;
                lastM = M;
                if (!first_visit(nchunk, M)) continue;
                pfnav_field_req rq = base;
                rq.chunk_r = Q.chunk_r; rq.chunk_c = Q.chunk_c; rq.target_type = PFNAV_TARGET_PORTAL;
                rq.port_r0 = Q.r0; rq.port_c0 = Q.c0; rq.port_r1 = Q.r1; rq.port_c1 = Q.c1;
                rq.next_r0 = P.r0; rq.next_c0 = P.c0; rq.next_r1 = P.r1; rq.next_c1 = P.c1;
                rq.next_chunk_r = P.chunk_r; rq.next_chunk_c = P.chunk_c;
                rq.port_iid = M; rq.next_iid = cur.li;
                const bool first = nodes_in_chunk[nchunk] == 0;
                if (!emit_flow(rq, nchunk)) { pfnav_set_error("pfnav_plan_goal: flow output too small"); return PFNAV_ERR_NOMEM; }
                if (first) {
                    if (*n_los >= max_los) { pfnav_set_error("pfnav_plan_goal: los output too small"); return PFNAV_ERR_NOMEM; }
                    pfnav_los_req lq;
                    memset(&lq, 0, sizeof(lq));
                    lq.chunk_r = Q.chunk_r; lq.chunk_c = Q.chunk_c; lq.layer = layer; lq.faction_id = PFNAV_FACTION_ID_NONE;
                    lq.tgt_chunk_r = tgt_chunk_r; lq.tgt_chunk_c = tgt_chunk_c; lq.tgt_tile_r = tgt_tile_r; lq.tgt_tile_c = tgt_tile_c;
                    lq.prev_index = los_index[cur.chunk];
                    lq.prev_chunk_r = P.chunk_r; lq.prev_chunk_c = P.chunk_c;
                    los_index[nchunk] = *n_los;
                    los_out[*n_los] = lq; los_chunk[*n_los] = nchunk; (*n_los)++;
                }
                S.q.push_back({nchunk, M});
            }
        }
    }
    return PFNAV_OK;
}

// The flow waves and the LOS dependency chains of a goal batch each get a context-owned stream (the flow kernels
// need ~100 KB of shared memory per CTA and would otherwise queue the caller's stream behind the persistent LOS
// CTAs that hold most of it).
// The LOS dependency chains of a goal batch are latency-bound (one thread per field replays the
// reference's heap) and read nothing the flow kernels write: they run on ctx->field_stream, forked
// after everything already queued on the caller's stream and joined (pf_fields_join) by whichever
// entry point next reads or writes LOS fields of the pool. The flow kernels, the position-index
// rebuild and the cohesion pass overlap them.
static int los_fork(pfnav_ctx *ctx, cudaStream_t st)
{
    // duration of the previous batch (fork -> done), if it has finished: input of the two-phase policy
    if (ctx->los_inflight && cudaEventQuery(ctx->ev_los) == cudaSuccess) {
        float ms = 0.0f;
        if (cudaEventElapsedTime(&ms, ctx->ev_fork, ctx->ev_los) == cudaSuccess) ctx->last_los_ms = ms;
    }
    cudaGetLastError();
    PF_CUDA(cudaEventRecord(ctx->ev_fork, st));
    PF_CUDA(cudaStreamWaitEvent(ctx->field_stream, ctx->ev_fork, 0));
    PF_CUDA(cudaStreamWaitEvent(ctx->flow_stream, ctx->ev_fork, 0));
    return 0;
}
static int los_forked(pfnav_ctx *ctx)
{
    PF_CUDA(cudaEventRecord(ctx->ev_flow, ctx->flow_stream));
    PF_CUDA(cudaEventRecord(ctx->ev_los, ctx->field_stream));
    ctx->los_inflight = true;
    return 0;
}

// ------------------------------------------------------------------------------------------
// Request staging (pfnav_internal.cuh: pf_stage_*). Every batch built on the host reaches its kernels the same way: it is
// written into the next of two pinned buffers, a ring whose buffer is reused once the copy that last read it is done,
// and copied on the batch's stream into one device buffer per context. The buffers only grow, by doubling.
// ------------------------------------------------------------------------------------------
struct pf_stager {
    uint8_t *host[2] = {nullptr, nullptr}; size_t host_bytes[2] = {0, 0}; cudaEvent_t host_ev[2] = {nullptr, nullptr};
    int next = 0;
    uint8_t *dev = nullptr; size_t dev_bytes = 0;
    cudaEvent_t read_ev = nullptr;            // pf_stage_done: after the last stream-ordered reader of `dev`
};

static pf_stager &stager_of(pfnav_ctx *ctx)
{
    if (!ctx->stager) ctx->stager = new pf_stager;
    return *(pf_stager *)ctx->stager;
}

int pf_stage_begin(pfnav_ctx *ctx, cudaStream_t st, size_t host_bytes, size_t dev_bytes, bool table, pf_stage *S)
{
    pf_stager &G = stager_of(ctx);
    const int ri = G.next;
    G.next ^= 1;
    const size_t hb = host_bytes + (table ? ctx->pool.table_bytes() : 0);
    if (!G.host_ev[ri]) PF_CUDA(cudaEventCreateWithFlags(&G.host_ev[ri], cudaEventDisableTiming));
    else PF_CUDA(cudaEventSynchronize(G.host_ev[ri]));
    if (G.host_bytes[ri] < hb) {
        cudaFreeHost(G.host[ri]);
        G.host[ri] = nullptr; G.host_bytes[ri] = 0;
        PF_CUDA(cudaMallocHost(&G.host[ri], hb * 2));
        G.host_bytes[ri] = hb * 2;
    }
    if (!G.read_ev) PF_CUDA(cudaEventCreateWithFlags(&G.read_ev, cudaEventDisableTiming));
    ctx->goal_batch.valid = false;            // the resident goal plan lives in `dev`
    if (dev_bytes) {
        PF_CUDA(pf_fields_join(ctx, st));
        PF_CUDA(cudaStreamWaitEvent(st, G.read_ev, 0));
        if (G.dev_bytes < dev_bytes) {
            PF_CUDA(pf_fields_sync(ctx));
            PF_CUDA(cudaEventSynchronize(G.read_ev));
            cudaFree(G.dev);
            G.dev = nullptr; G.dev_bytes = 0;
            PF_CUDA(cudaMalloc(&G.dev, dev_bytes * 2));
            G.dev_bytes = dev_bytes * 2;
        }
    }
    S->host = G.host[ri]; S->dev = G.dev; S->ri = ri;
    S->table = table ? S->host + host_bytes : nullptr;
    return PFNAV_OK;
}

int pf_stage_upload(pfnav_ctx *ctx, cudaStream_t st, const pf_stage &S, size_t bytes)
{
    if (bytes) PF_CUDA(cudaMemcpyAsync(S.dev, S.host, bytes, cudaMemcpyHostToDevice, st));
    if (S.table)
        if (int rc = pf_pool_stage_table(ctx, S.table, st)) return rc;
    PF_CUDA(cudaEventRecord(stager_of(ctx).host_ev[S.ri], st));
    return PFNAV_OK;
}

int pf_stage_done(pfnav_ctx *ctx, cudaStream_t st)
{
    PF_CUDA(cudaEventRecord(stager_of(ctx).read_ev, st));
    return PFNAV_OK;
}

void pf_stage_free(pfnav_ctx *ctx)
{
    pf_stager *G = (pf_stager *)ctx->stager;
    if (!G) return;
    for (int i = 0; i < 2; i++) {
        cudaFreeHost(G->host[i]);
        if (G->host_ev[i]) cudaEventDestroy(G->host_ev[i]);
    }
    cudaFree(G->dev);
    if (G->read_ev) cudaEventDestroy(G->read_ev);
    delete G;
    ctx->stager = nullptr;
}

int pf_waves_launch(pfnav_ctx *ctx, const uint8_t *dev, const pf_waves &W, uint8_t *flow_fields, uint8_t *los_fields,
                    cudaStream_t flow_st, cudaStream_t los_st)
{
    for (size_t w = 0; w + 1 < W.fwave_off.size(); w++) {
        const int first = W.fwave_off[w], cnt = W.fwave_off[w + 1] - first;
        if (cnt <= 0) continue;
        int rc = pfnav_flow_launch(ctx, (const pfnav_field_req *)dev + first, cnt, flow_fields,
                                   (const int32_t *)(dev + W.o_fs) + first, flow_st);
        if (rc) return rc;
    }
    return pfnav_los_launch(ctx, (const pfnav_los_req *)(dev + W.o_lr), W.nl, los_fields, (const int32_t *)(dev + W.o_ls),
                            los_st);
}

// Host side of a cold goal batch, owned by the context: persistent planner threads (created on the first batch,
// joined by pfnav_destroy) and per-goal / merge scratch that keeps its capacity across batches, so that a batch
// neither spawns threads nor allocates.
struct pf_planner {
    struct goal_plan { std::vector<pfnav_field_req> fr; std::vector<pfnav_los_req> lr; std::vector<int32_t> fc, fw, lc; int nf = 0, nl = 0, rc = 0; std::string err; };
    // the batch's requests (their destinations are the slots reserve_batch reserves) and keys: flow keys, then LOS keys
    struct merged {
        pf_wave_pack W; std::vector<size_t> keys, lkeys; std::vector<int32_t> slots;
        void clear() { W.clear(); keys.clear(); lkeys.clear(); }
    };
    std::vector<goal_plan> plans;
    merged batch;

    explicit pf_planner(int nworkers)
    {
        for (int i = 0; i < nworkers; i++) threads.emplace_back([this] { worker(); });
    }
    ~pf_planner()
    {
        { std::lock_guard<std::mutex> l(m); quit = true; }
        wake.notify_all();
        for (auto &t : threads) t.join();
    }
    // job(0) .. job(n - 1) on the workers and the calling thread; returns when all have finished
    void run(int n, std::function<void(int)> f)
    {
        if (n <= 1 || threads.empty()) { for (int g = 0; g < n; g++) f(g); return; }
        {
            std::lock_guard<std::mutex> l(m);
            job = std::move(f); njobs = n; next = 0; busy = (int)threads.size(); gen++;
        }
        wake.notify_all();
        drain();
        std::unique_lock<std::mutex> l(m);
        done.wait(l, [&] { return busy == 0; });
    }

private:
    std::vector<std::thread> threads;
    std::mutex m;
    std::condition_variable wake, done;
    std::function<void(int)> job;
    int njobs = 0, busy = 0;
    uint64_t gen = 0;
    bool quit = false;
    std::atomic<int> next{0};

    void drain() { for (int g = next.fetch_add(1); g < njobs; g = next.fetch_add(1)) job(g); }
    void worker()
    {
        uint64_t seen = 0;
        std::unique_lock<std::mutex> l(m);
        for (;;) {
            wake.wait(l, [&] { return quit || gen != seen; });
            if (quit) return;
            seen = gen;
            l.unlock();
            drain();
            l.lock();
            if (--busy == 0) done.notify_one();
        }
    }
};

static pf_planner &planner_of(pfnav_ctx *ctx)
{
    if (!ctx->planner) ctx->planner = new pf_planner(std::max(1, std::min((int)std::thread::hardware_concurrency(), 32)) - 1);
    return *(pf_planner *)ctx->planner;
}

void pf_planner_destroy(pfnav_ctx *ctx)
{
    delete (pf_planner *)ctx->planner;
    ctx->planner = nullptr;
}

// Plan every goal of a batch on the planner threads (independent read-only walks over the host mirrors) and merge what
// the batch writes into the planner's `batch`: every request, or with `missing_only` those whose (dest, chunk) field the
// pool does not hold. Changes nothing but the planner's scratch.
static int plan_batch(pfnav_ctx *ctx, int ngoals, const int32_t *dests, int layer, const int32_t *targets, bool missing_only,
                      pf_host_timer &ht)
{
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    pf_planner &PL = planner_of(ctx);
    const int cap = chunks * 8 + 8;
    if ((int)PL.plans.size() < ngoals) PL.plans.resize(ngoals);
    PL.run(ngoals, [&](int g) {
        pf_planner::goal_plan &P = PL.plans[g];
        if ((int)P.fr.size() < cap) { P.fr.resize(cap); P.lr.resize(cap); P.fc.resize(cap); P.fw.resize(cap); P.lc.resize(cap); }
        P.rc = pfnav_plan_goal(ctx, layer, targets[4 * g], targets[4 * g + 1], targets[4 * g + 2], targets[4 * g + 3],
                               P.fr.data(), P.fc.data(), P.fw.data(), cap, &P.nf, P.lr.data(), P.lc.data(), cap, &P.nl);
        if (P.rc) P.err = pfnav_last_error();          // the error text is thread-local
    });
    ht.lap(PF_HPROF_PLAN);
    pf_planner::merged &B = PL.batch;
    B.clear();
    for (int g = 0; g < ngoals; g++) {
        pf_planner::goal_plan &P = PL.plans[g];
        if (P.rc) { pfnav_set_error("%s", P.err.c_str()); return P.rc; }
        const size_t row = (size_t)dests[g] * chunks;
        const int32_t *fc = P.fc.data(), *lc = P.lc.data();
        // PFNAV_REQUEST_MISSING_ONLY: fields the pool still holds for this destination are kept, like a field-cache hit
        // (fieldcache.c:138-141); a rebuilt LOS field whose parent chunk is kept reads the parent out of its pool slot
        auto held = [&](int chunk, uint8_t bit) { return missing_only && (ctx->pool.has_of(row + chunk) & bit); };
        for (int i = 0; i < P.nf; i++) {
            if (held(fc[i], 1)) continue;
            B.W.flow(P.fr[i], P.fw[i], -1);
            B.keys.push_back(row + fc[i]);
        }
        B.W.los_chain(P.lr.data(), P.nl, [&](int i) { return !held(lc[i], 2); }, [&](int i) { B.lkeys.push_back(row + lc[i]); return -1; },
                      [&](int p) { return ctx->pool.slot_of(row + lc[p]); });
    }
    B.keys.insert(B.keys.end(), B.lkeys.begin(), B.lkeys.end());
    return PFNAV_OK;
}

// slots for everything a merged batch writes, all or nothing, and their `has` bits and flow requests
static int reserve_batch(pfnav_ctx *ctx, pf_planner::merged &B)
{
    pf_wave_pack &W = B.W;
    const int nf = (int)W.fr.size(), nl = (int)W.lr.size();
    B.slots.resize(B.keys.size());
    int rc = pf_pool_reserve(ctx, B.keys.data(), B.keys.size(), B.slots.data(), nullptr);
    if (rc) return rc;
    for (int i = 0; i < nf; i++) { W.fdst[i] = B.slots[i]; ctx->pool.built_flow(W.fdst[i], W.fr[i]); }
    for (int i = 0; i < nl; i++) { W.ldst[i] = B.slots[nf + i]; ctx->pool.built(W.ldst[i], 2); }
    return PFNAV_OK;
}

// n_request_path's field-building half, resident on the device, for a batch of goals: plan every
// goal, then run the flow waves and the LOS dependency waves of ALL goals together straight into the
// field pool (no host round trip of field bytes; one launch per wave, not per goal).
// targets: 4 ints per goal {chunk_r, chunk_c, tile_r, tile_c}. Asynchronous on `stream`.
extern "C" int pfnav_pool_request_goals(pfnav_ctx *ctx, int ngoals, const int32_t *dests, int layer,
                                        const int32_t *targets, void *stream, int *out_n_flow, int *out_n_los)
{
    return pfnav_pool_request_goals_ex(ctx, ngoals, dests, layer, targets, 0, stream, out_n_flow, out_n_los);
}

extern "C" int pfnav_pool_request_goals_ex(pfnav_ctx *ctx, int ngoals, const int32_t *dests, int layer,
                                           const int32_t *targets, uint32_t flags, void *stream, int *out_n_flow, int *out_n_los)
{
    const bool missing_only = (flags & PFNAV_REQUEST_MISSING_ONLY) != 0;
    PF_ARG(ctx && ctx->pool.d_slot, "pool not created");
    PF_NEED_DEVICE(ctx);
    PF_ARG(ngoals >= 0 && (ngoals == 0 || (dests && targets)), "goals");
    if (out_n_flow) *out_n_flow = 0;
    if (out_n_los) *out_n_los = 0;
    if (ngoals == 0) return PFNAV_OK;
    {   // fast path: the same batch on an unchanged map and pool -> the plan is still resident on the device
        auto &gb = ctx->goal_batch;
        if (!missing_only && gb.valid && gb.epoch == ctx->map_epoch && gb.layer == layer && (int)gb.dests.size() == ngoals &&
            memcmp(gb.dests.data(), dests, (size_t)ngoals * 4) == 0 && memcmp(gb.targets.data(), targets, (size_t)ngoals * 16) == 0) {
            PF_CUDA(cudaSetDevice(ctx->device));
            cudaStream_t st = pf_stream(ctx, stream);
            int rc = los_fork(ctx, st);          // the LOS chains do not read flow fields: fork before the flow waves
            if (rc) return rc;
            rc = pf_waves_launch(ctx, stager_of(ctx).dev, gb.waves, ctx->pool.d_flow, ctx->pool.d_los, ctx->flow_stream,
                                 ctx->field_stream);
            if (rc) return rc;
            rc = los_forked(ctx);
            if (rc) return rc;
            if (out_n_flow) *out_n_flow = gb.waves.nf;
            if (out_n_los) *out_n_los = gb.waves.nl;
            return PFNAV_OK;
        }
        gb.valid = false;
    }
    pf_host_timer ht(ctx);
    for (int g = 0; g < ngoals; g++) PF_ARG(dests[g] >= 0 && dests[g] < ctx->pool.ndests, "dest");
    int rc = plan_batch(ctx, ngoals, dests, layer, targets, missing_only, ht);
    if (rc) return rc;
    pf_planner::merged &B = planner_of(ctx).batch;
    pf_wave_pack &W = B.W;
    if (W.fr.empty() && W.lr.empty()) return PFNAV_OK;
    ht.lap(PF_HPROF_MERGE);
    if ((rc = reserve_batch(ctx, B))) return rc;       // all or nothing: nothing is published before this succeeds
    ht.lap(PF_HPROF_RESERVE);
    const size_t bytes = W.layout();
    PF_CUDA(cudaSetDevice(ctx->device));
    cudaStream_t st = pf_stream(ctx, stream);
    // the slot table and the `has` bytes travel in the same staging buffer, behind the plan; the plan stays in the
    // device buffer for the resident fast path
    pf_stage S;
    if ((rc = pf_stage_begin(ctx, st, bytes, bytes, true, &S))) return rc;
    ht.lap(PF_HPROF_WAIT);
    W.pack(S.host);
    ht.lap(PF_HPROF_PACK);
    PF_CUDA(pf_pool_refresh(ctx, st));       // after pfnav_pool_clear: reset the touch stamps (the table is uploaded below)
    if ((rc = pf_stage_upload(ctx, st, S, bytes))) return rc;
    ht.lap(PF_HPROF_UPLOAD);
    if ((rc = los_fork(ctx, st))) return rc;
    rc = pf_waves_launch(ctx, S.dev, W.out, ctx->pool.d_flow, ctx->pool.d_los, ctx->flow_stream, ctx->field_stream);
    if (rc) return rc;
    if ((rc = los_forked(ctx))) return rc;
    ht.lap(PF_HPROF_LAUNCH);
    {
        auto &gb = ctx->goal_batch;
        gb.valid = !missing_only; gb.epoch = ctx->map_epoch; gb.layer = layer;
        gb.dests.assign(dests, dests + ngoals); gb.targets.assign(targets, targets + 4 * (size_t)ngoals);
        gb.waves = W.out;
    }
    if (out_n_flow) *out_n_flow = W.out.nf;
    if (out_n_los) *out_n_los = W.out.nl;
    return PFNAV_OK;
}

extern "C" int pfnav_pool_request_goal(pfnav_ctx *ctx, int dest, int layer, int tgt_chunk_r, int tgt_chunk_c,
                                       int tgt_tile_r, int tgt_tile_c, void *stream, int *out_n_flow, int *out_n_los)
{
    const int32_t d = dest, t[4] = {tgt_chunk_r, tgt_chunk_c, tgt_tile_r, tgt_tile_c};
    return pfnav_pool_request_goals(ctx, 1, &d, layer, t, stream, out_n_flow, out_n_los);
}

// Order `stream` after the LOS chains that pfnav_pool_request_goals forked onto the context's field
// stream. pfnav_agents_tick and the pool entry points do this themselves.
extern "C" int pfnav_fields_join(pfnav_ctx *ctx, void *stream)
{
    PF_ARG(ctx, "ctx");
    PF_NEED_DEVICE(ctx);
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(pf_fields_join(ctx, pf_stream(ctx, stream)));
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// Goal batches of a multi-GPU job (pfnav_mgpu_request_goals_ex / pfnav_group_request_goals_ex; the exchanges are in
// pfnav_mgpu.cu). The map is replicated, so every member plans the same requests for the same goals; members differ
// only in which fields their pools still hold. For every goal ONE member, its owner, builds the union of the fields any
// member lacks into its segment of a staging buffer; the segments are exchanged and every member copies the fields IT
// lacks into its own slots. Each member reserves exactly the keys its solo call would (the same merged batch, the same
// pf_pool_reserve), so its slots, evictions and `has` bits are the solo call's. The bytes are the solo call's too: a
// field is a function of its request and the replicated map, and a field one member keeps equals the one the owner
// rebuilds for another member, because every commit that changed the map under it dropped it from every pool alike
// (pfnav_map_commit decides what to drop from the replicated map and the dirty chunks only) -- the premise
// PFNAV_REQUEST_MISSING_ONLY already rests on.
// ------------------------------------------------------------------------------------------

// one 4096-byte field per CTA: block it.src of the source buffer of its kind (0 flow, 1 LOS) to block it.dst of the
// destination buffer of that kind
__global__ void __launch_bounds__(256) k_field_copy(const uint8_t *flow_src, const uint8_t *los_src, uint8_t *flow_dst,
                                                    uint8_t *los_dst, const pf_field_copy *items)
{
    const pf_field_copy it = items[blockIdx.x];
    const uint4 *s = (const uint4 *)((it.kind ? los_src : flow_src) + (size_t)it.src * 4096);
    uint4 *d = (uint4 *)((it.kind ? los_dst : flow_dst) + (size_t)it.dst * 4096);
    d[threadIdx.x] = s[threadIdx.x];
}

static int field_copy_launch(pfnav_ctx *ctx, const uint8_t *flow_src, const uint8_t *los_src, uint8_t *flow_dst,
                             uint8_t *los_dst, const pf_field_copy *d_items, int n, cudaStream_t st)
{
    if (!n) return 0;
    k_field_copy<<<n, 4096 / sizeof(uint4), 0, st>>>(flow_src, los_src, flow_dst, los_dst, d_items);
    ctx->launches++;
    PF_CUDA(cudaGetLastError());
    return 0;
}

// a job's batch reads the replicated map: refused while this member holds device blocker ops its peers have not seen
int pf_job_check_state(pfnav_ctx *ctx)
{
    if (pf_mgpu_shares_blockers(ctx) && pf_blocker_ops_unexchanged(ctx)) {
        pfnav_set_error("batch of a job: device blocker ops decided since the last exchange have not been exchanged "
                        "(pfnav_mgpu_exchange_blocker_ops / pfnav_group_exchange_blocker_ops)");
        return PFNAV_ERR_STATE;
    }
    return PFNAV_OK;
}

int pf_job_plan(pfnav_ctx *ctx, pf_job &J)
{
    if (J.kind != PF_JOB_GOALS) return pf_aux_job_plan(ctx, J);
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    const bool missing_only = (J.flags & PFNAV_REQUEST_MISSING_ONLY) != 0;
    J.fits = true; J.nf = J.nl = 0;
    J.lack.assign((size_t)J.ngoals * chunks, 0);
    for (int g = 0; g < J.ngoals; g++) PF_ARG(J.dests[g] >= 0 && J.dests[g] < ctx->pool.ndests, "dest");
    PF_ARG(J.layer >= 0 && J.layer < ctx->nlayers, "layer");
    if (int rc = pf_job_check_state(ctx)) return rc;
    if (J.ngoals == 0) return PFNAV_OK;
    pf_host_timer ht(ctx);
    int rc = plan_batch(ctx, J.ngoals, J.dests, J.layer, J.targets, missing_only, ht);
    if (rc) return rc;
    const pf_planner::merged &B = planner_of(ctx).batch;
    J.nf = (int)B.W.fr.size(); J.nl = (int)B.W.lr.size();
    J.fits = pf_pool_fits(ctx->pool, B.keys.data(), B.keys.size());
    for (int g = 0; g < J.ngoals; g++)
        for (int c = 0; c < chunks; c++)
            J.lack[(size_t)g * chunks + c] = (uint8_t)(~(missing_only ? ctx->pool.has_of((size_t)J.dests[g] * chunks + c) : 0) & 3);
    return PFNAV_OK;
}

int pf_job_launch(pfnav_ctx *ctx, pf_job &J, const uint8_t *uni, int world, int rank, cudaStream_t st)
{
    if (J.kind != PF_JOB_GOALS) return pf_aux_job_launch(ctx, J, world, rank, st);
    const int chunks = ctx->chunk_w * ctx->chunk_h, ngoals = J.ngoals;
    pf_planner &PL = planner_of(ctx);
    pf_planner::merged &B = PL.batch;               // this member's solo batch, merged by pf_job_plan
    ctx->job_built[0] = ctx->job_built[1] = 0;
    J.nitems = 0; J.d_items = nullptr;
    // ---- owners: the goal with the longest LOS chain among its union fields first, to the member with the fewest union
    // fields so far, ties to the lower rank (a LOS chain's latency is per chain: this spreads chains, not just fields)
    std::vector<int> work(ngoals, 0), chain(ngoals, 0), depth, order;
    for (int g = 0; g < ngoals; g++) {
        const pf_planner::goal_plan &P = PL.plans[g];
        const uint8_t *u = uni + (size_t)g * chunks;
        for (int i = 0; i < P.nf; i++) work[g] += (u[P.fc[i]] & 1) != 0;
        depth.assign(P.nl, 0);
        for (int i = 0; i < P.nl; i++) {
            if (!(u[P.lc[i]] & 2)) continue;
            const int p = P.lr[i].prev_index;
            depth[i] = p >= 0 && (u[P.lc[p]] & 2) ? depth[p] + 1 : 0;
            chain[g] = std::max(chain[g], depth[i] + 1);
            work[g]++;
        }
        if (work[g]) order.push_back(g);
    }
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return chain[a] > chain[b]; });
    std::vector<int32_t> &owner = ctx->job_owner;
    owner.assign(ngoals, -1);
    std::vector<int64_t> load(world, 0);
    for (int g : order) {
        int r = 0;
        for (int k = 1; k < world; k++) if (load[k] < load[r]) r = k;
        owner[g] = r;
        load[r] += work[g];
    }
    // ---- staging blocks: owner by owner, goal by goal, a goal's union flow fields (one per chunk) then its LOS fields
    std::vector<int32_t> fblk((size_t)ngoals * chunks, -1), lblk((size_t)ngoals * chunks, -1);
    J.seg.assign(world + 1, 0);
    int32_t next = 0;
    for (int r = 0; r < world; r++) {
        J.seg[r] = (size_t)next;
        for (int g = 0; g < ngoals; g++) {
            if (owner[g] != r) continue;
            const pf_planner::goal_plan &P = PL.plans[g];
            const uint8_t *u = uni + (size_t)g * chunks;
            int32_t *fb = fblk.data() + (size_t)g * chunks, *lb = lblk.data() + (size_t)g * chunks;
            for (int i = 0; i < P.nf; i++)
                if ((u[P.fc[i]] & 1) && fb[P.fc[i]] < 0) fb[P.fc[i]] = next++;
            for (int i = 0; i < P.nl; i++)
                if (u[P.lc[i]] & 2) lb[P.lc[i]] = next++;
        }
    }
    J.seg[world] = (size_t)next;
    if (!next) return PFNAV_OK;                     // every member holds every field: nothing to build or copy
    // ---- what this member builds: its goals' union fields, into staging. A rebuilt LOS field whose parent is in the
    // union reads the parent from staging; a parent that every member keeps is copied from this member's pool into a
    // block behind the segments first, before anything of this batch is written.
    pf_wave_pack W;
    std::vector<pf_field_copy> parents;
    int32_t extra = next;
    for (int g = 0; g < ngoals; g++) {
        if (owner[g] != rank) continue;
        const pf_planner::goal_plan &P = PL.plans[g];
        const uint8_t *u = uni + (size_t)g * chunks;
        const size_t gi = (size_t)g * chunks, row = (size_t)J.dests[g] * chunks;
        for (int i = 0; i < P.nf; i++)
            if (u[P.fc[i]] & 1) W.flow(P.fr[i], P.fw[i], fblk[gi + P.fc[i]]);
        W.los_chain(P.lr.data(), P.nl, [&](int i) { return (u[P.lc[i]] & 2) != 0; }, [&](int i) { return lblk[gi + P.lc[i]]; },
                    [&](int p) { parents.push_back({ctx->pool.slot_of(row + P.lc[p]), extra, 1}); return extra++; });
    }
    // ---- this member's own slots, exactly as its solo call reserves them
    int rc = 0;
    if (!B.keys.empty() && (rc = reserve_batch(ctx, B))) return rc;
    // ---- the fields this member lacks: staging block -> its slot (a flow field once per (goal, chunk))
    std::vector<pf_field_copy> items;
    std::vector<uint8_t> seen((size_t)ngoals * chunks, 0);
    for (int g = 0; g < ngoals; g++) {
        const pf_planner::goal_plan &P = PL.plans[g];
        const size_t gi = (size_t)g * chunks, row = (size_t)J.dests[g] * chunks;
        for (int i = 0; i < P.nf; i++) {
            const int c = P.fc[i];
            if (!(J.lack[gi + c] & 1) || seen[gi + c]) continue;
            seen[gi + c] = 1;
            items.push_back({fblk[gi + c], ctx->pool.slot_of(row + c), 0});
        }
        for (int i = 0; i < P.nl; i++)
            if (J.lack[gi + P.lc[i]] & 2) items.push_back({lblk[gi + P.lc[i]], ctx->pool.slot_of(row + P.lc[i]), 1});
    }
    // ---- stage: the builds in wave / depth order, the copies, then the slot table and the `has` bytes
    const size_t b_pc = parents.size() * sizeof(pf_field_copy), b_it = items.size() * sizeof(pf_field_copy);
    const size_t o_pc = W.layout(), o_it = o_pc + pf_wave_pack::align16(b_pc), total = o_it + pf_wave_pack::align16(b_it);
    PF_CUDA(cudaSetDevice(ctx->device));
    // the job staging: the previous batch's builds, exchange and copies may still read it, so growing it waits for the
    // device and the forked field work (a group member's stream has waited for its peers' reads of its staging)
    if ((size_t)extra * 4096 > ctx->d_job_stage.cap) PF_CUDA(pf_fields_sync(ctx));
    if ((rc = ctx->d_job_stage.reserve((size_t)extra * 4096))) return rc;
    pf_stage S;
    if ((rc = pf_stage_begin(ctx, st, total, total, true, &S))) return rc;
    W.pack(S.host);
    memcpy(S.host + o_pc, parents.data(), b_pc);
    memcpy(S.host + o_it, items.data(), b_it);
    PF_CUDA(pf_pool_refresh(ctx, st));
    if ((rc = pf_stage_upload(ctx, st, S, total))) return rc;
    uint8_t *stage = ctx->d_job_stage;
    if ((rc = field_copy_launch(ctx, nullptr, ctx->pool.d_los, nullptr, stage, (const pf_field_copy *)(S.dev + o_pc),
                                (int)parents.size(), st)))
        return rc;
    // the owner's builds: flow waves and LOS chains on the context's field streams, as in the solo call; the exchange
    // that follows on `st` reads what they wrote
    if ((rc = los_fork(ctx, st))) return rc;
    if ((rc = pf_waves_launch(ctx, S.dev, W.out, stage, stage, ctx->flow_stream, ctx->field_stream))) return rc;
    if ((rc = los_forked(ctx))) return rc;
    PF_CUDA(pf_fields_join(ctx, st));
    ctx->job_built[0] = W.out.nf; ctx->job_built[1] = W.out.nl;
    J.d_items = S.dev + o_it; J.nitems = (int)items.size();
    return PFNAV_OK;
}

int pf_job_scatter(pfnav_ctx *ctx, pf_job &J, cudaStream_t st)
{
    if (J.seg.empty() || J.seg.back() == 0) return PFNAV_OK;
    PF_CUDA(cudaSetDevice(ctx->device));
    int rc = field_copy_launch(ctx, ctx->d_job_stage, ctx->d_job_stage, ctx->pool.d_flow, ctx->pool.d_los,
                               (const pf_field_copy *)J.d_items, J.nitems, st);
    if (rc) return rc;
    // the next pool reader on any stream joins the copies the way it joins a solo batch's forked builds
    PF_CUDA(cudaEventRecord(ctx->ev_flow, st));
    PF_CUDA(cudaEventRecord(ctx->ev_los, st));
    ctx->los_inflight = true;
    return PFNAV_OK;
}

// Zone and entity-field batches of a job (pfnav_region.cu: pf_aux_job_*). Neither batch skips a field the pool holds and
// neither field reads another pool field, so every member writes the same keys with the same bytes: the keys, their
// owners and the staging layout follow from the arguments alone.
void pf_job_layout(pfnav_ctx *ctx, pf_job &J, const std::vector<int32_t> &freq, const std::vector<size_t> &fkey,
                   const std::vector<int64_t> &fcost, int world, std::vector<int32_t> &blk)
{
    const size_t n = freq.size();
    // the last writer of every key: the last field of each run of equal keys, in (key, field) order
    std::vector<int32_t> ord(n);
    for (size_t f = 0; f < n; f++) ord[f] = (int32_t)f;
    std::sort(ord.begin(), ord.end(), [&](int32_t a, int32_t b) { return fkey[a] != fkey[b] ? fkey[a] < fkey[b] : a < b; });
    std::vector<uint8_t> kept(n, 0);
    for (size_t i = 0; i < n; i++) kept[ord[i]] = i + 1 == n || fkey[ord[i + 1]] != fkey[ord[i]];
    std::vector<int64_t> cost(J.m, 0);
    std::vector<uint8_t> writes(J.m, 0);
    for (size_t f = 0; f < n; f++) if (kept[f]) { cost[freq[f]] += fcost[f]; writes[freq[f]] = 1; }
    std::vector<int32_t> order;
    for (size_t i = 0; i < J.m; i++) if (writes[i]) order.push_back((int32_t)i);
    std::stable_sort(order.begin(), order.end(), [&](int32_t a, int32_t b) { return cost[a] > cost[b]; });
    std::vector<int32_t> &owner = ctx->job_owner;
    owner.assign(J.m, -1);
    std::vector<int64_t> load(world, 0);
    for (int32_t i : order) {
        int r = 0;
        for (int k = 1; k < world; k++) if (load[k] < load[r]) r = k;
        owner[i] = r;
        load[r] += cost[i];
    }
    blk.assign(n, -1);
    J.seg.assign(world + 1, 0);
    int32_t next = 0;
    for (int r = 0; r < world; r++) {
        J.seg[r] = (size_t)next;
        for (size_t f = 0; f < n; f++) if (kept[f] && owner[freq[f]] == r) blk[f] = next++;
    }
    J.seg[world] = (size_t)next;
}

int pf_job_stage(pfnav_ctx *ctx, pf_job &J, const std::vector<pf_field_copy> &items, int world, cudaStream_t st)
{
    const size_t o_items = J.seg[world] * 4096, b_items = items.size() * sizeof(pf_field_copy);
    if (o_items + b_items > ctx->d_job_stage.cap) PF_CUDA(pf_fields_sync(ctx));      // as in pf_job_launch
    if (int rc = ctx->d_job_stage.reserve(o_items + b_items)) return rc;
    pf_stage S;
    if (int rc = pf_stage_begin(ctx, st, b_items, 0, true, &S)) return rc;
    memcpy(S.host, items.data(), b_items);
    if (b_items) PF_CUDA(cudaMemcpyAsync(ctx->d_job_stage + o_items, S.host, b_items, cudaMemcpyHostToDevice, st));
    if (int rc = pf_stage_upload(ctx, st, S, 0)) return rc;
    J.d_items = ctx->d_job_stage + o_items; J.nitems = (int)items.size();
    return PFNAV_OK;
}

// TEST HOOK: the last batch of a job on this member, of any kind. Goal batches: the flow / LOS requests it built for the
// job, and the owner of every goal (-1: no member lacked a field of it). Zone and entity-field batches: the fields it
// built, 0, and the owner of every request (-1: the request writes no key last)
extern "C" int pfnav_mgpu_fields_stats(pfnav_ctx *ctx, int *out_n_flow, int *out_n_los, int32_t *out_owner, int max_goals)
{
    PF_ARG(ctx && max_goals >= 0 && (max_goals == 0 || out_owner), "args");
    if (out_n_flow) *out_n_flow = ctx->job_built[0];
    if (out_n_los) *out_n_los = ctx->job_built[1];
    for (int g = 0; g < max_goals; g++) out_owner[g] = g < (int)ctx->job_owner.size() ? ctx->job_owner[g] : -1;
    return PFNAV_OK;
}
