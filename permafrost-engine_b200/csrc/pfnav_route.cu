// pfnav_route.cu -- host-side, cost-faithful restatement of the reference's hierarchical path
// request (the part of the hot path that decides WHICH chunk fields a destination needs).
//
// Restates (reference file:line):
//   n_update_island_field / n_visit_island              src/navigation/nav.c:1731-1772, 856-901
//   n_link_chunk_portals + AStar_GridPath               src/navigation/nav.c:593-636, a_star.c:303-427
//   n_build_portal_travel_index + N_GridNeighbours      src/navigation/nav.c:1314-1363, 4878-4910
//   n_update_edge_states / n_local_ports_connected      src/navigation/nav.c:668-717
//   N_PortalReachableFromTile                           src/navigation/nav.c:4852
//   N_ClosestPathableLocalIsland                        src/navigation/nav.c:5131
//   n_closest_reachable_portal / _from_location         src/navigation/nav.c:1365, 1398
//   AStar_PortalGraphPath + neighbours_portal_graph     src/navigation/a_star.c:429-552, 212-262
//   n_request_path                                      src/navigation/nav.c:1774-2047
//   N_FlowFieldID                                       src/navigation/field.c:1952
//
// Everything here is pointer-heavy host logic over a tiny graph; the fields it asks for are built by
// the CUDA kernels. Float costs follow the reference's evaluation order exactly (same heap, same
// neighbour order), because the chosen portal path depends on them.
#include "pfnav_internal.cuh"
#include <algorithm>
#include <atomic>
#include <thread>
#include <deque>
#include <float.h>
#include <math.h>
#include <memory>
#include <string.h>
#include <unordered_map>

namespace {

struct coord { int r, c; };
struct tdesc { int chunk_r, chunk_c, tile_r, tile_c; };

// pqueue.h:109-208 (1-indexed heap, float priority, hole sift)
template <class T>
struct pq {
    struct node { float prio; T data; };
    std::vector<node> n{1};
    int size = 0;
    void push(float prio, const T &d)
    {
        if ((int)n.size() < size + 2) n.resize(std::max<size_t>(32, n.size() * 2));
        int curr = size + 1, parent = curr / 2;
        while (curr > 1 && n[parent].prio > prio) { n[curr] = n[parent]; curr = parent; parent /= 2; }
        n[curr].prio = prio; n[curr].data = d;
        size++;
    }
    T pop()
    {
        T out = n[1].data;
        n[1] = n[size--];
        int root = 1;
        while (root != size + 1) {
            int target = size + 1;
            const int l = root * 2, r = l + 1;
            if (l <= size && n[l].prio < n[target].prio) target = l;
            if (r <= size && n[r].prio < n[target].prio) target = r;
            n[root] = n[target];
            root = target;
        }
        return out;
    }
};

// N_GridNeighbours (nav.c:4878) == a_star.c neighbours_grid (:101)
static int grid_neighbours(const uint8_t *cost, coord at, coord *out, float *costs)
{
    int ret = 0;
    for (int r = -1; r <= 1; r++)
        for (int c = -1; c <= 1; c++) {
            const int ar = at.r + r, ac = at.c + c;
            if (ar < 0 || ar >= 64 || ac < 0 || ac >= 64) continue;
            if (r == 0 && c == 0) continue;
            if (cost[ar * 64 + ac] == 0xFF) continue;
            const bool diag = (r == c) || (r == -c);
            if (diag && cost[ar * 64 + at.c] == 0xFF && cost[at.r * 64 + ac] == 0xFF) continue;
            const float cost_mult = diag ? (float)sqrt(2) : 1.0f;
            out[ret] = {ar, ac};
            costs[ret] = cost[ar * 64 + ac] * cost_mult;
            ret++;
        }
    return ret;
}

// heuristic (a_star.c:282)
static float heuristic(coord a, coord b)
{
    const float D = 1.0f;
    const float D2 = sqrt(2) * D;
    const int dx = abs(a.r - b.r), dy = abs(a.c - b.c);
    return D * (dx + dy) + (D2 - 2 * D) * std::min(dx, dy);
}

// AStar_GridPath (a_star.c:303), cost only
static bool astar_grid_cost(const uint8_t *cost, coord start, coord finish, float *out_cost)
{
    pq<coord> frontier;
    float running[4096];
    bool has_cost[4096], has_from[4096];
    memset(has_cost, 0, sizeof(has_cost));
    memset(has_from, 0, sizeof(has_from));
    running[start.r * 64 + start.c] = 0.0f;
    has_cost[start.r * 64 + start.c] = true;
    frontier.push(0.0f, start);
    while (frontier.size > 0) {
        const coord curr = frontier.pop();
        if (curr.r == finish.r && curr.c == finish.c) break;
        coord nb[8]; float nc[8];
        const int n = grid_neighbours(cost, curr, nb, nc);
        for (int i = 0; i < n; i++) {
            const int k = nb[i].r * 64 + nb[i].c;
            const float new_cost = running[curr.r * 64 + curr.c] + nc[i];
            if (!has_cost[k] || new_cost < running[k]) {
                running[k] = new_cost; has_cost[k] = true;
                frontier.push(new_cost + heuristic(finish, nb[i]), nb[i]);
                has_from[k] = true;
            }
        }
    }
    if (!has_from[finish.r * 64 + finish.c]) return false;
    *out_cost = running[finish.r * 64 + finish.c];
    return true;
}

static inline uint16_t cost_pack(float cost)          // portal_cost_pack (nav_data.h:56)
{
    if (cost == FLT_MAX) return 0xffff;
    const float scaled = cost * 8 + 0.5f;
    if (scaled >= 0xffff) return 0xffff - 1;
    return (uint16_t)scaled;
}
static inline float cost_unpack(uint16_t p) { return p == 0xffff ? FLT_MAX : (float)p / 8; }

}   // namespace

struct pfnav_route_edge { int es; int nb; float cost; };          // nb: portal index in the same chunk
struct pfnav_route_chunk {
    std::vector<std::vector<pfnav_route_edge>> edges;             // per portal
    std::vector<uint16_t> travel;                                 // [nportals][4096]
};
struct pfnav_route_layer {
    bool built = false;
    uint64_t generation = 0;                                      // bumped by every pfnav_route_build: device copies follow it
    std::vector<pfnav_route_chunk> chunks;
    std::vector<uint16_t> islands;                                // global islands, chunk-blocked
};
// The routing structures live in the context (pfnav_ctx::route_state): two contexts driven from two threads
// (one per GPU in one process) share nothing.
typedef std::vector<pfnav_route_layer> route_vec;
static inline route_vec *routes_of(const pfnav_ctx *ctx) { return (route_vec *)ctx->route_state; }
// the built layer, or nullptr
static inline pfnav_route_layer *route_layer(const pfnav_ctx *ctx, int layer)
{
    route_vec *rv = routes_of(ctx);
    if (!rv || layer < 0 || layer >= (int)rv->size() || !(*rv)[layer].built) return nullptr;
    return &(*rv)[layer];
}

void pfnav_route_dev_forget(pfnav_ctx *ctx);
void pfnav_route_forget(pfnav_ctx *ctx) { pfnav_route_dev_forget(ctx); delete routes_of(ctx); ctx->route_state = nullptr; }
// the portal lists of `layer` were rebuilt: its edge / travel tables no longer describe them
void pfnav_route_invalidate_layer(pfnav_ctx *ctx, int layer)
{
    route_vec *rv = routes_of(ctx);
    if (rv && layer >= 0 && layer < (int)rv->size()) (*rv)[layer] = pfnav_route_layer();
}

static inline const uint8_t *L_cost(const pfnav_ctx *ctx, int layer, int chunk)
{ return ctx->h_cost.data() + ((size_t)layer * ctx->chunk_w * ctx->chunk_h + chunk) * 4096; }
static inline const uint16_t *L_blk(const pfnav_ctx *ctx, int layer, int chunk)
{ return ctx->h_blk.data() + ((size_t)layer * ctx->chunk_w * ctx->chunk_h + chunk) * 4096; }
static inline const uint16_t *L_liid(const pfnav_ctx *ctx, int layer, int chunk)
{ return ctx->h_liid.data() + ((size_t)layer * ctx->chunk_w * ctx->chunk_h + chunk) * 4096; }

// n_update_edge_states (nav.c:693) for one chunk
static void update_edge_states(pfnav_ctx *ctx, pfnav_route_layer &RL, int layer, int chunk)
{
    const auto &ports = ctx->portals[layer][chunk];
    const uint16_t *blk = L_blk(ctx, layer, chunk), *li = L_liid(ctx, layer, chunk);
    for (size_t i = 0; i < ports.size(); i++)
        for (auto &e : RL.chunks[chunk].edges[i]) {
            const auto &a = ports[i], &b = ports[e.nb];
            bool conn = false;
            for (int r1 = a.r0; r1 <= a.r1 && !conn; r1++)
                for (int c1 = a.c0; c1 <= a.c1 && !conn; c1++) {
                    if (blk[r1 * 64 + c1] > 0) continue;
                    for (int r2 = b.r0; r2 <= b.r1 && !conn; r2++)
                        for (int c2 = b.c0; c2 <= b.c1; c2++) {
                            if (blk[r2 * 64 + c2] > 0) continue;
                            if (li[r1 * 64 + c1] == li[r2 * 64 + c2]) { conn = true; break; }
                        }
                }
            e.es = conn ? 0 : 1;       // EDGE_STATE_ACTIVE : EDGE_STATE_BLOCKED
        }
}

// n_update_edge_states for one chunk after its islands changed; returns the number of flipped edges,
// or -1 when the routing structure of the layer has not been built.
int pfnav_route_refresh_edges(pfnav_ctx *ctx, int layer, int chunk)
{
    pfnav_route_layer *prl = route_layer(ctx, layer);
    if (!prl) return -1;
    auto &RL = *prl;
    std::vector<int> before;
    for (auto &ev : RL.chunks[chunk].edges) for (auto &e : ev) before.push_back(e.es);
    update_edge_states(ctx, RL, layer, chunk);
    int flipped = 0; size_t k = 0;
    for (auto &ev : RL.chunks[chunk].edges) for (auto &e : ev) flipped += (e.es != before[k++]);
    return flipped;
}

// The global islands of one layer as a row-major device image (ctx->d_gisl, [layer][H64][W64]) for the map queries.
// They ignore blockers, so only a rebuild changes them.
static int route_upload_islands(pfnav_ctx *ctx, int layer, const pfnav_route_layer &RL)
{
    const size_t ltiles = (size_t)ctx->W64 * ctx->H64;
    PF_CUDA(cudaSetDevice(ctx->device));
    if (int rc = ctx->d_gisl.reserve(ltiles * ctx->nlayers)) return rc;
    std::vector<uint16_t> img(ltiles);
    for (int ch = 0; ch < ctx->chunk_w * ctx->chunk_h; ch++)
        for (int r = 0; r < 64; r++)
            memcpy(img.data() + (size_t)((ch / ctx->chunk_w) * 64 + r) * ctx->W64 + (ch % ctx->chunk_w) * 64,
                   RL.islands.data() + (size_t)ch * 4096 + r * 64, 128);
    PF_CUDA(cudaDeviceSynchronize());          // a query on a non-blocking stream may still read the old image
    PF_CUDA(cudaMemcpy(ctx->d_gisl + ltiles * layer, img.data(), ltiles * 2, cudaMemcpyHostToDevice));
    PF_CUDA(cudaDeviceSynchronize());
    return PFNAV_OK;
}

// Build the routing structure of one layer (needs pfnav_map_build_nav first).
extern "C" int pfnav_route_build(pfnav_ctx *ctx, int layer)
{
    PF_ARG(ctx && ctx->d_cost, "map not created");
    PF_ARG(layer >= 0 && layer < ctx->nlayers, "layer");
    PF_ARG((size_t)layer < ctx->portals.size() && !ctx->portals[layer].empty(), "pfnav_map_build_nav not called for this layer");
    if (!ctx->route_state) ctx->route_state = new route_vec();
    auto &RV = *routes_of(ctx);
    if ((int)RV.size() < ctx->nlayers) RV.resize(ctx->nlayers);
    pfnav_route_layer &RL = RV[layer];
    const int cw = ctx->chunk_w, chh = ctx->chunk_h, chunks = cw * chh;
    RL.chunks.assign(chunks, {});
    // every chunk's portal edges and travel index depend on that chunk alone: spread the chunks over the host cores
    auto build_chunk = [&](int ch) {
        const auto &ports = ctx->portals[layer][ch];
        const uint8_t *cost = L_cost(ctx, layer, ch);
        auto &RC = RL.chunks[ch];
        RC.edges.assign(ports.size(), {});
        // n_link_chunk_portals (nav.c:593): A* between portal centres, i-major j-minor
        for (size_t i = 0; i < ports.size(); i++)
            for (size_t j = 0; j < ports.size(); j++) {
                if (i == j) continue;
                const coord a = {(ports[i].r0 + ports[i].r1) / 2, (ports[i].c0 + ports[i].c1) / 2};
                const coord b = {(ports[j].r0 + ports[j].r1) / 2, (ports[j].c0 + ports[j].c1) / 2};
                float c;
                if (astar_grid_cost(cost, a, b, &c)) RC.edges[i].push_back({0, (int)j, c});
            }
        // n_build_portal_travel_index (nav.c:1314): FIFO expansion, first visit fixes the cost
        RC.travel.assign(ports.size() * 4096, 0xffff);
        for (size_t pi = 0; pi < ports.size(); pi++) {
            bool visited[4096];
            memset(visited, 0, sizeof(visited));
            std::deque<std::pair<float, coord>> q;
            for (int r = ports[pi].r0; r <= ports[pi].r1; r++)
                for (int c = ports[pi].c0; c <= ports[pi].c1; c++) { q.push_back({0.0f, {r, c}}); visited[r * 64 + c] = true; }
            while (!q.empty()) {
                const auto cur = q.front();
                q.pop_front();
                RC.travel[pi * 4096 + cur.second.r * 64 + cur.second.c] = cost_pack(cur.first);
                coord nb[8]; float nc[8];
                const int n = grid_neighbours(cost, cur.second, nb, nc);
                for (int i = 0; i < n; i++) {
                    const int k = nb[i].r * 64 + nb[i].c;
                    if (visited[k]) continue;
                    q.push_back({cur.first + nc[i], nb[i]});
                    visited[k] = true;
                }
            }
        }
    };
    {
        const int nthreads = std::max(1, std::min({(int)std::thread::hardware_concurrency(), 32, chunks}));
        std::atomic<int> next{0};
        std::vector<std::thread> pool;
        for (int t = 1; t < nthreads; t++)
            pool.emplace_back([&]() { for (int ch = next.fetch_add(1); ch < chunks; ch = next.fetch_add(1)) build_chunk(ch); });
        for (int ch = next.fetch_add(1); ch < chunks; ch = next.fetch_add(1)) build_chunk(ch);
        for (auto &t : pool) t.join();
    }
    // n_update_island_field (nav.c:1731): global islands ignoring blockers, ids from 0
    RL.islands.assign((size_t)chunks * 4096, 0xffff);
    {
        uint16_t id = 0;
        std::deque<tdesc> q;
        for (int cr = 0; cr < chh; cr++)
            for (int cc = 0; cc < cw; cc++)
                for (int t = 0; t < 4096; t++) {
                    const int ch = cr * cw + cc;
                    if (RL.islands[(size_t)ch * 4096 + t] != 0xffff || L_cost(ctx, layer, ch)[t] == 0xFF) continue;
                    RL.islands[(size_t)ch * 4096 + t] = id;
                    q.push_back({cr, cc, t >> 6, t & 63});
                    while (!q.empty()) {
                        const tdesc cur = q.front();
                        q.pop_front();
                        const int dr[4] = {0, 0, -1, 1}, dc[4] = {-1, 1, 0, 0};
                        for (int e = 0; e < 4; e++) {
                            const int ar = cur.chunk_r * 64 + cur.tile_r + dr[e], ac = cur.chunk_c * 64 + cur.tile_c + dc[e];
                            if (ar < 0 || ar >= chh * 64 || ac < 0 || ac >= cw * 64) continue;
                            const int nch = (ar >> 6) * cw + (ac >> 6), nt = (ar & 63) * 64 + (ac & 63);
                            if (RL.islands[(size_t)nch * 4096 + nt] == 0xffff && L_cost(ctx, layer, nch)[nt] != 0xFF) {
                                RL.islands[(size_t)nch * 4096 + nt] = id;
                                q.push_back({ar >> 6, ac >> 6, ar & 63, ac & 63});
                            }
                        }
                    }
                    id++;
                }
    }
    for (int ch = 0; ch < chunks; ch++) update_edge_states(ctx, RL, layer, ch);
    { static std::atomic<uint64_t> next_generation{1}; RL.generation = next_generation++; }
    RL.built = ctx->device < 0 || route_upload_islands(ctx, layer, RL) == PFNAV_OK;
    return RL.built ? PFNAV_OK : PFNAV_ERR_CUDA;
}

// the device image of one layer's global islands, for pfnav_map_query
const uint16_t *pfnav_route_dev_islands(const pfnav_ctx *ctx, int layer)
{
    if (!route_layer(ctx, layer) || !ctx->d_gisl) return nullptr;
    return ctx->d_gisl + (size_t)layer * ctx->W64 * ctx->H64;
}

// Read-back for parity tests: islands and the edge table of one portal (neighbour ref, state, cost)
extern "C" int pfnav_route_islands_get(pfnav_ctx *ctx, int layer, uint16_t *out)
{
    PF_ARG(ctx && out, "args");
    const pfnav_route_layer *prl = route_layer(ctx, layer);
    PF_ARG(prl, "pfnav_route_build not called");
    memcpy(out, prl->islands.data(), prl->islands.size() * 2);
    return PFNAV_OK;
}

extern "C" int pfnav_route_edges_get(pfnav_ctx *ctx, int layer, int chunk, int portal, uint32_t *out, int maxout, int *out_n)
{
    PF_ARG(ctx && out && out_n, "args");
    const pfnav_route_layer *prl = route_layer(ctx, layer);
    PF_ARG(prl, "pfnav_route_build not called");
    const auto &RL = *prl;
    PF_ARG(chunk >= 0 && chunk < (int)RL.chunks.size() && portal >= 0 && portal < (int)RL.chunks[chunk].edges.size(), "chunk/portal");
    int n = 0;
    for (const auto &e : RL.chunks[chunk].edges[portal]) {
        if (n >= maxout) break;
        out[n * 3 + 0] = ((uint32_t)chunk << 8) | (uint32_t)e.nb;        // portal_ref_make (nav_data.h:90)
        out[n * 3 + 1] = (uint32_t)e.es;
        memcpy(&out[n * 3 + 2], &e.cost, 4);
        n++;
    }
    *out_n = n;
    return PFNAV_OK;
}

namespace {

struct Router {
    pfnav_ctx *ctx; pfnav_route_layer &RL; int layer; int cw, chh;
    const pfnav_ctx::portal_t &P(int chunk, int idx) const { return ctx->portals[layer][chunk][idx]; }
    int nports(int chunk) const { return (int)ctx->portals[layer][chunk].size(); }
    const uint16_t *li(int chunk) const { return L_liid(ctx, layer, chunk); }

    // N_PortalReachableFromTile (nav.c:4852)
    bool portal_reachable_from_tile(int chunk, int pi, coord tile) const
    {
        const auto &p = P(chunk, pi);
        const uint16_t *l = li(chunk);
        for (int r = p.r0; r <= p.r1; r++)
            for (int c = p.c0; c <= p.c1; c++) {
                if (l[r * 64 + c] == 0xffff) continue;
                for (int r1 = tile.r - 1; r1 <= tile.r + 1; r1++)
                    for (int c1 = tile.c - 1; c1 <= tile.c + 1; c1++) {
                        if (r1 < 0 || r1 >= 64 || c1 < 0 || c1 >= 64) continue;
                        if (l[r * 64 + c] == l[r1 * 64 + c1]) return true;
                    }
            }
        return false;
    }

    // N_ClosestPathableLocalIsland (nav.c:5131): note `visited[tile_r * tile_h + tile_c]`
    uint16_t closest_pathable_liid(int chunk, coord target) const
    {
        const uint16_t *l = li(chunk);
        if (l[target.r * 64 + target.c] != 0xffff) return l[target.r * 64 + target.c];
        bool visited[4096];
        memset(visited, 0, sizeof(visited));
        std::deque<coord> q;
        q.push_back(target);
        visited[target.r * 64 + target.c] = true;
        while (!q.empty()) {
            const coord cur = q.front();
            q.pop_front();
            const int dr[4] = {0, 0, -1, 1}, dc[4] = {-1, 1, 0, 0};
            for (int e = 0; e < 4; e++) {
                const int nr = cur.r + dr[e], nc = cur.c + dc[e];
                // M_Tile_RelativeDesc succeeds across chunk borders; tiles outside this chunk are skipped
                if (nr < 0 || nr >= 64 || nc < 0 || nc >= 64) continue;
                if (visited[nr * 64 + nc]) continue;
                if (l[nr * 64 + nc] != 0xffff) return l[nr * 64 + nc];
                visited[nr * 64 + nc] = true;
                q.push_back({nr, nc});
            }
        }
        return 0xffff;
    }

    // n_closest_reachable_portal (nav.c:1365)
    int closest_reachable_portal(int chunk, coord start, bool unblocked) const
    {
        int ret = -1;
        float min_cost = FLT_MAX;
        for (int i = 0; i < nports(chunk); i++) {
            const float cost = cost_unpack(RL.chunks[chunk].travel[(size_t)i * 4096 + start.r * 64 + start.c]);
            if (unblocked && !portal_reachable_from_tile(chunk, i, start)) continue;
            if (cost < min_cost) { ret = i; min_cost = cost; }
        }
        return ret;
    }

    struct hop { int chunk, pi; uint16_t liid; };
    static uint64_t hop_key(const hop &h) { return ((uint64_t)h.liid << 32) | ((uint64_t)h.chunk << 8) | (uint64_t)h.pi; }

    // neighbours_portal_graph (a_star.c:212) incl. portal_reachable_from_island (:138) and
    // portal_connected_liids (:151)
    int neighbours(const hop &cur, hop *out, float *costs) const
    {
        int ret = 0;
        const int maxout = 256;
        const uint16_t *l = li(cur.chunk);
        for (const auto &e : RL.chunks[cur.chunk].edges[cur.pi]) {
            if (ret == maxout) return ret;
            if (e.es == 1) continue;
            const auto &np = P(cur.chunk, e.nb);
            bool reach = false;
            for (int r = np.r0; r <= np.r1 && !reach; r++)
                for (int c = np.c0; c <= np.c1; c++)
                    if (l[r * 64 + c] == cur.liid) { reach = true; break; }
            if (!reach) continue;
            out[ret] = {cur.chunk, e.nb, cur.liid};
            costs[ret] = e.cost;
            ret++;
        }
        const auto &p = P(cur.chunk, cur.pi);
        const auto &conn = P(p.conn_chunk, p.conn_idx);
        const uint16_t *cl = li(p.conn_chunk);
        uint16_t conn_liids[256];
        int nconn = 0;
        for (int r1 = p.r0; r1 <= p.r1; r1++)
            for (int c1 = p.c0; c1 <= p.c1; c1++) {
                if (l[r1 * 64 + c1] != cur.liid) continue;
                // the reference scans every tile of the connected portal for Manhattan distance 1 (a_star.c:151);
                // only the four neighbours of (r1, c1) can qualify: visit those inside the portal's rectangle in the
                // same (row, column) order
                const int ar = p.chunk_r * 64 + r1, ac = p.chunk_c * 64 + c1;
                const int cand[4][2] = {{ar - 1, ac}, {ar, ac - 1}, {ar, ac + 1}, {ar + 1, ac}};
                for (int k = 0; k < 4; k++) {
                    const int r2 = cand[k][0] - conn.chunk_r * 64, c2 = cand[k][1] - conn.chunk_c * 64;
                    if (r2 < conn.r0 || r2 > conn.r1 || c2 < conn.c0 || c2 > conn.c1) continue;
                    if (nconn == 256) goto done_conn;
                    const uint16_t nl = cl[r2 * 64 + c2];
                    bool contains = false;
                    for (int i = 0; i < nconn; i++) if (conn_liids[i] == nl) { contains = true; break; }
                    if (!contains && nl != 0xffff) conn_liids[nconn++] = nl;
                }
            }
    done_conn:
        for (int i = 0; i < nconn; i++) {
            if (ret == maxout) return ret;
            out[ret] = {p.conn_chunk, p.conn_idx, conn_liids[i]};
            costs[ret] = 1;
            ret++;
        }
        return ret;
    }

    // AStar_PortalGraphPath (a_star.c:429)
    bool portal_graph_path(tdesc start, tdesc end, int fin_chunk, int fin_pi, std::vector<hop> &path, float *out_cost) const
    {
        const int bchunk = start.chunk_r * cw + start.chunk_c, echunk = end.chunk_r * cw + end.chunk_c;
        const uint16_t start_liid = closest_pathable_liid(bchunk, {start.tile_r, start.tile_c});
        if (start_liid == 0xffff) return false;
        const uint16_t end_liid = closest_pathable_liid(echunk, {end.tile_r, end.tile_c});
        if (end_liid == 0xffff) return false;
        pq<hop> frontier;
        std::unordered_map<uint64_t, float> running;
        std::unordered_map<uint64_t, hop> came_from;
        for (int i = 0; i < nports(bchunk); i++) {
            const coord tc = {start.tile_r, start.tile_c};
            if (!portal_reachable_from_tile(bchunk, i, tc)) continue;
            const float cost = cost_unpack(RL.chunks[bchunk].travel[(size_t)i * 4096 + tc.r * 64 + tc.c]);
            if (cost != FLT_MAX) {
                const hop h = {bchunk, i, start_liid};
                running[hop_key(h)] = cost;
                frontier.push(cost, h);
            }
        }
        const float penalty = (float)sqrt(pow(64, 2.0f) + pow(64, 2.0f));     // portal_node_penalty (a_star.c:298)
        while (frontier.size > 0) {
            const hop cur = frontier.pop();
            if (cur.chunk == fin_chunk && cur.pi == fin_pi && cur.liid == end_liid) break;
            hop nb[256]; float nc[256];
            const int n = neighbours(cur, nb, nc);
            for (int i = 0; i < n; i++) {
                const float new_cost = running[hop_key(cur)] + nc[i] + penalty;
                auto it = running.find(hop_key(nb[i]));
                if (it == running.end() || new_cost < it->second) {
                    running[hop_key(nb[i])] = new_cost;
                    frontier.push(new_cost, nb[i]);
                    came_from[hop_key(nb[i])] = cur;
                }
            }
        }
        const hop last = {fin_chunk, fin_pi, end_liid};
        if (came_from.find(hop_key(last)) == came_from.end()) return false;
        path.clear();
        hop cur = last;
        while (true) {
            path.push_back(cur);
            auto it = came_from.find(hop_key(cur));
            if (it == came_from.end()) break;
            cur = it->second;
        }
        std::reverse(path.begin(), path.end());
        *out_cost = running[hop_key(last)];
        return true;
    }

    // n_closest_reachable_from_location (nav.c:1398)
    int closest_reachable_from_location(int chunk, tdesc loc, tdesc *out_nearest) const
    {
        float shortest = FLT_MAX;
        int ret = -1;
        tdesc nearest = {0, 0, 0, 0};
        std::vector<hop> path;
        const uint16_t *l = li(chunk);
        for (int i = 0; i < nports(chunk); i++) {
            uint16_t liids[64];
            int nl = 0;
            const auto &p = P(chunk, i);
            for (int r = p.r0; r <= p.r1; r++)
                for (int c = p.c0; c <= p.c1; c++) {
                    const tdesc cur = {p.chunk_r, p.chunk_c, r, c};
                    const uint16_t cl = l[r * 64 + c];
                    bool contains = false;
                    for (int k = 0; k < nl; k++) if (liids[k] == cl) { contains = true; break; }
                    if (!contains && nl < 64) {
                        liids[nl++] = cl;
                        float cost;
                        if (portal_graph_path(loc, cur, chunk, i, path, &cost) && cost < shortest) {
                            nearest = cur; shortest = cost; ret = i;
                        }
                    }
                }
        }
        if (ret >= 0) *out_nearest = nearest;
        return ret;
    }

    bool blocked_off(int chunk, coord tile) const       // n_blocked_off (nav.c:1544)
    {
        for (int i = 0; i < nports(chunk); i++) if (portal_reachable_from_tile(chunk, i, tile)) return false;
        return true;
    }
    bool normally_reachable(int chunk, coord a, coord b) const      // n_normally_reachable (nav.c:1531)
    {
        for (int i = 0; i < nports(chunk); i++) {
            const bool ar = RL.chunks[chunk].travel[(size_t)i * 4096 + a.r * 64 + a.c] != 0xffff;
            const bool br = RL.chunks[chunk].travel[(size_t)i * 4096 + b.r * 64 + b.c] != 0xffff;
            if (ar != br) return false;
        }
        return true;
    }
};

// M_Tile_DescForPoint2D with the nav resolution (tile.c:547)
static bool desc_for_point(const pfnav_ctx *ctx, float px, float pz, tdesc *out)
{
    const float width = (float)(ctx->chunk_w * 256), height = (float)(ctx->chunk_h * 256);
    if (px > ctx->map_x || px < ctx->map_x - width) return false;
    if (pz < ctx->map_z || pz > ctx->map_z + height) return false;
    int chunk_r = (int)(fabs(ctx->map_z - pz) / 256.0f), chunk_c = (int)(fabs(ctx->map_x - px) / 256.0f);
    chunk_r = std::min(std::max(chunk_r, 0), ctx->chunk_h - 1);
    chunk_c = std::min(std::max(chunk_c, 0), ctx->chunk_w - 1);
    const float bx = ctx->map_x - (chunk_c * 256.0f), bz = ctx->map_z + (chunk_r * 256.0f);
    int tile_r = (int)(fabs(bz - pz) / 4), tile_c = (int)(fabs(bx - px) / 4);
    out->chunk_r = chunk_r; out->chunk_c = chunk_c;
    out->tile_r = std::min(std::max(tile_r, 0), 63); out->tile_c = std::min(std::max(tile_c, 0), 63);
    return true;
}

}   // namespace

// ------------------------------------------------------------------------------------------
// n_request_path (nav.c:1774-2047), split at the points where a batch of requests runs its parts in different places:
//   plan_begin        the global-island test, the same-chunk early outs and n_closest_reachable_portal: read-only walks
//                     over the routing structure, independent of the field pool (host threads in a batch);
//   search rounds     AStar_PortalGraphPath to the destination portal; when it fails, plan_after_search runs
//                     n_closest_reachable_from_location on the host and asks for a second search;
//   emit_plan         the flow / LOS requests, in the reference's order, given which (dest, chunk) entries the cache
//                     holds: the only part that depends on the requests before it.
// ------------------------------------------------------------------------------------------
namespace {

struct path_plan {
    tdesc src, dst, dst0;            // dst: where the path ends (moved by the second search's fallback); dst0: as requested
    uint32_t dest_id = 0;
    int schunk = 0, dchunk = 0, dst_port = -1;
    bool emit = false;               // same global island: the destination chunk's field and LOS are requested
    bool exists = false;             // a portal path was found: the fields along it are requested too
    int ok = 0;
    int search = 0;                  // the search round this plan waits for (1 or 2), 0 = decided
    std::vector<Router::hop> path;
    float cost = 0.0f;
};

static void plan_init(const pfnav_ctx *ctx, int layer, const tdesc &src, const tdesc &dst, path_plan &P)
{
    P.src = src; P.dst = dst; P.dst0 = dst;
    P.dest_id = (((uint32_t)dst.chunk_r & 0x3f) << 26) | (((uint32_t)dst.chunk_c & 0x3f) << 20) |
                (((uint32_t)dst.tile_r & 0x3f) << 14) | (((uint32_t)dst.tile_c & 0x3f) << 8) |
                (((uint32_t)layer & 0xf) << 4) | ((uint32_t)ctx->req_faction & 0xfu);      // n_dest_id (nav.c:839)
    P.schunk = src.chunk_r * ctx->chunk_w + src.chunk_c;
    P.dchunk = dst.chunk_r * ctx->chunk_w + dst.chunk_c;
}

// nav.c:1798-1880: up to the first portal-graph search
static void plan_begin(const Router &R, path_plan &P)
{
    const tdesc &src = P.src, &dst = P.dst;
    const int schunk = P.schunk, dchunk = P.dchunk;
    if (R.RL.islands[(size_t)schunk * 4096 + src.tile_r * 64 + src.tile_c] != R.RL.islands[(size_t)dchunk * 4096 + dst.tile_r * 64 + dst.tile_c])
        return;
    P.emit = true;
    const uint16_t dst_cl = R.closest_pathable_liid(dchunk, {dst.tile_r, dst.tile_c});
    if (schunk == dchunk && R.closest_pathable_liid(schunk, {src.tile_r, src.tile_c}) == dst_cl) { P.ok = 1; return; }
    if (schunk == dchunk) {
        const bool either = R.blocked_off(schunk, {src.tile_r, src.tile_c}) || R.blocked_off(schunk, {dst.tile_r, dst.tile_c});
        if (either && R.normally_reachable(schunk, {src.tile_r, src.tile_c}, {dst.tile_r, dst.tile_c})) { P.ok = 1; return; }
    }
    P.dst_port = R.closest_reachable_portal(dchunk, {dst.tile_r, dst.tile_c}, true);
    if (P.dst_port < 0) P.dst_port = R.closest_reachable_portal(dchunk, {dst.tile_r, dst.tile_c}, false);
    if (P.dst_port < 0) return;
    P.search = 1;
}

// nav.c:1882-1939: after search round P.search has set P.exists / P.path / P.cost
static void plan_after_search(const Router &R, path_plan &P)
{
    const int round = P.search;
    P.search = 0;
    if (round == 1 && !P.exists) {
        const tdesc orig = P.dst;
        tdesc nd = P.dst;
        P.dst_port = R.closest_reachable_from_location(P.dchunk, P.src, &nd);
        if (P.dst_port >= 0) P.dst = nd;
        if (R.closest_pathable_liid(P.dchunk, {P.dst.tile_r, P.dst.tile_c}) != R.closest_pathable_liid(P.dchunk, {orig.tile_r, orig.tile_c}) &&
            P.src.chunk_r == P.dst.chunk_r && P.src.chunk_c == P.dst.chunk_c) { P.ok = 1; return; }
        if (P.dst_port >= 0) { P.search = 2; return; }
    }
    if (!P.exists) {
        if (P.src.chunk_r == P.dst.chunk_r && P.src.chunk_c == P.dst.chunk_c) P.ok = 1;
        return;
    }
    P.ok = 1;
}

static void plan_search_host(const Router &R, path_plan &P)
{
    P.exists = R.portal_graph_path(P.src, P.dst, P.dchunk, P.dst_port, P.path, &P.cost);
}

// the flow and LOS requests of one plan
struct path_emit {
    std::vector<pfnav_field_req> fr; std::vector<uint64_t> fid; std::vector<int32_t> fc;
    std::vector<pfnav_los_req> lr; std::vector<int32_t> lc;
    void clear() { fr.clear(); fid.clear(); fc.clear(); lr.clear(); lc.clear(); }
};

// nav.c:1815-1847 (destination chunk) and 1941-2042 (the portal path, walked backwards). mapped[chunk]: the ff_id the
// cache maps (dest, chunk) to, or 0; los_have[chunk]: its LOS field exists. Both are updated as the cache would be.
// LOS prev_index: -1 destination chunk, >= 0 a request of this plan, -2 the previous chunk's field already exists.
static void emit_plan(const Router &R, const pfnav_ctx *ctx, int layer, const path_plan &P, uint64_t *mapped, uint8_t *los_have, path_emit &E)
{
    E.clear();
    if (!P.emit) return;
    const int cw = ctx->chunk_w, dchunk = P.dchunk;
    const tdesc &dst0 = P.dst0;
    std::vector<int> los_index(ctx->chunk_w * ctx->chunk_h, -1);
    auto emit_los = [&](int chunk, int prev_chunk, const tdesc &tgt) {
        pfnav_los_req q;
        memset(&q, 0, sizeof(q));
        q.chunk_r = chunk / cw; q.chunk_c = chunk % cw; q.layer = layer; q.faction_id = ctx->req_faction;
        q.tgt_chunk_r = tgt.chunk_r; q.tgt_chunk_c = tgt.chunk_c; q.tgt_tile_r = tgt.tile_r; q.tgt_tile_c = tgt.tile_c;
        q.prev_index = prev_chunk < 0 ? -1 : (los_index[prev_chunk] >= 0 ? los_index[prev_chunk] : -2);
        if (prev_chunk >= 0) { q.prev_chunk_r = prev_chunk / cw; q.prev_chunk_c = prev_chunk % cw; }
        los_index[chunk] = (int)E.lr.size();
        E.lr.push_back(q); E.lc.push_back(chunk);
        los_have[chunk] = 1;
    };
    auto emit_flow = [&](const pfnav_field_req &q, uint64_t id, int chunk) {
        E.fr.push_back(q); E.fid.push_back(id); E.fc.push_back(chunk);
        mapped[chunk] = id;
    };
    pfnav_field_req base;
    memset(&base, 0, sizeof(base));
    base.layer = layer; base.faction_id = ctx->req_faction;
    if (!mapped[dchunk]) {
        pfnav_field_req q = base;
        q.chunk_r = dst0.chunk_r; q.chunk_c = dst0.chunk_c; q.target_type = PFNAV_TARGET_TILE; q.init = 1;
        q.tile_r = dst0.tile_r; q.tile_c = dst0.tile_c;
        emit_flow(q, ((uint64_t)layer << 60) | ((uint64_t)1 << 56) | ((uint64_t)dst0.tile_r << 24) | ((uint64_t)dst0.tile_c << 16) |
                     ((uint64_t)(dchunk / cw) << 8) | (uint64_t)(dchunk % cw), dchunk);
    }
    if (!los_have[dchunk]) emit_los(dchunk, -1, dst0);
    if (!P.exists) return;
    const std::vector<Router::hop> &path = P.path;
    const tdesc &dst = P.dst;
    int prev_los_chunk = dst.chunk_r * cw + dst.chunk_c;
    const uint16_t dst_liid_now = R.closest_pathable_liid(dchunk, {dst.tile_r, dst.tile_c});
    for (int i = (int)path.size() - 1; i > 0; i--) {
        int next_hop_idx = i;
        if (i == 1 && path[i].chunk != P.schunk) next_hop_idx = 0;
        const Router::hop curr_hop = path[std::max(next_hop_idx - 1, 0)];
        const Router::hop next_hop = path[next_hop_idx];
        const auto &cp = R.P(curr_hop.chunk, curr_hop.pi);
        if (cp.conn_chunk == next_hop.chunk && cp.conn_idx == next_hop.pi) continue;
        if (curr_hop.chunk == dchunk && next_hop.chunk == dchunk && next_hop.pi == P.dst_port && next_hop.liid == dst_liid_now) continue;
        const int chunk = curr_hop.chunk;
        const auto &np = R.P(next_hop.chunk, next_hop.pi);
        const auto &nn = R.P(np.conn_chunk, np.conn_idx);
        pfnav_field_req q = base;
        q.chunk_r = chunk / cw; q.chunk_c = chunk % cw; q.target_type = PFNAV_TARGET_PORTAL;
        q.port_r0 = np.r0; q.port_c0 = np.c0; q.port_r1 = np.r1; q.port_c1 = np.c1;
        q.next_r0 = nn.r0; q.next_c0 = nn.c0; q.next_r1 = nn.r1; q.next_c1 = nn.c1;
        q.next_chunk_r = nn.chunk_r; q.next_chunk_c = nn.chunk_c;
        q.port_iid = next_hop.liid;
        q.next_iid = (i < (int)path.size() - 1) ? path[next_hop_idx + 1].liid : dst_liid_now;
        // N_FlowFieldID TARGET_PORTAL (field.c:1954)
        const uint64_t new_id = ((uint64_t)layer << 60) | ((uint64_t)0 << 56) | (((uint64_t)q.next_iid & 0xf) << 48) |
                                (((uint64_t)q.port_iid & 0xf) << 40) | ((uint64_t)np.r0 << 34) | ((uint64_t)np.c0 << 28) |
                                ((uint64_t)np.r1 << 22) | ((uint64_t)np.c1 << 16) | ((uint64_t)q.chunk_r << 8) | (uint64_t)q.chunk_c;
        if (mapped[chunk]) {
            if (mapped[chunk] != new_id) {
                q.init = 0;          // merge into the chunk's existing field (nav.c:1994-2010)
                emit_flow(q, new_id, chunk);
            }
        } else {
            q.init = 1;
            emit_flow(q, new_id, chunk);
        }
        if (!los_have[chunk]) emit_los(chunk, prev_los_chunk, dst);
        prev_los_chunk = chunk;
    }
}

template <class F>
static void parallel_for(int n, F f)
{
    const int nthreads = std::max(1, std::min({n, (int)std::thread::hardware_concurrency(), 32}));
    if (nthreads == 1) { for (int i = 0; i < n; i++) f(i); return; }
    std::atomic<int> next{0};
    std::vector<std::thread> pool;
    auto worker = [&]() { for (int i = next.fetch_add(1); i < n; i = next.fetch_add(1)) f(i); };
    for (int t = 1; t < nthreads; t++) pool.emplace_back(worker);
    worker();
    for (auto &t : pool) t.join();
}

}   // namespace

static int route_dev_search(pfnav_ctx *ctx, int layer, pfnav_route_layer &RL, const int32_t *req, int n, int32_t *out, int max_hops);

// A search round holding at least this many searches runs on the device (k_portal_graph_path_warp), a smaller one on
// host threads. tools/bench_route_dev.py on the C2 map, one H100 80GB HBM3 at a 400 W power limit, 16 host threads
// (DESIGN.md §5): 64 searches take 15.6 ms on the device and 8.6 ms on the host, 1024 take 21.4 ms and 62.2 ms. The
// device's time is mostly the latency of the longest search, so the two lines cross near 200 searches.
#define PF_ROUTE_DEVICE_MIN_SEARCHES 256

// One search round over the plans `idx` that wait for it (edge states current).
static int search_round(pfnav_ctx *ctx, const Router &R, int layer, std::vector<path_plan> &plans, const std::vector<int> &idx)
{
    const int n = (int)idx.size();
    if (n == 0) return PFNAV_OK;
    std::vector<uint8_t> on_host(n, 1);
    if (n >= PF_ROUTE_DEVICE_MIN_SEARCHES && ctx->device >= 0) {
        const int max_hops = 512;
        const size_t ostride = 4 + 3 * (size_t)max_hops;
        std::vector<int32_t> req((size_t)n * 8), out((size_t)n * ostride);
        for (int k = 0; k < n; k++) {
            const path_plan &P = plans[idx[k]];
            int32_t *q = &req[(size_t)k * 8];
            q[0] = P.schunk; q[1] = P.src.tile_r; q[2] = P.src.tile_c;
            q[3] = P.dchunk; q[4] = P.dst.tile_r; q[5] = P.dst.tile_c; q[6] = P.dchunk; q[7] = P.dst_port;
        }
        int rc = route_dev_search(ctx, layer, R.RL, req.data(), n, out.data(), max_hops);
        if (rc) return rc;
        for (int k = 0; k < n; k++) {
            const int32_t *o = &out[(size_t)k * ostride];
            if (o[0] < 0) continue;             // outgrew the device scratch: the host routine has no limits
            path_plan &P = plans[idx[k]];
            on_host[k] = 0;
            P.exists = o[0] == 1;
            P.path.clear();
            if (!P.exists) continue;
            memcpy(&P.cost, &o[2], 4);
            for (int h = 0; h < o[1]; h++) P.path.push_back({o[4 + 3 * h], o[4 + 3 * h + 1], (uint16_t)o[4 + 3 * h + 2]});
        }
    }
    parallel_for(n, [&](int k) { if (on_host[k]) plan_search_host(R, plans[idx[k]]); });
    return PFNAV_OK;
}

// Plans every request up to its emission: plan_begin, search round 1, the fallback, search round 2.
static int plan_requests(pfnav_ctx *ctx, const Router &R, int layer, std::vector<path_plan> &plans)
{
    const int n = (int)plans.size();
    parallel_for(n, [&](int i) { plan_begin(R, plans[i]); });
    for (int round = 1; round <= 2; round++) {
        std::vector<int> idx;
        for (int i = 0; i < n; i++) if (plans[i].search == round) idx.push_back(i);
        int rc = search_round(ctx, R, layer, plans, idx);
        if (rc) return rc;
        parallel_for((int)idx.size(), [&](int k) { plan_after_search(R, plans[idx[k]]); });
    }
    return PFNAV_OK;
}

// n_request_path (nav.c:1774-2047), request-generation half. Emits, in the reference's order, the
// flow requests (with the N_FlowFieldID of each, field.c:1952) and LOS requests a cold field cache
// would have to build for (src -> dst), given which (dest, chunk) entries `have_flow` / `have_los`
// already hold (arrays of `chunks` entries; have_flow holds the ff_id mapped for the chunk or 0).
// Returns 1 in *out_ok when a path exists (the function's bool), plus the dest_id.
extern "C" int pfnav_route_request_path(pfnav_ctx *ctx, int layer, float src_x, float src_z, float dst_x, float dst_z,
                                        const uint64_t *have_flow, const uint8_t *have_los,
                                        pfnav_field_req *flow_out, uint64_t *flow_ffid, int32_t *flow_chunk, int max_flow,
                                        int *n_flow, pfnav_los_req *los_out, int32_t *los_chunk, int max_los, int *n_los,
                                        uint32_t *out_dest_id, int *out_ok)
{
    PF_ARG(ctx && n_flow && n_los && out_ok && out_dest_id, "args");
    pfnav_route_layer *prl = route_layer(ctx, layer);
    PF_ARG(prl, "pfnav_route_build not called");
    pfnav_route_layer &RL = *prl;
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    Router R{ctx, RL, layer, ctx->chunk_w, ctx->chunk_h};
    *n_flow = 0; *n_los = 0; *out_ok = 0;
    // n_update_dirty_local_islands + n_update_all_edge_states (nav.c:1786-1787)
    for (int ch = 0; ch < chunks; ch++) update_edge_states(ctx, RL, layer, ch);
    tdesc src, dst;
    PF_ARG(desc_for_point(ctx, src_x, src_z, &src) && desc_for_point(ctx, dst_x, dst_z, &dst), "position outside the map");
    path_plan P;
    plan_init(ctx, layer, src, dst, P);
    *out_dest_id = P.dest_id;
    plan_begin(R, P);
    while (P.search) { plan_search_host(R, P); plan_after_search(R, P); }
    std::vector<uint64_t> mapped(have_flow, have_flow + chunks);
    std::vector<uint8_t> los_have(have_los, have_los + chunks);
    path_emit E;
    emit_plan(R, ctx, layer, P, mapped.data(), los_have.data(), E);
    const int nf = std::min((int)E.fr.size(), std::max(max_flow, 0)), nl = std::min((int)E.lr.size(), std::max(max_los, 0));
    for (int i = 0; i < nf; i++) { flow_out[i] = E.fr[i]; flow_ffid[i] = E.fid[i]; flow_chunk[i] = E.fc[i]; }
    for (int i = 0; i < nl; i++) { los_out[i] = E.lr[i]; los_chunk[i] = E.lc[i]; }
    *n_flow = nf; *n_los = nl;
    if (nf < (int)E.fr.size()) { pfnav_set_error("flow output too small"); return PFNAV_ERR_NOMEM; }
    if (nl < (int)E.lr.size()) { pfnav_set_error("los output too small"); return PFNAV_ERR_NOMEM; }
    *out_ok = P.ok;
    return PFNAV_OK;
}

namespace {

// The flow waves and LOS requests of consecutive requests of a batch that go to the device together. Within one
// segment no pool slot changes owner, so (dest, chunk) keys and slots correspond one to one.
struct path_segment {
    pf_wave_pack W;                                   // flow requests by wave, LOS requests with their parents
    std::unordered_map<int32_t, int> writes;          // slot -> flow writes to it so far: the next one goes a wave later
    std::unordered_map<size_t, int> los_at;           // (dest, chunk) -> its LOS request in W
    std::vector<std::pair<int32_t, size_t>> used;     // (slot, key) of every slot written or read
    void clear() { W.clear(); writes.clear(); los_at.clear(); used.clear(); }
};

// Stage a segment's requests and launch its flow waves and its one LOS launch on `st`.
static int launch_segment(pfnav_ctx *ctx, cudaStream_t st, path_segment &S)
{
    pf_wave_pack &W = S.W;
    if (W.fr.empty() && W.lr.empty()) return PFNAV_OK;
    const size_t bytes = W.layout();
    pf_stage G;
    int rc = pf_stage_begin(ctx, st, bytes, bytes, false, &G);
    if (rc) return rc;
    W.pack(G.host);
    if ((rc = pf_stage_upload(ctx, st, G, bytes))) return rc;
    if ((rc = pf_waves_launch(ctx, G.dev, W.out, ctx->pool.d_flow, ctx->pool.d_los, st, st))) return rc;
    return pf_stage_done(ctx, st);
}

}   // namespace

// The staged form of a path-request batch (pfnav_internal.cuh): every request planned up front, then emitted against
// the pool mirrors one by one in the caller's order, reserved, and staged into a segment for the device.
struct pf_path_batch {
    pfnav_ctx *ctx = nullptr;
    cudaStream_t st = nullptr;
    std::vector<int32_t> dests, layers;
    std::vector<path_plan> plans;
    std::vector<uint8_t> planned;              // the request's layer is routed and both of its points are on the map
    path_segment S;
    path_emit E;                               // the emission of the last probed request
    int probed = -1;
    std::vector<size_t> keys;                  // its (dest, chunk) keys: flow writes, LOS writes, LOS parents read
    std::vector<uint64_t> mapped;
    std::vector<uint8_t> los_have, row_touched;
    bool any_evicted = false;
};

int pf_path_batch_begin(pfnav_ctx *ctx, int n, const int32_t *dests, const int32_t *layers, const float *src_xz,
                        const float *dst_xz, cudaStream_t st, pf_path_batch **out)
{
    *out = nullptr;
    PF_CUDA(cudaSetDevice(ctx->device));
    PF_CUDA(pf_fields_sync(ctx));
    PF_CUDA(pf_pool_refresh(ctx, st));
    std::unique_ptr<pf_path_batch> B(new pf_path_batch);
    B->ctx = ctx; B->st = st;
    B->dests.assign(dests, dests + n); B->layers.assign(layers, layers + n);
    B->plans.resize(n); B->planned.assign(n, 0);
    const int cw = ctx->chunk_w, chunks = cw * ctx->chunk_h;
    B->mapped.resize(chunks); B->los_have.resize(chunks); B->row_touched.assign(ctx->pool.ndests, 0);
    std::vector<tdesc> s(n), d(n);
    std::set<int> used_layers;
    for (int i = 0; i < n; i++) {
        B->planned[i] = route_layer(ctx, layers[i]) && desc_for_point(ctx, src_xz[2 * i], src_xz[2 * i + 1], &s[i]) &&
                        desc_for_point(ctx, dst_xz[2 * i], dst_xz[2 * i + 1], &d[i]);
        if (B->planned[i]) used_layers.insert(layers[i]);
    }
    for (int layer : used_layers) {
        pfnav_route_layer &RL = *route_layer(ctx, layer);
        // n_update_all_edge_states (nav.c:1787): the map does not change between the requests of a batch
        for (int ch = 0; ch < chunks; ch++) update_edge_states(ctx, RL, layer, ch);
        Router R{ctx, RL, layer, cw, ctx->chunk_h};
        std::vector<int> idx;
        for (int i = 0; i < n; i++) if (B->planned[i] && layers[i] == layer) idx.push_back(i);
        std::vector<path_plan> plans(idx.size());
        for (size_t k = 0; k < idx.size(); k++) plan_init(ctx, layer, s[idx[k]], d[idx[k]], plans[k]);
        int rc = plan_requests(ctx, R, layer, plans);
        if (rc) return rc;
        for (size_t k = 0; k < idx.size(); k++) B->plans[idx[k]] = std::move(plans[k]);
    }
    *out = B.release();
    return PFNAV_OK;
}

void pf_path_batch_end(pf_path_batch *B) { delete B; }

bool pf_path_batch_planned(const pf_path_batch *B, int i) { return B->planned[i] != 0; }

int pf_path_batch_probe(pf_path_batch *B, int i, pf_path_probe *out)
{
    pfnav_ctx *ctx = B->ctx;
    PF_ARG(B->planned[i], "pfnav_route_build not called, or a position outside the map");
    const int layer = B->layers[i], cw = ctx->chunk_w, chunks = cw * ctx->chunk_h;
    const size_t row = (size_t)B->dests[i] * chunks;
    for (int c = 0; c < chunks; c++) B->los_have[c] = (ctx->pool.has_of(row + c) & 2) ? 1 : 0;
    memcpy(B->mapped.data(), ctx->pool.ffid.data() + row, (size_t)chunks * 8);
    Router R{ctx, *route_layer(ctx, layer), layer, cw, ctx->chunk_h};
    path_emit &E = B->E;
    emit_plan(R, ctx, layer, B->plans[i], B->mapped.data(), B->los_have.data(), E);
    const int nf = (int)E.fr.size(), nl = (int)E.lr.size();
    B->probed = i;
    out->dest_id = B->plans[i].dest_id; out->ok = B->plans[i].ok; out->nf = nf; out->nl = nl;
    out->would_evict = false;
    out->write_slots.clear();
    // slots for everything this request writes (and the previous-chunk LOS fields it reads), all or nothing
    std::vector<size_t> &keys = B->keys;
    keys.clear();
    for (int k = 0; k < nf; k++) keys.push_back(row + E.fc[k]);
    for (int k = 0; k < nl; k++) keys.push_back(row + E.lc[k]);
    for (int k = 0; k < nl; k++)
        if (E.lr[k].prev_index == -2) keys.push_back(row + E.lr[k].prev_chunk_r * cw + E.lr[k].prev_chunk_c);
    for (size_t k = 0; k < (size_t)(nf + nl); k++) {
        const int32_t s = ctx->pool.slot_of(keys[k]);
        if (s >= 0) out->write_slots.push_back(s);
    }
    std::vector<size_t> fresh;
    pf_pool_fresh(ctx->pool, keys.data(), keys.size(), fresh);
    out->would_evict = fresh.size() > ctx->pool.avail();
    return PFNAV_OK;
}

int pf_path_batch_commit(pf_path_batch *B, std::vector<int32_t> *out_slots)
{
    pfnav_ctx *ctx = B->ctx;
    const path_emit &E = B->E;
    const int dest = B->dests[B->probed], cw = ctx->chunk_w;
    const size_t row = (size_t)dest * cw * ctx->chunk_h;
    const int nf = (int)E.fr.size(), nl = (int)E.lr.size();
    if (out_slots) out_slots->clear();
    if (nf == 0 && nl == 0) return PFNAV_OK;
    const std::vector<size_t> &keys = B->keys;
    std::vector<int32_t> slots(keys.size());
    bool evicted = false;
    int rc = pf_pool_reserve(ctx, keys.data(), keys.size(), slots.data(), &evicted);
    if (rc) return rc;
    path_segment &S = B->S;
    B->any_evicted |= evicted;
    B->row_touched[dest] = 1;
    if (evicted) {
        // a slot this segment writes or reads now belongs to another (dest, chunk): launch the segment first, so
        // that its writes and reads stay ordered before this request's
        bool moved = false;
        for (const auto &u : S.used) moved |= ctx->pool.owner[u.first] != (int64_t)u.second;
        if (moved) { rc = launch_segment(ctx, B->st, S); if (rc) return rc; S.clear(); }
    }
    for (size_t k = 0; k < keys.size(); k++) S.used.push_back({slots[k], keys[k]});
    for (int i = 0; i < nf; i++) {
        const int32_t s = slots[i];
        ctx->pool.built_flow(s, E.fr[i]);
        ctx->pool.ffid[row + E.fc[i]] = E.fid[i];
        S.W.flow(E.fr[i], S.writes[s]++, s);
    }
    const int l0 = (int)S.W.lr.size();
    for (int i = 0; i < nl; i++) {
        const int32_t s = slots[nf + i];
        ctx->pool.built(s, 2);
        pfnav_los_req q = E.lr[i];
        if (q.prev_index >= 0) q.prev_index += l0;
        else if (q.prev_index == -2) {
            const size_t pkey = row + q.prev_chunk_r * cw + q.prev_chunk_c;
            auto it = S.los_at.find(pkey);
            if (it != S.los_at.end()) q.prev_index = it->second;        // built earlier in this segment
            else q._pad = ctx->pool.slot_of(pkey);                      // absolute pool slot of prev_los
        }
        S.los_at[row + E.lc[i]] = S.W.los(q, s);
    }
    if (out_slots) out_slots->assign(slots.begin(), slots.begin() + nf + nl);
    return PFNAV_OK;
}

int pf_path_batch_flush(pf_path_batch *B)
{
    pfnav_ctx *ctx = B->ctx;
    cudaStream_t st = B->st;
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    int rc = launch_segment(ctx, st, B->S);
    if (rc) return rc;
    B->S.clear();
    if (B->any_evicted)      // entries of other destinations lost their slots
        PF_CUDA(cudaMemcpyAsync(ctx->pool.d_slot, ctx->pool.slot.data(), ctx->pool.slot.size() * 4, cudaMemcpyHostToDevice, st));
    else
        for (int d = 0; d < ctx->pool.ndests; d++)
            if (B->row_touched[d])
                PF_CUDA(cudaMemcpyAsync(ctx->pool.d_slot + (size_t)d * chunks, ctx->pool.slot.data() + (size_t)d * chunks,
                                        (size_t)chunks * 4, cudaMemcpyHostToDevice, st));
    bool any_touched = B->any_evicted;
    for (uint8_t t : B->row_touched) any_touched |= t != 0;
    if (any_touched)
        PF_CUDA(cudaMemcpyAsync(ctx->pool.d_has, ctx->pool.has.data(), ctx->pool.max,
                                cudaMemcpyHostToDevice, st));
    std::fill(B->row_touched.begin(), B->row_touched.end(), 0);
    B->any_evicted = false;
    return PFNAV_OK;
}

// pfnav_pool_request_paths once its arguments are checked: plan every request, then emit and reserve request by
// request in order -- what the serial calls would do to the pool mirrors -- and launch the device work per segment.
static int pool_request_paths(pfnav_ctx *ctx, int n, const int32_t *dests, int layer, const float *src_xz, const float *dst_xz,
                              void *stream, uint32_t *out_dest_ids, int32_t *out_ok, int32_t *out_n_flow, int32_t *out_n_los,
                              int *out_ndone)
{
    const std::vector<int32_t> layers(n, layer);
    pf_path_batch *pb = nullptr;
    int rc = pf_path_batch_begin(ctx, n, dests, layers.data(), src_xz, dst_xz, pf_stream(ctx, stream), &pb);
    if (rc) return rc;
    std::unique_ptr<pf_path_batch, void (*)(pf_path_batch *)> B(pb, pf_path_batch_end);
    pf_path_probe pr;
    int done = 0;
    for (; done < n; done++) {
        if ((rc = pf_path_batch_probe(pb, done, &pr))) break;
        if (out_dest_ids) out_dest_ids[done] = pr.dest_id;
        if (out_ok) out_ok[done] = pr.ok;
        if (out_n_flow) out_n_flow[done] = pr.nf;
        if (out_n_los) out_n_los[done] = pr.nl;
        if ((rc = pf_path_batch_commit(pb, nullptr))) break;
    }
    int lrc = pf_path_batch_flush(pb);
    if (lrc) return lrc;
    if (out_ndone) *out_ndone = done;
    return rc;
}

// N_RequestPath (nav.c:3386) for a batch of requests on one layer against the device field pool (pfnav.h).
extern "C" int pfnav_pool_request_paths(pfnav_ctx *ctx, int n, const int32_t *dests, int layer, const float *src_xz,
                                        const float *dst_xz, void *stream, uint32_t *out_dest_ids, int32_t *out_ok,
                                        int32_t *out_n_flow, int32_t *out_n_los, int *out_ndone)
{
    if (out_ndone) *out_ndone = 0;
    PF_ARG(ctx, "ctx");
    PF_ARG(n >= 0 && (n == 0 || (dests && src_xz && dst_xz)), "n / null arrays");
    PF_ARG(route_layer(ctx, layer), "pfnav_route_build not called");
    for (int i = 0; i < n; i++) {
        tdesc t;
        PF_ARG(dests[i] >= 0, "dest");
        PF_ARG(desc_for_point(ctx, src_xz[2 * i], src_xz[2 * i + 1], &t) && desc_for_point(ctx, dst_xz[2 * i], dst_xz[2 * i + 1], &t),
               "position outside the map");
    }
    PF_NEED_DEVICE(ctx);
    PF_ARG(ctx->pool.d_slot, "pool not created");
    for (int i = 0; i < n; i++) PF_ARG(dests[i] < ctx->pool.ndests, "dest");
    if (n == 0) return PFNAV_OK;
    return pool_request_paths(ctx, n, dests, layer, src_xz, dst_xz, stream, out_dest_ids, out_ok, out_n_flow, out_n_los, out_ndone);
}

// pfnav_pool_request_paths with endpoints that may name resident entities (pfnav.h): k_resident_xz writes the named
// records' positions over the given ones in the request staging, one copy back and one wait, then the batch as given.
extern "C" int pfnav_pool_request_paths_resident(pfnav_ctx *ctx, int n, const int32_t *dests, int layer, const uint32_t *src_uids,
                                                 const float *src_xz, const uint32_t *dst_uids, const float *dst_xz, void *stream,
                                                 uint32_t *out_dest_ids, int32_t *out_ok, int32_t *out_n_flow, int32_t *out_n_los,
                                                 int *out_ndone)
{
    if (out_ndone) *out_ndone = 0;
    PF_ARG(ctx, "ctx");
    PF_ARG(n >= 0, "n");
    pf_resident_points P;
    if (int rc = pf_resident_points_begin(ctx, "path requests", (size_t)n, src_uids, src_xz != nullptr, dst_uids,
                                          dst_xz != nullptr, P))
        return rc;
    if (P.entry.empty())
        return pfnav_pool_request_paths(ctx, n, dests, layer, src_xz, dst_xz, stream, out_dest_ids, out_ok, out_n_flow,
                                        out_n_los, out_ndone);
    // the staging holds the pairs, then the sources and the destinations as given (2n floats each)
    const size_t o_xz = (P.bytes() + 15) & ~(size_t)15, nxz = (size_t)n * 8, need = o_xz + 2 * nxz;
    PF_NEED_DEVICE(ctx);
    PF_CUDA(cudaSetDevice(ctx->device));
    const cudaStream_t st = pf_stream(ctx, stream);
    pf_stage S;
    if (int rc = pf_stage_begin(ctx, st, need, need, false, &S)) return rc;
    P.pack(S.host);
    if (src_xz) memcpy(S.host + o_xz, src_xz, nxz);
    if (dst_xz) memcpy(S.host + o_xz + nxz, dst_xz, nxz);
    if (int rc = pf_stage_upload(ctx, st, S, need)) return rc;
    if (int rc = pf_resident_xz_launch(ctx, st, S.dev, P, 2, 0, 2 * n, (float *)(S.dev + o_xz))) return rc;
    PF_CUDA(cudaMemcpyAsync(S.host + o_xz, S.dev + o_xz, 2 * nxz, cudaMemcpyDeviceToHost, st));
    if (int rc = pf_stage_done(ctx, st)) return rc;
    PF_CUDA(cudaStreamSynchronize(st));
    std::vector<float> xz(4 * (size_t)n);
    memcpy(xz.data(), S.host + o_xz, 2 * nxz);
    return pfnav_pool_request_paths(ctx, n, dests, layer, xz.data(), xz.data() + 2 * (size_t)n, stream, out_dest_ids, out_ok,
                                    out_n_flow, out_n_los, out_ndone);
}

// N_RequestPath (nav.c:3386) against the device field pool: route src -> dst exactly as the reference
// does, then build only the fields the pool does not hold yet, in place, on the device. The one-request batch.
extern "C" int pfnav_pool_request_path(pfnav_ctx *ctx, int dest, int layer, float src_x, float src_z, float dst_x,
                                       float dst_z, void *stream, uint32_t *out_dest_id, int *out_ok, int *out_n_flow,
                                       int *out_n_los)
{
    PF_ARG(ctx && ctx->pool.d_slot, "pool not created");
    PF_NEED_DEVICE(ctx);
    PF_ARG(dest >= 0 && dest < ctx->pool.ndests, "dest");
    PF_ARG(route_layer(ctx, layer), "pfnav_route_build not called");
    const float s[2] = {src_x, src_z}, d[2] = {dst_x, dst_z};
    tdesc t;
    PF_ARG(desc_for_point(ctx, src_x, src_z, &t) && desc_for_point(ctx, dst_x, dst_z, &t), "position outside the map");
    uint32_t did = 0;
    int32_t ok = 0, nf = 0, nl = 0;
    int ndone = 0;
    const int rc = pool_request_paths(ctx, 1, &dest, layer, s, d, stream, &did, &ok, &nf, &nl, &ndone);
    if (out_dest_id) *out_dest_id = did;
    if (out_ok) *out_ok = ok;
    if (out_n_flow) *out_n_flow = nf;
    if (out_n_los) *out_n_los = nl;
    return rc;
}

// ------------------------------------------------------------------------------------------
// arrived() support (movement.c:2170-2196): the two map searches it makes depend only on the flock
// target and the layer, not on the entity, so they are evaluated once per (flock, layer) on the host
// mirrors and handed to the state-update kernel as constants:
//   * N_ClosestPathable (nav.c:4126): nearest not-blocked tile to the target, breadth-first over the
//     4-neighbourhood in the order {0,-1} {0,+1} {-1,0} {+1,0}; result = M_Tile_Bounds corner (x, z)
//   * N_IsMaximallyClose (nav.c:4707) -> n_closest_island_tiles (nav.c:1226, ignore_blockers = false):
//     the tiles of the target's global island, without blockers, at the smallest Manhattan distance
//     from the target (the target tile itself is never reported: it is marked visited up front and the
//     {0,0} delta is skipped), as "tile centres" map_pos -/+ (abs tile index) * 4 (nav.c:4729-4732)
// ------------------------------------------------------------------------------------------
int pfnav_arrival_consts(pfnav_ctx *ctx, int layer, float tx, float tz, pf_arrival_consts *out, int which)
{
    out->nearest_ok = 0; out->nearest[0] = out->nearest[1] = 0.0f; out->mc_n = 0;
    const pfnav_route_layer *prl = route_layer(ctx, layer);
    if (!prl && (which & PF_ARRIVAL_MC)) {
        pfnav_set_error("pfnav_agents_compute_updates: pfnav_route_build(layer %d) is needed (global islands, nav.c:1731)", layer);
        return PFNAV_ERR_ARG;
    }
    tdesc t;
    if (!desc_for_point(ctx, tx, tz, &t)) return PFNAV_OK;       // target outside the map: the reference asserts
    const int cw = ctx->chunk_w, chh = ctx->chunk_h, W = cw * 64, H = chh * 64;
    auto blocked = [&](int ar, int ac) {
        const int ch = (ar >> 6) * cw + (ac >> 6), tt = (ar & 63) * 64 + (ac & 63);
        return L_cost(ctx, layer, ch)[tt] == 0xFF || L_blk(ctx, layer, ch)[tt] > 0;
    };
    const int tr = t.chunk_r * 64 + t.tile_r, tc = t.chunk_c * 64 + t.tile_c;
    // ---- N_ClosestPathable ----
    const bool nearest = which & PF_ARRIVAL_NEAREST;
    if (nearest && !blocked(tr, tc)) {
        out->nearest_ok = 1; out->nearest[0] = tx; out->nearest[1] = tz;
    } else if (nearest) {
        std::vector<uint8_t> vis((size_t)W * H, 0);
        std::vector<int> q; q.push_back(tr * W + tc);
        for (size_t qi = 0; qi < q.size(); qi++) {
            const int ar = q[qi] / W, ac = q[qi] % W;
            if (!blocked(ar, ac)) {
                // M_Tile_Bounds (tile.c:356): x decreases with the column, z increases with the row
                out->nearest_ok = 1;
                out->nearest[0] = (ctx->map_x - (float)((ac >> 6) * 256)) - (float)((ac & 63) * 4);
                out->nearest[1] = (ctx->map_z + (float)((ar >> 6) * 256)) + (float)((ar & 63) * 4);
                break;
            }
            const int dr[4] = {0, 0, -1, 1}, dc[4] = {-1, 1, 0, 0};
            for (int e = 0; e < 4; e++) {
                const int nr = ar + dr[e], nc = ac + dc[e];
                if (nr < 0 || nr >= H || nc < 0 || nc >= W) continue;
                if (vis[(size_t)nr * W + nc]) continue;
                vis[(size_t)nr * W + nc] = 1;
                q.push_back(nr * W + nc);
            }
        }
    }
    // ---- n_closest_island_tiles(target, giid(target), ignore_blockers = false, maxout = 256) ----
    if (which & PF_ARRIVAL_MC) {
        const pfnav_route_layer &RL = *prl;
        const uint16_t giid = RL.islands[(size_t)(t.chunk_r * cw + t.chunk_c) * 4096 + t.tile_r * 64 + t.tile_c];
        std::vector<uint8_t> vis((size_t)W * H, 0);
        std::vector<int> q; q.push_back(tr * W + tc);
        vis[(size_t)tr * W + tc] = 1;
        int first_mh = -1, n = 0;
        bool done = false;
        for (size_t qi = 0; qi < q.size() && !done; qi++) {
            const int ar = q[qi] / W, ac = q[qi] % W;
            const int dr[9] = {0, 0, 0, -1, 1, -1, -1, 1, 1}, dc[9] = {0, -1, 1, 0, 0, -1, 1, -1, 1};
            for (int e = 0; e < 9; e++) {
                const int nr = ar + dr[e], nc = ac + dc[e];
                if (nr < 0 || nr >= H || nc < 0 || nc >= W) continue;
                if (vis[(size_t)nr * W + nc]) continue;
                const int ch = (nr >> 6) * cw + (nc >> 6), tt = (nr & 63) * 64 + (nc & 63);
                bool skip = RL.islands[(size_t)ch * 4096 + tt] != giid;
                if (L_blk(ctx, layer, ch)[tt] > 0) skip = true;
                const int mh = abs(tr - nr) + abs(tc - nc);
                if (first_mh > 0 && mh > first_mh) { done = true; break; }
                if (!skip) {
                    out->mc[n][0] = ctx->map_x - (float)nc * 4.0f;      // (chunk_c*64 + tile_c) * tile_dims.x
                    out->mc[n][1] = ctx->map_z + (float)nr * 4.0f;
                    n++;
                    if (first_mh == -1) first_mh = mh;
                    if (n == PF_ARRIVAL_MC_MAX) { done = true; break; }
                }
                vis[(size_t)nr * W + nc] = 1;
                q.push_back(nr * W + nc);
            }
        }
        out->mc_n = n;
    }
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// Seeds of the repair chain of N_DesiredPointSeekVelocity (nav.c:3508-3554), host side (they need the
// global islands and breadth-first ring searches over the chunk; the integration itself runs on the
// device, k_repair_chain):
//   kind 0  N_FlowFieldUpdateToNearestPathable (field.c:2247): the passable tiles that border the
//           non-passable blob containing (start_r, start_c)   (field_passable_frontier, field.c:1441)
//   kind 1  N_FlowFieldUpdateIslandToNearest (field.c:2307): the tiles of local island `local_iid`
//           nearest (Manhattan) to the field's own frontier     (field_closest_tiles_local, field.c:1010)
// mask: 64 rows of 64 bits. The chain builds kind-0 seeds itself (pfnav_repair_kernel.cuh); the host search of kind 0
// is the reference pfnav_repair_seed_mask exposes.
// ------------------------------------------------------------------------------------------
// The argument checks of a kind-0 repair.
static int pfnav_repair_start_check(pfnav_ctx *ctx, const pfnav_field_req &q, int arg)
{
    const int chunk = q.chunk_r * ctx->chunk_w + q.chunk_c;
    const uint8_t *cost = L_cost(ctx, q.layer, chunk);
    const uint16_t *blk = L_blk(ctx, q.layer, chunk);
    const int sr = arg >> 8, sc = arg & 0xFF;
    PF_ARG(sr >= 0 && sr < 64 && sc >= 0 && sc < 64, "repair start tile");
    PF_ARG(!(cost[sr * 64 + sc] != 0xFF && blk[sr * 64 + sc] == 0),
           "N_FlowFieldUpdateToNearestPathable needs a non-passable start tile (field.c:1455)");
    return PFNAV_OK;
}

static int pfnav_repair_seeds(pfnav_ctx *ctx, const pfnav_field_req &q, int kind, int arg, uint64_t *mask)
{
    memset(mask, 0, 64 * sizeof(uint64_t));
    const int layer = q.layer, cw = ctx->chunk_w;
    const int chunk = q.chunk_r * cw + q.chunk_c;
    const uint8_t *cost = L_cost(ctx, layer, chunk);
    const uint16_t *blk = L_blk(ctx, layer, chunk), *liid = L_liid(ctx, layer, chunk);
    auto passable = [&](int r, int c) { return cost[r * 64 + c] != 0xFF && blk[r * 64 + c] == 0; };
    static const int dr4[4] = {0, 0, -1, 1}, dc4[4] = {-1, 1, 0, 0};
    if (kind == 0) {
        const int sr = arg >> 8, sc = arg & 0xFF;
        int rc = pfnav_repair_start_check(ctx, q, arg);
        if (rc) return rc;
        std::vector<uint8_t> vis(4096, 0);
        std::vector<int> fq; fq.push_back(sr * 64 + sc);
        vis[sr * 64 + sc] = 1;
        for (size_t qi = 0; qi < fq.size(); qi++) {
            const int r = fq[qi] >> 6, c = fq[qi] & 63;
            if (passable(r, c)) { mask[r] |= 1ull << c; continue; }
            for (int e = 0; e < 4; e++) {
                const int ar = r + dr4[e], ac = c + dc4[e];
                if (ar < 0 || ar >= 64 || ac < 0 || ac >= 64 || vis[ar * 64 + ac]) continue;
                vis[ar * 64 + ac] = 1;
                fq.push_back(ar * 64 + ac);
            }
        }
        return PFNAV_OK;
    }
    // ---- kind 1 ----
    const pfnav_route_layer *prl = route_layer(ctx, layer);
    PF_ARG(prl, "pfnav_route_build(layer) is needed (global islands, nav.c:1731)");
    const uint16_t *gisl = prl->islands.data() + (size_t)chunk * 4096;
    const uint16_t local_iid = (uint16_t)arg;
    std::vector<int> init;
    if ((q.target_type & 0xFF) >= 2) {
        // TARGET_ENEMIES / TARGET_ENTITY field of pool destination q._pad: the entities' own tiles inside the chunk
        int rc = pfnav_aux_chunk_seeds(ctx, q._pad, q.chunk_r, q.chunk_c, init);
        if (rc) return rc;
    } else if ((q.target_type & 0xFF) == PFNAV_TARGET_TILE) {
        // field_tile_initial_frontier (field.c:1096); when the tile is blocked the reference retries with
        // ignoreblock (field.c:2367) -- either way the frontier is the tile itself
        init.push_back(q.tile_r * 64 + q.tile_c);
    } else {
        const uint16_t *nliid = L_liid(ctx, layer, q.next_chunk_r * cw + q.next_chunk_c);
        for (int r = q.port_r0; r <= q.port_r1; r++)
            for (int c = q.port_c0; c <= q.port_c1; c++) {
                if (!passable(r, c)) continue;
                if (q.port_iid != PFNAV_ISLAND_NONE && liid[r * 64 + c] != q.port_iid) continue;
                bool adj = false;
                for (int r2 = q.next_r0; r2 <= q.next_r1 && !adj; r2++)
                    for (int c2 = q.next_c0; c2 <= q.next_c1; c2++) {
                        const int ddr = (q.next_chunk_r * 64 + r2) - (q.chunk_r * 64 + r);
                        const int ddc = (q.next_chunk_c * 64 + c2) - (q.chunk_c * 64 + c);
                        if (abs(ddr) + abs(ddc) == 1 && nliid[r2 * 64 + c2] == q.next_iid) { adj = true; break; }
                    }
                if (adj) init.push_back(r * 64 + c);
            }
    }
    int min_mh = INT_MAX;
    std::vector<int> newf;
    std::vector<uint8_t> vis(4096);
    std::vector<int> fq, tmp;
    for (int t0 : init) {
        const int r0 = t0 >> 6, c0 = t0 & 63;
        const uint16_t cg = gisl[t0], cl = liid[t0];
        if (cl == local_iid) {
            if (min_mh > 0) newf.clear();
            min_mh = 0;
            newf.push_back(t0);
            continue;
        }
        // field_closest_tiles_local(chunk, curr, local_iid, curr_giid)
        std::fill(vis.begin(), vis.end(), 0);
        fq.clear(); tmp.clear();
        fq.push_back(t0); vis[t0] = 1;
        int first = -1;
        const size_t cap = 4096 - newf.size();
        for (size_t qi = 0; qi < fq.size(); qi++) {
            const int r = fq[qi] >> 6, c = fq[qi] & 63;
            for (int e = 0; e < 4; e++) {
                const int ar = r + dr4[e], ac = c + dc4[e];
                if (ar < 0 || ar >= 64 || ac < 0 || ac >= 64 || vis[ar * 64 + ac]) continue;
                vis[ar * 64 + ac] = 1;
                fq.push_back(ar * 64 + ac);
            }
            const int mh = abs(r0 - r) + abs(c0 - c);
            if (first > -1 && mh > first) break;
            if (cost[r * 64 + c] == 0xFF) continue;
            if (blk[r * 64 + c] > 0) continue;
            if (cg != PFNAV_ISLAND_NONE && gisl[r * 64 + c] != cg) continue;
            if (local_iid != PFNAV_ISLAND_NONE && liid[r * 64 + c] != local_iid) continue;
            if (first == -1) first = mh;
            tmp.push_back(r * 64 + c);
            if (tmp.size() == cap) break;
        }
        if (tmp.empty()) continue;
        const int mh = abs((tmp[0] >> 6) - r0) + abs((tmp[0] & 63) - c0);
        if (mh < min_mh) { min_mh = mh; newf.clear(); }
        if (mh > min_mh) continue;
        newf.insert(newf.end(), tmp.begin(), tmp.end());
    }
    for (int t : newf) mask[t >> 6] |= 1ull << (t & 63);
    return PFNAV_OK;
}

int pf_chain_item_seeds(pfnav_ctx *ctx, pf_chain_item &it, std::vector<uint64_t> &masks)
{
    if (it.kind == 0) {
        if (int rc = pfnav_repair_start_check(ctx, it.q, it.arg)) return rc;
        it.mask = -1;
        return PFNAV_OK;
    }
    uint64_t mask[64];
    if (int rc = pfnav_repair_seeds(ctx, it.q, it.kind, it.arg, mask)) return rc;
    it.mask = (int32_t)(masks.size() / 64);
    masks.insert(masks.end(), mask, mask + 64);
    return PFNAV_OK;
}

// The seeds of a repair of a TARGET_TILE field (pfnav.h), host side; works on host-only contexts.
extern "C" int pfnav_repair_seed_mask(pfnav_ctx *ctx, int layer, int chunk_r, int chunk_c, int kind, int arg, uint64_t *out_rows)
{
    PF_ARG(ctx && out_rows && ctx->chunk_w > 0, "map not created");
    PF_ARG(layer >= 0 && layer < ctx->nlayers && chunk_r >= 0 && chunk_r < ctx->chunk_h && chunk_c >= 0 && chunk_c < ctx->chunk_w,
           "layer / chunk");
    PF_ARG(kind == PFNAV_REPAIR_NEAREST_PATHABLE || kind == PFNAV_REPAIR_ISLAND_TO_NEAREST, "repair kind");
    pfnav_field_req q;
    memset(&q, 0, sizeof(q));
    q.layer = layer; q.chunk_r = chunk_r; q.chunk_c = chunk_c; q.target_type = PFNAV_TARGET_TILE;
    return pfnav_repair_seeds(ctx, q, kind, arg, out_rows);
}

// N_RequestPathAttacking (nav.c:3393): the faction carried by the path requests that follow -- packed into the
// dest_id and forwarded to every flow / LOS request, exactly what n_request_path does with its faction_id.
extern "C" int pfnav_request_faction(pfnav_ctx *ctx, int faction_id)
{
    PF_ARG(ctx, "ctx");
    PF_ARG(faction_id == PFNAV_FACTION_ID_NONE || (faction_id >= 0 && faction_id < 15), "faction_id");
    ctx->req_faction = faction_id;
    return PFNAV_OK;
}

// Inspection / test entry: the per-(target, layer) constants of arrived() (movement.c:2170) that
// pfnav_agents_compute_updates uploads: N_ClosestPathable's answer and the tile centres N_IsMaximallyClose
// compares with. out_mc: up to cap (x, z) pairs. Host structure code; needs pfnav_route_build(layer).
extern "C" int pfnav_route_arrival_consts(pfnav_ctx *ctx, int layer, float tx, float tz, int32_t *out_nearest_ok,
                                          float *out_nearest_xz, float *out_mc_xz, size_t cap, int32_t *out_mc_n)
{
    PF_ARG(ctx && out_nearest_ok && out_nearest_xz && out_mc_n, "null argument");
    pf_arrival_consts c;
    int rc = pfnav_arrival_consts(ctx, layer, tx, tz, &c);
    if (rc) return rc;
    *out_nearest_ok = c.nearest_ok; out_nearest_xz[0] = c.nearest[0]; out_nearest_xz[1] = c.nearest[1];
    *out_mc_n = c.mc_n;
    for (int i = 0; i < c.mc_n && (size_t)i < cap && out_mc_xz; i++) { out_mc_xz[2 * i] = c.mc[i][0]; out_mc_xz[2 * i + 1] = c.mc[i][1]; }
    return PFNAV_OK;
}

// ------------------------------------------------------------------------------------------
// Device-side AStar_PortalGraphPath (a_star.c:429; SURVEY 8f-2): a batch of portal-graph searches, one warp per search.
// The search itself is the reference's, statement for statement -- N_ClosestPathableLocalIsland (nav.c:5131) for both
// ends, N_PortalReachableFromTile (:4852) + the travel-cost index for the start portals, neighbours_portal_graph
// (a_star.c:212), portal_node_penalty (:298), and the 1-indexed binary heap of pqueue.h:109-208 whose tie order decides
// between equal-cost paths -- over device copies of the portal table, the intra-chunk edges with their states, the
// travel-cost index and the local-island image.
// Heap pushes and pops, and the cost-table updates that decide them, stay in the reference's serial order on lane 0.
// The lanes share what surrounds them: the start-portal tests, each expansion's edge tests (compacted in edge order
// with ballots), the portal_connected_liids scan (an order-preserving dedupe with match / ballot) and the cost-table
// lookups of the neighbours. The cost / predecessor table is stamped per launch instead of being cleared.
// Per-search scratch (heap, cost / predecessor table, flood queue) lives in HBM.
// ------------------------------------------------------------------------------------------
namespace {

struct dev_portal { int16_t r0, c0, r1, c1, chunk_r, chunk_c; int32_t conn_chunk, conn_idx, edge_off, edge_cnt; };
struct dev_edge { int32_t nb, es; float cost; };
struct dev_route {
    const dev_portal *ports;      // [chunks][64]
    const int32_t *nports;        // [chunks]
    const int32_t *port_base;     // [chunks]: first row of the chunk's portals in `travel`
    const dev_edge *edges;
    const uint16_t *travel;       // [port_base[chunk] + i][4096]
    const uint16_t *liid;         // image of the layer [H64][W64]
    int cw, chh, W64;
    float penalty;
};
#define GP_HT 16384               // cost / predecessor table slots (open addressing, at most 3/4 used)
#define GP_PQ 16384               // heap capacity
#define GP_WARPS 4                // searches per CTA
#define GP_NONE (~0ull)           // no predecessor (a key never has its top bits set)
struct gp_slot { uint64_t key, from; float cost; uint32_t stamp; };       // stamp != the launch's: free
struct gp_scratch {
    gp_slot h[GP_HT];
    float pprio[GP_PQ]; uint64_t pdata[GP_PQ];
    uint32_t visited[1024];       // 4096 flags
    uint16_t queue[4096];
};
struct route_dev_state {
    pf_dbuf<dev_portal> d_ports; pf_dbuf<int32_t> d_nports, d_port_base; pf_dbuf<dev_edge> d_edges;
    pf_dbuf<uint16_t> d_travel; size_t travel_rows = 0;
    pf_dbuf<gp_scratch> d_scratch; uint32_t stamp = 0;
    pf_dbuf<int32_t> d_req, d_out;
    int layer = -1; uint64_t epoch = ~0ull, generation = 0;
};

__device__ __forceinline__ uint16_t gp_li(const dev_route &R, int chunk, int r, int c)
{
    return R.liid[(size_t)((chunk / R.cw) * 64 + r) * R.W64 + (chunk % R.cw) * 64 + c];
}
__device__ __forceinline__ uint64_t gp_key(int chunk, int pi, uint16_t liid) { return ((uint64_t)liid << 32) | ((uint64_t)chunk << 8) | (uint64_t)pi; }

// N_ClosestPathableLocalIsland (nav.c:5131). The flood returns the first island tile in the serial queue order, so it
// stays on lane 0; the lanes clear its visited flags.
__device__ uint16_t gp_closest_liid(const dev_route &R, gp_scratch &S, int chunk, int tr, int tc, int lane)
{
    const uint16_t own = gp_li(R, chunk, tr, tc);
    if (own != 0xffff) return own;
    for (int i = lane; i < 1024; i += 32) S.visited[i] = 0;
    __syncwarp();
    uint16_t found = 0xffff;
    if (lane == 0) {
        uint8_t *vis = (uint8_t *)S.visited;
        int head = 0, tail = 0;
        S.queue[tail++] = (uint16_t)(tr * 64 + tc);
        vis[tr * 64 + tc] = 1;
        while (head < tail && found == 0xffff) {
            const int cur = S.queue[head++], r = cur >> 6, c = cur & 63;
            const int dr[4] = {0, 0, -1, 1}, dc[4] = {-1, 1, 0, 0};
            for (int e = 0; e < 4; e++) {
                const int nr = r + dr[e], nc = c + dc[e];
                if (nr < 0 || nr >= 64 || nc < 0 || nc >= 64) continue;
                if (vis[nr * 64 + nc]) continue;
                const uint16_t l = gp_li(R, chunk, nr, nc);
                if (l != 0xffff) { found = l; break; }
                vis[nr * 64 + nc] = 1;
                S.queue[tail++] = (uint16_t)(nr * 64 + nc);
            }
        }
    }
    return (uint16_t)__shfl_sync(0xffffffffu, (int)found, 0);
}

// N_PortalReachableFromTile (nav.c:4852)
__device__ bool gp_portal_reachable(const dev_route &R, int chunk, const dev_portal &p, int tr, int tc)
{
    for (int r = p.r0; r <= p.r1; r++)
        for (int c = p.c0; c <= p.c1; c++) {
            const uint16_t l = gp_li(R, chunk, r, c);
            if (l == 0xffff) continue;
            for (int r1 = tr - 1; r1 <= tr + 1; r1++)
                for (int c1 = tc - 1; c1 <= tc + 1; c1++) {
                    if (r1 < 0 || r1 >= 64 || c1 < 0 || c1 >= 64) continue;
                    if (l == gp_li(R, chunk, r1, c1)) return true;
                }
        }
    return false;
}

__device__ __forceinline__ int gp_find(const gp_scratch &S, uint64_t key, uint32_t stamp)   // slot of key, or the first free one
{
    uint32_t h = (uint32_t)((key * 0x9E3779B97F4A7C15ull) >> 50) & (GP_HT - 1);
    while (S.h[h].stamp == stamp && S.h[h].key != key) h = (h + 1) & (GP_HT - 1);
    return (int)h;
}
// pq push / pop: pqueue.h:165-208 (strict comparisons, hole sift)
__device__ __forceinline__ bool gp_push(gp_scratch &S, int &size, float prio, uint64_t d)
{
    if (size + 2 >= GP_PQ) return false;
    int curr = size + 1, parent = curr / 2;
    while (curr > 1 && S.pprio[parent] > prio) { S.pprio[curr] = S.pprio[parent]; S.pdata[curr] = S.pdata[parent]; curr = parent; parent /= 2; }
    S.pprio[curr] = prio; S.pdata[curr] = d;
    size++;
    return true;
}
__device__ __forceinline__ uint64_t gp_pop(gp_scratch &S, int &size)
{
    const uint64_t out = S.pdata[1];
    const float xp = S.pprio[size]; const uint64_t xd = S.pdata[size];
    size--;
    int root = 1;
    while (true) {
        const int l = root * 2, r = l + 1;
        int target = 0; float tp = xp;
        if (l <= size && S.pprio[l] < tp) { target = l; tp = S.pprio[l]; }
        if (r <= size && S.pprio[r] < tp) { target = r; tp = S.pprio[r]; }
        if (!target) break;
        S.pprio[root] = S.pprio[target]; S.pdata[root] = S.pdata[target];
        root = target;
    }
    S.pprio[root] = xp; S.pdata[root] = xd;
    return out;
}

// req: {start chunk, start tile_r, start tile_c, end chunk, end tile_r, end tile_c, finish chunk, finish portal}
// out (per search, 4 + 3 * max_hops ints): {status (1 found, 0 none, -1 scratch overflow), nhops, cost bits, 0, hops (chunk, portal, liid)...}
// stamp: nonzero, different from every earlier launch over the same scratch.
__global__ void __launch_bounds__(GP_WARPS * 32) k_portal_graph_path_warp(dev_route R, const int32_t *__restrict__ req, int n,
                                                                         gp_scratch *scratch, int32_t *out, int max_hops, uint32_t stamp)
{
    const unsigned FULL = 0xffffffffu;
    __shared__ uint64_t s_key[GP_WARPS][256];       // this expansion's neighbours, in neighbours_portal_graph's order
    __shared__ float s_cost[GP_WARPS][256];         // edge cost, then the relaxed cost (< 0: no update)
    __shared__ int32_t s_slot[GP_WARPS][256];       // the neighbour's table slot when it holds the key, else -1
    __shared__ uint16_t s_conn[GP_WARPS][256];      // portal_connected_liids
    const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
    const int i = blockIdx.x * GP_WARPS + w;
    if (i >= n) return;
    gp_scratch &S = scratch[i];
    const int32_t *q = req + (size_t)i * 8;
    int32_t *o = out + (size_t)i * (4 + 3 * max_hops);
    if (lane < 4) o[lane] = 0;
    const int bchunk = q[0], echunk = q[3], fin_chunk = q[6], fin_pi = q[7];
    const uint16_t start_liid = gp_closest_liid(R, S, bchunk, q[1], q[2], lane);
    if (start_liid == 0xffff) return;
    const uint16_t end_liid = gp_closest_liid(R, S, echunk, q[4], q[5], lane);
    if (end_liid == 0xffff) return;
    // start portals: reachability and travel cost on the lanes, pushed in portal order
    const int np = R.nports[bchunk];
    for (int p = lane; p < np; p += 32) {
        const dev_portal P = R.ports[bchunk * 64 + p];
        float c = -1.0f;
        if (gp_portal_reachable(R, bchunk, P, q[1], q[2])) {
            const uint16_t t = R.travel[(size_t)(R.port_base[bchunk] + p) * 4096 + q[1] * 64 + q[2]];
            if (t != 0xffff) c = (float)t / 8;
        }
        s_cost[w][p] = c;
    }
    __syncwarp();
    int size = 0, nkeys = 0;          // lane 0's
    bool overflow = false;
    if (lane == 0)
        for (int p = 0; p < np; p++) {
            const float cost = s_cost[w][p];
            if (cost < 0.0f) continue;
            const uint64_t key = gp_key(bchunk, p, start_liid);
            const int s = gp_find(S, key, stamp);
            if (S.h[s].stamp != stamp) { S.h[s].stamp = stamp; S.h[s].key = key; S.h[s].from = GP_NONE; nkeys++; }
            S.h[s].cost = cost;
            overflow |= !gp_push(S, size, cost, key);
        }
    const uint64_t last = gp_key(fin_chunk, fin_pi, end_liid);
    while (true) {
        uint64_t cur = 0;
        int go = 0;
        if (lane == 0 && size > 0 && !overflow) { cur = gp_pop(S, size); go = cur != last; }
        if (!__shfl_sync(FULL, go, 0)) break;
        cur = __shfl_sync(FULL, cur, 0);
        const int cchunk = (int)((cur >> 8) & 0xffffff), cpi = (int)(cur & 0xff);
        const uint16_t cli = (uint16_t)(cur >> 32);
        const dev_portal P = R.ports[cchunk * 64 + cpi];
        // neighbours_portal_graph (a_star.c:212): the chunk's own portals over active edges whose portal touches the island ...
        int nout = 0;
        for (int e0 = 0; e0 < P.edge_cnt && nout < 256; e0 += 32) {
            const int e = e0 + lane;
            bool acc = false;
            dev_edge E = {0, 1, 0.0f};
            if (e < P.edge_cnt) {
                E = R.edges[P.edge_off + e];
                if (E.es != 1) {
                    const dev_portal NP = R.ports[cchunk * 64 + E.nb];
                    for (int r = NP.r0; r <= NP.r1 && !acc; r++)
                        for (int c = NP.c0; c <= NP.c1; c++)
                            if (gp_li(R, cchunk, r, c) == cli) { acc = true; break; }
                }
            }
            const unsigned m = __ballot_sync(FULL, acc);
            const int pos = nout + __popc(m & ((1u << lane) - 1));
            if (acc && pos < 256) { s_key[w][pos] = gp_key(cchunk, E.nb, cli); s_cost[w][pos] = E.cost; }
            nout = min(256, nout + __popc(m));
        }
        // ... then the islands of the connected chunk that touch this one across the portal (portal_connected_liids, :151):
        // candidates (portal tile on the island, row-major) x (its four neighbours, in order) inside the connected portal
        if (nout < 256) {
            const dev_portal C = R.ports[P.conn_chunk * 64 + P.conn_idx];
            const int pw = P.c1 - P.c0 + 1, ncand = pw * (P.r1 - P.r0 + 1) * 4;
            int nconn = 0;
            for (int t0 = 0; t0 < ncand && nconn < 256; t0 += 32) {
                const int t = t0 + lane;
                bool valid = false;
                uint16_t nl = 0xffff;
                if (t < ncand) {
                    const int tile = t >> 2, k = t & 3, r1 = P.r0 + tile / pw, c1 = P.c0 + tile % pw;
                    if (gp_li(R, cchunk, r1, c1) == cli) {
                        const int ar = P.chunk_r * 64 + r1 + (k == 0 ? -1 : k == 3 ? 1 : 0);
                        const int ac = P.chunk_c * 64 + c1 + (k == 1 ? -1 : k == 2 ? 1 : 0);
                        const int r2 = ar - C.chunk_r * 64, c2 = ac - C.chunk_c * 64;
                        if (r2 >= C.r0 && r2 <= C.r1 && c2 >= C.c0 && c2 <= C.c1) {
                            nl = gp_li(R, P.conn_chunk, r2, c2);
                            valid = nl != 0xffff;
                        }
                    }
                }
                // new: valid, first of its id in this round, and not listed by an earlier round
                const unsigned same = __match_any_sync(FULL, valid ? (unsigned)nl : 0x10000u + lane);
                bool fresh = valid && (same & ((1u << lane) - 1)) == 0;
                for (int j = 0; j < nconn && fresh; j++) if (s_conn[w][j] == nl) fresh = false;
                const unsigned m = __ballot_sync(FULL, fresh);
                const int pos = nconn + __popc(m & ((1u << lane) - 1));
                if (fresh && pos < 256) s_conn[w][pos] = nl;
                nconn = min(256, nconn + __popc(m));
                __syncwarp();
            }
            for (int j = lane; j < nconn && nout + j < 256; j += 32) {
                s_key[w][nout + j] = gp_key(P.conn_chunk, P.conn_idx, s_conn[w][j]);
                s_cost[w][nout + j] = 1.0f;
            }
            nout = min(256, nout + nconn);
        }
        __syncwarp();
        // the neighbours' keys are distinct: look them up on the lanes, then relax in order on lane 0
        const float base = S.h[gp_find(S, cur, stamp)].cost;
        for (int j = lane; j < nout; j += 32) {
            const float new_cost = base + s_cost[w][j] + R.penalty;
            const int s = gp_find(S, s_key[w][j], stamp);
            const bool held = S.h[s].stamp == stamp;
            s_slot[w][j] = held ? s : -1;
            s_cost[w][j] = (!held || new_cost < S.h[s].cost) ? new_cost : -1.0f;
        }
        __syncwarp();
        if (lane == 0)
            for (int j = 0; j < nout && !overflow; j++) {
                const float new_cost = s_cost[w][j];
                if (new_cost < 0.0f) continue;
                const uint64_t nk = s_key[w][j];
                int s = s_slot[w][j];
                if (s < 0) {
                    if (nkeys + 1 >= GP_HT * 3 / 4) { overflow = true; break; }
                    s = gp_find(S, nk, stamp);
                    S.h[s].stamp = stamp; S.h[s].key = nk; nkeys++;
                }
                S.h[s].cost = new_cost; S.h[s].from = cur;
                overflow |= !gp_push(S, size, new_cost, nk);
            }
        __syncwarp();
    }
    if (lane != 0) return;
    if (overflow) { o[0] = -1; return; }
    const int ls = gp_find(S, last, stamp);
    if (S.h[ls].stamp != stamp || S.h[ls].from == GP_NONE) return;       // came_from holds no entry for the finish node
    int nh = 0;
    for (uint64_t cur = last; cur != GP_NONE; cur = S.h[gp_find(S, cur, stamp)].from) nh++;
    o[1] = nh; o[2] = __float_as_int(S.h[ls].cost);
    if (nh > max_hops) { o[0] = -1; return; }
    int k = nh;
    for (uint64_t cur = last; cur != GP_NONE; cur = S.h[gp_find(S, cur, stamp)].from) {
        k--;
        o[4 + 3 * k] = (int)((cur >> 8) & 0xffffff); o[4 + 3 * k + 1] = (int)(cur & 0xff); o[4 + 3 * k + 2] = (int)(cur >> 32);
    }
    o[0] = 1;
}

static route_dev_state *route_dev(pfnav_ctx *ctx)
{
    if (!ctx->route_dev_state) ctx->route_dev_state = new route_dev_state();
    return (route_dev_state *)ctx->route_dev_state;
}

}   // namespace

void pfnav_route_dev_forget(pfnav_ctx *ctx)
{
    route_dev_state *D = (route_dev_state *)ctx->route_dev_state;
    if (!D) return;
    if (ctx->device >= 0) cudaSetDevice(ctx->device);
    delete D;
    ctx->route_dev_state = nullptr;
}

// device copies of the routing tables of one layer; the travel-cost index follows the costs (re-sent when the layer was
// rebuilt), the portal table + edge states follow every commit (map_epoch)
static int route_dev_sync(pfnav_ctx *ctx, int layer, pfnav_route_layer &RL, route_dev_state *D)
{
    const int chunks = ctx->chunk_w * ctx->chunk_h;
    if (D->layer == layer && D->epoch == ctx->map_epoch && D->generation == RL.generation) return 0;
    std::vector<dev_portal> ports((size_t)chunks * 64);
    std::vector<int32_t> nports(chunks), base(chunks);
    std::vector<dev_edge> edges;
    size_t rows = 0;
    for (int ch = 0; ch < chunks; ch++) {
        const auto &pp = ctx->portals[layer][ch];
        nports[ch] = (int32_t)pp.size(); base[ch] = (int32_t)rows; rows += pp.size();
        for (size_t i = 0; i < pp.size(); i++) {
            dev_portal d;
            d.r0 = pp[i].r0; d.c0 = pp[i].c0; d.r1 = pp[i].r1; d.c1 = pp[i].c1; d.chunk_r = pp[i].chunk_r; d.chunk_c = pp[i].chunk_c;
            d.conn_chunk = pp[i].conn_chunk; d.conn_idx = pp[i].conn_idx;
            d.edge_off = (int32_t)edges.size(); d.edge_cnt = (int32_t)RL.chunks[ch].edges[i].size();
            for (const auto &e : RL.chunks[ch].edges[i]) edges.push_back({e.nb, e.es, e.cost});
            ports[(size_t)ch * 64 + i] = d;
        }
    }
    const bool retravel = D->layer != layer || D->generation != RL.generation || D->travel_rows != rows;
    int rc;
    if ((rc = D->d_ports.reserve(ports.size())) || (rc = D->d_nports.reserve(chunks)) || (rc = D->d_port_base.reserve(chunks)) ||
        (rc = D->d_edges.reserve(std::max<size_t>(edges.size(), 1))))
        return rc;
    PF_CUDA(cudaMemcpy(D->d_ports, ports.data(), ports.size() * sizeof(dev_portal), cudaMemcpyHostToDevice));
    PF_CUDA(cudaMemcpy(D->d_nports, nports.data(), (size_t)chunks * 4, cudaMemcpyHostToDevice));
    PF_CUDA(cudaMemcpy(D->d_port_base, base.data(), (size_t)chunks * 4, cudaMemcpyHostToDevice));
    if (!edges.empty()) PF_CUDA(cudaMemcpy(D->d_edges, edges.data(), edges.size() * sizeof(dev_edge), cudaMemcpyHostToDevice));
    if (retravel) {
        if ((rc = D->d_travel.reserve(std::max<size_t>(rows, 1) * 4096))) return rc;
        for (int ch = 0; ch < chunks; ch++)
            if (nports[ch])
                PF_CUDA(cudaMemcpy(D->d_travel + (size_t)base[ch] * 4096, RL.chunks[ch].travel.data(), (size_t)nports[ch] * 4096 * 2,
                                   cudaMemcpyHostToDevice));
        D->travel_rows = rows;
    }
    D->layer = layer; D->epoch = ctx->map_epoch; D->generation = RL.generation;
    return 0;
}

// n portal-graph searches on the device (k_portal_graph_path_warp), in the layout of pfnav_route_graph_paths. The host
// edge states must be current; the local islands are the device image, which pfnav_map_commit keeps equal to the host's.
static int route_dev_search(pfnav_ctx *ctx, int layer, pfnav_route_layer &RL, const int32_t *req, int n, int32_t *out, int max_hops)
{
    PF_CUDA(cudaSetDevice(ctx->device));
    route_dev_state *D = route_dev(ctx);
    D->epoch = ~0ull;                                                                  // edge states were just refreshed
    if (int rc = route_dev_sync(ctx, layer, RL, D)) return rc;
    const size_t ostride = 4 + 3 * (size_t)max_hops;
    const int batch = 4096;                                                            // 588 KB of scratch per search in flight
    const int want = std::min(std::max(n, 1), batch);
    bool grew;
    if (int rc = D->d_scratch.reserve((size_t)want, &grew)) return rc;
    if (grew) {
        PF_CUDA(cudaMemset(D->d_scratch, 0, D->d_scratch.cap * sizeof(gp_scratch)));     // no slot carries a stamp yet
        D->stamp = 0;
    }
    if (int rc = D->d_req.reserve((size_t)batch * 8)) return rc;
    if (int rc = D->d_out.reserve((size_t)batch * ostride)) return rc;
    dev_route R;
    R.ports = D->d_ports; R.nports = D->d_nports; R.port_base = D->d_port_base; R.edges = D->d_edges; R.travel = D->d_travel;
    R.liid = ctx->d_liid + (size_t)ctx->W64 * ctx->H64 * layer; R.cw = ctx->chunk_w; R.chh = ctx->chunk_h; R.W64 = ctx->W64;
    R.penalty = (float)sqrt(pow(64, 2.0f) + pow(64, 2.0f));                          // portal_node_penalty (a_star.c:298)
    PF_CUDA(cudaDeviceSynchronize());
    for (int b0 = 0; b0 < n; b0 += batch) {
        const int nb = std::min(batch, n - b0);
        if (++D->stamp == 0) {                                                         // the stamps wrapped: start the tables over
            PF_CUDA(cudaMemset(D->d_scratch, 0, D->d_scratch.cap * sizeof(gp_scratch)));
            D->stamp = 1;
        }
        PF_CUDA(cudaMemcpy(D->d_req, req + (size_t)b0 * 8, (size_t)nb * 32, cudaMemcpyHostToDevice));
        k_portal_graph_path_warp<<<(nb + GP_WARPS - 1) / GP_WARPS, GP_WARPS * 32>>>(R, D->d_req, nb, D->d_scratch,
                                                                                  D->d_out, max_hops, D->stamp);
        ctx->launches++;
        PF_CUDA(cudaGetLastError());
        PF_CUDA(cudaMemcpy(out + (size_t)b0 * ostride, D->d_out, (size_t)nb * ostride * 4, cudaMemcpyDeviceToHost));
    }
    return PFNAV_OK;
}

// AStar_PortalGraphPath for n searches. req: 8 ints per search {start chunk index, start tile r, c, end chunk index, end tile
// r, c, finish chunk index, finish portal index}; out: (4 + 3 * max_hops) ints per search {status, nhops, cost (float
// bits), 0, then (chunk, portal, local island) per hop, start to finish}; status 1 = path, 0 = none, -1 = the search
// outgrew its scratch (heap 16 k entries / 12 k nodes) or max_hops. on_device != 0: the kernel (k_portal_graph_path_warp);
// 0: the host planner's own routine (what pfnav_route_request_path runs) on host threads, for comparison.
extern "C" int pfnav_route_graph_paths(pfnav_ctx *ctx, int layer, const int32_t *req, int n, int32_t *out, int max_hops, int on_device)
{
    PF_ARG(ctx && req && out && n >= 0 && max_hops > 0, "args");
    pfnav_route_layer *prl = route_layer(ctx, layer);
    PF_ARG(prl, "pfnav_route_build not called");
    const int cw = ctx->chunk_w, chunks = cw * ctx->chunk_h;
    for (int i = 0; i < n; i++) {
        const int32_t *q = req + (size_t)i * 8;
        PF_ARG(q[0] >= 0 && q[0] < chunks && q[3] >= 0 && q[3] < chunks && q[6] >= 0 && q[6] < chunks, "chunk index");
        PF_ARG(q[1] >= 0 && q[1] < 64 && q[2] >= 0 && q[2] < 64 && q[4] >= 0 && q[4] < 64 && q[5] >= 0 && q[5] < 64, "tile");
        PF_ARG(q[7] >= 0 && q[7] < (int)ctx->portals[layer][q[6]].size(), "finish portal");
    }
    const size_t ostride = 4 + 3 * (size_t)max_hops;
    if (!on_device) {
        Router R{ctx, *prl, layer, cw, ctx->chunk_h};
        for (int ch = 0; ch < chunks; ch++) update_edge_states(ctx, *prl, layer, ch);
        parallel_for(n, [&](int i) {          // on host threads, as a batch's search round below the device threshold
            const int32_t *q = req + (size_t)i * 8;
            int32_t *o = out + (size_t)i * ostride;
            memset(o, 0, ostride * 4);
            std::vector<Router::hop> path;
            float cost = 0.0f;
            const tdesc s = {q[0] / cw, q[0] % cw, q[1], q[2]}, e = {q[3] / cw, q[3] % cw, q[4], q[5]};
            if (!R.portal_graph_path(s, e, q[6], q[7], path, &cost)) return;
            o[1] = (int32_t)path.size(); memcpy(&o[2], &cost, 4);
            if ((int)path.size() > max_hops) { o[0] = -1; return; }
            for (size_t k = 0; k < path.size(); k++) { o[4 + 3 * k] = path[k].chunk; o[4 + 3 * k + 1] = path[k].pi; o[4 + 3 * k + 2] = path[k].liid; }
            o[0] = 1;
        });
        return PFNAV_OK;
    }
    PF_NEED_DEVICE(ctx);
    PF_CUDA(cudaSetDevice(ctx->device));
    { int rc = pfnav_blockers_flush(ctx); if (rc) return rc; }
    for (int ch = 0; ch < chunks; ch++) update_edge_states(ctx, *prl, layer, ch);      // n_update_all_edge_states (nav.c:1787)
    return route_dev_search(ctx, layer, *prl, req, n, out, max_hops);
}
