/*
 * oracle/pf_oracle.c -- TEST INFRASTRUCTURE ONLY (see pf_oracle.h).
 *
 * Plain-C restatement of the reference's hot path. Every function cites the reference
 * file:line it follows (paths relative to the reference checkout's src/). Serial, scalar,
 * written for clarity: it is a checker, not a product path. Compile with -ffp-contract=off so
 * float expressions round exactly as the reference's x86-64 SSE build does.
 */
#include "pf_oracle.h"
#include <math.h>
#include <stdbool.h>
#include <stdlib.h>
#include <string.h>

#define RES 64
#define COST_IMPASSABLE 0xff
#define ISLAND_NONE 0xffff
#define TARGET_PORTAL 0
#define TARGET_TILE 1
enum { FD_NONE = 0, FD_NW, FD_N, FD_NE, FD_W, FD_E, FD_SW, FD_S, FD_SE };

/* ------------------------------------------------------------------------------------------
 * lib/public/pqueue.h:109-208 -- 1-indexed binary min-heap, float priority, hole-based sift
 * ---------------------------------------------------------------------------------------- */
typedef struct { float prio; int r, c; } pq_node;
typedef struct { pq_node *nodes; int size, cap; } pq;

static void pq_init(pq *q) { q->nodes = NULL; q->size = 0; q->cap = 0; }
static void pq_free(pq *q) { free(q->nodes); q->nodes = NULL; }

static void pq_push(pq *q, float prio, int r, int c)
{
    if(q->size + 1 >= q->cap) {
        q->cap = q->cap ? q->cap * 2 : 32;
        q->nodes = realloc(q->nodes, q->cap * sizeof(pq_node));
    }
    int curr = q->size + 1, parent = curr / 2;
    while(curr > 1 && q->nodes[parent].prio > prio) {
        q->nodes[curr] = q->nodes[parent];
        curr = parent;
        parent = parent / 2;
    }
    q->nodes[curr].prio = prio; q->nodes[curr].r = r; q->nodes[curr].c = c;
    q->size++;
}

static void pq_pop(pq *q, int *r, int *c)
{
    *r = q->nodes[1].r; *c = q->nodes[1].c;
    q->nodes[1] = q->nodes[q->size--];
    int root = 1;
    while(root != q->size + 1) {        /* _pq_balance */
        int target = q->size + 1;
        int l = root * 2, rr = l + 1;
        if(l <= q->size && q->nodes[l].prio < q->nodes[target].prio) target = l;
        if(rr <= q->size && q->nodes[rr].prio < q->nodes[target].prio) target = rr;
        q->nodes[root] = q->nodes[target];
        root = target;
    }
}

static bool pq_contains(const pq *q, int r, int c)
{
    for(int i = 1; i <= q->size; i++)
        if(q->nodes[i].r == r && q->nodes[i].c == c) return true;
    return false;
}

/* ------------------------------------------------------------------------------------------
 * chunk accessors
 * ---------------------------------------------------------------------------------------- */
static const uint8_t *chunk_cost(const pfo_map *m, int cr, int cc) { return m->cost + ((size_t)cr * m->chunk_w + cc) * 4096; }
static uint16_t chunk_blk(const pfo_map *m, int cr, int cc, int r, int c)
{ return m->blockers ? m->blockers[((size_t)cr * m->chunk_w + cc) * 4096 + r * RES + c] : 0; }
static uint16_t chunk_liid(const pfo_map *m, int cr, int cc, int r, int c)
{ return m->local_islands[((size_t)cr * m->chunk_w + cc) * 4096 + r * RES + c]; }

/* field_tile_passable (navigation/field.c:117) */
static bool tile_passable(const pfo_map *m, int cr, int cc, int r, int c)
{
    if(chunk_cost(m, cr, cc)[r * RES + c] == COST_IMPASSABLE) return false;
    if(chunk_blk(m, cr, cc, r, c) > 0) return false;
    return true;
}

/* field_tile_passable_no_enemies (field.c:179) when the request carries a faction, else field_tile_passable */
static bool tile_passable_f(const pfo_map *m, int faction, int cr, int cc, int r, int c)
{
    if(faction == 0xF || !m->factions) return tile_passable(m, cr, cc, r, c);
    if(chunk_cost(m, cr, cc)[r * RES + c] == COST_IMPASSABLE) return false;
    const uint8_t *fac = m->factions + ((size_t)cr * m->chunk_w + cc) * 15 * 4096;
    const uint16_t enemies = m->enemies[faction & 0xF];
    bool enemies_only = true;
    for(int i = 0; i < 15; i++)
        if(fac[(size_t)i * 4096 + r * RES + c] && !(enemies & (1u << i))) { enemies_only = false; break; }
    if(enemies_only) return true;
    return chunk_blk(m, cr, cc, r, c) == 0;
}

/* field_flow_dir (navigation/field.c:355): note the selection at :405-428 re-tests only equality
 * with min_cost, not the "both side tiles finite" admissibility used to compute min_cost. */
static int flow_dir(const float intf[RES][RES], int r, int c)
{
    float min_cost = INFINITY;
#define MINF(a, b) ((a) < (b) ? (a) : (b))
    if(r > 0) min_cost = MINF(min_cost, intf[r-1][c]);
    if(r < RES-1) min_cost = MINF(min_cost, intf[r+1][c]);
    if(c > 0) min_cost = MINF(min_cost, intf[r][c-1]);
    if(c < RES-1) min_cost = MINF(min_cost, intf[r][c+1]);
    if(r > 0 && c > 0 && intf[r-1][c] < INFINITY && intf[r][c-1] < INFINITY) min_cost = MINF(min_cost, intf[r-1][c-1]);
    if(r > 0 && c < RES-1 && intf[r-1][c] < INFINITY && intf[r][c+1] < INFINITY) min_cost = MINF(min_cost, intf[r-1][c+1]);
    if(r < RES-1 && c > 0 && intf[r+1][c] < INFINITY && intf[r][c-1] < INFINITY) min_cost = MINF(min_cost, intf[r+1][c-1]);
    if(r < RES-1 && c < RES-1 && intf[r+1][c] < INFINITY && intf[r][c+1] < INFINITY) min_cost = MINF(min_cost, intf[r+1][c+1]);
    if(r > 0 && intf[r-1][c] == min_cost) return FD_N;
    else if(r < RES-1 && intf[r+1][c] == min_cost) return FD_S;
    else if(c < RES-1 && intf[r][c+1] == min_cost) return FD_E;
    else if(c > 0 && intf[r][c-1] == min_cost) return FD_W;
    else if(r > 0 && c > 0 && intf[r-1][c-1] == min_cost) return FD_NW;
    else if(r > 0 && c < RES-1 && intf[r-1][c+1] == min_cost) return FD_NE;
    else if(r < RES-1 && c > 0 && intf[r+1][c-1] == min_cost) return FD_SW;
    else if(r < RES-1 && c < RES-1 && intf[r+1][c+1] == min_cost) return FD_SE;
    return 0;
}

/* N_FlowFieldInit + N_FlowFieldUpdate (navigation/field.c:2020-2083) for one request */
static void flow_field_update(const pfo_map *m, const pfo_field_req *q, uint8_t *inout)
{
    if(q->init) memset(inout, FD_NONE, 4096);
    float intf[RES][RES];
    float (*f)[RES] = intf;
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++) f[r][c] = INFINITY;
    pq frontier; pq_init(&frontier);
    const int cr = q->chunk_r, cc = q->chunk_c;

    if(q->target_type == TARGET_TILE) {
        /* field_tile_initial_frontier (field.c:1096) */
        if(tile_passable_f(m, q->faction_id, cr, cc, q->tile_r, q->tile_c)) {
            pq_push(&frontier, 0.0f, q->tile_r, q->tile_c);
            f[q->tile_r][q->tile_c] = 0.0f;
        }
    }else{
        /* field_portal_initial_frontier (field.c:1160) + field_tile_adjacent_to_next_iid (:1131) */
        for(int r = q->port_r0; r <= q->port_r1; r++) {
        for(int c = q->port_c0; c <= q->port_c1; c++) {
            if(!tile_passable_f(m, q->faction_id, cr, cc, r, c)) continue;
            if(q->port_iid != ISLAND_NONE && chunk_liid(m, cr, cc, r, c) != q->port_iid) continue;
            bool adj = false;
            for(int r2 = q->next_r0; r2 <= q->next_r1 && !adj; r2++) {
            for(int c2 = q->next_c0; c2 <= q->next_c1; c2++) {
                int dr = (q->next_chunk_r * RES + r2) - (cr * RES + r);
                int dc = (q->next_chunk_c * RES + c2) - (cc * RES + c);
                if(abs(dr) + abs(dc) == 1 && chunk_liid(m, q->next_chunk_r, q->next_chunk_c, r2, c2) == q->next_iid) {
                    adj = true; break;
                }
            }}
            if(!adj) continue;
            pq_push(&frontier, 0.0f, r, c);
            f[r][c] = 0.0f;
        }}
    }
    /* field_build_integration (field.c:539) with field_neighbours_grid (:203): 4-connected,
     * edge weight = cost_base of the tile entered, accumulated in float */
    const uint8_t *cost = chunk_cost(m, cr, cc);
    while(frontier.size > 0) {
        int r, c; pq_pop(&frontier, &r, &c);
        for(int dr = -1; dr <= 1; dr++) {
        for(int dc = -1; dc <= 1; dc++) {
            int ar = r + dr, ac = c + dc;
            if(ar < 0 || ar >= RES || ac < 0 || ac >= RES) continue;
            if(dr == 0 && dc == 0) continue;
            if(dr == dc || dr == -dc) continue;
            if(!tile_passable_f(m, q->faction_id, cr, cc, ar, ac)) continue;
            float total = f[r][c] + cost[ar * RES + ac];
            if(total < f[ar][ac]) { f[ar][ac] = total; pq_push(&frontier, total, ar, ac); }
        }}
    }
    pq_free(&frontier);
    /* field_build_flow (field.c:734) */
    for(int r = 0; r < RES; r++) {
    for(int c = 0; c < RES; c++) {
        if(f[r][c] == INFINITY) continue;
        if(f[r][c] == 0.0f) { inout[r * RES + c] = FD_NONE; continue; }
        inout[r * RES + c] = (uint8_t)flow_dir((const float(*)[RES])f, r, c);
    }}
    /* field_fixup_portal_edges (field.c:830) */
    if(q->target_type == TARGET_PORTAL) {
        bool up = q->next_chunk_r < cr, down = q->next_chunk_r > cr, left = q->next_chunk_c < cc;
        uint8_t d = up ? FD_N : down ? FD_S : left ? FD_W : FD_E;
        for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++)
            if(f[r][c] == 0.0f) inout[r * RES + c] = d;
    }
}

void pfo_flow_fields_update(const pfo_map *map, const pfo_field_req *reqs, size_t n, uint8_t *inout)
{
    for(size_t i = 0; i < n; i++) flow_field_update(map, &reqs[i], inout + i * 4096);
}

/* ------------------------------------------------------------------------------------------
 * LOS field
 * ---------------------------------------------------------------------------------------- */
typedef struct { uint8_t vis[RES][RES], blk[RES][RES]; } los_t;

/* field_create_wavefront_blocked_line (field.c:463) with M_Tile_Bounds (map/tile.c:356) */
static void blocked_line(const pfo_map *m, const pfo_los_req *q, int r, int c, los_t *out)
{
    float tbx = (m->map_x - (float)(q->tgt_chunk_c * 256)) - (float)(q->tgt_tile_c * 4);
    float tbz = (m->map_z + (float)(q->tgt_chunk_r * 256)) + (float)(q->tgt_tile_r * 4);
    float cbx = (m->map_x - (float)(q->chunk_c * 256)) - (float)(c * 4);
    float cbz = (m->map_z + (float)(q->chunk_r * 256)) + (float)(r * 4);
    float tcx = tbx - 4.0f / 2.0f, tcz = tbz + 4.0f / 2.0f;
    float ccx = cbx - 4.0f / 2.0f, ccz = cbz + 4.0f / 2.0f;
    float sx_ = tcx - ccx, sz_ = tcz - ccz;
    float len = (float)sqrt(sx_ * sx_ + sz_ * sz_);
    sx_ = sx_ / len; sz_ = sz_ / len;
    int dx = abs((int)(sx_ * 1000));
    int dy = -abs((int)(sz_ * 1000));
    int sx = sx_ > 0.0f ? 1 : -1;
    int sy = sz_ < 0.0f ? 1 : -1;
    int err = dx + dy, e2;
    do {
        out->blk[r][c] = 1;
        e2 = 2 * err;
        if(e2 >= dy) { err += dy; c += sx; }
        if(e2 <= dx) { err += dx; r += sy; }
    }while(r >= 0 && r < RES && c >= 0 && c < RES);
}

static bool blocked_or_impass(const pfo_map *m, int cr, int cc, int r, int c) { return !tile_passable(m, cr, cc, r, c); }

/* field_is_los_corner (field.c:435) */
static bool is_los_corner(const pfo_map *m, int cr, int cc, int r, int c)
{
    if(r > 0 && r < RES-1) {
        bool a = blocked_or_impass(m, cr, cc, r-1, c), b = blocked_or_impass(m, cr, cc, r+1, c);
        if(a ^ b) return true;
    }
    if(c > 0 && c < RES-1) {
        bool a = blocked_or_impass(m, cr, cc, r, c-1), b = blocked_or_impass(m, cr, cc, r, c+1);
        if(a ^ b) return true;
    }
    return false;
}

/* N_LOSFieldCreate (field.c:2085) */
static void los_field_create(const pfo_map *m, const pfo_los_req *q, const uint8_t *prev, uint8_t *outb)
{
    los_t out; memset(&out, 0, sizeof(out));
    float intf[RES][RES];
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++) intf[r][c] = INFINITY;
    pq frontier; pq_init(&frontier);
    const int cr = q->chunk_r, cc = q->chunk_c;
    const uint8_t *cost = chunk_cost(m, cr, cc);

    if(cr == q->tgt_chunk_r && cc == q->tgt_chunk_c) {
        pq_push(&frontier, 0.0f, q->tgt_tile_r, q->tgt_tile_c);
        intf[q->tgt_tile_r][q->tgt_tile_c] = 0.0f;
    }else{
        bool horizontal; int curr_edge, prev_edge;
        if(q->prev_chunk_r < cr)      { horizontal = false; curr_edge = 0;     prev_edge = RES-1; }
        else if(q->prev_chunk_r > cr) { horizontal = false; curr_edge = RES-1; prev_edge = 0; }
        else if(q->prev_chunk_c < cc) { horizontal = true;  curr_edge = 0;     prev_edge = RES-1; }
        else                          { horizontal = true;  curr_edge = RES-1; prev_edge = 0; }
        for(int e = 0; e < RES; e++) {
            int r = horizontal ? e : curr_edge, c = horizontal ? curr_edge : e;
            uint8_t pv = horizontal ? prev[e * RES + prev_edge] : prev[prev_edge * RES + e];
            out.vis[r][c] = pv & 1; out.blk[r][c] = (pv >> 1) & 1;
            if(out.blk[r][c]) blocked_line(m, q, r, c, &out);
            if(out.vis[r][c]) { pq_push(&frontier, 0.0f, r, c); intf[r][c] = 0.0f; }
        }
    }
    while(frontier.size > 0) {
        int r, c; pq_pop(&frontier, &r, &c);
        /* field_neighbours_grid_los (field.c:304): the neighbour list -- including the
         * wavefront_blocked filter -- is collected BEFORE any neighbour is processed, so a line drawn
         * while handling an earlier neighbour does not remove a later one from this pop */
        int nbr[4][2], nn = 0;
        for(int dr = -1; dr <= 1; dr++) {
        for(int dc = -1; dc <= 1; dc++) {
            int ar = r + dr, ac = c + dc;
            if(ar < 0 || ar >= RES || ac < 0 || ac >= RES) continue;
            if(dr == 0 && dc == 0) continue;
            if(dr == dc || dr == -dc) continue;
            if(out.blk[ar][ac]) continue;
            nbr[nn][0] = ar; nbr[nn][1] = ac; nn++;
        }}
        for(int i = 0; i < nn; i++) {
        {
            int ar = nbr[i][0], ac = nbr[i][1];
            uint8_t ncost = cost[ar * RES + ac];
            if(!tile_passable_f(m, q->faction_id, cr, cc, ar, ac)) ncost = COST_IMPASSABLE;
            if(ncost > 1) {
                if(!is_los_corner(m, cr, cc, ar, ac)) continue;
                blocked_line(m, q, ar, ac, &out);
            }else{
                float new_cost = intf[r][c] + 1;
                out.vis[ar][ac] = 1;
                if(new_cost < intf[ar][ac]) {
                    intf[ar][ac] = new_cost;
                    if(!pq_contains(&frontier, ar, ac)) pq_push(&frontier, new_cost, ar, ac);
                }
            }
        }}
    }
    pq_free(&frontier);
    /* field_pad_wavefront (field.c:519) */
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++) {
        if(!out.blk[r][c]) continue;
        for(int rr = r-1; rr <= r+1; rr++) for(int c2 = c-1; c2 <= c+1; c2++) {
            if(rr < 0 || rr > RES-1 || c2 < 0 || c2 > RES-1) continue;
            out.vis[rr][c2] = 0;
        }
    }
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++)
        outb[r * RES + c] = (uint8_t)(out.vis[r][c] | (out.blk[r][c] << 1));
}

void pfo_los_fields_create(const pfo_map *map, const pfo_los_req *reqs, size_t n, uint8_t *out)
{
    for(size_t i = 0; i < n; i++) {
        const uint8_t *prev = reqs[i].prev_index >= 0 ? out + (size_t)reqs[i].prev_index * 4096 : NULL;
        los_field_create(map, &reqs[i], prev, out + i * 4096);
    }
}

/* ------------------------------------------------------------------------------------------
 * vec2 (pf_math.c:58-94)
 * ---------------------------------------------------------------------------------------- */
typedef struct { float x, z; } v2;
static v2 v2_add(v2 a, v2 b) { return (v2){a.x + b.x, a.z + b.z}; }
static v2 v2_sub(v2 a, v2 b) { return (v2){a.x - b.x, a.z - b.z}; }
static v2 v2_scale(v2 a, float s) { return (v2){a.x * s, a.z * s}; }
static float v2_dot(v2 a, v2 b) { return a.x * b.x + a.z * b.z; }
static float v2_len(v2 a) { return sqrt(a.x * a.x + a.z * a.z); }
static v2 v2_normal(v2 a) { float l = v2_len(a); return (v2){a.x / l, a.z / l}; }
static v2 v2_truncate(v2 a, float max_len)       /* game/movement.c:643 */
{
    if(v2_len(a) > max_len) { a = v2_normal(a); a = v2_scale(a, max_len); }
    return a;
}

/* ------------------------------------------------------------------------------------------
 * tiles (map/tile.c:547, map/map.c:817-845)
 * ---------------------------------------------------------------------------------------- */
typedef struct { int chunk_r, chunk_c, tile_r, tile_c; } tdesc;
#define CLAMP(a, lo, hi) ((a) < (lo) ? (lo) : (a) > (hi) ? (hi) : (a))

static bool desc_for_point(const pfo_map *m, float px, float pz, tdesc *out)
{
    float width = m->chunk_w * 256.0f, height = m->chunk_h * 256.0f;
    if(px > m->map_x || px < m->map_x - width) return false;
    if(pz < m->map_z || pz > m->map_z + height) return false;
    int chunk_r = fabs(m->map_z - pz) / 256.0f;
    int chunk_c = fabs(m->map_x - px) / 256.0f;
    chunk_r = CLAMP(chunk_r, 0, m->chunk_h - 1);
    chunk_c = CLAMP(chunk_c, 0, m->chunk_w - 1);
    float base_x = m->map_x - (chunk_c * 256.0f);
    float base_z = m->map_z + (chunk_r * 256.0f);
    int tile_r = fabs(base_z - pz) / 4;
    int tile_c = fabs(base_x - px) / 4;
    out->chunk_r = chunk_r; out->chunk_c = chunk_c;
    out->tile_r = CLAMP(tile_r, 0, RES-1); out->tile_c = CLAMP(tile_c, 0, RES-1);
    return true;
}

static void probe(const pfo_map *m, float px, float pz, bool *pathable, bool *blocked)
{
    tdesc t; *pathable = false; *blocked = false;
    if(!desc_for_point(m, px, pz, &t)) return;
    *pathable = chunk_cost(m, t.chunk_r, t.chunk_c)[t.tile_r * RES + t.tile_c] != COST_IMPASSABLE;
    *blocked = chunk_blk(m, t.chunk_r, t.chunk_c, t.tile_r, t.tile_c) > 0;
}

static v2 flow_dir_vec(int dir)     /* N_FlowDir (navigation/field.c:2429) */
{
    float d = 1.0f / sqrt(2.0f);
    switch(dir) {
    case FD_NW: return (v2){d, -d};   case FD_N: return (v2){0.0f, -1.0f}; case FD_NE: return (v2){-d, -d};
    case FD_W:  return (v2){1.0f, 0.0f}; case FD_E: return (v2){-1.0f, 0.0f};
    case FD_SW: return (v2){d, d};    case FD_S: return (v2){0.0f, 1.0f};  case FD_SE: return (v2){-d, d};
    default: return (v2){0.0f, 0.0f};
    }
}

/* N_DesiredPointSeekVelocity happy path + n_interpolated_flow_dir (navigation/nav.c:3468, 3407)
 * and N_HasDestLOS (nav.c:4026); the n_request_path-on-miss branches are the host planner's job. */
void pfo_desired_velocity(const pfo_map *m, const pfo_agent *agents, const pfo_flock *flocks,
                          const uint32_t *work, size_t nwork, const int32_t *slot,
                          const uint8_t *flow, const uint8_t *los, float *out_vdes, uint8_t *out_los)
{
    const int chunks = m->chunk_w * m->chunk_h;
    for(size_t w = 0; w < nwork; w++) {
        const pfo_agent *a = &agents[work[w]];
        v2 vdes = {0.0f, 0.0f}; uint8_t l = 0;
        int dest = a->flock >= 0 ? flocks[a->flock].dest : -1;
        if(dest >= 0) {
            const int32_t *sl = slot + (size_t)dest * chunks;
            tdesc t;
            if(los && desc_for_point(m, a->prev_pos[0], a->prev_pos[1], &t)) {
                int s = sl[t.chunk_r * m->chunk_w + t.chunk_c];
                if(s >= 0) l = los[(size_t)s * 4096 + t.tile_r * RES + t.tile_c] & 1;
            }
            if(desc_for_point(m, a->pos[0], a->pos[1], &t)) {
                int s = sl[t.chunk_r * m->chunk_w + t.chunk_c];
                if(s >= 0) {
                    const uint8_t *base_ff = flow + (size_t)s * 4096;
                    int base_dir = base_ff[t.tile_r * RES + t.tile_c] & 0xf;
                    float bx = (m->map_x - (float)(t.chunk_c * 256)) - (float)(t.tile_c * 4);
                    float bz = (m->map_z + (float)(t.chunk_r * 256)) + (float)(t.tile_r * 4);
                    float cx = bx - 4.0f / 2.0f, cz = bz + 4.0f / 2.0f;
                    float dx = a->pos[0] - cx, dz = a->pos[1] - cz;
                    int dc = (dx < 0.0f) ? 1 : -1, dr = (dz > 0.0f) ? 1 : -1;
                    float wc = fmin(fabs(dx) / 4.0f, 1.0f), wr = fmin(fabs(dz) / 4.0f, 1.0f);
                    const int sdc[4] = {0, dc, 0, dc}, sdr[4] = {0, 0, dr, dr};
                    const float sw[4] = {(1.0f - wc) * (1.0f - wr), wc * (1.0f - wr), (1.0f - wc) * wr, wc * wr};
                    v2 acc = {0.0f, 0.0f}; float wsum = 0.0f;
                    for(int i = 0; i < 4; i++) {
                        if(sw[i] <= 0.0f) continue;
                        int ar = t.chunk_r * RES + t.tile_r + sdr[i], ac = t.chunk_c * RES + t.tile_c + sdc[i];
                        if(ar < 0 || ar >= m->chunk_h * RES || ac < 0 || ac >= m->chunk_w * RES) continue;
                        const uint8_t *ff = base_ff;
                        if(ar / RES != t.chunk_r || ac / RES != t.chunk_c) {
                            int s2 = sl[(ar / RES) * m->chunk_w + ac / RES];
                            if(s2 < 0) continue;
                            ff = flow + (size_t)s2 * 4096;
                        }
                        int dir = ff[(ar % RES) * RES + ac % RES] & 0xf;
                        if(dir == FD_NONE) continue;
                        acc = v2_add(acc, v2_scale(flow_dir_vec(dir), sw[i]));
                        wsum += sw[i];
                    }
                    if(wsum < 1e-6f || v2_len(acc) < 1e-6f) vdes = flow_dir_vec(base_dir);
                    else vdes = v2_normal(acc);
                }
            }
        }
        out_vdes[2*w] = vdes.x; out_vdes[2*w+1] = vdes.z;
        if(out_los) out_los[w] = l;
    }
}

/* ------------------------------------------------------------------------------------------
 * position index (lib/public/bitmap_grid.h; game/position.c:264, 359, 379)
 * ---------------------------------------------------------------------------------------- */
struct pfo_world {
    pfo_map map;
    const pfo_agent *agents; size_t n;
    const pfo_flock *flocks; size_t nflocks;
    int hz;
    int grid_w, grid_h; int32_t origin_x, origin_y;
    uint32_t *cell_start;        /* [ncells+1] */
    uint32_t *sid; int32_t *six, *siy;
    uint32_t *flock_start, *flock_members;
    const pfo_formation *forms;          /* per uid, may be NULL */
    const pfo_movestate_ext *exts;       /* per uid, may be NULL */
};

void pfo_world_set_states(pfo_world *w, const pfo_formation *forms, const pfo_movestate_ext *exts)
{
    w->forms = forms; w->exts = exts;
}

static int32_t bg_scale(float x) { return (int32_t)lrintf(x * 256.0f); }
static int cell_of(int32_t i, int32_t origin, int n) { int c = (i - origin) >> 12; return c < 0 ? 0 : c >= n ? n - 1 : c; }

pfo_world *pfo_world_create(const pfo_map *map, const pfo_agent *agents, size_t n,
                            const pfo_flock *flocks, size_t nflocks, int hz)
{
    pfo_world *w = calloc(1, sizeof(*w));
    w->map = *map; w->agents = agents; w->n = n; w->flocks = flocks; w->nflocks = nflocks; w->hz = hz;
    float W = map->chunk_w * 256.0f, H = map->chunk_h * 256.0f;
    float cx = map->map_x - W / 2.0f, cz = map->map_z + H / 2.0f;
    float xmin = cx - W / 2.0f, xmax = cx + W / 2.0f, zmin = cz - H / 2.0f, zmax = cz + H / 2.0f;
    w->origin_x = bg_scale(xmin); w->origin_y = bg_scale(zmin);
    int32_t span_x = bg_scale(xmax) - w->origin_x, span_y = bg_scale(zmax) - w->origin_y;
    w->grid_w = (int)(((uint32_t)span_x + 4095u) >> 12); if(w->grid_w < 1) w->grid_w = 1;
    w->grid_h = (int)(((uint32_t)span_y + 4095u) >> 12); if(w->grid_h < 1) w->grid_h = 1;
    size_t ncells = (size_t)w->grid_w * w->grid_h;
    w->cell_start = calloc(ncells + 1, 4);
    w->sid = malloc((n ? n : 1) * 4); w->six = malloc((n ? n : 1) * 4); w->siy = malloc((n ? n : 1) * 4);
    uint32_t *cnt = calloc(ncells + 1, 4);
    for(size_t i = 0; i < n; i++) {
        int c = cell_of(bg_scale(agents[i].pos[1]), w->origin_y, w->grid_h) * w->grid_w
              + cell_of(bg_scale(agents[i].pos[0]), w->origin_x, w->grid_w);
        cnt[c]++;
    }
    for(size_t c = 0; c < ncells; c++) w->cell_start[c + 1] = w->cell_start[c] + cnt[c];
    memset(cnt, 0, (ncells + 1) * 4);
    /* insert in uid order then bg_cleanup: each cell holds its members in DESCENDING uid order
     * (LIFO overflow chain, bitmap_grid.h:1110-1130, 1477-1540) */
    for(size_t k = n; k-- > 0;) {
        int c = cell_of(bg_scale(agents[k].pos[1]), w->origin_y, w->grid_h) * w->grid_w
              + cell_of(bg_scale(agents[k].pos[0]), w->origin_x, w->grid_w);
        uint32_t slot = w->cell_start[c] + cnt[c]++;
        w->sid[slot] = (uint32_t)k; w->six[slot] = bg_scale(agents[k].pos[0]); w->siy[slot] = bg_scale(agents[k].pos[1]);
    }
    free(cnt);
    w->flock_start = calloc(nflocks + 1, 4); w->flock_members = malloc((n ? n : 1) * 4);
    for(size_t i = 0; i < n; i++) if(agents[i].flock >= 0) w->flock_start[agents[i].flock + 1]++;
    for(size_t f = 0; f < nflocks; f++) w->flock_start[f + 1] += w->flock_start[f];
    uint32_t *cur = malloc((nflocks + 1) * 4); memcpy(cur, w->flock_start, (nflocks + 1) * 4);
    for(size_t i = 0; i < n; i++) if(agents[i].flock >= 0) w->flock_members[cur[agents[i].flock]++] = (uint32_t)i;
    free(cur);
    return w;
}

void pfo_world_destroy(pfo_world *w)
{
    if(!w) return;
    free(w->cell_start); free(w->sid); free(w->six); free(w->siy); free(w->flock_start); free(w->flock_members);
    free(w);
}

/* bg_ent_inrange_circle (bitmap_grid.h:1376) */
static int bg_inrange_circle(const pfo_world *w, float x, float z, float range, uint32_t *out, int maxout)
{
    if(maxout <= 0 || range < 0.0f) return 0;
    int32_t icx = bg_scale(x), icy = bg_scale(z), ir = bg_scale(range);
    int64_t ir2 = (int64_t)ir * ir;
    int32_t imnx = icx - ir, imxx = icx + ir, imny = icy - ir, imxy = icy + ir;
    if(imxx < w->origin_x || imxy < w->origin_y) return 0;
    if(imnx >= w->origin_x + (w->grid_w << 12) || imny >= w->origin_y + (w->grid_h << 12)) return 0;
    int cx_lo = (imnx - w->origin_x) >> 12, cx_hi = (imxx - w->origin_x) >> 12;
    int cy_lo = (imny - w->origin_y) >> 12, cy_hi = (imxy - w->origin_y) >> 12;
    if(cx_lo < 0) cx_lo = 0; if(cy_lo < 0) cy_lo = 0;
    if(cx_hi >= w->grid_w) cx_hi = w->grid_w - 1; if(cy_hi >= w->grid_h) cy_hi = w->grid_h - 1;
    int written = 0;
    int64_t extent = (int64_t)(cx_hi - cx_lo + 1) * (cy_hi - cy_lo + 1), total = (int64_t)w->grid_w * w->grid_h;
    if(extent * 4 >= total * 3) {       /* wide query: whole pool in pool order */
        for(size_t i = 0; i < w->n; i++) {
            int64_t dx = (int64_t)w->six[i] - icx, dy = (int64_t)w->siy[i] - icy;
            if(dx * dx + dy * dy <= ir2) { out[written++] = w->sid[i]; if(written >= maxout) return maxout; }
        }
        return written;
    }
    for(int cyc = cy_lo >> 3; cyc <= cy_hi >> 3; cyc++) {
    for(int cxc = cx_lo >> 3; cxc <= cx_hi >> 3; cxc++) {
        int fy0 = cyc * 8, fy1 = fy0 + 8, fx0 = cxc * 8, fx1 = fx0 + 8;
        if(fy0 < cy_lo) fy0 = cy_lo; if(fy1 > cy_hi + 1) fy1 = cy_hi + 1;
        if(fx0 < cx_lo) fx0 = cx_lo; if(fx1 > cx_hi + 1) fx1 = cx_hi + 1;
        for(int fy = fy0; fy < fy1; fy++) {
        for(int fx = fx0; fx < fx1; fx++) {
            int c = fy * w->grid_w + fx;
            for(uint32_t i = w->cell_start[c]; i < w->cell_start[c + 1]; i++) {
                int64_t dx = (int64_t)w->six[i] - icx, dy = (int64_t)w->siy[i] - icy;
                if(dx * dx + dy * dy <= ir2) { out[written++] = w->sid[i]; if(written >= maxout) return maxout; }
            }
        }}
    }}
    return written;
}

/* G_Pos_EntsInCircleFrom (position.c:379): the raw grid query, then filter_garrisoned
 * (position.c:100-119) -- a swap-remove from the back, which REORDERS the survivors. */
#define FLAG_GARRISONED_Q (1u << 18)
int pfo_ents_in_circle(const pfo_world *w, float x, float z, float range, uint32_t *out, int maxout)
{
    int count = bg_inrange_circle(w, x, z, range, out, maxout);
    int ret = count;
    for(int i = count - 1; i >= 0; i--) {
        if(w->agents[out[i]].flags & FLAG_GARRISONED_Q) {
            out[i] = out[ret - 1];
            ret--;
        }
    }
    return ret;
}

/* ------------------------------------------------------------------------------------------
 * ClearPath (game/clearpath.c) + line intersections (phys/collision.c:820-875)
 * ---------------------------------------------------------------------------------------- */
#define EPSILON (1.0 / 1024)
#define EPSILON_F (1.0f / 1024)
#define MAX_NEIGHBOURS 32
typedef struct { v2 point, dir; } line2;
typedef struct { v2 pos, vel; float radius; } cpent;

static bool infinite_line_isect(line2 l1, line2 l2, v2 *out)      /* collision.c:820 */
{
    float s1 = fabs(l1.dir.x) < EPSILON_F ? NAN : (l1.dir.z / l1.dir.x);
    float s2 = fabs(l2.dir.x) < EPSILON_F ? NAN : (l2.dir.z / l2.dir.x);
    if(isnan(s1) && isnan(s2)) return false;
    if(fabs(s1 - s2) < EPSILON_F) return false;
    if(isnan(s1) && !isnan(s2)) {
        out->x = l1.point.x;
        out->z = (l1.point.x - l2.point.x) * s2 + l2.point.z;
    }else if(!isnan(s1) && isnan(s2)) {
        out->x = l2.point.x;
        out->z = (l2.point.x - l1.point.x) * s1 + l2.point.z;     /* sic: l2.point (collision.c:839-840) */
    }else{
        out->x = (s1 * l1.point.x - s2 * l2.point.x + l2.point.z - l1.point.z) / (s1 - s2);
        out->z = s2 * (out->x - l2.point.x) + l2.point.z;
    }
    return true;
}

static bool ray_ray_isect(line2 l1, line2 l2, v2 *out)            /* collision.c:854 */
{
    v2 p;
    if(!infinite_line_isect(l1, l2, &p)) return false;
    if((p.x - l1.point.x) / l1.dir.x < 0.0f) return false;
    if((p.z - l1.point.z) / l1.dir.z < 0.0f) return false;
    if((p.x - l2.point.x) / l2.dir.x < 0.0f) return false;
    if((p.z - l2.point.z) / l2.dir.z < 0.0f) return false;
    *out = p;
    return true;
}

static bool inside_pcr(const line2 *rays, int n_rays, v2 test)    /* clearpath.c:249 */
{
    for(int i = 0; i < n_rays; i += 2) {
        v2 ptt = v2_sub(test, rays[i].point);
        if(v2_len(ptt) < EPSILON) continue;
        ptt = v2_normal(ptt);
        float left_det = (ptt.z * rays[i].dir.x) - (ptt.x * rays[i].dir.z);
        if(left_det < EPSILON) continue;
        ptt = v2_sub(test, rays[i+1].point);
        if(v2_len(ptt) < EPSILON) continue;
        ptt = v2_normal(ptt);
        float right_det = (ptt.z * rays[i+1].dir.x) - (ptt.x * rays[i+1].dir.z);
        if(right_det > -EPSILON) continue;
        return true;
    }
    return false;
}

static void vo_edges(cpent ent, cpent nb, v2 *right, v2 *left)    /* clearpath.c:130 */
{
    v2 e2n = v2_normal(v2_sub(nb.pos, ent.pos));
    v2 r = {-e2n.z, e2n.x};
    r = v2_scale(r, nb.radius + ent.radius + 0.0f);
    v2 rt = v2_add(nb.pos, r), lt = v2_sub(nb.pos, r);
    *right = v2_normal(v2_sub(rt, ent.pos));
    *left = v2_normal(v2_sub(lt, ent.pos));
}

/* clearpath_new_velocity (clearpath.c:552) */
static bool clearpath_new_velocity(cpent ent, v2 des_v, const cpent *dyn, int ndyn, const cpent *stat, int nstat, v2 *out)
{
    line2 rays[4 * MAX_NEIGHBOURS];
    int n_rays = 0;
    for(int i = 0; i < ndyn; i++) {     /* compute_all_hrvos :232 -> compute_hrvo :174 */
        cpent nb = dyn[i];
        if(v2_len(v2_sub(nb.pos, ent.pos)) < EPSILON) continue;
        v2 right, left; vo_edges(ent, nb, &right, &left);
        v2 rvo_apex = v2_add(ent.pos, v2_scale(v2_add(ent.vel, nb.vel), 0.5f));
        v2 centerline = v2_add(left, right);
        v2 vo_apex = v2_add(ent.pos, nb.vel);
        float det = (centerline.x * ent.vel.z) - (centerline.z * ent.vel.x);
        v2 apex = rvo_apex, p;
        if(det > EPSILON) { if(infinite_line_isect((line2){rvo_apex, left}, (line2){vo_apex, right}, &p)) apex = p; }
        else if(det < -EPSILON) { if(infinite_line_isect((line2){rvo_apex, right}, (line2){vo_apex, left}, &p)) apex = p; }
        rays[n_rays++] = (line2){apex, left};
        rays[n_rays++] = (line2){apex, right};
    }
    for(int i = 0; i < nstat; i++) {    /* compute_all_vos :216 */
        cpent nb = stat[i];
        if(v2_len(v2_sub(nb.pos, ent.pos)) < EPSILON) continue;
        v2 right, left; vo_edges(ent, nb, &right, &left);
        v2 apex = v2_add(ent.pos, nb.vel);
        rays[n_rays++] = (line2){apex, left};
        rays[n_rays++] = (line2){apex, right};
    }
    v2 des_v_ws = v2_add(ent.pos, des_v);
    if(!inside_pcr(rays, n_rays, des_v_ws)) { *out = des_v; return true; }
    /* compute_vo_xpoints :321, compute_vdes_proj_points :344, compute_vnew :368 (fused) */
    float min_dist = INFINITY; v2 ret = {0.0f, 0.0f}; int npoints = 0;
    for(int i = 0; i < n_rays; i++) for(int j = 0; j < n_rays; j++) {
        if(i == j) continue;
        v2 p;
        if(!ray_ray_isect(rays[i], rays[j], &p)) continue;
        if(inside_pcr(rays, n_rays, p)) continue;
        npoints++;
        v2 curr = v2_sub(p, ent.pos); float len = v2_len(v2_sub(des_v, curr));
        if(len < min_dist) { min_dist = len; ret = curr; }
    }
    for(int i = 0; i < n_rays; i++) {
        float len = v2_dot(rays[i].dir, des_v);
        v2 proj = v2_add(rays[i].point, v2_scale(rays[i].dir, len));
        if(inside_pcr(rays, n_rays, proj)) continue;
        npoints++;
        v2 curr = v2_sub(proj, ent.pos); float l2 = v2_len(v2_sub(des_v, curr));
        if(l2 < min_dist) { min_dist = l2; ret = curr; }
    }
    if(npoints == 0) return false;
    *out = ret;
    return true;
}

/* G_ClearPath_NewVelocity (clearpath.c:694) incl. remove_furthest (:390) */
static v2 clearpath(cpent ent, v2 des_v, cpent *dyn, int ndyn, cpent *stat, int nstat)
{
    do {
        v2 ret;
        if(clearpath_new_velocity(ent, des_v, dyn, ndyn, stat, nstat, &ret)) return ret;
        float max_dist = -INFINITY; int which = -1, idx = -1;
        for(int j = 0; j < ndyn; j++) { float l = v2_len(v2_sub(ent.pos, dyn[j].pos)); if(l > max_dist) { max_dist = l; which = 0; idx = j; } }
        for(int j = 0; j < nstat; j++) { float l = v2_len(v2_sub(ent.pos, stat[j].pos)); if(l > max_dist) { max_dist = l; which = 1; idx = j; } }
        if(which == 0) dyn[idx] = dyn[--ndyn];
        else if(which == 1) stat[idx] = stat[--nstat];
    }while(ndyn > 0 && nstat > 0);
    return (v2){0.0f, 0.0f};
}

void pfo_clearpath(const float *self5, const float *vpref2, const float *dyn5, int ndyn, const float *stat5, int nstat,
                   float max_len, float *out2)
{
    cpent self = {{self5[0], self5[1]}, {self5[2], self5[3]}, self5[4]};
    cpent dyn[MAX_NEIGHBOURS], stat[MAX_NEIGHBOURS];
    for(int i = 0; i < ndyn; i++) dyn[i] = (cpent){{dyn5[5*i], dyn5[5*i+1]}, {dyn5[5*i+2], dyn5[5*i+3]}, dyn5[5*i+4]};
    for(int i = 0; i < nstat; i++) stat[i] = (cpent){{stat5[5*i], stat5[5*i+1]}, {stat5[5*i+2], stat5[5*i+3]}, stat5[5*i+4]};
    v2 nv = v2_truncate(clearpath(self, (v2){vpref2[0], vpref2[1]}, dyn, ndyn, stat, nstat), max_len);
    out2[0] = nv.x; out2[1] = nv.z;
}

void pfo_inside_pcr(const float *rays4, int n_rays, const float *pts2, long n, uint8_t *out)
{
    line2 rays[4 * MAX_NEIGHBOURS];
    for(int i = 0; i < n_rays; i++) rays[i] = (line2){{rays4[4*i], rays4[4*i+1]}, {rays4[4*i+2], rays4[4*i+3]}};
    for(long i = 0; i < n; i++) out[i] = inside_pcr(rays, n_rays, (v2){pts2[2*i], pts2[2*i+1]});
}

void pfo_line_isect(const float *lines4, long n, float *out3)
{
    for(long i = 0; i < n; i++) {
        const float *l = lines4 + 8 * i;
        v2 p = {0.0f, 0.0f};
        bool ok = infinite_line_isect((line2){{l[0], l[1]}, {l[2], l[3]}}, (line2){{l[4], l[5]}, {l[6], l[7]}}, &p);
        out3[3*i] = ok ? 1.0f : 0.0f; out3[3*i+1] = p.x; out3[3*i+2] = p.z;
    }
}

/* ------------------------------------------------------------------------------------------
 * move_velocity_work (game/movement.c:3395): the state picks the steering variant (movement.c:3414-3448)
 *   STATE_TURNING                  no preferred velocity, ClearPath only
 *   STATE_SEEK_ENEMIES             enemy_seek_vpref (movement.c:1946)
 *   STATE_ARRIVING_TO_CELL         cell_arrival_seek_vpref (movement.c:1908)
 *   STATE_MOVING_IN_FORMATION      formation_seek_vpref (movement.c:1985)
 *   every other state              point_seek_vpref (movement.c:1870)
 * The formation variants read struct formation_state (movement.c:215-225); an entity without an assignment stands
 * still (movement.c:3426, 3438) and a formation drag caps the speed at 75 % (movement.c:1940, 2017).
 * The variants beyond point_seek_vpref are NOT an independent restatement: they were written without a reference
 * checkout and follow k_agent_velocity (pfnav_agents.cu); they stay unpinned until tests/test_oracle.py's
 * test_port_all_states_vs_ref runs against oracle/_ref (tests/golden/README.md).
 * ---------------------------------------------------------------------------------------- */
#define FLAG_MOVABLE (1u << 3)
#define FLAG_AIR (1u << 15)
#define FLAG_COMBAT_HELD (1u << 21)
#define STATE_MOVING_IN_FORMATION 1
#define STATE_ARRIVED 2
#define STATE_SEEK_ENEMIES 3
#define STATE_WAITING 4
#define STATE_TURNING 7
#define STATE_ARRIVING_TO_CELL 8
#define FORM_HAS_FORMATION (1u << 0)
#define FORM_ASSIGNMENT_READY (1u << 1)
#define FORM_ASSIGNED_TO_CELL (1u << 2)
#define FORM_IN_RANGE_OF_CELL (1u << 3)
#define FORM_ARRIVED_AT_CELL (1u << 4)
#define CELL_ARRIVAL_RADIUS 30.0f           /* movement.c:1769 */
#define MOVE_ARRIVE_FORCE_SCALE 0.5f
#define MOVE_COHESION_FORCE_SCALE 0.15f
#define MOVE_SEPARATION_FORCE_SCALE 0.6f
#define MOVE_ALIGN_FORCE_SCALE 0.15f

typedef struct {                    /* what the steering functions of one work item read */
    const pfo_world *w;
    const pfo_agent *a;
    uint32_t uid;
    v2 pos, velocity, vdes;
    float smf; double smf_d;
    pfo_formation fs;               /* zero when the world has no formation table */
} steer_in;

/* separation_force (movement.c:1690) */
static v2 separation_force(const steer_in *s)
{
    uint32_t near_ents[128];
    int num_near = pfo_ents_in_circle(s->w, s->pos.x, s->pos.z, 30.0f, near_ents, 128);
    v2 separation = {0.0f, 0.0f};
    for(int i = 0; i < num_near; i++) {
        uint32_t curr = near_ents[i];
        const pfo_agent *o = &s->w->agents[curr];
        if(curr == s->uid) continue;
        if(!(o->flags & FLAG_MOVABLE)) continue;
        if((s->a->flags & FLAG_AIR) != (o->flags & FLAG_AIR)) continue;
        v2 diff = v2_sub((v2){o->pos[0], o->pos[1]}, s->pos);
        float radius = s->a->radius + o->radius + 0.0f;
        if(v2_len(diff) < EPSILON_F) continue;
        float t = (v2_len(diff) - radius * 0.85f) / v2_len(diff);
        float mt = -20.0f * t;
        float scale = exp(mt < 40.0f ? mt : 40.0f);
        separation = v2_add(separation, v2_scale(diff, scale));
    }
    if(num_near == 0) return (v2){0.0f, 0.0f};
    separation = v2_scale(separation, -1.0f);
    return v2_truncate(separation, s->smf);
}

/* arrive_force_point (movement.c:1546) */
static v2 arrive_force_point(const steer_in *s)
{
    const pfo_agent *a = s->a;
    const int hz = s->w->hz;
    v2 target = a->flock >= 0 ? (v2){s->w->flocks[a->flock].target[0], s->w->flocks[a->flock].target[1]} : s->pos;
    v2 desired;
    if(a->has_dest_los) {
        desired = v2_sub(target, s->pos);
        float distance = v2_len(desired);
        desired = v2_normal(desired);
        desired = v2_scale(desired, a->max_speed / hz);
        if(distance < 10.0f) desired = v2_scale(desired, distance / 10.0f);
    }else desired = v2_scale(s->vdes, a->max_speed / hz);
    return v2_truncate(v2_sub(desired, s->velocity), s->smf);
}

/* arrive_force_cell (movement.c:1571): the desired velocity itself, not a correction of the current one */
static v2 arrive_force_cell(const steer_in *s)
{
    v2 desired = v2_sub((v2){s->fs.cell_pos[0], s->fs.cell_pos[1]}, s->pos);
    float distance = v2_len(desired);
    if(distance < 10.0f) return v2_scale(desired, distance / 10.0f);
    return v2_scale(s->vdes, s->a->max_speed / s->w->hz);
}

/* arrive_force_enemies (movement.c:1593) */
static v2 arrive_force_enemies(const steer_in *s)
{
    v2 desired = v2_scale(s->vdes, s->a->max_speed / s->w->hz);
    return v2_truncate(v2_sub(desired, s->velocity), s->smf);
}

/* cohesion_force (movement.c:1653), flock members in ascending uid */
static v2 cohesion_force(const steer_in *s)
{
    const pfo_world *w = s->w;
    const int32_t flock = s->a->flock;
    if(flock < 0) return (v2){0.0f, 0.0f};
    v2 com = {0.0f, 0.0f}; size_t cnt = 0;
    for(uint32_t k = w->flock_start[flock]; k < w->flock_start[flock + 1]; k++) {
        uint32_t cu = w->flock_members[k];
        if(cu == s->uid) continue;
        v2 cp = {w->agents[cu].pos[0], w->agents[cu].pos[1]};
        v2 diff = v2_sub(cp, s->pos);
        float t = (v2_len(diff) - 50.0f * 0.75) / 50.0f;
        float scale = exp(-6.0f * t);
        com = v2_add(com, v2_scale(cp, scale));
        cnt++;
    }
    if(!cnt) return (v2){0.0f, 0.0f};
    com = v2_scale(com, 1.0f / cnt);
    return v2_truncate(v2_sub(com, s->pos), s->smf);
}

/* nullify_impass_components (movement.c:1831): the tile probes a steering force may not point into */
typedef struct { bool on_blocked, lp, lb, rp, rb, tp, tb, bp, bb; } impass_probes;
static impass_probes impass_probe(const pfo_map *m, v2 pos)
{
    impass_probes q; bool d0;
    probe(m, pos.x, pos.z, &d0, &q.on_blocked);
    probe(m, pos.x + 4.0f, pos.z, &q.lp, &q.lb); probe(m, pos.x - 4.0f, pos.z, &q.rp, &q.rb);
    probe(m, pos.x, pos.z + 4.0f, &q.tp, &q.tb); probe(m, pos.x, pos.z - 4.0f, &q.bp, &q.bb);
    return q;
}
static v2 nullify_impass_components(const impass_probes *q, v2 f)
{
    if(f.x > 0 && (!q->lp || (!q->on_blocked && q->lb))) f.x = 0.0f;
    if(f.x < 0 && (!q->rp || (!q->on_blocked && q->rb))) f.x = 0.0f;
    if(f.z > 0 && (!q->tp || (!q->on_blocked && q->tb))) f.z = 0.0f;
    if(f.z < 0 && (!q->bp || (!q->on_blocked && q->bb))) f.z = 0.0f;
    return f;
}

/* the shared tail of point_seek_vpref / cell_arrival_seek_vpref / formation_seek_vpref (movement.c:1870-1905,
 * 1908-1944, 1985-2021): the total force first, then separation alone, then arrival alone, each with its impassable
 * components removed, until one is longer than 1 % of SCALED_MAX_FORCE (a double comparison, movement.c:1895) */
static v2 prioritized_vpref(const steer_in *s, v2 total, v2 separation, v2 arrive)
{
    const impass_probes q = impass_probe(&s->w->map, s->pos);
    const v2 forces[3] = {total, separation, arrive};
    v2 steer = {0.0f, 0.0f};
    for(int prio = 0; prio < 3; prio++) {
        steer = nullify_impass_components(&q, forces[prio]);
        if(v2_len(steer) > s->smf_d * 0.01) break;
    }
    v2 accel = v2_scale(steer, 1.0f / 1.0f);
    return v2_truncate(v2_add(s->velocity, accel), s->a->speed / s->w->hz);
}

/* formation_vpref_limits: the drag cap (movement.c:1940, 2017), then no motion without an assignment (:3426, :3438) */
static v2 formation_vpref_limits(const steer_in *s, v2 vpref)
{
    if(v2_len((v2){s->fs.drag[0], s->fs.drag[1]}) > EPSILON_F)
        vpref = v2_truncate(vpref, (float)(((double)s->a->speed * 0.75) / (double)s->w->hz));
    if(!(s->fs.flags & FORM_ASSIGNMENT_READY)) vpref = (v2){0.0f, 0.0f};
    return vpref;
}

/* point_seek_vpref (movement.c:1870) with point_seek_total_force (:1745) */
static v2 point_seek_vpref(const steer_in *s)
{
    v2 separation = separation_force(s), arrive = arrive_force_point(s), cohesion = cohesion_force(s);
    v2 ret = {0.0f, 0.0f};
    ret = v2_add(ret, v2_scale(arrive, MOVE_ARRIVE_FORCE_SCALE));
    ret = v2_add(ret, v2_scale(separation, MOVE_SEPARATION_FORCE_SCALE));
    ret = v2_add(ret, v2_scale(cohesion, MOVE_COHESION_FORCE_SCALE));
    return prioritized_vpref(s, v2_truncate(ret, s->smf), separation, arrive);
}

/* formation_seek_vpref (movement.c:1985) with formation_point_seek_total_force (:1960): the formation's own cohesion
 * force in the place of the flock's */
static v2 formation_seek_vpref(const steer_in *s)
{
    v2 separation = separation_force(s), arrive = arrive_force_point(s);
    v2 cohesion = {s->fs.cohesion[0], s->fs.cohesion[1]};
    v2 ret = {0.0f, 0.0f};
    ret = v2_add(ret, v2_scale(arrive, MOVE_ARRIVE_FORCE_SCALE));
    ret = v2_add(ret, v2_scale(separation, MOVE_SEPARATION_FORCE_SCALE));
    ret = v2_add(ret, v2_scale(cohesion, MOVE_COHESION_FORCE_SCALE));
    return formation_vpref_limits(s, prioritized_vpref(s, v2_truncate(ret, s->smf), separation, arrive));
}

/* cell_arrival_seek_vpref (movement.c:1908) with cell_seek_total_force (:1769): cohesion and alignment only while the
 * cell is farther than CELL_ARRIVAL_RADIUS */
static v2 cell_arrival_seek_vpref(const steer_in *s)
{
    v2 separation = separation_force(s), arrive = arrive_force_cell(s);
    v2 ret = {0.0f, 0.0f};
    ret = v2_add(ret, v2_scale(arrive, MOVE_ARRIVE_FORCE_SCALE));
    ret = v2_add(ret, v2_scale(separation, MOVE_SEPARATION_FORCE_SCALE));
    if(v2_len(v2_sub((v2){s->fs.cell_pos[0], s->fs.cell_pos[1]}, s->pos)) > CELL_ARRIVAL_RADIUS) {
        ret = v2_add(ret, v2_scale((v2){s->fs.cohesion[0], s->fs.cohesion[1]}, MOVE_COHESION_FORCE_SCALE));
        ret = v2_add(ret, v2_scale((v2){s->fs.align[0], s->fs.align[1]}, MOVE_ALIGN_FORCE_SCALE));
    }
    return formation_vpref_limits(s, prioritized_vpref(s, v2_truncate(ret, s->smf), separation, arrive));
}

/* enemy_seek_vpref (movement.c:1946) with enemy_seek_total_force (:1801): arrival and separation, no cohesion, no
 * impassable-component pass and no fall-backs */
static v2 enemy_seek_vpref(const steer_in *s)
{
    v2 separation = separation_force(s), arrive = arrive_force_enemies(s);
    v2 ret = {0.0f, 0.0f};
    ret = v2_add(ret, v2_scale(arrive, MOVE_ARRIVE_FORCE_SCALE));
    ret = v2_add(ret, v2_scale(separation, MOVE_SEPARATION_FORCE_SCALE));
    v2 accel = v2_scale(v2_truncate(ret, s->smf), 1.0f / 1.0f);
    return v2_truncate(v2_add(s->velocity, accel), s->a->speed / s->w->hz);
}

void pfo_velocity_work(const pfo_world *w, const uint32_t *work, size_t nwork, float *out_vel, float *out_vpref)
{
    const int hz = w->hz;
    /* SCALED_MAX_FORCE (movement.c:93): (MAX_FORCE / hz_count * 20.0) is a double */
    const double smf_d = (double)(0.75f / hz) * 20.0;
    const float smf = (float)smf_d;
    for(size_t wi = 0; wi < nwork; wi++) {
        const uint32_t uid = work[wi];
        const pfo_agent *a = &w->agents[uid];
        const uint32_t ent_flags = a->flags;
        if(ent_flags & FLAG_COMBAT_HELD) {
            out_vel[2*wi] = out_vel[2*wi+1] = 0.0f;
            if(out_vpref) out_vpref[2*wi] = out_vpref[2*wi+1] = 0.0f;
            continue;
        }
        v2 pos = {a->pos[0], a->pos[1]}, velocity = {a->velocity[0], a->velocity[1]};
        steer_in s = {w, a, uid, pos, velocity, {a->vdes[0], a->vdes[1]}, smf, smf_d, {{0}}};
        if(w->forms) s.fs = w->forms[uid];
        v2 vpref = {0.0f, 0.0f};
        switch(a->state) {
        case STATE_TURNING:             break;
        case STATE_SEEK_ENEMIES:        vpref = enemy_seek_vpref(&s); break;
        case STATE_ARRIVING_TO_CELL:    vpref = cell_arrival_seek_vpref(&s); break;
        case STATE_MOVING_IN_FORMATION: vpref = formation_seek_vpref(&s); break;
        default:                        vpref = point_seek_vpref(&s); break;
        }
        /* find_neighbours (movement.c:2768) */
        uint32_t near_ents[512];
        int num_near = pfo_ents_in_circle(w, pos.x, pos.z, 10.0f, near_ents, 512);
        cpent dyn[MAX_NEIGHBOURS], stat[MAX_NEIGHBOURS]; int ndyn = 0, nstat = 0;
        for(int i = 0; i < num_near; i++) {
            uint32_t curr = near_ents[i];
            const pfo_agent *o = &w->agents[curr];
            if(curr == uid) continue;
            if(!(o->flags & FLAG_MOVABLE)) continue;
            if(o->radius == 0.0f) continue;
            if((ent_flags & FLAG_AIR) != (o->flags & FLAG_AIR)) continue;
            cpent nd = {{o->pos[0], o->pos[1]}, {o->velocity[0], o->velocity[1]}, o->radius};
            bool still = (o->state == STATE_ARRIVED || o->state == STATE_WAITING);
            if(still || v2_len(nd.vel) < 0.3f) { nd.vel = (v2){0.0f, 0.0f}; if(nstat < MAX_NEIGHBOURS) stat[nstat++] = nd; }
            else { if(ndyn < MAX_NEIGHBOURS) dyn[ndyn++] = nd; }
        }
        cpent self = {{a->prev_pos[0], a->prev_pos[1]}, velocity, a->radius};
        v2 nv = clearpath(self, vpref, dyn, ndyn, stat, nstat);
        nv = v2_truncate(nv, a->max_speed / hz);
        out_vel[2*wi] = nv.x; out_vel[2*wi+1] = nv.z;
        if(out_vpref) { out_vpref[2*wi] = vpref.x; out_vpref[2*wi+1] = vpref.z; }
    }
}

/* ------------------------------------------------------------------------------------------
 * Tile attributes -> cost_base: n_set_cost_for_tile (nav.c:267-344) + n_make_cliff_edges
 * (nav.c:431-475) with n_tile_pathable / n_tile_water_pathable / n_height_pathable
 * (nav.c:215-233, 258-265) and the corner heights of M_Tile_{NW,NE,SW,SE}Height
 * (map/tile.c:117-180). M_Tile_HeightAtPos (tile.c:249) is only consulted for corner tiles at
 * the four tile corners, where its ray/plane construction returns 4*corner_height up to float
 * rounding; the int conversion and the comparison against -1 make that rounding irrelevant
 * (|error| << 1 around multiples of 4), so the integer corner height is used.
 * attrs: int32[chunk_h*32][chunk_w*32][4] = {pathable, type, base_height, ramp_height}.
 * out: [chunks][64][64] chunk-blocked (the reference's layout).
 * ------------------------------------------------------------------------------------------ */
enum { TT_FLAT = 0, TT_RAMP_SN, TT_RAMP_NS, TT_RAMP_EW, TT_RAMP_WE, TT_CC_SW, TT_CV_SW, TT_CC_SE, TT_CV_SE,
       TT_CC_NW, TT_CV_NW, TT_CC_NE, TT_CV_NE };

static int tile_corner_raised(int type, int sub_r, int sub_c)
{
    /* bit sets of tile types whose {NW, NE, SW, SE} corner is raised (tile.c:117-180) */
    static const unsigned raised[2][2] = {
        { (1u<<TT_RAMP_SN)|(1u<<TT_RAMP_EW)|(1u<<TT_CV_SW)|(1u<<TT_CV_SE)|(1u<<TT_CC_SE)|(1u<<TT_CV_NE),   /* NW */
          (1u<<TT_RAMP_SN)|(1u<<TT_RAMP_WE)|(1u<<TT_CV_SW)|(1u<<TT_CC_SW)|(1u<<TT_CV_SE)|(1u<<TT_CV_NW) }, /* NE */
        { (1u<<TT_RAMP_NS)|(1u<<TT_RAMP_EW)|(1u<<TT_CV_SE)|(1u<<TT_CV_NW)|(1u<<TT_CC_NE)|(1u<<TT_CV_NE),   /* SW */
          (1u<<TT_RAMP_NS)|(1u<<TT_RAMP_WE)|(1u<<TT_CV_SW)|(1u<<TT_CV_NE)|(1u<<TT_CC_NW)|(1u<<TT_CV_NW) }, /* SE */
    };
    return (raised[sub_r][sub_c] >> type) & 1u;
}

static int tile_path_bit(int type, int sub_r, int sub_c)
{
    /* the 2x2 "tile_path_map" of n_set_cost_for_tile (nav.c:276-322) */
    switch(type) {
    case TT_CC_SW: case TT_CV_NE: return sub_r == 1 && sub_c == 0;   /* bl */
    case TT_CC_SE: case TT_CV_NW: return sub_r == 1 && sub_c == 1;   /* br */
    case TT_CC_NW: case TT_CV_SE: return sub_r == 0 && sub_c == 0;   /* tl */
    case TT_CC_NE: case TT_CV_SW: return sub_r == 0 && sub_c == 1;   /* tr */
    default: return 0;
    }
}

void pfo_cost_from_tiles(int chunk_w, int chunk_h, const int32_t *attrs, int ref_layer, uint8_t *out)
{
    const int H = chunk_h * 32, W = chunk_w * 32;
    const int group = ref_layer / 4;     /* 0 ground, 1 water, 2 air (nav.h enum nav_layer) */
    for(int r = 0; r < H; r++)
    for(int c = 0; c < W; c++) {
        const int32_t *t = attrs + ((size_t)r * W + c) * 4;
        const int path = t[0] != 0, type = t[1], base = t[2], ramp = t[3];
        int pathable;
        if(group == 0)      pathable = path && base >= -1 && !(type != TT_FLAT && ramp > 1);
        else if(group == 1) pathable = path && !(base + ramp > -1);
        else                pathable = 1;
        for(int sr = 0; sr < 2; sr++)
        for(int sc = 0; sc < 2; sc++) {
            const int h = (tile_corner_raised(type, sr, sc) ? base + ramp : base) * 4;
            const int hp = group == 1 ? (h <= -1) : group == 2 ? 1 : (h >= -1);
            uint8_t v = pathable ? 1 : (tile_path_bit(type, sr, sc) && hp) ? 1 : 0xFF;
            /* cliff edges: both tiles FLAT with different base heights. Note n_set_cost_edge blocks
             * the half of the tile where its map is ZERO (nav.c:415), i.e. EDGE_BOT blocks the top
             * sub-row and EDGE_RIGHT the left sub-column. */
            if(type == TT_FLAT) {
                #define CLIFF(rr, cc) ((rr) >= 0 && (rr) < H && (cc) >= 0 && (cc) < W \
                    && attrs[((size_t)(rr) * W + (cc)) * 4 + 1] == TT_FLAT \
                    && attrs[((size_t)(rr) * W + (cc)) * 4 + 2] != base)
                if(CLIFF(r + 1, c) && sr == 0) v = 0xFF;
                if(CLIFF(r - 1, c) && sr == 1) v = 0xFF;
                if(CLIFF(r, c - 1) && sc == 1) v = 0xFF;
                if(CLIFF(r, c + 1) && sc == 0) v = 0xFF;
                #undef CLIFF
            }
            const int nr = 2 * r + sr, nc = 2 * c + sc;
            out[((size_t)(nr / 64) * chunk_w + nc / 64) * 4096 + (nr % 64) * 64 + nc % 64] = v;
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * Repair chain of N_DesiredPointSeekVelocity (nav.c:3508-3554) for an entity standing on a tile whose
 * cached flow direction is FD_NONE although a path exists.
 * ---------------------------------------------------------------------------------------- */

/* N_FlowFieldUpdateToNearestPathable (field.c:2247): the entity sits on a non-passable tile. Frontier =
 * the passable tiles that border the impassable blob containing `start` (field_passable_frontier,
 * field.c:1441: 4-connected flood over non-passable tiles, chunk-local); Dijkstra over NON-passable
 * tiles only (field_build_integration_nonpass, field.c:643: edge weight = cost_base of the tile
 * entered); directions are written for 0 < cost < INF only. */
void pfo_flow_update_nearest_pathable(const pfo_map *m, int cr, int cc, int start_r, int start_c, uint8_t *inout)
{
    float intf[RES][RES];
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++) intf[r][c] = INFINITY;
    pq frontier; pq_init(&frontier);
    {
        static const int dr[4] = {0, 0, -1, 1}, dc[4] = {-1, 1, 0, 0};
        bool visited[RES][RES]; memset(visited, 0, sizeof(visited));
        int q[RES * RES][2], head = 0, tail = 0;
        q[tail][0] = start_r; q[tail][1] = start_c; tail++;
        visited[start_r][start_c] = true;
        while(head < tail) {
            int r = q[head][0], c = q[head][1]; head++;
            if(tile_passable(m, cr, cc, r, c)) {
                pq_push(&frontier, 0.0f, r, c);
                intf[r][c] = 0.0f;
                continue;
            }
            for(int e = 0; e < 4; e++) {
                int ar = r + dr[e], ac = c + dc[e];
                if(ar < 0 || ar >= RES || ac < 0 || ac >= RES) continue;
                if(visited[ar][ac]) continue;
                visited[ar][ac] = true;
                q[tail][0] = ar; q[tail][1] = ac; tail++;
            }
        }
    }
    const uint8_t *cost = chunk_cost(m, cr, cc);
    while(frontier.size > 0) {
        int r, c; pq_pop(&frontier, &r, &c);
        for(int dr = -1; dr <= 1; dr++) {
        for(int dc = -1; dc <= 1; dc++) {
            int ar = r + dr, ac = c + dc;
            if(ar < 0 || ar >= RES || ac < 0 || ac >= RES) continue;
            if(dr == 0 && dc == 0) continue;
            if(dr == dc || dr == -dc) continue;
            if(tile_passable(m, cr, cc, ar, ac)) continue;
            float total = intf[r][c] + cost[ar * RES + ac];
            if(total < intf[ar][ac]) { intf[ar][ac] = total; pq_push(&frontier, total, ar, ac); }
        }}
    }
    pq_free(&frontier);
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++) {
        if(intf[r][c] == INFINITY || intf[r][c] == 0.0f) continue;
        inout[r * RES + c] = (uint8_t)flow_dir((const float(*)[RES])intf, r, c);
    }
}

/* field_closest_tiles_local (field.c:1010): breadth-first rings around `target` inside the chunk; the
 * tiles of the first Manhattan ring that holds a passable, unblocked tile of the wanted islands. */
static int closest_tiles_local(const pfo_map *m, const uint16_t *gisl, int cr, int cc, int tr, int tc,
                               uint16_t local_iid, uint16_t global_iid, int (*out)[2], int maxout)
{
    static const int dr[4] = {0, 0, -1, 1}, dc[4] = {-1, 1, 0, 0};
    bool visited[RES][RES]; memset(visited, 0, sizeof(visited));
    int q[RES * RES][2], head = 0, tail = 0, ret = 0, first = -1;
    q[tail][0] = tr; q[tail][1] = tc; tail++;
    visited[tr][tc] = true;
    const uint8_t *cost = chunk_cost(m, cr, cc);
    const uint16_t *gi = gisl + ((size_t)cr * m->chunk_w + cc) * 4096;
    while(head < tail) {
        int r = q[head][0], c = q[head][1]; head++;
        for(int e = 0; e < 4; e++) {
            int ar = r + dr[e], ac = c + dc[e];
            if(ar < 0 || ar >= RES || ac < 0 || ac >= RES) continue;
            if(visited[ar][ac]) continue;
            visited[ar][ac] = true;
            q[tail][0] = ar; q[tail][1] = ac; tail++;
        }
        int mh = abs(tr - r) + abs(tc - c);
        if(first > -1 && mh > first) break;
        if(cost[r * RES + c] == COST_IMPASSABLE) continue;
        if(chunk_blk(m, cr, cc, r, c) > 0) continue;
        if(global_iid != ISLAND_NONE && gi[r * RES + c] != global_iid) continue;
        if(local_iid != ISLAND_NONE && chunk_liid(m, cr, cc, r, c) != local_iid) continue;
        if(first == -1) first = mh;
        out[ret][0] = r; out[ret][1] = c; ret++;
        if(ret == maxout) break;
    }
    return ret;
}

/* N_FlowFieldUpdateIslandToNearest (field.c:2307) for TARGET_TILE / TARGET_PORTAL fields: the entity's
 * local island was cut off from the field's frontier by blockers. New frontier = the tiles of that
 * island nearest (Manhattan) to the original frontier; then the ordinary integration + flow + fixup.
 * q = the request that built the field (its target); gisl = global islands [chunks][64][64]. */
void pfo_flow_update_island_to_nearest(const pfo_map *m, const uint16_t *gisl, const pfo_field_req *q,
                                       uint16_t local_iid, uint8_t *inout)
{
    const int cr = q->chunk_r, cc = q->chunk_c;
    int init[RES * RES][2], ninit = 0;
    if(q->target_type == TARGET_TILE) {
        /* field_tile_initial_frontier (field.c:1096), then again with ignoreblock (field.c:2367) */
        init[0][0] = q->tile_r; init[0][1] = q->tile_c; ninit = 1;
    }else{
        for(int r = q->port_r0; r <= q->port_r1; r++) {
        for(int c = q->port_c0; c <= q->port_c1; c++) {
            if(!tile_passable(m, cr, cc, r, c)) continue;
            if(q->port_iid != ISLAND_NONE && chunk_liid(m, cr, cc, r, c) != q->port_iid) continue;
            bool adj = false;
            for(int r2 = q->next_r0; r2 <= q->next_r1 && !adj; r2++) {
            for(int c2 = q->next_c0; c2 <= q->next_c1; c2++) {
                int dr = (q->next_chunk_r * RES + r2) - (cr * RES + r);
                int dc = (q->next_chunk_c * RES + c2) - (cc * RES + c);
                if(abs(dr) + abs(dc) == 1 && chunk_liid(m, q->next_chunk_r, q->next_chunk_c, r2, c2) == q->next_iid) {
                    adj = true; break;
                }
            }}
            if(!adj) continue;
            init[ninit][0] = r; init[ninit][1] = c; ninit++;
        }}
    }
    const uint16_t *gi = gisl + ((size_t)cr * m->chunk_w + cc) * 4096;
    int min_mh = INT32_MAX, nnew = 0;
    static int newf[RES * RES][2], tmp[RES * RES][2];
    for(int i = 0; i < ninit; i++) {
        int r = init[i][0], c = init[i][1];
        uint16_t cg = gi[r * RES + c], cl = chunk_liid(m, cr, cc, r, c);
        if(cl == local_iid) {
            if(min_mh > 0) nnew = 0;
            min_mh = 0;
            newf[nnew][0] = r; newf[nnew][1] = c; nnew++;
            continue;
        }
        int nextra = closest_tiles_local(m, gisl, cr, cc, r, c, local_iid, cg, tmp, RES * RES - nnew);
        if(!nextra) continue;
        int mh = abs(tmp[0][0] - r) + abs(tmp[0][1] - c);
        if(mh < min_mh) { min_mh = mh; nnew = 0; }
        if(mh > min_mh) continue;
        memcpy(newf + nnew, tmp, nextra * sizeof(tmp[0]));
        nnew += nextra;
    }
    float intf[RES][RES];
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++) intf[r][c] = INFINITY;
    pq frontier; pq_init(&frontier);
    for(int i = 0; i < nnew; i++) { pq_push(&frontier, 0.0f, newf[i][0], newf[i][1]); intf[newf[i][0]][newf[i][1]] = 0.0f; }
    const uint8_t *cost = chunk_cost(m, cr, cc);
    while(frontier.size > 0) {
        int r, c; pq_pop(&frontier, &r, &c);
        for(int dr = -1; dr <= 1; dr++) {
        for(int dc = -1; dc <= 1; dc++) {
            int ar = r + dr, ac = c + dc;
            if(ar < 0 || ar >= RES || ac < 0 || ac >= RES) continue;
            if(dr == 0 && dc == 0) continue;
            if(dr == dc || dr == -dc) continue;
            if(!tile_passable(m, cr, cc, ar, ac)) continue;
            float total = intf[r][c] + cost[ar * RES + ac];
            if(total < intf[ar][ac]) { intf[ar][ac] = total; pq_push(&frontier, total, ar, ac); }
        }}
    }
    pq_free(&frontier);
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++) {
        if(intf[r][c] == INFINITY) continue;
        if(intf[r][c] == 0.0f) { inout[r * RES + c] = FD_NONE; continue; }
        inout[r * RES + c] = (uint8_t)flow_dir((const float(*)[RES])intf, r, c);
    }
    if(q->target_type == TARGET_PORTAL) {
        bool up = q->next_chunk_r < cr, down = q->next_chunk_r > cr, left = q->next_chunk_c < cc;
        uint8_t d = up ? FD_N : down ? FD_S : left ? FD_W : FD_E;
        for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++)
            if(intf[r][c] == 0.0f) inout[r * RES + c] = d;
    }
}

/* ------------------------------------------------------------------------------------------
 * Region ("cell arrival" / "group arrival") fields: dim x dim tiles that may straddle chunks and
 * the map edge; the output packs two directions per byte (set_flow_cell, field.c:790: even column
 * -> high nibble). All tile coordinates are absolute: chunk * 64 + tile.
 * ---------------------------------------------------------------------------------------- */
static bool abs_exists(const pfo_map *m, int ar, int ac)     /* M_Tile_RelativeDesc's bounds (tile.c:391) */
{ return ar >= 0 && ar < m->chunk_h * RES && ac >= 0 && ac < m->chunk_w * RES; }
static bool abs_passable(const pfo_map *m, int ar, int ac)   /* field_tile_passable (field.c:117) */
{ return tile_passable(m, ar / RES, ac / RES, ar % RES, ac % RES); }
static uint8_t abs_cost(const pfo_map *m, int ar, int ac)
{ return chunk_cost(m, ar / RES, ac / RES)[(ar % RES) * RES + (ac % RES)]; }
/* field_tile_passable_no_enemies (field.c:179) with an explicit enemy mask */
static bool abs_passable_mask(const pfo_map *m, int ar, int ac, uint16_t enemies)
{
    if(enemies == 0 || !m->factions) return abs_passable(m, ar, ac);
    const int cr = ar / RES, cc = ac / RES, r = ar % RES, c = ac % RES;
    if(chunk_cost(m, cr, cc)[r * RES + c] == COST_IMPASSABLE) return false;
    const uint8_t *fac = m->factions + ((size_t)cr * m->chunk_w + cc) * 15 * 4096;
    for(int i = 0; i < 15; i++)
        if(fac[(size_t)i * 4096 + r * RES + c] && !(enemies & (1u << i)))
            return chunk_blk(m, cr, cc, r, c) == 0;
    return true;
}

/* field_flow_dir (field.c:355) for a dim x dim integration field (row stride = rdim = dim) */
static int flow_dir_n(const float *f, int n, int r, int c)
{
    float mc = INFINITY;
#define F(rr, cc) f[(rr) * n + (cc)]
    if(r > 0) mc = MINF(mc, F(r-1, c));
    if(r < n-1) mc = MINF(mc, F(r+1, c));
    if(c > 0) mc = MINF(mc, F(r, c-1));
    if(c < n-1) mc = MINF(mc, F(r, c+1));
    if(r > 0 && c > 0 && F(r-1, c) < INFINITY && F(r, c-1) < INFINITY) mc = MINF(mc, F(r-1, c-1));
    if(r > 0 && c < n-1 && F(r-1, c) < INFINITY && F(r, c+1) < INFINITY) mc = MINF(mc, F(r-1, c+1));
    if(r < n-1 && c > 0 && F(r+1, c) < INFINITY && F(r, c-1) < INFINITY) mc = MINF(mc, F(r+1, c-1));
    if(r < n-1 && c < n-1 && F(r+1, c) < INFINITY && F(r, c+1) < INFINITY) mc = MINF(mc, F(r+1, c+1));
    if(r > 0 && F(r-1, c) == mc) return FD_N;
    else if(r < n-1 && F(r+1, c) == mc) return FD_S;
    else if(c < n-1 && F(r, c+1) == mc) return FD_E;
    else if(c > 0 && F(r, c-1) == mc) return FD_W;
    else if(r > 0 && c > 0 && F(r-1, c-1) == mc) return FD_NW;
    else if(r > 0 && c < n-1 && F(r-1, c+1) == mc) return FD_NE;
    else if(r < n-1 && c > 0 && F(r+1, c-1) == mc) return FD_SW;
    else if(r < n-1 && c < n-1 && F(r+1, c+1) == mc) return FD_SE;
#undef F
    return 0;
}

static void set_cell(int v, int r, int c, int n, uint8_t *buf)   /* set_flow_cell (field.c:790) */
{
    const size_t b = (size_t)r * (n / 2) + c / 2;
    if(c % 2 == 1) buf[b] = (uint8_t)((buf[b] & 0xf0) | v);
    else           buf[b] = (uint8_t)((buf[b] & 0x0f) | (v << 4));
}

static void overlay_mask(const int32_t *ov, int nov, int base_r, int base_c, int n, bool *mask)   /* build_overlay_mask (field.c:571) */
{
    memset(mask, 0, (size_t)n * n);
    for(int i = 0; i < nov; i++) {
        int dr = ov[2*i] - base_r, dc = ov[2*i+1] - base_c;
        if(dr >= 0 && dr < n && dc >= 0 && dc < n) mask[dr * n + dc] = true;
    }
}

/* N_CellArrivalFieldCreate (field.c:2445; cell_mode = 1: one target, the base is shifted when the target
 * falls one past the far edge, :2477-2482) and the tile-space part of N_GroupArrivalFieldCreate
 * (field.c:2525; cell_mode = 0: every seed inside the region is a zero-cost source). Dijkstra over passable
 * tiles (field_build_integration_region, field.c:587; field_neighbours_grid_global, :253: 4-neighbourhood,
 * edge weight = cost_base of the tile entered, overlay-blocked tiles are never entered). */
void pfo_region_field_create(const pfo_map *m, int dim, uint16_t enemies, int cell_mode, const int32_t *seeds, int nseeds,
                             int center_r, int center_c, const int32_t *overlay, int noverlay, uint8_t *out)
{
    memset(out, 0, (size_t)dim * dim / 2);
    int base_r = center_r - dim / 2, base_c = center_c - dim / 2;
    if(cell_mode) {
        if(seeds[0] - base_r >= dim) base_r = seeds[0] - (dim - 1);
        if(seeds[1] - base_c >= dim) base_c = seeds[1] - (dim - 1);
    }
    float *intf = malloc(sizeof(float) * dim * dim);
    bool *mask = malloc((size_t)dim * dim);
    for(int i = 0; i < dim * dim; i++) intf[i] = INFINITY;
    pq frontier; pq_init(&frontier);
    for(int i = 0; i < (cell_mode ? 1 : nseeds); i++) {
        int dr = seeds[2*i] - base_r, dc = seeds[2*i+1] - base_c;
        if(dr < 0 || dr >= dim || dc < 0 || dc >= dim) continue;     /* tile_outside_region (field.c:126) */
        pq_push(&frontier, 0.0f, seeds[2*i], seeds[2*i+1]);
        intf[dr * dim + dc] = 0.0f;
    }
    const bool have_ov = overlay && noverlay > 0;
    if(have_ov) overlay_mask(overlay, noverlay, base_r, base_c, dim, mask);
    while(frontier.size > 0) {
        int ar, ac; pq_pop(&frontier, &ar, &ac);
        const int dr = ar - base_r, dc = ac - base_c;
        for(int e = 0; e < 4; e++) {
            static const int er[4] = {-1, 0, 0, 1}, ec[4] = {0, -1, 1, 0};
            const int nr = ar + er[e], nc = ac + ec[e];
            if(!abs_exists(m, nr, nc)) continue;
            if(!abs_passable_mask(m, nr, nc, enemies)) continue;
            const int ndr = nr - base_r, ndc = nc - base_c;
            if(ndr < 0 || ndr >= dim || ndc < 0 || ndc >= dim) continue;
            if(have_ov && mask[ndr * dim + ndc]) continue;
            float total = intf[dr * dim + dc] + abs_cost(m, nr, nc);
            if(total < intf[ndr * dim + ndc]) { intf[ndr * dim + ndc] = total; pq_push(&frontier, total, nr, nc); }
        }
    }
    pq_free(&frontier);
    for(int r = 0; r < dim; r++) for(int c = 0; c < dim; c++) {      /* field_build_flow_unaligned (field.c:804) */
        if(intf[r * dim + c] == INFINITY) continue;
        if(intf[r * dim + c] == 0.0f) { set_cell(FD_NONE, r, c, dim, out); continue; }
        set_cell(flow_dir_n(intf, dim, r, c), r, c, dim, out);
    }
    free(intf); free(mask);
}

/* N_GroupArrivalFieldCreate (field.c:2525): world-space targets and centre */
void pfo_group_arrival_field(const pfo_map *m, int dim, uint16_t enemies, const float *targets_xz, int ntargets,
                             const float *center_xz, const int32_t *overlay, int noverlay, uint8_t *out)
{
    memset(out, 0, (size_t)dim * dim / 2);
    tdesc ct;
    if(!desc_for_point(m, center_xz[0], center_xz[1], &ct)) return;
    int32_t *seeds = malloc(sizeof(int32_t) * 2 * (ntargets ? ntargets : 1));
    int ns = 0;
    for(int i = 0; i < ntargets; i++) {
        tdesc t;
        if(!desc_for_point(m, targets_xz[2*i], targets_xz[2*i+1], &t)) continue;
        seeds[2*ns] = t.chunk_r * RES + t.tile_r; seeds[2*ns+1] = t.chunk_c * RES + t.tile_c; ns++;
    }
    pfo_region_field_create(m, dim, enemies, 0, seeds, ns, ct.chunk_r * RES + ct.tile_r, ct.chunk_c * RES + ct.tile_c,
                            overlay, noverlay, out);
    free(seeds);
}

/* N_CellArrivalFieldUpdateToNearestPathable (field.c:2603). The flood that finds the passable rim of the
 * blocked island around `start` (field_passable_frontier, field.c:1441) runs inside the map-clamped region
 * (clamped_region, field.c:1892: its extents are end - base, so the last row / column of a clamped edge is
 * left out) and indexes its visited array with stride region.r (visited_idx, field.c:1431) -- when the
 * clamped region has fewer rows than columns distinct tiles alias, so the flood order is kept literally.
 * Then Dijkstra over non-passable or overlay-blocked tiles (field_build_integration_nonpass_region,
 * field.c:678) from that rim; only 0 < cost < INF cells are rewritten. The unclamped base here is
 * center - dim/2: the target shift of the create call is NOT repeated. */
void pfo_region_field_update_to_nearest_pathable(const pfo_map *m, int dim, int start_r, int start_c, int center_r, int center_c,
                                                 const int32_t *overlay, int noverlay, uint8_t *inout)
{
    const int max_r = m->chunk_h * RES, max_c = m->chunk_w * RES;
    const int cb_r = (center_r - dim / 2 >= 0) ? center_r - dim / 2 : 0;
    const int cb_c = (center_c - dim / 2 >= 0) ? center_c - dim / 2 : 0;
    const int ce_r = (center_r + dim / 2 < max_r) ? center_r + dim / 2 : max_r - 1;
    const int ce_c = (center_c + dim / 2 < max_c) ? center_c + dim / 2 : max_c - 1;
    const int reg_r = ce_r - cb_r, reg_c = ce_c - cb_c;
    const int nelems = (reg_r > reg_c ? reg_r : reg_c) * (reg_r > reg_c ? reg_r : reg_c);
    const int base_r = center_r - dim / 2, base_c = center_c - dim / 2;

    float *intf = malloc(sizeof(float) * dim * dim);
    for(int i = 0; i < dim * dim; i++) intf[i] = INFINITY;
    pq frontier; pq_init(&frontier);
    {
        static const int er[4] = {0, 0, -1, 1}, ec[4] = {-1, 1, 0, 0};
        bool *visited = calloc(nelems ? nelems : 1, 1);
        int (*q)[2] = malloc(sizeof(int[2]) * (nelems ? nelems : 1));
        int head = 0, tail = 0;
        q[tail][0] = start_r; q[tail][1] = start_c; tail++;
        visited[(start_r - cb_r) * reg_r + (start_c - cb_c)] = true;
        while(head < tail) {
            int r = q[head][0], c = q[head][1]; head++;
            if(abs_passable(m, r, c)) {
                int dr = r - base_r, dc = c - base_c;
                if(dr < 0 || dr >= dim || dc < 0 || dc >= dim) continue;
                pq_push(&frontier, 0.0f, r, c);
                intf[dr * dim + dc] = 0.0f;
                continue;
            }
            for(int e = 0; e < 4; e++) {
                int nr = r + er[e], nc = c + ec[e];
                if(!abs_exists(m, nr, nc)) continue;
                int dr = nr - cb_r, dc = nc - cb_c;
                if(dr < 0 || dr >= reg_r || dc < 0 || dc >= reg_c) continue;
                if(visited[dr * reg_r + dc]) continue;
                visited[dr * reg_r + dc] = true;
                q[tail][0] = nr; q[tail][1] = nc; tail++;
            }
        }
        free(visited); free(q);
    }
    bool *mask = malloc((size_t)dim * dim);
    const bool have_ov = overlay && noverlay > 0;
    if(have_ov) overlay_mask(overlay, noverlay, base_r, base_c, dim, mask);
    while(frontier.size > 0) {
        int ar, ac; pq_pop(&frontier, &ar, &ac);
        const int dr = ar - base_r, dc = ac - base_c;
        for(int e = 0; e < 4; e++) {
            static const int er[4] = {-1, 0, 0, 1}, ec[4] = {0, -1, 1, 0};
            const int nr = ar + er[e], nc = ac + ec[e];
            if(!abs_exists(m, nr, nc)) continue;
            const int ndr = nr - base_r, ndc = nc - base_c;
            if(ndr < 0 || ndr >= dim || ndc < 0 || ndc >= dim) continue;
            const bool ovb = have_ov && mask[ndr * dim + ndc];
            if(abs_passable(m, nr, nc) && !ovb) continue;
            float total = intf[dr * dim + dc] + abs_cost(m, nr, nc);
            if(total < intf[ndr * dim + ndc]) { intf[ndr * dim + ndc] = total; pq_push(&frontier, total, nr, nc); }
        }
    }
    pq_free(&frontier);
    for(int r = 0; r < dim; r++) for(int c = 0; c < dim; c++) {
        if(!abs_exists(m, base_r + r, base_c + c)) continue;
        if(intf[r * dim + c] == INFINITY || intf[r * dim + c] == 0.0f) continue;
        set_cell(flow_dir_n(intf, dim, r, c), r, c, dim, inout);
    }
    free(intf); free(mask);
}

/* ------------------------------------------------------------------------------------------
 * TARGET_ZONE chunk fields (the group arrival fields a flock follows into the open slots around its goal):
 * N_FlowFieldUpdate -> field_update_zone (field.c:1810) over the chunk padded by half a chunk on every side.
 * ---------------------------------------------------------------------------------------- */
/* field_zone_initial_frontier (field.c:1683): (1) snap to the nearest open tile, best-first by squared
 * distance from the centre, stepping through blocked tiles; (2) best-first flood of the connected open
 * footprint from that tile (pushed at priority 0) until `budget` tiles are collected. Both use the
 * reference's binary heap, whose tie order decides which tiles of the last distance class make the budget. */
static int zone_initial_frontier(const pfo_map *m, int centre_r, int centre_c, int base_r, int base_c, int dim,
                                 int32_t *out, int budget)
{
    static const int er[8] = {0, 0, -1, 1, -1, -1, 1, 1}, ec[8] = {-1, 1, 0, 0, -1, 1, -1, 1};
    const int cdr = centre_r - base_r, cdc = centre_c - base_c;
    if(cdr < 0 || cdr >= dim || cdc < 0 || cdc >= dim) return 0;
    bool *visited = calloc((size_t)dim * dim, 1);
    pq frontier; pq_init(&frontier);
    visited[cdr * dim + cdc] = true;
    pq_push(&frontier, 0.0f, centre_r, centre_c);
    int start_r = 0, start_c = 0; bool have_start = false;
    while(frontier.size > 0) {
        int r, c; pq_pop(&frontier, &r, &c);
        if(abs_passable(m, r, c)) { start_r = r; start_c = c; have_start = true; break; }
        for(int e = 0; e < 8; e++) {
            int nr = r + er[e], nc = c + ec[e];
            if(!abs_exists(m, nr, nc)) continue;
            int dr = nr - base_r, dc = nc - base_c;
            if(dr < 0 || dr >= dim || dc < 0 || dc >= dim) continue;
            if(visited[dr * dim + dc]) continue;
            visited[dr * dim + dc] = true;
            int ndr = nr - centre_r, ndc = nc - centre_c;
            pq_push(&frontier, (float)(ndr * ndr + ndc * ndc), nr, nc);
        }
    }
    int ret = 0;
    if(have_start) {
        frontier.size = 0;
        memset(visited, 0, (size_t)dim * dim);
        visited[(start_r - base_r) * dim + (start_c - base_c)] = true;
        pq_push(&frontier, 0.0f, start_r, start_c);
        while(frontier.size > 0 && ret < budget) {
            int r, c; pq_pop(&frontier, &r, &c);
            if(abs_passable(m, r, c)) { out[2*ret] = r; out[2*ret+1] = c; ret++; }
            for(int e = 0; e < 8; e++) {
                int nr = r + er[e], nc = c + ec[e];
                if(!abs_exists(m, nr, nc)) continue;
                int dr = nr - base_r, dc = nc - base_c;
                if(dr < 0 || dr >= dim || dc < 0 || dc >= dim) continue;
                if(visited[dr * dim + dc]) continue;
                visited[dr * dim + dc] = true;
                if(!abs_passable(m, nr, nc)) continue;
                int ndr = nr - centre_r, ndc = nc - centre_c;
                pq_push(&frontier, (float)(ndr * ndr + ndc * ndc), nr, nc);
            }
        }
    }
    pq_free(&frontier); free(visited);
    return ret;
}

/* the zone's seed tiles alone (for the device path's parity tests): out = (r, c) pairs, returns the count */
int pfo_zone_seeds(const pfo_map *m, int chunk_r, int chunk_c, int centre_r, int centre_c, int radius, int32_t *out)
{
    const int dim = (m->chunk_h > 1 && m->chunk_w > 1) ? 2 * RES : RES;
    const int base_r = chunk_r > 0 ? chunk_r * RES - RES / 2 : 0, base_c = chunk_c > 0 ? chunk_c * RES - RES / 2 : 0;
    size_t budget = (size_t)(M_PI * radius * radius + 0.5);
    if(budget > (size_t)(dim * dim)) budget = dim * dim;
    return zone_initial_frontier(m, centre_r, centre_c, base_r, base_c, dim, out, (int)budget);
}

/* The shared tail of field_update_zone / _entity / _enemies (field.c:1810, 1609, 1540): `seeds` (absolute tiles inside
 * the padded region) at cost 0, field_build_integration_region (:587) with plain passability and no overlay, then
 * field_build_flow_region (:762) over the chunk's window. pfo_flow_field_zone =
 * N_FlowFieldUpdate for TARGET_ZONE (field.c:2050 -> field_update_zone, :1810), in place on `inout` (64 x 64
 * direction bytes): the integration runs over the padded region (plain passability, no overlay) and
 * field_build_flow_region (field.c:762) writes the chunk's window, leaving unreached tiles as they were. Only the
 * square cases are defined: 128 x 128 on maps with more than one chunk row AND column, 64 x 64 on a 1 x 1 map
 * (with one of the two the reference's row stride overruns its buffer). */
void pfo_chunk_field_seeded(const pfo_map *m, int chunk_r, int chunk_c, const int32_t *seeds, int ns, uint8_t *inout)
{
    const int dim = (m->chunk_h > 1 && m->chunk_w > 1) ? 2 * RES : RES;
    const int base_r = chunk_r > 0 ? chunk_r * RES - RES / 2 : 0, base_c = chunk_c > 0 ? chunk_c * RES - RES / 2 : 0;
    const int roff = chunk_r > 0 ? RES / 2 : 0, coff = chunk_c > 0 ? RES / 2 : 0;
    float *intf = malloc(sizeof(float) * dim * dim);
    for(int i = 0; i < dim * dim; i++) intf[i] = INFINITY;
    pq frontier; pq_init(&frontier);
    for(int i = 0; i < ns; i++) {
        pq_push(&frontier, 0.0f, seeds[2*i], seeds[2*i+1]);
        intf[(seeds[2*i] - base_r) * dim + (seeds[2*i+1] - base_c)] = 0.0f;
    }
    while(frontier.size > 0) {
        int ar, ac; pq_pop(&frontier, &ar, &ac);
        const int dr = ar - base_r, dc = ac - base_c;
        for(int e = 0; e < 4; e++) {
            static const int er[4] = {-1, 0, 0, 1}, ec[4] = {0, -1, 1, 0};
            const int nr = ar + er[e], nc = ac + ec[e];
            if(!abs_exists(m, nr, nc) || !abs_passable(m, nr, nc)) continue;
            const int ndr = nr - base_r, ndc = nc - base_c;
            if(ndr < 0 || ndr >= dim || ndc < 0 || ndc >= dim) continue;
            float total = intf[dr * dim + dc] + abs_cost(m, nr, nc);
            if(total < intf[ndr * dim + ndc]) { intf[ndr * dim + ndc] = total; pq_push(&frontier, total, nr, nc); }
        }
    }
    pq_free(&frontier);
    for(int r = 0; r < RES; r++) for(int c = 0; c < RES; c++) {
        const int ir = r + roff, ic = c + coff;
        if(intf[ir * dim + ic] == INFINITY) continue;
        if(intf[ir * dim + ic] == 0.0f) { inout[r * RES + c] = FD_NONE; continue; }
        inout[r * RES + c] = (uint8_t)flow_dir_n(intf, dim, ir, ic);
    }
    free(intf);
}

void pfo_flow_field_zone(const pfo_map *m, int chunk_r, int chunk_c, int centre_r, int centre_c, int radius, uint8_t *inout)
{
    const int dim = (m->chunk_h > 1 && m->chunk_w > 1) ? 2 * RES : RES;
    int32_t *seeds = malloc(sizeof(int32_t) * 2 * dim * dim);
    const int ns = pfo_zone_seeds(m, chunk_r, chunk_c, centre_r, centre_c, radius, seeds);
    pfo_chunk_field_seeded(m, chunk_r, chunk_c, seeds, ns, inout);
    free(seeds);
}

/* N_DesiredGroupArrivalVelocity (nav.c:3561) against caller-held zone fields: fields[chunk] = 64 x 64 direction
 * bytes or NULL-equivalent (has[chunk] == 0). out_vel 2 floats, out_flags bit0 = returned true, bit1 = at_slot */
void pfo_group_arrival_velocity(const pfo_map *m, const uint8_t *fields, const uint8_t *has, const float *centre_xz, int radius,
                                const float *pos_xz, int n, float *out_vel, uint8_t *out_flags)
{
    tdesc ct;
    const bool cok = desc_for_point(m, centre_xz[0], centre_xz[1], &ct);
    for(int i = 0; i < n; i++) {
        out_vel[2*i] = out_vel[2*i+1] = 0.0f; out_flags[i] = 0;
        tdesc t;
        if(!desc_for_point(m, pos_xz[2*i], pos_xz[2*i+1], &t) || !cok) continue;
        const int chunk = t.chunk_r * m->chunk_w + t.chunk_c;
        if(!has[chunk]) continue;
        const int dir = fields[(size_t)chunk * 4096 + t.tile_r * RES + t.tile_c];
        v2 d = flow_dir_vec(dir);
        out_vel[2*i] = d.x; out_vel[2*i+1] = d.z;
        out_flags[i] = 1;
        if(dir == FD_NONE) {
            const int dr = (t.chunk_r * RES + t.tile_r) - (ct.chunk_r * RES + ct.tile_r);
            const int dc = (t.chunk_c * RES + t.tile_c) - (ct.chunk_c * RES + ct.tile_c);
            if(dr * dr + dc * dc <= radius * radius) out_flags[i] |= 2;
        }
    }
}

/* ------------------------------------------------------------------------------------------
 * State update: entity_compute_update (game/movement.c:2303-2670), all nine movement states, no arrival group. The
 * quaternion helpers keep the reference's mix of float and double arithmetic (pf_math.c). The states beyond point
 * seeking, and the movestate_ext part of the apply, are NOT an independent restatement: they were written without a
 * reference checkout and follow k_entity_update / k_entity_apply (pfnav_agents.cu), including the heading gate's state
 * set (MOVING_IN_FORMATION ungated, unverified, DESIGN.md §4); they stay unpinned until test_port_all_states_vs_ref runs
 * against oracle/_ref.
 * The map of the world holds ONE layer: it stands for the layer Entity_NavLayerWithRadius picks (entity.c:554).
 * ---------------------------------------------------------------------------------------- */
typedef struct { float x, y, z, w; } pquat;
#define PFO_PI_D 3.14159265358979323846
#define PFO_HIST 14

/* first column of PFM_Mat4x4_RotFromQuat (pf_math.c:324) applied to (1,0,0,1), as PFM_Quat_PitchDiff uses it (:677) */
static void quat_front(pquat q, float *dx, float *dz)
{
    *dx = (float)(1 - 2 * ((double)q.y * (double)q.y) - 2 * ((double)q.z * (double)q.z));
    *dz = 2 * q.x * q.z + 2 * q.w * q.y;
}
static float quat_pitch_diff(pquat a, pquat b)            /* PFM_Quat_PitchDiff (pf_math.c:677-704) */
{
    float ax, az, bx, bz;
    quat_front(a, &ax, &az); quat_front(b, &bx, &bz);
    const float dot = ax * bx + az * bz, det = ax * bz - az * bx;
    return (float)atan2((double)det, (double)dot);
}
static pquat dir_quat_from_velocity(v2 v)                  /* movement.c:1411 */
{
    const float angle_rad = (float)(atan2((double)v.z, (double)v.x) - PFO_PI_D / 2.0f);
    pquat q = {0.0f, (float)(1.0f * sin((double)(angle_rad / 2.0f))), 0.0f, (float)cos((double)(angle_rad / 2.0f))};
    return q;
}
/* turn_toward (movement.c:2249): PFM_Mat4x4_MakeRotY -> PFM_Quat_FromRotMat -> PFM_Quat_MultQuat -> PFM_Quat_Normal */
static pquat turn_toward(pquat cur, pquat target, float max_deg)
{
    float angle_deg = (float)((double)quat_pitch_diff(cur, target) * (180.0f / PFO_PI_D));
    if(180.0f - fabs((double)angle_deg) < 1.0f) angle_deg = 180.0f;
    const double mn = ((double)max_deg < fabs((double)angle_deg)) ? (double)max_deg : fabs((double)angle_deg);
    const int sg = (angle_deg > 0) - (angle_deg < 0);
    const float turn_deg = (float)(mn * -sg);
    const float radians = (float)((double)turn_deg * (PFO_PI_D / 180.0f));
    const float c = (float)cos((double)radians), sn = (float)sin((double)radians);
    const float m00 = c, m02 = -sn, m20 = sn, m22 = c, m11 = 1.0f;
    pquat rot;
    const float tr = m00 + m11 + m22;
    if(tr > 0) {
        const float S = (float)(sqrt((double)tr + 1.0) * 2);
        rot.w = (float)(0.25 * (double)S); rot.x = (0.0f - 0.0f) / S; rot.y = (m02 - m20) / S; rot.z = (0.0f - 0.0f) / S;
    }else if((m00 > m11) && (m00 > m22)) {
        const float S = (float)(sqrt(1.0 + (double)m00 - (double)m11 - (double)m22) * 2);
        rot.w = (0.0f - 0.0f) / S; rot.x = (float)(0.25 * (double)S); rot.y = (0.0f + 0.0f) / S; rot.z = (m02 + m20) / S;
    }else if(m11 > m22) {
        const float S = (float)(sqrt(1.0 + (double)m11 - (double)m00 - (double)m22) * 2);
        rot.w = (m02 - m20) / S; rot.x = (0.0f + 0.0f) / S; rot.y = (float)(0.25 * (double)S); rot.z = (0.0f + 0.0f) / S;
    }else{
        const float S = (float)(sqrt(1.0 + (double)m22 - (double)m00 - (double)m11) * 2);
        rot.w = (0.0f - 0.0f) / S; rot.x = (m02 + m20) / S; rot.y = (0.0f + 0.0f) / S; rot.z = (float)(0.25 * (double)S);
    }
    pquat f;                                                /* PFM_Quat_MultQuat(&rot, &cur) (pf_math.c:639) */
    f.x = ( rot.x * cur.w) + (rot.y * cur.z) - (rot.z * cur.y) + (rot.w * cur.x);
    f.y = (-rot.x * cur.z) + (rot.y * cur.w) + (rot.z * cur.x) + (rot.w * cur.y);
    f.z = ( rot.x * cur.y) - (rot.y * cur.x) + (rot.z * cur.w) + (rot.w * cur.z);
    f.w = (-rot.x * cur.x) - (rot.y * cur.y) - (rot.z * cur.z) + (rot.w * cur.w);
    const float len = (float)sqrt((double)(f.x * f.x + f.y * f.y + f.z * f.z + f.w * f.w));
    f.x = f.x / len; f.y = f.y / len; f.z = f.z / len; f.w = f.w / len;
    return f;
}

enum { ST_MOVING = 0, ST_MOVING_IN_FORMATION, ST_ARRIVED, ST_SEEK_ENEMIES, ST_WAITING, ST_SURROUND, ST_ENTER_RANGE,
       ST_TURNING, ST_ARRIVING_TO_CELL };
enum { UP_STATE = 1 << 0, UP_VELOCITY = 1 << 1, UP_POSITION = 1 << 2, UP_ROTATION = 1 << 3, UP_NEXT_POS = 1 << 4,
       UP_PREV_POS = 1 << 5, UP_STEP = 1 << 6, UP_LEFT = 1 << 7, UP_NEXT_ROT = 1 << 8, UP_PREV_ROT = 1 << 9,
       UP_DEST = 1 << 10, UP_TARGET_PREV = 1 << 11, UP_MOVING = 1 << 12, UP_TARGET_DIR = 1 << 13, UP_TURNING_IN_PLACE = 1 << 14 };
enum { TODO_SURROUND_QUERY = 1 << 0, TODO_USE_SURROUND_FIELD = 1 << 1, TODO_DROP_SURROUND_FIELD = 1 << 2 };
#define NULL_UID 0xffffffffu
#define WAIT_TICKS 60                       /* movement.c:97 */
#define ADJACENCY_SEP_DIST 5.0f             /* movement.c:953 */
#define FL_WATER (1u << 14)
#define FL_AIR (1u << 15)
#define FL_GARRISONED (1u << 18)
#define FL_COMBAT_HELD (1u << 21)

/* M_NavIsAdjacentToImpassable (nav.c:4745): a 4-neighbour of the tile under `pos` is not passable */
static bool adjacent_to_impassable(const pfo_map *m, v2 pos)
{
    tdesc td;
    if(!desc_for_point(m, pos.x, pos.z, &td)) return false;
    const int ar = td.chunk_r * RES + td.tile_r, ac = td.chunk_c * RES + td.tile_c;
    static const int dr[4] = {-1, 0, 0, 1}, dc[4] = {0, -1, 1, 0};
    for(int e = 0; e < 4; e++) {
        const int nr = ar + dr[e], nc = ac + dc[e];
        if(nr < 0 || nr >= m->chunk_h * RES || nc < 0 || nc >= m->chunk_w * RES) continue;
        if(!abs_passable(m, nr, nc)) return true;
    }
    return false;
}

/* M_NavIsMaximallyClose (nav.c:4707) over the precomputed tile centres: one within `tol` of `pos` */
static bool maximally_close(const pfo_arrival *ac, v2 pos, float tol)
{
    for(int i = 0; i < ac->mc_n; i++)
        if(v2_len((v2){ac->mc[2 * i] - pos.x, ac->mc[2 * i + 1] - pos.z}) <= tol) return true;
    return false;
}

/* arrived() (movement.c:2170) then adjacent_flock_members (movement.c:953): a flock member within r + r' +
 * ADJACENCY_SEP_DIST of the CURRENT position that has ARRIVED */
static bool entity_arrived(const pfo_world *w, const pfo_agent *a, uint32_t uid, const pfo_arrival *ac, v2 new_pos, v2 curr)
{
    const pfo_flock *fl = &w->flocks[a->flock];
    const float thresh = a->radius * 1.5f;
    if(v2_len(v2_sub((v2){fl->target[0], fl->target[1]}, new_pos)) < thresh) return true;
    if(adjacent_to_impassable(&w->map, new_pos) && maximally_close(ac, new_pos, thresh)) return true;
    if(ac->nearest_ok && v2_len((v2){ac->nearest[0] - new_pos.x, ac->nearest[1] - new_pos.z}) < thresh) return true;
    for(size_t o = 0; o < w->n; o++) {
        if(o == uid) continue;
        const pfo_agent *b = &w->agents[o];
        if(b->state != ST_ARRIVED || b->flock != a->flock) continue;
        if(v2_len((v2){curr.x - b->pos[0], curr.z - b->pos[1]}) <= a->radius + b->radius + ADJACENCY_SEP_DIST) return true;
    }
    return false;
}

static void set_state(pfo_patch *p, int next, int block) { p->flags |= UP_STATE; p->next_state = next; p->next_block = block; }

void pfo_entity_updates(const pfo_world *w, const pfo_movestate *mss, const pfo_arrival *arr, const pfo_arrival *tarr,
                        const uint32_t *work, size_t nwork, const float *new_vel_xz, const float *vdes_xz, pfo_patch *out)
{
    const pfo_map *m = &w->map;
    const float EPS = 1.0f / 1024;
    const float turn_rate = (float)((double)(15.0f / (float)w->hz) * 20.0);     /* SCALED_MAX_TURN_RATE (movement.c:434) */
    for(size_t wi = 0; wi < nwork; wi++) {
        const uint32_t uid = work[wi];
        const pfo_agent *a = &w->agents[uid];
        const pfo_movestate *ms = &mss[uid];
        pfo_patch p;
        memset(&p, 0, sizeof(p));
        p.next_state = -1;
        pfo_movestate_ext ex;
        if(w->exts) ex = w->exts[uid];
        else { memset(&ex, 0, sizeof(ex)); ex.surround_target_uid = NULL_UID; ex.rot[3] = 1.0f; }
        pfo_formation fs;
        if(w->forms) fs = w->forms[uid]; else memset(&fs, 0, sizeof(fs));
        p.wait_ticks_left = ex.wait_ticks_left;
        const pquat ms_rot = {ms->next_rot[0], ms->next_rot[1], ms->next_rot[2], ms->next_rot[3]};
        v2 new_vel = {new_vel_xz[2 * wi], new_vel_xz[2 * wi + 1]};
        const v2 vdes = {vdes_xz[2 * wi], vdes_xz[2 * wi + 1]};
        const v2 ms_vel = {a->velocity[0], a->velocity[1]};
        const v2 curr_xz = {a->pos[0], a->pos[1]};
        const uint32_t state = a->state;

        if(ms->left > 0) {                                   /* flush an unfinished interpolation (movement.c:2311) */
            p.flags |= UP_POSITION | UP_ROTATION | UP_LEFT;
            memcpy(p.next_pos, ms->next_pos, sizeof(p.next_pos));
            p.next_rot[0] = ms_rot.x; p.next_rot[1] = ms_rot.y; p.next_rot[2] = ms_rot.z; p.next_rot[3] = ms_rot.w;
            p.next_left = 0;
        }
        bool turn_to_move = false;                           /* heading gate (movement.c:2323-2335) */
        pquat travel_dir = ms_rot;
        const bool gated = state == ST_MOVING || state == ST_SEEK_ENEMIES || state == ST_SURROUND || state == ST_ENTER_RANGE;
        if(v2_len(new_vel) > EPS && gated) {
            travel_dir = dir_quat_from_velocity(v2_len(vdes) > EPS ? vdes : new_vel);
            const float heading_err = (float)fabs((double)quat_pitch_diff(ms_rot, travel_dir) * (180.0f / PFO_PI_D));
            const float tolerance = (v2_len(ms_vel) > EPS) ? 90.0f : 10.0f;
            if(heading_err > tolerance) { turn_to_move = true; new_vel = (v2){0.0f, 0.0f}; }
        }
        v2 new_pos_xz = v2_add(curr_xz, new_vel);
        const bool still = state == ST_ARRIVED || state == ST_WAITING;
        if(a->flags & FL_GARRISONED) {
            if(!still) { p.flags |= UP_STATE; p.next_state = ST_ARRIVED; p.next_block = 0; }
            out[wi] = p;
            continue;
        }
        bool dummy, on_blocked, np_path, np_blocked;
        probe(m, curr_xz.x, curr_xz.z, &dummy, &on_blocked);
        probe(m, new_pos_xz.x, new_pos_xz.z, &np_path, &np_blocked);
        if(v2_len(new_vel) > 0 && np_path && (on_blocked || !np_blocked)) {
            /* unit_height (movement.c:2198) with M_HeightAtPoint == 0 (terrain height is render state) */
            const float y = (a->flags & FL_WATER) ? 0.0f : (a->flags & FL_AIR) ? 20.0f : 0.0f;
            p.flags |= UP_PREV_POS | UP_NEXT_POS | UP_STEP | UP_LEFT;
            memcpy(p.next_ppos, ms->next_pos, sizeof(p.next_ppos));
            p.next_npos[0] = new_pos_xz.x; p.next_npos[1] = y; p.next_npos[2] = new_pos_xz.z;
            p.next_step = 1.0f / (20 / w->hz);
            p.next_left = (float)((20 / w->hz) - 1);
            p.flags |= UP_POSITION;
            if((20 / w->hz) - 1 == 0) {
                p.next_pos[0] = new_pos_xz.x; p.next_pos[1] = y; p.next_pos[2] = new_pos_xz.z;
            }else{                                           /* interpolate_positions (movement.c:2221) */
                float ix, iy, iz;
                if(fabs(1.0 - (double)ms->step) < EPS) { ix = p.next_npos[0]; iy = p.next_npos[1]; iz = p.next_npos[2]; }
                else {
                    ix = p.next_ppos[0] + (p.next_npos[0] - p.next_ppos[0]) * ms->step;
                    iy = p.next_ppos[1] + (p.next_npos[1] - p.next_ppos[1]) * ms->step;
                    iz = p.next_ppos[2] + (p.next_npos[2] - p.next_ppos[2]) * ms->step;
                }
                new_pos_xz = (v2){ix, iz};
                p.next_pos[0] = ix; p.next_pos[1] = iy; p.next_pos[2] = iz;
            }
            p.flags |= UP_VELOCITY;
            p.next_velocity[0] = new_vel.x; p.next_velocity[1] = new_vel.z;
            p.flags |= UP_PREV_ROT | UP_NEXT_ROT | UP_ROTATION;
            p.next_prot[0] = ms_rot.x; p.next_prot[1] = ms_rot.y; p.next_prot[2] = ms_rot.z; p.next_prot[3] = ms_rot.w;
            v2 wma = {0.0f, 0.0f};                           /* orient_to_velocity_history (:2291) over vel_wma (:2067) */
            float denom = 0.0f;
            for(int i = 0; i < PFO_HIST; i++) {
                const int k = (ms->vel_hist_idx + i) % PFO_HIST;
                const float wgt = (float)(PFO_HIST - i);
                wma.x = wma.x + ms->vel_hist[k][0] * wgt;
                wma.z = wma.z + ms->vel_hist[k][1] * wgt;
                denom += wgt;
            }
            if(denom > EPS) { const float inv = 1.0f / denom; wma.x = wma.x * inv; wma.z = wma.z * inv; }
            pquat nrot = ms_rot;
            if(v2_len(wma) > EPS) nrot = turn_toward(ms_rot, dir_quat_from_velocity(wma), turn_rate);
            p.next_nrot[0] = nrot.x; p.next_nrot[1] = nrot.y; p.next_nrot[2] = nrot.z; p.next_nrot[3] = nrot.w;
            p.next_rot[0] = ms_rot.x; p.next_rot[1] = ms_rot.y; p.next_rot[2] = ms_rot.z; p.next_rot[3] = ms_rot.w;
        }else{
            p.flags |= UP_VELOCITY;
            p.next_velocity[0] = 0.0f; p.next_velocity[1] = 0.0f;
            const bool held = (a->flags & FL_COMBAT_HELD) != 0;
            if(held || turn_to_move) {
                p.flags |= UP_PREV_ROT | UP_NEXT_ROT | UP_ROTATION | UP_TURNING_IN_PLACE;
                const pquat cf = {ms->combat_facing[0], ms->combat_facing[1], ms->combat_facing[2], ms->combat_facing[3]};
                const pquat nrot = turn_toward(ms_rot, held ? cf : travel_dir, turn_rate);
                p.next_prot[0] = ms_rot.x; p.next_prot[1] = ms_rot.y; p.next_prot[2] = ms_rot.z; p.next_prot[3] = ms_rot.w;
                p.next_nrot[0] = nrot.x; p.next_nrot[1] = nrot.y; p.next_nrot[2] = nrot.z; p.next_nrot[3] = nrot.w;
                p.next_rot[0] = ms_rot.x; p.next_rot[1] = ms_rot.y; p.next_rot[2] = ms_rot.z; p.next_rot[3] = ms_rot.w;
            }
        }
        bool cur_path, cur_blk;                              /* stuck on non-pathable terrain: keep the state (:2417) */
        probe(m, new_pos_xz.x, new_pos_xz.z, &cur_path, &cur_blk);
        if(!cur_path) { out[wi] = p; continue; }

        const bool has_fid = (fs.flags & FORM_HAS_FORMATION) != 0;
        const bool ready = (fs.flags & FORM_ASSIGNMENT_READY) != 0;
        switch(state) {
        case ST_MOVING:
        case ST_MOVING_IN_FORMATION:                         /* movement.c:2421-2500 */
            if(has_fid && !ready) break;                     /* wait for the formation's cell assignment */
            if(has_fid && (fs.flags & FORM_ASSIGNED_TO_CELL) && (fs.flags & FORM_IN_RANGE_OF_CELL)) {
                set_state(&p, ST_ARRIVING_TO_CELL, 0);
                break;
            }
            if(a->flock < 0) break;
            if(entity_arrived(w, a, uid, &arr[a->flock], new_pos_xz, curr_xz)) set_state(&p, ST_ARRIVED, 1);
            else if(v2_len(vdes) < EPS) set_state(&p, ST_WAITING, 1);
            break;
        case ST_SEEK_ENEMIES:                                /* movement.c:2501: retried every tick */
            break;
        case ST_SURROUND:                                    /* movement.c:2505-2567 */
            if(ex.surround_target_uid == NULL_UID) set_state(&p, ST_ARRIVED, 1);
            else p.engine_todo |= TODO_SURROUND_QUERY;       /* the target's geometry is the engine's (deviation 4) */
            break;
        case ST_ENTER_RANGE: {                               /* movement.c:2569-2603 */
            if(ex.surround_target_uid == NULL_UID) { set_state(&p, ST_ARRIVED, 1); break; }
            const pfo_agent *t = &w->agents[ex.surround_target_uid];
            const v2 xz_target = {t->pos[0], t->pos[1]};
            bool in_range = v2_len(v2_sub(new_pos_xz, xz_target)) <= ex.target_range;
            /* M_NavIsAdjacentToImpassable && M_NavIsMaximallyClose(.., tolerance 0.0f) (movement.c:2584) */
            if(!in_range && tarr && adjacent_to_impassable(m, new_pos_xz)) in_range = maximally_close(&tarr[wi], new_pos_xz, 0.0f);
            if(in_range) { set_state(&p, ST_WAITING, 1); break; }
            if(v2_len(v2_sub(xz_target, (v2){ex.target_prev_pos[0], ex.target_prev_pos[1]})) > 5.0f) {
                /* the target moved: re-issue the move order towards it (G_Move_SetDest, attack = false) */
                p.flags |= UP_DEST | UP_TARGET_PREV;
                p.next_dest[0] = xz_target.x; p.next_dest[1] = xz_target.z; p.next_attack = 0;
                p.next_target_prev[0] = xz_target.x; p.next_target_prev[1] = xz_target.z;
            }
            break;
        }
        case ST_TURNING: {                                   /* movement.c:2605-2627 */
            const pquat ent_rot = {ex.rot[0], ex.rot[1], ex.rot[2], ex.rot[3]};
            const pquat tdir = {ex.target_dir[0], ex.target_dir[1], ex.target_dir[2], ex.target_dir[3]};
            const float degrees = (float)((double)quat_pitch_diff(ent_rot, tdir) * (180.0f / PFO_PI_D));
            if(fabs((double)degrees) <= 5.0f) { set_state(&p, ST_ARRIVED, 1); break; }
            const pquat r = turn_toward(ent_rot, tdir, turn_rate);
            p.flags |= UP_ROTATION | UP_PREV_ROT;
            p.next_rot[0] = r.x; p.next_rot[1] = r.y; p.next_rot[2] = r.z; p.next_rot[3] = r.w;
            p.next_prot[0] = r.x; p.next_prot[1] = r.y; p.next_prot[2] = r.z; p.next_prot[3] = r.w;
            break;
        }
        case ST_WAITING:                                     /* movement.c:2630-2645: the countdown, then the old state */
            p.wait_ticks_left = ex.wait_ticks_left - 1;
            if(p.wait_ticks_left == 0) { p.flags |= UP_MOVING; p.next_state = ex.wait_prev; }
            break;
        case ST_ARRIVING_TO_CELL:                            /* movement.c:2648-2670 */
            if(!has_fid) { set_state(&p, ST_MOVING, 0); break; }
            if(!ready) break;
            if(!(fs.flags & FORM_IN_RANGE_OF_CELL)) { set_state(&p, ST_MOVING_IN_FORMATION, 0); break; }
            if(fs.flags & FORM_ARRIVED_AT_CELL) {
                set_state(&p, ST_TURNING, 0);
                p.flags |= UP_TARGET_DIR;
                memcpy(p.next_target_dir, fs.target_orientation, sizeof(p.next_target_dir));
            }
            break;
        default:                                             /* ST_ARRIVED */
            break;
        }
        /* ent_update_using_surround_field (movement.c:2672-2691), on the tick's snapshot positions, for the state the
         * entity is in after this update: start using the surround field inside a third of a chunk of the target, stop
         * outside half a chunk */
        const uint32_t after = (p.flags & (UP_STATE | UP_MOVING)) ? (uint32_t)p.next_state : state;
        if(after == ST_SURROUND && ex.surround_target_uid != NULL_UID) {
            const pfo_agent *t = &w->agents[ex.surround_target_uid];
            const float dx = (float)fabs((double)(t->pos[0] - curr_xz.x)), dz = (float)fabs((double)(t->pos[1] - curr_xz.z));
            const float low = (float)(256.0 / 3.0f), high = (float)(256.0 / 2.0f);
            if(!ex.using_surround_field) { if(dx < low && dz < low) p.engine_todo |= TODO_USE_SURROUND_FIELD; }
            else if(dx >= high || dz >= high) p.engine_todo |= TODO_DROP_SURROUND_FIELD;
        }
        out[wi] = p;
    }
}

/* The movestate part of entity_apply_update (movement.c:2693-2757) for one patch: the waiting countdown, the state
 * (entity_finish_moving, movement.c:685, clears the velocity and a stop to WAITING records the state it leaves and
 * WAIT_TICKS), velocity + velocity history (update_vel_hist :2025, seed_vel_hist_facing :2046 / facing_dir :2040),
 * interpolation fields, rotations, the ENTER_ENTITY_RANGE / TURNING targets, SET_MOVING (move_notify_motion_start wipes
 * the history unless combat-held) and the surround-field bit. agents / mss / exts are updated in place. */
void pfo_entity_apply(pfo_agent *agents, pfo_movestate *mss, pfo_movestate_ext *exts, const uint32_t *work, size_t nwork,
                      const pfo_patch *patches)
{
    const float EPS = 1.0f / 1024;
    for(size_t wi = 0; wi < nwork; wi++) {
        pfo_agent *a = &agents[work[wi]];
        pfo_movestate *ms = &mss[work[wi]];
        pfo_movestate_ext *ex = exts ? &exts[work[wi]] : NULL;
        const pfo_patch *p = &patches[wi];
        if(a->flags & FL_GARRISONED) continue;                                   /* movement.c:2697 */
        if(ex) ex->wait_ticks_left = p->wait_ticks_left;
        if(p->flags & UP_STATE) {
            if(p->next_state == ST_ARRIVED || p->next_state == ST_WAITING) {
                if(ex && p->next_state == ST_WAITING) { ex->wait_prev = (int32_t)a->state; ex->wait_ticks_left = WAIT_TICKS; }
                a->velocity[0] = 0.0f; a->velocity[1] = 0.0f;
            }
            a->state = (uint32_t)p->next_state;
        }
        if(p->flags & UP_VELOCITY) {
            a->velocity[0] = p->next_velocity[0]; a->velocity[1] = p->next_velocity[1];
            if(p->flags & UP_TURNING_IN_PLACE) {
                memset(ms->vel_hist, 0, sizeof(ms->vel_hist));
            }else{
                bool empty = true;
                for(int i = 0; i < PFO_HIST; i++)
                    if(sqrtf(ms->vel_hist[i][0] * ms->vel_hist[i][0] + ms->vel_hist[i][1] * ms->vel_hist[i][1]) > EPS) empty = false;
                const float vl = sqrtf(a->velocity[0] * a->velocity[0] + a->velocity[1] * a->velocity[1]);
                if(empty && vl > EPS) {
                    const float theta = (float)(2.0 * atan2((double)ms->next_rot[1], (double)ms->next_rot[3]));
                    const float dx = (float)(-sin((double)theta)), dz = (float)cos((double)theta);
                    for(int i = 0; i < PFO_HIST; i++) { ms->vel_hist[i][0] = dx * vl; ms->vel_hist[i][1] = dz * vl; }
                }
                ms->vel_hist[ms->vel_hist_idx][0] = a->velocity[0]; ms->vel_hist[ms->vel_hist_idx][1] = a->velocity[1];
                ms->vel_hist_idx = (ms->vel_hist_idx + 1) % PFO_HIST;
            }
        }
        if(p->flags & UP_POSITION) { a->pos[0] = p->next_pos[0]; a->pos[1] = p->next_pos[2]; }
        if(p->flags & UP_PREV_POS) { a->prev_pos[0] = p->next_ppos[0]; a->prev_pos[1] = p->next_ppos[2]; }
        if(p->flags & UP_NEXT_POS) memcpy(ms->next_pos, p->next_npos, sizeof(ms->next_pos));
        if(p->flags & UP_STEP) ms->step = p->next_step;
        if(p->flags & UP_LEFT) ms->left = (int)p->next_left;
        if(p->flags & UP_NEXT_ROT) memcpy(ms->next_rot, p->next_nrot, sizeof(ms->next_rot));
        if(ex) {
            if(p->flags & UP_ROTATION) memcpy(ex->rot, p->next_rot, sizeof(ex->rot));                  /* Entity_SetRot */
            if(p->flags & UP_TARGET_PREV) memcpy(ex->target_prev_pos, p->next_target_prev, sizeof(ex->target_prev_pos));
            if(p->flags & UP_TARGET_DIR) memcpy(ex->target_dir, p->next_target_dir, sizeof(ex->target_dir));
        }
        if(p->flags & UP_MOVING) {
            if(!(a->flags & FL_COMBAT_HELD)) memset(ms->vel_hist, 0, sizeof(ms->vel_hist));
            a->state = (uint32_t)p->next_state;
        }
        if(ex && a->state == ST_SURROUND) {
            if(p->engine_todo & TODO_USE_SURROUND_FIELD) ex->using_surround_field = 1;
            if(p->engine_todo & TODO_DROP_SURROUND_FIELD) ex->using_surround_field = 0;
        }
    }
}
