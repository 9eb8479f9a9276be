/*
 * oracle/pf_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement ("port") of the reference algorithms on the hot path, in plain C99. It is the
 * checker for the CUDA path when the compiled reference (oracle/_ref) is not at hand, and is
 * itself pinned against oracle/_ref and the committed golden vectors (tests/test_oracle.py).
 * Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may
 * load it; libpfnav.so never links or calls anything here.
 *
 * Request structs are layout-identical to include/pfnav.h so that one numpy record array feeds
 * both sides.
 */
#ifndef PF_ORACLE_H
#define PF_ORACLE_H
#include <stddef.h>
#include <stdint.h>

typedef struct pfo_map {
    int chunk_w, chunk_h;
    float map_x, map_z;
    const uint8_t  *cost;            /* [chunks][64][64], one layer */
    const uint16_t *blockers;        /* may be NULL (all zero) */
    const uint16_t *local_islands;   /* may be NULL when no TARGET_PORTAL request is made */
    const uint8_t  *factions;        /* [chunks][15][64][64] per-faction blocker refcounts, may be NULL */
    uint16_t enemies[16];            /* enemies[f] = bit mask of the factions at war with f (field.c:151) */
} pfo_map;

typedef struct pfo_field_req {       /* == pfnav_field_req */
    int32_t chunk_r, chunk_c, layer, faction_id, target_type, init, tile_r, tile_c;
    int16_t port_r0, port_c0, port_r1, port_c1, next_r0, next_c0, next_r1, next_c1;
    int32_t next_chunk_r, next_chunk_c;
    uint16_t port_iid, next_iid;
    int32_t _pad;
} pfo_field_req;

typedef struct pfo_los_req {         /* == pfnav_los_req */
    int32_t chunk_r, chunk_c, layer, faction_id, tgt_chunk_r, tgt_chunk_c, tgt_tile_r, tgt_tile_c;
    int32_t prev_index, prev_chunk_r, prev_chunk_c, _pad;
} pfo_los_req;

typedef struct pfo_agent {           /* == pfnav_agent */
    float pos[2], prev_pos[2], velocity[2], vdes[2];
    float radius, max_speed, speed;
    uint32_t state, flags;
    int32_t flock;
    uint32_t has_dest_los, _pad;
} pfo_agent;

typedef struct pfo_flock {           /* == pfnav_flock */
    float target[2];
    int32_t dest, layer;
} pfo_flock;

/* N_FlowFieldInit + N_FlowFieldUpdate, TARGET_TILE / TARGET_PORTAL (field.c:2020-2083) */
void pfo_flow_fields_update(const pfo_map *map, const pfo_field_req *reqs, size_t n, uint8_t *inout);
/* N_LOSFieldCreate (field.c:2085-2245); requests may chain through prev_index */
void pfo_los_fields_create(const pfo_map *map, const pfo_los_req *reqs, size_t n, uint8_t *out);

/* Position index + velocity update (position.c:379, bitmap_grid.h:1376; movement.c:3395-3466;
 * clearpath.c:694). Agents are indexed by uid; cohesion sums flock members in ascending uid. */
typedef struct pfo_world pfo_world;
pfo_world *pfo_world_create(const pfo_map *map, const pfo_agent *agents, size_t n,
                            const pfo_flock *flocks, size_t nflocks, int hz);
void pfo_world_destroy(pfo_world *w);
/* The inputs of the states beyond point seeking, per uid (layout-identical to pfnav_formation_in / pfnav_movestate_ext):
 * struct formation_state + cell_pos + cell_arrival_vdes of struct move_work_in (movement.c:215-225, 264-276) and the
 * rest of struct movestate (movement.c:146-215). Either may be NULL: no formation / NULL_UID targets, zero counters. The
 * world keeps the pointers; the caller keeps the arrays alive. */
typedef struct pfo_formation {
    float cell_pos[2], cell_arrival_vdes[2], cohesion[2], align[2], drag[2], target_orientation[4];
    uint32_t flags, _pad;
} pfo_formation;
typedef struct pfo_movestate_ext {
    int32_t wait_prev, wait_ticks_left;
    uint32_t surround_target_uid, using_surround_field;
    float target_range, target_prev_pos[2], _padf, target_dir[4], rot[4];
} pfo_movestate_ext;
void pfo_world_set_states(pfo_world *w, const pfo_formation *forms, const pfo_movestate_ext *exts);
int  pfo_ents_in_circle(const pfo_world *w, float x, float z, float range, uint32_t *out, int maxout);
/* vdes / has_dest_los are taken from the agent records (for STATE_ARRIVING_TO_CELL the caller puts cell_arrival_vdes
 * there, ent_desired_velocity, movement.c:1507). The state picks the steering variant (movement.c:3414-3448).
 * out_vel/out_vpref: 2 floats per work item */
void pfo_velocity_work(const pfo_world *w, const uint32_t *work, size_t nwork, float *out_vel,
                       float *out_vpref);
/* G_ClearPath_NewVelocity (clearpath.c:694) then vec2_truncate(max_len) (movement.c:3464), as pfo_velocity_work runs it.
 * self5 / dyn5 / stat5: {px, pz, vx, vz, radius}; ndyn, nstat <= 32 */
void pfo_clearpath(const float *self5, const float *vpref2, const float *dyn5, int ndyn, const float *stat5, int nstat,
                   float max_len, float *out2);
/* inside_pcr (clearpath.c:249) over a ray table rays4 = [n_rays] {px, pz, dx, dz} (left, right per obstacle) */
void pfo_inside_pcr(const float *rays4, int n_rays, const float *pts2, long n, uint8_t *out);
/* C_InfiniteLineIntersection (collision.c:820): lines4 = [n][2] {px, pz, dx, dz}; out3 = {ok, x, z} */
void pfo_line_isect(const float *lines4, long n, float *out3);
/* N_DesiredPointSeekVelocity + N_HasDestLOS against caller-supplied fields: slot[dest*chunks+chunk]
 * indexes flow/los (4096 B each), -1 = absent (nav.c:3468, 4026, 3407) */
void pfo_desired_velocity(const pfo_map *map, const pfo_agent *agents, const pfo_flock *flocks,
                          const uint32_t *work, size_t nwork, const int32_t *slot,
                          const uint8_t *flow, const uint8_t *los, float *out_vdes, uint8_t *out_los);
/* Repair chain of N_DesiredPointSeekVelocity (nav.c:3508-3554): in-place updates of one cached field.
 * N_FlowFieldUpdateToNearestPathable (field.c:2247) / N_FlowFieldUpdateIslandToNearest (field.c:2307);
 * q = the request that built the field; gisl = global islands [chunks][64][64] */
void pfo_flow_update_nearest_pathable(const pfo_map *m, int chunk_r, int chunk_c, int start_r, int start_c, uint8_t *inout);
void pfo_flow_update_island_to_nearest(const pfo_map *m, const uint16_t *gisl, const pfo_field_req *q,
                                       uint16_t local_iid, uint8_t *inout);
/* n_set_cost_for_tile + n_make_cliff_edges (nav.c:267, 431): attrs int32[chunk_h*32][chunk_w*32][4]
 * = {pathable, type, base_height, ramp_height}; ref_layer = the reference's enum nav_layer (0..11);
 * out = cost_base [chunks][64][64] */
void pfo_cost_from_tiles(int chunk_w, int chunk_h, const int32_t *attrs, int ref_layer, uint8_t *out);
/* Region fields (dim x dim tiles around `center`, two directions per byte; absolute tile coordinates
 * = chunk * 64 + tile; seeds / overlay = (r, c) pairs): N_CellArrivalFieldCreate (field.c:2445, cell_mode 1),
 * N_GroupArrivalFieldCreate (field.c:2525) and N_CellArrivalFieldUpdateToNearestPathable (field.c:2603) */
void pfo_region_field_create(const pfo_map *m, int dim, uint16_t enemies, int cell_mode, const int32_t *seeds, int nseeds,
                             int center_r, int center_c, const int32_t *overlay, int noverlay, uint8_t *out);
void pfo_group_arrival_field(const pfo_map *m, int dim, uint16_t enemies, const float *targets_xz, int ntargets,
                             const float *center_xz, const int32_t *overlay, int noverlay, uint8_t *out);
void pfo_region_field_update_to_nearest_pathable(const pfo_map *m, int dim, int start_r, int start_c, int center_r, int center_c,
                                                 const int32_t *overlay, int noverlay, uint8_t *inout);
/* State update: entity_compute_update (movement.c:2303-2670), all nine movement states. Records are layout-identical to
 * pfnav_movestate / pfnav_patch (160 B, struct movestate_patch, movement.c:245-262). arr[flock]: the two map searches of
 * arrived() (movement.c:2170) for the flock's target: N_ClosestPathable (nav.c:4126) and the tile centres
 * N_IsMaximallyClose compares with (nav.c:4707, n_closest_island_tiles :1226), mc = 2 floats per tile. tarr[work item]
 * (may be NULL): the same tile centres for the target entity's position of a STATE_ENTER_ENTITY_RANGE item
 * (movement.c:2584). The STATE_WAITING countdown is reported in the patch's wait_ticks_left, the movestate_ext records
 * are not modified. out: one patch per work item. */
typedef struct pfo_movestate {
    float next_pos[3], step, next_rot[4], combat_facing[4], vel_hist[14][2];
    int32_t left, vel_hist_idx, _pad[2];
} pfo_movestate;
typedef struct pfo_patch {
    uint32_t flags; int32_t next_state, next_block, next_attack;
    float next_velocity[2], next_pos[3], next_rot[4], next_ppos[3], next_npos[3], next_step, next_left, next_nrot[4], next_prot[4];
    int32_t wait_ticks_left; uint32_t engine_todo; float _padf;
    float next_dest[2], next_target_prev[2], next_target_dir[4];
} pfo_patch;
typedef struct pfo_arrival { int32_t nearest_ok; float nearest[2]; int32_t mc_n; const float *mc; } pfo_arrival;
void pfo_entity_updates(const pfo_world *w, const pfo_movestate *mss, const pfo_arrival *arr, const pfo_arrival *tarr,
                        const uint32_t *work, size_t nwork, const float *new_vel_xz, const float *vdes_xz, pfo_patch *out);
/* the movestate part of entity_apply_update (movement.c:2693-2757), in place on agents / movestate / movestate_ext records
 * (exts may be NULL) */
void pfo_entity_apply(pfo_agent *agents, pfo_movestate *mss, pfo_movestate_ext *exts, const uint32_t *work, size_t nwork,
                      const pfo_patch *patches);
/* TARGET_ZONE chunk fields: N_FlowFieldUpdate -> field_update_zone (field.c:2050, 1810), its seed flood
 * field_zone_initial_frontier (field.c:1683) and the per-entity consumer N_DesiredGroupArrivalVelocity (nav.c:3561).
 * centre in absolute tile coordinates; inout = 64 x 64 direction bytes of chunk (chunk_r, chunk_c). */
int  pfo_zone_seeds(const pfo_map *m, int chunk_r, int chunk_c, int centre_r, int centre_c, int radius, int32_t *out);
void pfo_chunk_field_seeded(const pfo_map *m, int chunk_r, int chunk_c, const int32_t *seeds, int ns, uint8_t *inout);
void pfo_flow_field_zone(const pfo_map *m, int chunk_r, int chunk_c, int centre_r, int centre_c, int radius, uint8_t *inout);
void pfo_group_arrival_velocity(const pfo_map *m, const uint8_t *fields, const uint8_t *has, const float *centre_xz, int radius,
                                const float *pos_xz, int n, float *out_vel, uint8_t *out_flags);
#endif
