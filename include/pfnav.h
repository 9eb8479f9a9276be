/*
 * pfnav.h -- C ABI of libpfnav.so: the H100 (sm_90a) implementation of permafrost-engine's
 * per-tick navigation + crowd-movement hot path.
 *
 * Plain C, plain pointers and sizes; no CUDA or torch types in any signature (streams are passed
 * as an opaque `void*` that is a cudaStream_t / CUstream, NULL = the legacy default stream).
 * All functions return 0 on success and a negative pfnav_status on failure;
 * pfnav_last_error() returns a thread-local human-readable message.  There is NO CPU fallback:
 * if no sm_90 (H100) device is usable, pfnav_create() fails.
 *
 * Each entry point cites the reference interface (file:line under the reference checkout) that
 * it replaces; INTEGRATION.md shows the binding a maintainer adds on the engine side.
 *
 * Conventions (identical to the reference):
 *   - a map is chunk_w x chunk_h chunks; a chunk is 64x64 nav tiles (FIELD_RES_R/C,
 *     src/navigation/nav_data.h:45-46); a nav tile is 4x4 world units; chunk = 256x256 wu.
 *   - world X DEcreases with the column index, Z increases with the row index
 *     (src/map/tile.c:547-592); map_pos is the (x,z) of the top-left corner.
 *   - chunk-blocked grids are [chunk_r][chunk_c][64][64], the order of N_CopyCostBasePacked
 *     (src/navigation/nav.c:2432).
 *   - a flow field is 4096 bytes, one `dir_idx` (enum flow_dir 0..8, nav.h:94-104) per tile,
 *     byte-identical to `struct flow_field::field` (src/navigation/field.h:103-109).
 *   - a LOS field is 4096 bytes, bit0 = visible, bit1 = wavefront_blocked, byte-identical to
 *     `struct LOS_field::field` (field.h:48-54).
 */
#ifndef PFNAV_H
#define PFNAV_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define PFNAV_FIELD_RES        64
#define PFNAV_FIELD_TILES      4096
#define PFNAV_COST_IMPASSABLE  0xff     /* nav_data.h:47 */
#define PFNAV_ISLAND_NONE      0xffff   /* nav_data.h:48 */
#define PFNAV_FACTION_ID_NONE  0xf      /* nav_data.h:49 */
#define PFNAV_NAV_LAYER_MAX    12       /* nav.h:78-92 */
#define PFNAV_MAX_NEIGHBOURS   32       /* movement.c:437 */

typedef enum pfnav_status {
    PFNAV_OK            =  0,
    PFNAV_ERR_ARG       = -1,
    PFNAV_ERR_CUDA      = -2,
    PFNAV_ERR_NO_DEVICE = -3,
    PFNAV_ERR_STATE     = -4,
    PFNAV_ERR_NOMEM     = -5
} pfnav_status;

/* enum flow_dir, src/navigation/public/nav.h:94-104 */
enum pfnav_flow_dir { PFNAV_FD_NONE = 0, PFNAV_FD_NW, PFNAV_FD_N, PFNAV_FD_NE, PFNAV_FD_W,
                      PFNAV_FD_E, PFNAV_FD_SW, PFNAV_FD_S, PFNAV_FD_SE };

/* field_target.type, src/navigation/field.h:78-91 (only the chunk-local kinds) */
enum pfnav_target_type { PFNAV_TARGET_PORTAL = 0, PFNAV_TARGET_TILE = 1 };

typedef struct pfnav_ctx pfnav_ctx;

/* ---------------------------------------------------------------------------------------- */
/* Context + map state (replaces struct nav_private / nav_chunk, nav_private.h:52, nav_data.h:118)
 * ---------------------------------------------------------------------------------------- */

const char *pfnav_last_error(void);
int  pfnav_version(void);

/* device: CUDA ordinal. Fails (PFNAV_ERR_NO_DEVICE) without a usable GPU. */
/* Streams: every `void *stream` argument is a cudaStream_t. NULL names the context's own
 * non-blocking stream -- NOT the legacy default stream (work queued there would not be ordered
 * against the context's stream). Calls on one stream are ordered as issued. */
int  pfnav_create(int device, pfnav_ctx **out);
void pfnav_destroy(pfnav_ctx *ctx);

/* N_NewCtxForMapData (nav.c:2284): allocate device grids for chunk_w x chunk_h chunks and
 * `nlayers` navigation layers (cost_base u8, blockers u16, local_islands u16 per layer). */
int  pfnav_map_create(pfnav_ctx *ctx, int chunk_w, int chunk_h, int nlayers,
                      float map_x, float map_z);

/* map->pos: the world (x, z) of the map's top-left corner, when it is only known after the grids (a caller that
 * mirrors an existing nav context learns it with the first world-space call). Grids are unaffected. */
int  pfnav_map_set_pos(pfnav_ctx *ctx, float map_x, float map_z);

/* Upload one layer from HOST chunk-blocked arrays ([chunk_r][chunk_c][64][64]).
 * blockers / local_islands may be NULL (treated as all 0 / left unchanged).
 * Same packed layout as N_CopyCostBasePacked / N_CopyBlockersPacked (nav.c:2432, 2462). */
int  pfnav_map_upload_layer(pfnav_ctx *ctx, int layer, const uint8_t *cost_base,
                            const uint16_t *blockers, const uint16_t *local_islands);

/* Cost pass of N_NewCtxForMapData for one layer ON THE DEVICE (nav.c:2311-2336): n_set_cost_for_tile
 * (nav.c:267) for every tile type incl. corner tiles (M_Tile_{NW,NE,SW,SE}Height, map/tile.c:117-180)
 * + n_make_cliff_edges (nav.c:431); blockers of the layer are cleared (nav.c:2332). Bit-exact.
 *   chunk_tiles[chunk_r*chunk_w + chunk_c] -> 32x32 records of `tile_stride` bytes whose first 16
 *   bytes are the head of the engine's `struct tile` (map/public/tile.h:101): bool pathable @0,
 *   enum tiletype @4, int base_height @8, int ramp_height @12. Pass the engine's own
 *   `const struct tile **chunk_tiles` with tile_stride = sizeof(struct tile) (36).
 *   ref_layer: the reference's enum nav_layer (0-3 ground, 4-7 water, 8-11 air; nav.h:78-92) whose
 *   pathability rule applies to `layer`. Follow with pfnav_map_build_nav(layer). */
int  pfnav_map_cost_from_tiles(pfnav_ctx *ctx, int layer, int ref_layer, const void *const *chunk_tiles,
                               size_t tile_stride);
/* PFMAP terrain ingestion (SURVEY.md 8f-4; docs/pfmap.txt). pfnav_tile is the head of the engine's `struct tile`
 * (map/public/tile.h:101) as pfnav_map_cost_from_tiles reads it (tile_stride = sizeof(pfnav_tile)).
 * pfnav_pfmap_parse: al_parse_pfmap_header (asset_load.c:168) + the material / splat lines + m_al_read_pfchunk /
 * m_al_parse_tile (map_asset_load.c:181, 103) over a memory image of the file. out_tiles = [chunk][32][32], chunks in
 * row-major order, cap_tiles records; NULL reads the header only. Malformed input -> PFNAV_ERR_ARG. Host only.
 * pfnav_map_load_pfmap: parse + pfnav_map_create(num_cols, num_rows, nlayers) + for every layer i the device cost
 * pass under the reference layer ref_layers[i] + pfnav_map_build_nav(i) -- N_NewCtxForMapData (nav.c:2284). */
typedef struct pfnav_tile { int32_t pathable, type, base_height, ramp_height; } pfnav_tile;
int  pfnav_pfmap_parse(const char *text, size_t len, int *out_chunk_rows, int *out_chunk_cols, pfnav_tile *out_tiles,
                       size_t cap_tiles);
int  pfnav_map_load_pfmap(pfnav_ctx *ctx, const char *text, size_t len, int nlayers, const int32_t *ref_layers,
                          float map_x, float map_z);
/* Read one layer's DEVICE grids back in the packed chunk-blocked layout of N_CopyCostBasePacked /
 * N_CopyBlockersPacked (nav.c:2432, 2462). Any out pointer may be NULL. */
int  pfnav_map_get_layer(pfnav_ctx *ctx, int layer, uint8_t *cost_base, uint16_t *blockers,
                         uint16_t *local_islands);

/* Sparse update of one chunk (what N_BlockersIncref/Decref + N_Update change, nav.c:4663-4705,
 * 2119): any pointer may be NULL to keep that grid. HOST pointers, [64][64] each. */
int  pfnav_map_update_chunk(pfnav_ctx *ctx, int layer, int chunk_r, int chunk_c,
                            const uint8_t *cost_base, const uint16_t *blockers,
                            const uint16_t *local_islands);

/* Structural part of N_NewCtxForMapData for one layer (nav.c:2284), computed on the host from the
 * uploaded cost_base + blockers: local islands (n_update_local_islands, nav.c:967: ids from 1 in
 * row-major discovery order) and the portal table (n_create_portals / n_link_chunks, nav.c:563,
 * 477: identical indices and endpoints). The islands are pushed to the device. */
int  pfnav_map_build_nav(pfnav_ctx *ctx, int layer);
/* n_update_dirty_local_islands (nav.c:986) for one chunk after pfnav_map_update_chunk changed
 * its blockers; pushes the refreshed islands to the device. */
int  pfnav_map_refresh_chunk(pfnav_ctx *ctx, int layer, int chunk_r, int chunk_c);
/* Read back: local islands ([chunk][64][64] u16) and portals (10 ints per portal: chunk_r, chunk_c,
 * index, endpoints[0].r/.c, endpoints[1].r/.c, connected chunk index, connected portal index, 0). */
int  pfnav_local_islands_get(pfnav_ctx *ctx, int layer, uint16_t *out);
int  pfnav_portals_get(pfnav_ctx *ctx, int layer, int32_t *out, int maxout, int *out_n);

/* "Attacking" requests (N_RequestPathAttacking, nav.c:3393): a field / LOS request whose faction_id is not
 * PFNAV_FACTION_ID_NONE treats a blocked tile as passable when every faction holding a blocker refcount on it
 * is at war with the requesting faction (field_tile_passable_no_enemies, field.c:179).
 *   pfnav_set_enemy_factions: G_GetEnemyFactions (game.h:184), bit i of the mask = faction i is an enemy.
 *   pfnav_map_upload_factions: chunk->factions of one layer, u8 [chunk][15][64][64]; pfnav_blockers_incref /
 *   decref maintain the same counts when given a faction id in 0..14 (nav.c:1032). */
int  pfnav_set_enemy_factions(pfnav_ctx *ctx, int faction_id, uint16_t enemies_mask);
int  pfnav_map_upload_factions(pfnav_ctx *ctx, int layer, const uint8_t *factions);
/* N_BlockersIncref / N_BlockersDecref (nav.c:4663-4683): reference-count the tiles under a circle
 * (M_Tile_AllUnderCircle, tile.c:687) plus 1/2/3 contour rings (M_Tile_Contour, tile.c:759) for the
 * 3x3/5x5/7x7 layers, on the ground AND water layers for non-air entities, air layers otherwise.
 * Layers the context does not hold are skipped. Host-side; the device sees the change at commit. */
int  pfnav_blockers_incref(pfnav_ctx *ctx, float x, float z, float range, int faction_id, uint32_t flags);
int  pfnav_blockers_decref(pfnav_ctx *ctx, float x, float z, float range, int faction_id, uint32_t flags);
/* N_BlockersIncrefOBB / N_BlockersDecrefOBB (nav.c:4685-4705): building footprints. corners_xz = the bottom
 * face of the engine's `struct obb`: corners[0], [1], [5], [4] as 4 (x, z) pairs (M_Tile_AllUnderObj,
 * tile.c:594-599). All four corners must lie inside the map. */
int  pfnav_blockers_incref_obb(pfnav_ctx *ctx, const float *corners_xz, int faction_id, uint32_t flags);
int  pfnav_blockers_decref_obb(pfnav_ctx *ctx, const float *corners_xz, int faction_id, uint32_t flags);
/* a tick's worth of the two calls above, applied in order (delta = +1 incref, -1 decref) */
typedef struct pfnav_blocker_op { float x, z, range; int32_t faction_id; uint32_t flags; int32_t delta; } pfnav_blocker_op;
int  pfnav_blockers_batch(pfnav_ctx *ctx, const pfnav_blocker_op *ops, size_t n);
int  pfnav_blockers_get(pfnav_ctx *ctx, int layer, uint16_t *out);
/* nav_chunk::factions of one layer: out = u8 [chunks][15][64][64] */
int  pfnav_blockers_get_factions(pfnav_ctx *ctx, int layer, uint8_t *out);
/* N_Update + N_ApplyDeferredInvalidations (nav.c:2119-2223): for every chunk whose occupancy
 * changed, recompute the local islands, refresh the portal edge states, push the chunk's blockers +
 * islands to the device, and invalidate the pool: entries AT the chunk, and -- when an edge state
 * flipped -- every field of every destination routed THROUGH it (fieldcache.c:460-545).
 * The ops pfnav_agents_apply_updates_ex / pfnav_agents_set_blocking left on the device are applied here too, after the
 * host-queued ones; it reads their count back (and the few whose circle is wider than the device's bit window, which
 * take the host rasteriser). */
int  pfnav_map_commit(pfnav_ctx *ctx, int *out_ndirty);

/* ---------------------------------------------------------------------------------------- */
/* Flow fields + LOS fields (seam B2: src/navigation/field.h:115-202)
 * ---------------------------------------------------------------------------------------- */

/* One N_FlowFieldUpdate call (field.c:2030). 64 bytes. Mirrors struct field_work_in
 * (nav.c:126-131) with the portal_desc pointers resolved to plain coordinates. */
typedef struct pfnav_field_req {
    int32_t  chunk_r, chunk_c;      /* struct coord chunk_coord */
    int32_t  layer;                 /* enum nav_layer */
    int32_t  faction_id;            /* PFNAV_FACTION_ID_NONE for non-attacking paths */
    int32_t  target_type;           /* enum pfnav_target_type */
    int32_t  init;                  /* !=0: N_FlowFieldInit first (field.c:2020); 0: update the
                                     * existing `inout` field in place (nav.c:1998-2008) */
    /* TARGET_TILE: struct coord tile */
    int32_t  tile_r, tile_c;
    /* TARGET_PORTAL: struct portal_desc (field.h:68-73) */
    int16_t  port_r0, port_c0, port_r1, port_c1;   /* pd.port->endpoints[0..1] */
    int16_t  next_r0, next_c0, next_r1, next_c1;   /* pd.next->endpoints[0..1] */
    int32_t  next_chunk_r, next_chunk_c;           /* pd.next->chunk (== port->connected chunk) */
    uint16_t port_iid, next_iid;                   /* pd.port_iid, pd.next_iid */
    int32_t  _pad;
} pfnav_field_req;

/* Batch of N_FlowFieldUpdate (+ optional N_FlowFieldInit). reqs and inout_fields are HOST
 * buffers (inout_fields: n x 4096 bytes). Synchronous: results are in inout_fields on return. */
int  pfnav_flow_fields_update(pfnav_ctx *ctx, const pfnav_field_req *reqs, size_t n,
                              uint8_t *inout_fields);

/* Repair chain of N_DesiredPointSeekVelocity (nav.c:3508-3554) for an entity standing on a tile whose
 * cached direction is FD_NONE, applied in place to HOST fields (4096 bytes each):
 *   PFNAV_REPAIR_NEAREST_PATHABLE  N_FlowFieldUpdateToNearestPathable (field.c:2247): args[i] =
 *       start_r << 8 | start_c, a NON-passable tile of the chunk; directions lead out of the blocked blob
 *   PFNAV_REPAIR_ISLAND_TO_NEAREST N_FlowFieldUpdateIslandToNearest (field.c:2307): args[i] = the local
 *       island id cut off from the field's frontier; needs pfnav_route_build(layer) (global islands)
 * targets[i] = the request that built field i (its chunk, layer and target). */
enum pfnav_repair_kind { PFNAV_REPAIR_NEAREST_PATHABLE = 0, PFNAV_REPAIR_ISLAND_TO_NEAREST = 1 };
int  pfnav_flow_fields_repair(pfnav_ctx *ctx, const pfnav_field_req *targets, const int32_t *kinds,
                              const int32_t *args, size_t n, uint8_t *inout_fields);

/* Same, DEVICE-resident reqs / fields, asynchronous on `stream`. */
int  pfnav_flow_fields_update_dev(pfnav_ctx *ctx, const pfnav_field_req *d_reqs, size_t n,
                                  uint8_t *d_inout_fields, void *stream);

/* One N_LOSFieldCreate call (field.c:2085). 48 bytes. */
#define PFNAV_LOS_PREV_INPLACE (-3)
typedef struct pfnav_los_req {
    int32_t  chunk_r, chunk_c;          /* chunk the field is for */
    int32_t  layer;
    int32_t  faction_id;
    int32_t  tgt_chunk_r, tgt_chunk_c;  /* struct tile_desc target */
    int32_t  tgt_tile_r, tgt_tile_c;
    int32_t  prev_index;                /* -1: destination chunk (prev_los == NULL); >= 0: index,
                                         * within the same batch, of the request whose output is
                                         * prev_los (must be < this request's own index);
                                         * PFNAV_LOS_PREV_INPLACE (host API): prev_los is a field the
                                         * caller holds -- its 4096 bytes are passed in out_fields[i]
                                         * and replaced by the result (N_LOSFieldCreate's `prev`).  */
    int32_t  prev_chunk_r, prev_chunk_c;/* prev_los->chunk */
    int32_t  _pad;
} pfnav_los_req;

/* Batch of N_LOSFieldCreate. Requests are processed in dependency order (a request may name an
 * earlier one as its prev_los). HOST buffers; out_fields: n x 4096 bytes. */
int  pfnav_los_fields_create(pfnav_ctx *ctx, const pfnav_los_req *reqs, size_t n,
                             uint8_t *out_fields);
/* Same, DEVICE-resident d_reqs / d_out_fields (n x 4096 bytes, field i at block i), asynchronous on
 * `stream` (NULL: the context's own stream). The requests are taken in the caller's order, which
 * need not be sorted by depth. They are not validated on the host: prev_index must be -1 on the
 * destination chunk and an index < i elsewhere. PFNAV_LOS_PREV_INPLACE is for the host call only:
 * a device request off the destination chunk with a negative prev_index reads block _pad of
 * d_out_fields as its parent. A request that names itself or a later one as its parent never
 * finishes: the kernel waits on it.
 * h_wave_offsets[0 .. n_waves] is a HOST array, checked and otherwise unused: it must start at 0,
 * not decrease and end at n (PFNAV_ERR_ARG otherwise). LOS launches of one context run one after
 * another, on whatever streams they are queued. */
int  pfnav_los_fields_create_dev(pfnav_ctx *ctx, const pfnav_los_req *d_reqs, size_t n,
                                 uint8_t *d_out_fields, int n_waves, const int32_t *h_wave_offsets,
                                 void *stream);

/* Goal planner (the request-generation half of n_request_path, nav.c:1774-2047): emits, for every
 * chunk connected to the goal tile, the TARGET_TILE / TARGET_PORTAL flow request and the chained
 * LOS request that guide agents there. Breadth-first over (chunk, local island) nodes, i.e. it
 * minimises portal hops rather than AStar_PortalGraphPath's travel cost (a_star.c:429).
 *   flow_chunk[i] / los_chunk[i] : chunk index (r*chunk_w+c) a request's output belongs to
 *   flow_wave[i]                 : 0 for a chunk's first request (init=1); k>0 for the k-th further
 *                                  target merged into the same field (init=0, nav.c:1998-2008);
 *                                  wave k must run after wave k-1 on that chunk's field.
 *   los requests are emitted parent-before-child with prev_index into los_out. */
int  pfnav_plan_goal(pfnav_ctx *ctx, int layer, int tgt_chunk_r, int tgt_chunk_c, int tgt_tile_r,
                     int tgt_tile_c, pfnav_field_req *flow_out, int32_t *flow_chunk,
                     int32_t *flow_wave, int max_flow, int *n_flow, pfnav_los_req *los_out,
                     int32_t *los_chunk, int max_los, int *n_los);

/* Cost-faithful routing structure of one layer (after pfnav_map_build_nav): portal edges with
 * AStar_GridPath costs (nav.c:593, a_star.c:303), per-portal travel index (nav.c:1314), global
 * islands (nav.c:1731), edge states (nav.c:693). Host-side; bit-identical costs and ids. */
int  pfnav_route_build(pfnav_ctx *ctx, int layer);
int  pfnav_route_islands_get(pfnav_ctx *ctx, int layer, uint16_t *out);
/* edges of one portal, 3 u32 per edge {neighbour portal_ref, edge_state, cost float bits} */
int  pfnav_route_edges_get(pfnav_ctx *ctx, int layer, int chunk, int portal, uint32_t *out, int maxout,
                           int *out_n);
/* n_request_path (nav.c:1774-2047), request-generation half: the flow requests (with their
 * N_FlowFieldID, field.c:1952) and LOS requests, in the reference's order, that the path src -> dst
 * needs given what (dest, chunk) entries already exist: have_flow[chunk] = mapped ff_id or 0,
 * have_los[chunk] = 0/1. LOS prev_index: -1 destination chunk, >= 0 index in this batch, -2 the
 * previous chunk's field pre-exists (caller supplies it). *out_ok = the function's bool result. */
int  pfnav_route_request_path(pfnav_ctx *ctx, int layer, float src_x, float src_z, float dst_x,
                              float dst_z, const uint64_t *have_flow, const uint8_t *have_los,
                              pfnav_field_req *flow_out, uint64_t *flow_ffid, int32_t *flow_chunk,
                              int max_flow, int *n_flow, pfnav_los_req *los_out, int32_t *los_chunk,
                              int max_los, int *n_los, uint32_t *out_dest_id, int *out_ok);
/* N_RequestPathAttacking (nav.c:3393): the faction applied to the path requests that follow (route + pool
 * entry points); PFNAV_FACTION_ID_NONE restores N_RequestPath. It is packed into the dest_id (nav.c:853) and
 * forwarded to every flow / LOS request, which is all n_request_path does with it. */
int  pfnav_request_faction(pfnav_ctx *ctx, int faction_id);
/* N_RequestPath (nav.c:3386) against the device field pool: route src -> dst exactly as the
 * reference does and build, on the device, the fields the pool does not hold yet for `dest`
 * (cached (dest, chunk) entries and their ff_ids are honoured like the field cache's). */
int  pfnav_pool_request_path(pfnav_ctx *ctx, int dest, int layer, float src_x, float src_z,
                             float dst_x, float dst_z, void *stream, uint32_t *out_dest_id,
                             int *out_ok, int *out_n_flow, int *out_n_los);
/* N_RequestPath (nav.c:3386) for a batch of n requests on one layer against the device field pool. Equivalent, field
 * for field, to calling pfnav_pool_request_path(ctx, dests[i], layer, src_xz[2i], src_xz[2i+1], dst_xz[2i],
 * dst_xz[2i+1], ...) for i = 0 .. n-1 in order: a later request sees (reuses, merges into, chains its LOS onto) the
 * fields an earlier one produced. Per-request outputs may be NULL. Arguments are validated before anything changes
 * (PFNAV_ERR_ARG: nothing done). If the pool cannot hold request k's fields, requests 0 .. k-1 are done exactly as the
 * serial calls would have left them, *out_ndone = k and PFNAV_ERR_NOMEM is returned. Launches are asynchronous on
 * `stream`, like pfnav_pool_request_path's. The portal-graph searches of a large batch run on the device. */
int  pfnav_pool_request_paths(pfnav_ctx *ctx, int n, const int32_t *dests, int layer, const float *src_xz,
                              const float *dst_xz, void *stream, uint32_t *out_dest_ids, int32_t *out_ok,
                              int32_t *out_n_flow, int32_t *out_n_los, int *out_ndone);
/* Positions named by resident entities. pfnav_pool_request_paths_resident, pfnav_map_query_resident and
 * pfnav_group_arrival_velocity_resident take, in place of a host position, the uid of an entity of the device-resident
 * population, so that the device-resident loop issues orders, map queries and arrival velocities without reading
 * positions back (pfnav_agents_read_state). They share these rules:
 * - Equivalence: the call leaves everything exactly as the plain entry point (pfnav_pool_request_paths,
 *   pfnav_map_query, pfnav_group_arrival_velocity) leaves it when called with each named position replaced by the
 *   x, z of that entity's 24-byte record: pool, slots, ff_ids, LRU state, outputs, *out_ndone and the return code. On a
 *   single context after an index build that is the pos pfnav_agents_read_state reports. The plain call's rules then
 *   hold unchanged: a path endpoint off the map is PFNAV_ERR_ARG with nothing done, a query point off the map gives
 *   ok = 0, an arrival position off the map clears flag bit 0.
 * - Errors, in this order, with nothing changed and the outputs untouched: PFNAV_ERR_ARG for a uid not below the
 *   population, n not below 2^24, or a NULL array the rules of the call forbid; PFNAV_ERR_STATE when n > 0 and records
 *   were written since the last index build (as pfnav_ents_in_circles: the call goes after pfnav_agents_rebuild_index
 *   or a gather); then every error of the plain entry point.
 * - Multi-GPU: a job member resolves any uid (global uids) from its own record column, which the gather made whole, and
 *   answers as one context holding the whole population would. There is no job form and no collective.
 * - Host waits: map queries and arrival velocities wait only where the plain call does; path requests wait once more,
 *   to read the resolved endpoints back for the host route planner.
 * pfnav_pool_request_paths_resident: request i's source is the resident position of src_uids[i] unless src_uids is
 * NULL or src_uids[i] == PFNAV_NULL_UID; then it is src_xz[2i, 2i+1]. The same holds for the destination with
 * dst_uids / dst_xz. src_xz (dst_xz) may be NULL only when every src_uids (dst_uids) entry names a uid. */
int  pfnav_pool_request_paths_resident(pfnav_ctx *ctx, int n, const int32_t *dests, int layer,
                                       const uint32_t *src_uids, const float *src_xz, const uint32_t *dst_uids,
                                       const float *dst_xz, void *stream, uint32_t *out_dest_ids, int32_t *out_ok,
                                       int32_t *out_n_flow, int32_t *out_n_los, int *out_ndone);
/* Read one pool entry back (4096 B each, pointers may be NULL). *out_has: bit0 flow, bit1 LOS;
 * *out_ffid: the N_FlowFieldID currently mapped for (dest, chunk). */
int  pfnav_pool_get(pfnav_ctx *ctx, int dest, int chunk_r, int chunk_c, uint8_t *flow_out,
                    uint8_t *los_out, int *out_has, uint64_t *out_ffid);
/* Host-only context for the HOST-side structure code above (islands, portals, routing) on a
 * machine without a GPU. It has no compute path: kernel-launching entry points fail with
 * PFNAV_ERR_NO_DEVICE. */
int  pfnav_create_hostonly(pfnav_ctx **out);

/* Selects how the 64x64 tiles are staged into shared memory: 1 = TMA tensor maps
 * (cp.async.bulk.tensor), 0 = plain coalesced loads. Default 1. */
int  pfnav_set_tma(pfnav_ctx *ctx, int enable);

/* ---------------------------------------------------------------------------------------- */
/* Field pool: device-resident (dest_id, chunk) -> {flow field, LOS field}
 * (replaces the fieldcache lookups done per agent: fieldcache.c N_FC_GetDestFFMapping /
 *  N_FC_FlowFieldAt / N_FC_LOSFieldAt, called from nav.c:3483-3506, 4044-4052)
 * ---------------------------------------------------------------------------------------- */

/* Size the pool for `ndests` destinations (flocks). Slot table is ndests x chunks. */
int  pfnav_pool_create(pfnav_ctx *ctx, int ndests, int max_fields);
/* Store field bytes (HOST, 4096 each; either may be NULL) for (dest, chunk). */
int  pfnav_pool_put(pfnav_ctx *ctx, int dest, int chunk_r, int chunk_c,
                    const uint8_t *flow_field, const uint8_t *los_field);
/* Empty the pool. Does not block and queues no device work: the host mirrors are reset now, the device copies by the
 * next entry point that uses the pool, ordered on that call's stream. */
int  pfnav_pool_clear(pfnav_ctx *ctx);
/* N_RequestPath's field-building half (nav.c:1819-2042), resident on the device: plan the goal
 * (pfnav_plan_goal), then run the flow waves and the LOS chain straight into the pool slots of
 * destination `dest`. No field bytes cross PCIe. Launches are asynchronous on `stream`. */
int  pfnav_pool_request_goal(pfnav_ctx *ctx, int dest, int layer, int tgt_chunk_r, int tgt_chunk_c,
                             int tgt_tile_r, int tgt_tile_c, void *stream, int *out_n_flow,
                             int *out_n_los);
/* The same for a batch of goals (the reference runs up to 256 field tasks concurrently, nav.c:88):
 * the flow waves and the LOS dependency waves of all goals are launched together.
 * dests[ngoals]; targets: 4 ints per goal {chunk_r, chunk_c, tile_r, tile_c}. */
int  pfnav_pool_request_goals(pfnav_ctx *ctx, int ngoals, const int32_t *dests, int layer,
                              const int32_t *targets, void *stream, int *out_n_flow, int *out_n_los);
/* PFNAV_REQUEST_MISSING_ONLY: (dest, chunk) fields the pool still holds are kept -- the field cache's hit path
 * (fieldcache.c:138-141) -- and only the missing ones (never built, invalidated by pfnav_map_commit, or evicted)
 * are planned and built; a rebuilt LOS field reads a kept parent chunk's field out of the pool. */
#define PFNAV_REQUEST_MISSING_ONLY (1u << 0)
int  pfnav_pool_request_goals_ex(pfnav_ctx *ctx, int ngoals, const int32_t *dests, int layer, const int32_t *targets,
                                 uint32_t flags, void *stream, int *out_n_flow, int *out_n_los);
/* pfnav_pool_request_goals runs the LOS dependency chains on a context-owned stream so that work which
 * does not read fields (position index, cohesion) overlaps them; pfnav_agents_tick and the pool entry
 * points order themselves after it. A caller that reads pool LOS fields through raw device pointers
 * on its own stream calls this first. */
/* Test / tuning hook: LOS kernel variant, 0 = bit rows, 1 (default) = one state byte per tile. Same results. */
int  pfnav_set_los_variant(pfnav_ctx *ctx, int variant);
/* Profiling aid: per-field trace of the LOS launches. enable != 0 arms it for the following launches; with
 * out != NULL the trace of the last traced launch is returned first: out[4i..4i+3] = {taken, dependency
 * satisfied, finished} in %globaltimer nanoseconds and 1 + heap pops (0 = zero-filled early out). */
int  pfnav_los_trace(pfnav_ctx *ctx, int enable, unsigned long long *out, size_t cap, size_t *out_n);
int  pfnav_fields_join(pfnav_ctx *ctx, void *stream);
/* On-miss chain of N_DesiredPointSeekVelocity (nav.c:3484-3554) for the uploaded work list, against the pool:
 * every work agent whose own tile has no direction (field absent or FD_NONE) is collected on the device; per
 * (dest, chunk, local island | blocked tile), in work order, the host then (1) requests the path from that
 * agent's position (n_request_path, nav.c:3486/3499 == pfnav_pool_request_path), and if the tile is still
 * FD_NONE (2) repairs the field in place: N_FlowFieldUpdateToNearestPathable when the tile is non-passable,
 * N_FlowFieldUpdateIslandToNearest otherwise. Blocking; needs pfnav_route_build. The caller re-runs the tick. */
int  pfnav_pool_repair(pfnav_ctx *ctx, int *out_nrequests, int *out_nrepairs);
/* pfnav_pool_repair in device rounds: the same representatives, requests and repairs in the same order, leaving exactly
 * the pool pfnav_pool_repair leaves (flow and LOS bytes, `has` bits, ff_ids, slot mapping and LRU state, entity-field
 * footprints) and the same *out_nrequests / *out_nrepairs. The LOS-state requests are one request batch; the
 * desired-velocity requests and repairs run in rounds of one request batch and one launch of predicated repairs (a
 * repair applies only if its tile still has no direction when its turn comes); the enemy-seek / surround repairs are one
 * launch. A round ends only where a request's emission depends on a byte written earlier in the round, would write a
 * slot with a pending repair, or would evict. *out_nrounds: the rounds that launched work. Pointers may be NULL.
 * Ordered on `stream` (NULL: the context's stream) after forked field work and pfnav_pool_clear; it waits for the device
 * only when its scratch has to grow and to read back each phase's representatives and the bytes they stand on, at round boundaries (the round's request
 * upload and its gather) and once at the end, never per entity. Errors as
 * pfnav_pool_repair's: PFNAV_ERR_ARG (no agents / pool, pfnav_route_build missing where a request needs it),
 * PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_NOMEM at representative k leaves 0 .. k-1 done as the serial
 * loop leaves them. */
int  pfnav_pool_repair_batch(pfnav_ctx *ctx, void *stream, int *out_nrequests, int *out_nrepairs, int *out_nrounds);
/* TEST / MEASUREMENT HOOK, not part of the engine-facing API: what the last pfnav_pool_repair_batch call did.
 * out6[0..2] = representatives (distinct misses) of phase 0 (LOS state), 1 (desired velocity), 2 (enemy-seek /
 * surround); out6[3..5] = rounds the desired-velocity phase ended by rule (i) a request needing a byte written earlier in
 * the round, (ii) a request writing a slot with a pending repair, (iii) a reservation that would evict. */
int  pfnav_pool_repair_batch_stats(pfnav_ctx *ctx, int *out6);
/* TEST HOOK, not part of the engine-facing API: the seeds (64 rows of 64 bits, bit c = column c) of a repair of a TARGET_TILE field of chunk
 * (chunk_r, chunk_c) on `layer`, as the host builds them (kind / arg as in pfnav_flow_fields_repair). Works on a
 * host-only context. */
int  pfnav_repair_seed_mask(pfnav_ctx *ctx, int layer, int chunk_r, int chunk_c, int kind, int arg, uint64_t *out_rows);

/* ---------------------------------------------------------------------------------------- */
/* Region fields (SURVEY.md 8f-1): the dim x dim "cell arrival" fields a formation builds for every cell and
 * every arriving group (formation.c:3152-3176 builds CELL_ARRIVAL_FIELD_RES = 96 squares per cell). The region
 * is centred on `center`, may straddle chunks and hang over the map edge, and its directions are packed two
 * per byte (set_flow_cell, field.c:790: even column -> high nibble); a field is dim * dim / 2 bytes, row-major.
 * All tile coordinates are ABSOLUTE nav tiles (chunk * 64 + tile) as (r, c) int32 pairs.
 *   PFNAV_REGION_CREATE  N_CellArrivalFieldCreate (field.c:2445) / N_GroupArrivalFieldCreate (field.c:2525):
 *                        zero the field, seed seeds[seed_off .. seed_off + seed_n) (those inside the region) at
 *                        cost 0, Dijkstra over passable tiles (enemy-mask rule when enemies != 0; overlay tiles
 *                        are never entered), derive directions.
 *   PFNAV_REGION_CELL    with CREATE: one seed (the cell's tile); the region base shifts when the tile lies one
 *                        past the far edge (field.c:2477-2482). seed_n must be 1.
 *   PFNAV_REGION_FIXUP   N_CellArrivalFieldUpdateToNearestPathable (field.c:2603), after CREATE when both are
 *                        set (cell_field_fixup_task, formation.c:3171): directions off the blocked island that
 *                        holds (start_r, start_c), a NON-passable tile inside the map-clamped region.
 * Without PFNAV_REGION_CREATE the field is updated in place (the caller supplies it). */
enum { PFNAV_REGION_CREATE = 1, PFNAV_REGION_FIXUP = 2, PFNAV_REGION_CELL = 4 };
#define PFNAV_REGION_DIM_MAX 128
typedef struct pfnav_region_req {      /* 40 bytes */
    int32_t  layer;
    int32_t  center_r, center_c;
    int32_t  start_r, start_c;         /* PFNAV_REGION_FIXUP only */
    int32_t  seed_off, seed_n;         /* pairs, into seeds_rc */
    int32_t  overlay_off, overlay_n;   /* pairs, into overlay_rc (struct nav_cell_overlay, nav.h:695) */
    uint16_t enemies;                  /* enemy faction bit mask, 0 = plain passability */
    uint16_t flags;
} pfnav_region_req;
/* HOST buffers; synchronous. inout_fields: n * dim * dim / 2 bytes. dim even, <= PFNAV_REGION_DIM_MAX. */
int  pfnav_region_fields(pfnav_ctx *ctx, int dim, const pfnav_region_req *reqs, size_t n, const int32_t *seeds_rc,
                         size_t nseeds, const int32_t *overlay_rc, size_t noverlay, uint8_t *inout_fields);
/* DEVICE buffers (requests already validated by the caller), asynchronous on `stream`. */
int  pfnav_region_fields_dev(pfnav_ctx *ctx, int dim, const pfnav_region_req *d_reqs, size_t n,
                             const int32_t *d_seeds_rc, const int32_t *d_overlay_rc, uint8_t *d_inout_fields,
                             void *stream);
/* N_GroupArrivalFieldCreate (field.c:2525) with its world-space arguments: targets_xz[ntargets][2], center_xz[2].
 * A centre outside the map yields the zero field, targets outside the map or the region are skipped. */
int  pfnav_group_arrival_field(pfnav_ctx *ctx, int layer, int dim, uint16_t enemies, const float *targets_xz,
                               size_t ntargets, const float *center_xz, const int32_t *overlay_rc, size_t noverlay,
                               uint8_t *out_field);

/* Group arrival (TARGET_ZONE) fields: a flock arriving at its goal follows one shared field per chunk into the
 * open tiles around the goal (arrival.c:859 -> N_RequestAsyncGroupArrivalField nav.c:3921 -> field task ->
 * N_FlowFieldUpdate field.c:2050 -> field_update_zone :1810). The seeds are the first pi * radius^2 open tiles of a
 * best-first flood from the centre (field_zone_initial_frontier, field.c:1683, in the reference's heap order: on the
 * host in pfnav_zone_seeds / pfnav_zone_fields, on the device in the pool requests), the integration runs on the device
 * over the chunk padded by half a chunk, and the
 * chunk's 64 x 64 window is written one direction per byte. Call pfnav_map_commit first when blockers changed.
 * Only maps with more than one chunk row AND column (or exactly 1 x 1) are accepted: with one of the two the
 * reference indexes its padded buffer out of bounds. centre_r / centre_c: absolute nav tile of the zone centre. */
int  pfnav_zone_seeds(pfnav_ctx *ctx, int layer, int chunk_r, int chunk_c, int centre_r, int centre_c, int radius,
                      int32_t *out_rc, size_t cap, size_t *out_n);
/* chunks_rc: n (chunk_r, chunk_c) pairs; out_fields: HOST, n * 4096 bytes. Synchronous. */
int  pfnav_zone_fields(pfnav_ctx *ctx, int layer, int centre_r, int centre_c, int radius, const int32_t *chunks_rc,
                       size_t n, uint8_t *out_fields);
/* N_RequestAsyncGroupArrivalField + N_AwaitAsyncFields (nav.c:3921, 3958): the zone fields of every chunk within
 * reach (2 * radius tiles) of the world-space centre go into pool destination `dest` as its flow fields. A centre
 * outside the map requests nothing. Returns when the fields are in the pool. The one-request case of
 * pfnav_pool_request_zones followed by a synchronise of `stream`. */
int  pfnav_pool_request_zone(pfnav_ctx *ctx, int dest, int layer, const float *centre_xz, int radius, void *stream,
                             int *out_nfields);
/* One request of pfnav_pool_request_zones: the arguments of one pfnav_pool_request_zone call. */
typedef struct pfnav_zone_req {        /* 24 bytes */
    int32_t dest, layer;
    float   centre_x, centre_z;        /* world space, as pfnav_pool_request_zone's centre_xz */
    int32_t radius;                    /* 0 .. 0xFFFF */
    int32_t _pad;
} pfnav_zone_req;
/* N_RequestAsyncGroupArrivalField calls queued during a tick and built at once by N_AwaitAsyncFields: m zone requests
 * against the device field pool in one call.
 * - Equivalence: the pool ends exactly as pfnav_pool_request_zone(ctx, reqs[i].dest, ...) leaves it when called for
 *   i = 0 .. m-1 in order: flow bytes, `has` bits, the (dest, chunk) -> slot mapping pfnav_pool_get exposes, ff_ids and
 *   the pool's remaining capacity. Zone fields take a fresh slot for a (dest, chunk) without one; they never evict and
 *   never reuse slots freed by eviction. A repeated (dest, chunk) ends with the last request's field.
 *   out_nfields[i] (may be NULL) = the fields request i put in the pool.
 * - A centre outside the map requests nothing: out_nfields[i] = 0, and the request counts as done.
 * - The whole batch is validated before anything changes: dest, layer, radius, null pointers, and a map shape the padded
 *   chunk fields support (more than one chunk row and column, or 1 x 1) when any centre lies on the map. Failure:
 *   PFNAV_ERR_ARG, *out_ndone = 0, nothing changed. This differs from pfnav_pool_request_zone before the batch existed:
 *   on a map with one chunk row or column it reserved its pool slots before rejecting the request.
 * - If chunk j of request k does not fit the pool, requests 0 .. k-1 are done, request k's chunks before j stay reserved
 *   without fields (as the single call leaves them), *out_ndone = k (may be NULL) and PFNAV_ERR_NOMEM is returned.
 * - Launches are asynchronous on `stream` (NULL: the context's stream) and ordered after the field work forked by
 *   pfnav_pool_request_goals and after pfnav_pool_clear. The inputs are copied before the call returns. The call does not
 *   wait for the device. The seed floods (field_zone_initial_frontier, field.c:1683) run on the device, or on the host
 *   when the batch's flood budgets add up to at most ten times its largest one (a few large zones, a single request):
 *   a device flood runs on one lane and the batch waits for its longest flood. Results are identical either way.
 * - Host-only context: PFNAV_ERR_NO_DEVICE. */
int  pfnav_pool_request_zones(pfnav_ctx *ctx, const pfnav_zone_req *reqs, size_t m, void *stream,
                              int32_t *out_nfields, int *out_ndone);
/* N_DesiredGroupArrivalVelocity (nav.c:3561) for n world positions against pool destination `dest`:
 * out_vel[n][2] = N_FlowDir of the tile's direction; out_flags[n]: bit 0 = the call returned true (position and centre on
 * the map, chunk field present), bit 1 = *out_at_slot (FD_NONE within `radius` tiles of the centre). HOST buffers. */
int  pfnav_group_arrival_velocity(pfnav_ctx *ctx, int dest, const float *centre_xz, int radius, const float *pos_xz,
                                  size_t n, float *out_vel, uint8_t *out_flags);
/* pfnav_group_arrival_velocity for n resident entities: position k is that of uids[k] (every entry names a uid). The
 * rules of pfnav_pool_request_paths_resident apply. A whole arriving flock goes in one call. */
int  pfnav_group_arrival_velocity_resident(pfnav_ctx *ctx, int dest, const float *centre_xz, int radius,
                                           const uint32_t *uids, size_t n, float *out_vel, uint8_t *out_flags);

/* TARGET_ENTITY / TARGET_ENEMIES chunk fields (N_FlowFieldUpdate field.c:2040-2048 -> field_update_entity :1609,
 * field_update_enemies :1540; consumers N_DesiredSurroundVelocity / N_DesiredEnemySeekVelocity nav.c:3683, 3603).
 * Same padded-chunk integration as the zone fields; the zero-cost frontier is the set of tiles under the target
 * entity (field_entity_initial_frontier, field.c:1317) or under every enemy near the chunk
 * (field_enemies_initial_frontier, field.c:1209). What field.c reads about an entity through its
 * nav_unit_query_ctx is passed in a pfnav_footprint; WHICH entities count as enemies (faction, COMBATABLE,
 * diplomacy, not dying: field_enemy_ent field.c:963) is engine state and is decided by the caller. */
typedef struct pfnav_footprint {       /* 48 bytes */
    float    x, z;                     /* ent_pos_xz */
    float    sel_radius;               /* ent_sel_radius; used unless is_building */
    uint32_t is_building;              /* ENTITY_FLAG_BUILDING: the footprint is the bottom face of ent_curr_obb ... */
    float    corners_xz[8];            /* ... as 4 (x, z) pairs, like pfnav_blockers_incref_obb; all inside the map */
} pfnav_footprint;
enum { PFNAV_TARGET_ENTITY = 0, PFNAV_TARGET_ENEMIES = 1 };
/* Seed tiles of one chunk's field (host structure code, no device needed). ref_layer = the reference's enum
 * nav_layer of `layer`, which fixes the number of contour rings (ENTITY: 3x3 -> 1, 5x5 -> 1, 7x7 and above -> 2;
 * ENEMIES: 1 / 2 / 3). ENEMIES keeps only the entities whose position lies in the chunk's search rectangle
 * (the chunk grown by half a chunk + 16 units, field.c:1229-1243) and returns each tile once, row-major. */
int  pfnav_entity_seeds(pfnav_ctx *ctx, int ref_layer, int target_kind, const pfnav_footprint *ents, size_t nents,
                        int chunk_r, int chunk_c, int32_t *out_rc, size_t cap, size_t *out_n);
/* N_FlowFieldInit + N_FlowFieldUpdate for the listed chunks; out_fields: HOST, n * 4096 bytes. Synchronous. */
int  pfnav_entity_fields(pfnav_ctx *ctx, int layer, int ref_layer, int target_kind, const pfnav_footprint *ents,
                         size_t nents, const int32_t *chunks_rc, size_t n, uint8_t *out_fields);

/* ---------------------------------------------------------------------------------------- */
/* Per-tick agent velocity update (seam B1: the reference's own GPU back-end calls
 * R_GL_MoveUploadData / R_GL_MoveDispatchWork / R_GL_MoveReadNewVelocities,
 * src/render/public/render.h:619-691, computing what move_velocity_work computes on the CPU,
 * src/game/movement.c:3395-3466)
 * ---------------------------------------------------------------------------------------- */

/* enum move_state, movement.c:117-142 */
enum pfnav_move_state { PFNAV_STATE_MOVING = 0, PFNAV_STATE_MOVING_IN_FORMATION, PFNAV_STATE_ARRIVED,
                        PFNAV_STATE_SEEK_ENEMIES, PFNAV_STATE_WAITING, PFNAV_STATE_SURROUND_ENTITY,
                        PFNAV_STATE_ENTER_ENTITY_RANGE, PFNAV_STATE_TURNING, PFNAV_STATE_ARRIVING_TO_CELL };

/* Entity flags the path reads: the engine's own bit values (src/entity.h:59-82), so the
 * entity flag word can be passed through verbatim. Only the low 24 bits are kept. */
#define PFNAV_FLAG_MOVABLE      (1u << 3)
#define PFNAV_FLAG_WATER        (1u << 14)
#define PFNAV_FLAG_AIR          (1u << 15)
#define PFNAV_FLAG_GARRISONED   (1u << 18)
#define PFNAV_FLAG_COMBAT_HELD  (1u << 21)

/* One entity as the movement tick sees it: struct gpu_ent_desc (movement.c:350-369) plus the
 * two things the CPU path uses and the GLSL record lacks (prev_pos, SURVEY 8a-6). 64 bytes. */
typedef struct pfnav_agent {
    float    pos[2];        /* xz, gamestate snapshot position            */
    float    prev_pos[2];   /* ms->prev_pos: ClearPath self position + LOS sample (movement.c:4351,4137) */
    float    velocity[2];   /* ms->velocity, world units per tick          */
    float    vdes[2];       /* in: ignored when the tick computes vdes from the field pool */
    float    radius;        /* selection radius                            */
    float    max_speed;     /* ms->max_speed (wu/s)                        */
    float    speed;         /* entity_speed() (wu/s)                       */
    uint32_t state;         /* enum pfnav_move_state                       */
    uint32_t flags;         /* PFNAV_FLAG_*                                */
    int32_t  flock;         /* index into flocks, -1 = none                */
    uint32_t has_dest_los;  /* in: ignored when computed from the pool     */
    uint32_t aux_dest1;     /* 1 + field-pool destination of this entity's TARGET_ENEMIES fields (STATE_SEEK_ENEMIES,
                             * M_NavDesiredEnemySeekVelocity) or TARGET_ENTITY fields (STATE_SURROUND_ENTITY,
                             * M_NavDesiredSurroundVelocity), built with pfnav_pool_request_entity_fields; 0 = none */
} pfnav_agent;

typedef struct pfnav_flock {
    float    target[2];     /* flock->target_xz (movement.c:193)           */
    int32_t  dest;          /* field-pool destination index, -1 = none     */
    int32_t  layer;         /* N_DestLayer(dest_id)                        */
} pfnav_flock;

/* move_copy_gamestate (movement.c:3607): upload the entity snapshot. HOST pointers.
 * uid == index. Rebuilds the device spatial index (position.c:359 G_Pos_CopyBitmapGrid). */
int  pfnav_agents_upload(pfnav_ctx *ctx, const pfnav_agent *agents, size_t n,
                         const pfnav_flock *flocks, size_t nflocks, int hz);

/* ---------------------------------------------------------------------------------------- */
/* Multi-GPU (SURVEY.md 8e). Entities are partitioned by contiguous index range -- the reference's own fork-join
 * split of the work array (movement.c:3751-3762) -- one range per GPU; each GPU updates its own range and needs the
 * 24-byte neighbour record {pos, vel, radius, state | flags} of every other entity: ONE all-gather of those records
 * per tick, nothing else. The map is replicated; a rank's field pool holds the destinations of its own flocks.
 *
 *   one process per GPU (NCCL over NVLink / NVSwitch; libnccl.so.2 is resolved with dlopen at run time):
 *       rank 0: pfnav_mgpu_unique_id(id) -> the host program hands the 128 bytes to every rank
 *       all   : pfnav_mgpu_init(ctx, rank, world, id)
 *       upload: pfnav_agents_upload_shard(ctx, own records, lo, hi, n_total, ...)   [lo, hi) = pfnav_mgpu_shard_range
 *       tick  : pfnav_mgpu_gather(ctx, stream); pfnav_agents_tick(...); [compute / apply updates]; repeat
 *   one process driving several contexts from one thread (how the engine itself would use 8 GPUs):
 *       pfnav_group_create(ctxs, n, &g); per context pfnav_agents_upload_shard; pfnav_group_gather(g); ticks ...
 *
 * uids stay global (index into the whole population); work lists, movestate uploads, velocity / patch / state
 * read-backs of a context cover its OWN range only.
 *
 * A job that shares blockers (pfnav_mgpu_share_blockers / pfnav_group_share_blockers) lets each member take its own
 * entities' blockers on the device; per tick and member, in this order:
 *       pfnav_agents_compute_updates -> pfnav_agents_apply_updates_ex(PFNAV_APPLY_BLOCKERS)
 *       -> pfnav_agents_set_blocking for commands, on the rank that owns the uids
 *       -> pfnav_mgpu_exchange_blocker_ops (every rank) / pfnav_group_exchange_blocker_ops (once)
 *       -> pfnav_blockers_* / pfnav_blockers_batch for host ops (buildings, load-time blocks), on every rank
 *       -> pfnav_map_commit -> pfnav_mgpu_gather / pfnav_group_gather
 * The engine's orders reach a job as one batch of deltas that every member receives whole (pfnav_mgpu_commands /
 * pfnav_group_commands, after pfnav_agents_commands), before the blocking calls of those commands:
 *       apply_updates_ex -> job commands + pfnav_agents_set_blocking -> exchange -> pfnav_map_commit -> gather
 *       -> pfnav_agents_set_work_dev -> tick
 * After a gather every member holds the whole record column and position index, so any member answers
 * pfnav_ents_in_circles for any query, with global uids as centres, without a collective. */
typedef struct pfnav_group pfnav_group;
#define PFNAV_MGPU_ID_BYTES 128
int  pfnav_mgpu_shard_range(size_t n_total, int rank, int world, size_t *lo, size_t *hi);
int  pfnav_mgpu_unique_id(void *out_id /* PFNAV_MGPU_ID_BYTES */);
int  pfnav_mgpu_init(pfnav_ctx *ctx, int rank, int world, const void *id);
int  pfnav_mgpu_finalize(pfnav_ctx *ctx);
/* The per-tick collective: all-gather of the neighbour records (plus the flock id column after an upload that may
 * have changed membership), then the spatial index over the whole population (G_Pos_CopyBitmapGrid, position.c:359)
 * on this rank. Asynchronous on `stream` (blocks only when member lists are rebuilt). */
int  pfnav_mgpu_gather(pfnav_ctx *ctx, void *stream);
int  pfnav_group_create(pfnav_ctx **ctxs, int world, pfnav_group **out);
int  pfnav_group_gather(pfnav_group *g);       /* on every member's own context stream */
void pfnav_group_destroy(pfnav_group *g);
/* Opt-in: the members of this job take their owned entities' blockers on the device. Call on every rank (NCCL)
 * or once per group; it only sets state. Afterwards the blocking entry points work on the members, and a member's
 * device-decided ops must go through an exchange before they are applied:
 *   - the blocking table of a member covers its own range [shard_lo, shard_hi), like pfnav_agents_upload_movestate,
 *     pfnav_agents_read_state and pfnav_agents_set_work: pfnav_agents_upload_blocking takes shard_hi - shard_lo
 *     records, pfnav_agents_read_blocking returns that range, pfnav_agents_set_blocking rejects a uid outside it with
 *     PFNAV_ERR_ARG (nothing changed), and PFNAV_APPLY_BLOCKERS works on the member's work list (owned uids);
 *   - no commit before the exchange: while a member holds device-decided ops that were not exchanged, every entry point
 *     that would apply them (pfnav_map_commit, pfnav_blockers_get, pfnav_blockers_get_factions, field and path
 *     requests that apply queued ops first) returns PFNAV_ERR_STATE and applies nothing;
 *   - ops queued on the host (pfnav_blockers_*, pfnav_blockers_batch) are not exchanged: the engine sends them to
 *     every rank, as without the opt-in.
 * Without the opt-in nothing changes: the blocking entry points return PFNAV_ERR_STATE on a member of a job.
 * Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_STATE on a context in no job; PFNAV_ERR_ARG for
 * pfnav_mgpu_share_blockers on a group member, or group members holding populations of different sizes;
 * pfnav_group_share_blockers: PFNAV_ERR_STATE when two distinct member devices cannot access each other's memory
 * (checked up front, so that an exchange never fails halfway). pfnav_group_destroy / pfnav_mgpu_finalize end the
 * opt-in with the job. */
int  pfnav_mgpu_share_blockers(pfnav_ctx *ctx);
int  pfnav_group_share_blockers(pfnav_group *g);
/* Every member ends up with every member's pending device ops (its own first, then the others' in rank order; ops a
 * previous exchange already delivered are not sent again). Blocking, like pfnav_map_commit: it waits for each member's
 * device first. NCCL: a collective that every rank calls (an all-gather of the op counts, one read of them, then a
 * group of broadcasts on `stream`). Group: peer copies on the members' context streams; before it returns, each
 * member's stream waits until every peer has finished reading its ops.
 * Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_STATE when the context is in no job or its job has not
 * opted in; PFNAV_ERR_ARG for pfnav_mgpu_exchange_blocker_ops on a group member, or group members holding populations
 * of different sizes. */
int  pfnav_mgpu_exchange_blocker_ops(pfnav_ctx *ctx, void *stream);
int  pfnav_group_exchange_blocker_ops(pfnav_group *g);
/* pfnav_pool_request_goals_ex for a whole job: the members' flocks may head for the same destinations, and each
 * (dest, chunk) field is built on ONE member and copied to the members that need it. Every rank calls the NCCL form with
 * the same arguments; the group form is called once.
 *   - Equivalence: every member's pool ends exactly as pfnav_pool_request_goals_ex(member, same arguments) would leave
 *     it: flow and LOS bytes, `has` bits, the (dest, chunk) -> slot mapping and the ff_ids pfnav_pool_get reports, and
 *     the member's own LRU choices and evictions. Members keep their own pools, slots and eviction histories (their
 *     ticks read different slots, so their device touch stamps differ). out_n_flow / out_n_los are the member's solo
 *     counts; the group form takes arrays of `world` entries, member i's at [i] (either may be NULL).
 *   - Each field is built once: every goal has one owner member, which builds every field of the goal that any member
 *     lacks (the union of the members' missing (dest, chunk) sets; with flags == 0 the goal's whole plan). Each member
 *     writes only the fields it lacks. Owners follow from the plan, which every member computes alike from the
 *     replicated map: the goal with the longest LOS chain first, to the member with the fewest fields so far, ties to
 *     the lower rank. A field one member keeps equals the one the owner rebuilds for another member: every commit that
 *     changed the map under it dropped it from every pool alike -- the premise PFNAV_REQUEST_MISSING_ONLY rests on.
 *     As in the solo call, a destination repeated in one batch must name the same target each time.
 *   - All or nothing across the job: every member validates the arguments and its state (dest, layer, no device blocker
 *     ops decided since the last exchange) and dry-runs its reservation before any pool changes. If any member's pool
 *     cannot hold its fields, EVERY member returns PFNAV_ERR_NOMEM and no pool changes -- unlike the solo call, where
 *     only the member that does not fit fails. An argument or state error on one rank is returned by every rank.
 *   - Streams: asynchronous on the device like the solo call, with one host wait: NCCL all-gathers one record per member
 *     on `stream` and reads it (a group reads its members' host state). The owners' flow waves and LOS chains run on the
 *     context's field streams and are joined on `stream` before the exchange: NCCL broadcasts the owners' staging
 *     segments on `stream`; a group member pulls them with peer copies on its context stream, and its stream waits
 *     until the peers have finished reading its own segment. The copies into the pool follow on the same stream; the
 *     next pool reader joins them like a solo batch's LOS chains.
 *   - Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_STATE on a context in no job, for the NCCL form on
 *     a group member, for device blocker ops not yet exchanged, and for a group whose members sit on distinct devices
 *     without peer access (refused up front); PFNAV_ERR_ARG for bad arguments or members whose maps or pools differ in
 *     shape; PFNAV_ERR_NOMEM as above. The single-context entry points are unchanged. */
int  pfnav_mgpu_request_goals_ex(pfnav_ctx *ctx, int ngoals, const int32_t *dests, int layer, const int32_t *targets,
                                 uint32_t flags, void *stream, int *out_n_flow, int *out_n_los);
int  pfnav_group_request_goals_ex(pfnav_group *g, int ngoals, const int32_t *dests, int layer, const int32_t *targets,
                                  uint32_t flags, int *out_n_flow, int *out_n_los);
/* pfnav_pool_request_zones for a whole job: a flock arriving as a group needs its zone fields on every member that holds
 * one of its units, and each (dest, chunk) field is built on ONE member and copied to every member. Every rank calls the
 * NCCL form with the same arguments; the group form is called once. pfnav_mgpu_request_entity_fields_batch /
 * pfnav_group_request_entity_fields_batch (below, after pfnav_pool_request_entity_fields_batch) do the same for
 * enemy-seek and surround fields, with the same contract.
 *   - Equivalence: every member's pool ends exactly as the solo call with the same arguments would leave it: flow bytes,
 *     `has` bits, the (dest, chunk) -> slot mapping and the ff_ids pfnav_pool_get reports, and the member's own slot
 *     choices (pool_used order for zones, which are never evicted; LRU evictions for entity fields). For entity fields
 *     also the footprints each destination remembers, which pfnav_pool_repair / pfnav_pool_repair_batch start from.
 *     Members keep their own pools and histories, so their slots may differ. out_nfields (zones) is per request and the
 *     same on every member; the group form takes one array of m entries.
 *   - Each field is built once. A field depends on its request and the replicated map only (centre, radius, layer and
 *     chunk; footprints, kind, layer, ref_layer and chunk), and neither batch skips a field the pool holds: every member
 *     writes the same keys with the same bytes, the last request naming a key deciding them. Every written key has one
 *     owner, computed alike on every member from the arguments: each request costs the flood budgets
 *     (min(pi r^2, dim^2)) of its fields whose window holds the centre (zones) or its field count (entity fields),
 *     counting only the keys it writes last; the most expensive request goes first, to the member with the least cost
 *     so far, ties to the lower rank. A request's keys are built by its owner into a staging buffer, and every member
 *     copies every key it holds at the end into its own slot.
 *   - All or nothing across the job: every member validates the arguments and its state (pool created, no device
 *     blocker ops decided since the last exchange) and dry-runs its reservation before any pool changes. If one member
 *     refuses, every member returns that error; if one member's pool cannot hold the batch, EVERY member returns
 *     PFNAV_ERR_NOMEM. Either way no pool changes -- unlike the solo calls, which keep the requests before the one that
 *     did not fit (out_ndone). NCCL all-gathers one {verdict, fits} record per member on `stream` and reads it on the
 *     host; nothing else is exchanged before the builds.
 *   - Streams: the owners' builds run on `stream` (NCCL) or the context stream (group), as the solo call's do. NCCL
 *     broadcasts the owners' staging segments on `stream` (grouped); a group member pulls them with peer copies on its
 *     context stream, and its stream waits until the peers have finished reading its own segment. The copies into the
 *     pool follow on the same stream, and the next pool reader joins them like a goal batch's.
 *   - Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_STATE on a context in no job, for the NCCL form on
 *     a group member, for device blocker ops not yet exchanged, and for a group whose members sit on distinct devices
 *     without peer access; PFNAV_ERR_ARG for bad arguments or members whose maps or pools differ in shape;
 *     PFNAV_ERR_NOMEM as above. The single-context entry points are unchanged. */
int  pfnav_mgpu_request_zones(pfnav_ctx *ctx, const pfnav_zone_req *reqs, size_t m, void *stream, int32_t *out_nfields);
int  pfnav_group_request_zones(pfnav_group *g, const pfnav_zone_req *reqs, size_t m, int32_t *out_nfields);
/* TEST HOOK: this member's part in its last job batch of any kind. Goal batches: the flow / LOS requests it built for
 * the job (*out_n_flow, *out_n_los) and the owner rank of goals 0 .. max_goals - 1 (-1: no member lacked a field of the
 * goal). Zone and entity-field batches: the fields it built, 0, and the owner rank of requests 0 .. max_goals - 1 (-1:
 * the request writes no key -- centred off the map, or every key it names is written again by a later request). */
int  pfnav_mgpu_fields_stats(pfnav_ctx *ctx, int *out_n_flow, int *out_n_los, int32_t *out_owner, int max_goals);
/* move_copy_gamestate (movement.c:3607) for this context's own range [lo, hi) of a population of n_total entities;
 * shard[i] is entity lo + i, `flock` fields index the GLOBAL flock table. The snapshot is complete after the next
 * pfnav_mgpu_gather / pfnav_group_gather. On a context outside any multi-GPU job lo = 0, hi = n_total is the whole
 * population (== pfnav_agents_upload).
 * PFNAV_UPLOAD_SAME_FLOCKS: only positions, velocities, states and speeds changed since the previous upload of the
 * same range -- flock membership, selection radii, layers, the GARRISONED flag and the flock table are as before --
 * so the per-entity host pass and the member-list rebuild are skipped (the engine pushes deltas, SURVEY.md 7). */
#define PFNAV_UPLOAD_SAME_FLOCKS (1u << 0)
int  pfnav_agents_upload_shard(pfnav_ctx *ctx, const pfnav_agent *shard, size_t lo, size_t hi, size_t n_total,
                               const pfnav_flock *flocks, size_t nflocks, int hz, uint32_t flags);

/* Work list (move_push_work, movement.c:3741): the uids that take a velocity update this tick.
 * NULL = every agent whose state is not ARRIVED/WAITING (ent_still, movement.c:652). */
int  pfnav_agents_set_work(pfnav_ctx *ctx, const uint32_t *uids, size_t nwork);

/* ---------------------------------------------------------------------------------------- */
/* State update (SURVEY 8 a-8): entity_compute_update (game/movement.c:2303-2650) on the device, one
 * `struct movestate_patch` (movement.c:245-262) per work item, for every movement state (the formation inputs
 * and the state beyond point seeking arrive through pfnav_formation_in / pfnav_movestate_ext). The engine applies the patches on
 * its main thread (entity_apply_update, movement.c:2693: blockers, events, G_Pos_Set);
 * pfnav_agents_apply_updates is the device-side equivalent for the movestate fields so that
 * consecutive ticks can run without a host round trip. */
#define PFNAV_VEL_HIST_LEN 14           /* VEL_HIST_LEN, movement.c:94 */
typedef struct pfnav_movestate {        /* the part of struct movestate (movement.c:146-215) the update reads */
    float   next_pos[3];                /* ms->next_pos                                  */
    float   step;                       /* ms->step                                      */
    float   next_rot[4];                /* ms->next_rot, quaternion {x, y, z, w}          */
    float   combat_facing[4];           /* ms->combat_facing                             */
    float   vel_hist[PFNAV_VEL_HIST_LEN][2];
    int32_t left;                       /* ms->left                                      */
    int32_t vel_hist_idx;
    int32_t _pad[2];
} pfnav_movestate;                      /* 176 bytes */

/* The formation inputs of one work item: struct formation_state + cell_pos + cell_arrival_vdes of struct move_work_in
 * (movement.c:215-225, 264-276). formation.c computes them on the main thread (G_Formation_*); the velocity pass and
 * the state update read them (STATE_MOVING_IN_FORMATION / STATE_ARRIVING_TO_CELL). 64 bytes. */
#define PFNAV_FORM_HAS_FORMATION    (1u << 0)   /* fstate.fid != NULL_FID */
#define PFNAV_FORM_ASSIGNMENT_READY (1u << 1)
#define PFNAV_FORM_ASSIGNED_TO_CELL (1u << 2)
#define PFNAV_FORM_IN_RANGE_OF_CELL (1u << 3)
#define PFNAV_FORM_ARRIVED_AT_CELL  (1u << 4)
typedef struct pfnav_formation_in {
    float    cell_pos[2];            /* in->cell_pos                                   */
    float    cell_arrival_vdes[2];   /* in->cell_arrival_vdes: the desired velocity of STATE_ARRIVING_TO_CELL */
    float    cohesion[2];            /* fstate.normal_cohesion_force                   */
    float    align[2];               /* fstate.normal_align_force                      */
    float    drag[2];                /* fstate.normal_drag_force                       */
    float    target_orientation[4];  /* fstate.target_orientation                      */
    uint32_t flags;                  /* PFNAV_FORM_*                                   */
    uint32_t _pad;
} pfnav_formation_in;
/* HOST array, one record per entity of this context's own range (uid order). Optional: without it every entity is
 * outside any formation (fid == NULL_FID). */
int  pfnav_agents_upload_formation(pfnav_ctx *ctx, const pfnav_formation_in *f, size_t n);
/* Inspection: read the own range's formation table back (at most maxout records; waits for the device).
 * PFNAV_ERR_ARG when no table exists. */
int  pfnav_agents_read_formation(pfnav_ctx *ctx, pfnav_formation_in *out, size_t maxout);

/* The rest of struct movestate (movement.c:146-215) that the states beyond point seeking read. 64 bytes. */
#define PFNAV_NULL_UID 0xffffffffu
typedef struct pfnav_movestate_ext {
    int32_t  wait_prev;              /* ms->wait_prev (enum pfnav_move_state)          */
    int32_t  wait_ticks_left;
    uint32_t surround_target_uid;    /* PFNAV_NULL_UID = none; also the target of STATE_ENTER_ENTITY_RANGE */
    uint32_t using_surround_field;
    float    target_range;           /* STATE_ENTER_ENTITY_RANGE                       */
    float    target_prev_pos[2];
    float    _padf;
    float    target_dir[4];          /* STATE_TURNING: ms->target_dir                  */
    float    rot[4];                 /* Entity_GetRot(uid), what Entity_SetRot last set */
} pfnav_movestate_ext;
/* HOST array, own range, uid order. Optional: zero / NULL_UID defaults. */
int  pfnav_agents_upload_movestate_ext(pfnav_ctx *ctx, const pfnav_movestate_ext *ms, size_t n);
/* Inspection: read the own range's movestate_ext table back (at most maxout records; waits for the device).
 * PFNAV_ERR_ARG when no table was uploaded. */
int  pfnav_agents_read_movestate_ext(pfnav_ctx *ctx, pfnav_movestate_ext *out, size_t maxout);

/* enum movestate_flags (movement.c:226-242), same bit values */
#define PFNAV_UPDATE_SET_STATE        (1u << 0)
#define PFNAV_UPDATE_SET_VELOCITY     (1u << 1)
#define PFNAV_UPDATE_SET_POSITION     (1u << 2)
#define PFNAV_UPDATE_SET_ROTATION     (1u << 3)
#define PFNAV_UPDATE_SET_NEXT_POS     (1u << 4)
#define PFNAV_UPDATE_SET_PREV_POS     (1u << 5)
#define PFNAV_UPDATE_SET_STEP         (1u << 6)
#define PFNAV_UPDATE_SET_LEFT         (1u << 7)
#define PFNAV_UPDATE_SET_NEXT_ROT     (1u << 8)
#define PFNAV_UPDATE_SET_PREV_ROT     (1u << 9)
#define PFNAV_UPDATE_SET_DEST         (1u << 10)
#define PFNAV_UPDATE_SET_TARGET_PREV  (1u << 11)
#define PFNAV_UPDATE_SET_MOVING       (1u << 12)
#define PFNAV_UPDATE_SET_TARGET_DIR   (1u << 13)
#define PFNAV_UPDATE_TURNING_IN_PLACE (1u << 14)
/* engine_todo: what the device pass leaves to the engine for this work item */
#define PFNAV_TODO_SURROUND_QUERY     (1u << 0)  /* STATE_SURROUND_ENTITY with a live target: the branch decisions of
                                                  * movement.c:2513-2567 need the target's geometry (M_NavObjAdjacentFrom,
                                                  * M_NavClosestReachableAdjacentPosFrom: OBBs, entity tables) -- the movement
                                                  * part of the patch is complete, the state decision is the engine's */
#define PFNAV_TODO_USE_SURROUND_FIELD  (1u << 1) /* ent_update_using_surround_field (movement.c:2672): ms->using_surround_field */
#define PFNAV_TODO_DROP_SURROUND_FIELD (1u << 2) /* ... switches on / off (low / high water marks of the distance to the target) */

typedef struct pfnav_patch {            /* struct movestate_patch (movement.c:245-262); unselected fields are 0 */
    uint32_t flags;
    int32_t  next_state;                /* -1 unless SET_STATE / SET_MOVING               */
    int32_t  next_block;
    int32_t  next_attack;
    float    next_velocity[2];
    float    next_pos[3];               /* y: 0 (AIR_UNIT_HEIGHT for air units); terrain height
                                         * (M_HeightAtPoint) is render state, added by the engine  */
    float    next_rot[4];
    float    next_ppos[3];
    float    next_npos[3];
    float    next_step;
    float    next_left;
    float    next_nrot[4];
    float    next_prot[4];
    int32_t  wait_ticks_left;           /* ms->wait_ticks_left after the call (entity_compute_update counts it down in place) */
    uint32_t engine_todo;               /* PFNAV_TODO_*                                    */
    float    _padf;
    float    next_dest[2];              /* UPDATE_SET_DEST: the engine re-issues the move order (G_Move_SetDest) */
    float    next_target_prev[2];
    float    next_target_dir[4];
} pfnav_patch;                          /* 160 bytes */

/* Inspection / test entry: the two map searches of arrived() (movement.c:2170) for a flock target on `layer`, as
 * pfnav_agents_compute_updates precomputes them per (flock, layer): N_ClosestPathable (nav.c:4126) and the tile
 * centres N_IsMaximallyClose compares with (nav.c:4707). out_mc_xz: up to cap (x, z) pairs. Host code; needs
 * pfnav_route_build(layer). */
int  pfnav_route_arrival_consts(pfnav_ctx *ctx, int layer, float tx, float tz, int32_t *out_nearest_ok,
                                float *out_nearest_xz, float *out_mc_xz, size_t cap, int32_t *out_mc_n);
/* Map point queries (seam B3, src/navigation/public/nav.h), answered in batches on the device. */
enum pfnav_map_query_kind {
    PFNAV_QUERY_PATHABLE = 0,            /* N_PositionPathable (nav.c:4055): the tile under (x, z) is not 0xFF        */
    PFNAV_QUERY_BLOCKED,                 /* N_PositionBlocked (nav.c:4070): the tile under (x, z) holds a blocker     */
    PFNAV_QUERY_ADJACENT_IMPASSABLE,     /* N_IsAdjacentToImpassable (nav.c:4745): one of the 4 neighbours of the tile
                                          * under (x, z) has cost 0xFF or a blocker                                   */
    PFNAV_QUERY_CLOSEST_PATHABLE,        /* N_ClosestPathable (nav.c:4126): the nearest tile to (x, z) that is
                                          * neither impassable nor blocked                                            */
    PFNAV_QUERY_MAXIMALLY_CLOSE,         /* N_IsMaximallyClose (nav.c:4707) of (x, z) to (dst_x, dst_z)               */
    PFNAV_QUERY_DEST_ID                  /* N_DestIDForPos / N_DestIDForPosAttacking (nav.c:839) of (x, z)            */
};
typedef struct pfnav_map_query_req {         /* 32 bytes */
    int32_t kind, layer;                 /* enum pfnav_map_query_kind; 0 <= layer < nlayers                            */
    float   x, z;                        /* the position (CLOSEST_PATHABLE: the target, DEST_ID: the destination)     */
    float   dst_x, dst_z;                /* MAXIMALLY_CLOSE: the destination                                          */
    float   tolerance;                   /* MAXIMALLY_CLOSE: finite                                                   */
    int32_t faction_id;                  /* DEST_ID: PFNAV_FACTION_ID_NONE = N_DestIDForPos, 0..14 = ...Attacking      */
} pfnav_map_query_req;
typedef struct pfnav_map_query_result {  /* 16 bytes */
    int32_t  ok;                         /* the reference function's bool (DEST_ID, CLOSEST_PATHABLE: a tile exists)  */
    uint32_t dest_id;                    /* DEST_ID: the dest_id_t                                                    */
    float    x, z;                       /* CLOSEST_PATHABLE: *out -- the query point when its tile is free, else the
                                          * M_Tile_Bounds corner of the tile found                                    */
} pfnav_map_query_result;
/* n map queries against the COMMITTED map: blocker counts as the last pfnav_map_commit left them (the state the
 * reader contexts and the tick see), costs as last uploaded. pfnav_blockers_* changes not yet committed are not seen.
 * - Buffers are on the host; the call returns when out[0 .. n) is filled.
 * - Work is queued on `stream` (NULL: the context's stream), ordered after pfnav_map_commit and after the field work
 *   forked by pfnav_pool_request_goals, like the pool entry points.
 * - A query point outside the map box gives ok = 0 for every kind.
 * - CLOSEST_PATHABLE: breadth-first from the tile under (x, z), neighbours (0,-1) (0,+1) (-1,0) (+1,0); the first tile
 *   dequeued whose cost is not 0xFF and that holds no blocker. ok = 0 when there is none.
 * - MAXIMALLY_CLOSE: ok = some tile centre n_closest_island_tiles (nav.c:1226) lists for the destination -- the
 *   closest tiles of its global island without blockers, at most 256 -- lies within `tolerance` of (x, z). It does not
 *   include the N_IsAdjacentToImpassable test that arrived() (movement.c:2170) adds; combine the two kinds for that.
 * - The searches run on the device: over a window around the start tile, then over the whole layer for a search that
 *   leaves it. Results are identical either way.
 * - Everything is validated before anything runs: null pointers (n > 0), kind, layer, a finite tolerance and
 *   pfnav_route_build(layer) (the global islands) for MAXIMALLY_CLOSE, faction_id in 0..15 for DEST_ID. Failure:
 *   PFNAV_ERR_ARG, out untouched. n == 0 is valid. Host-only context: PFNAV_ERR_NO_DEVICE. */
int  pfnav_map_query(pfnav_ctx *ctx, const pfnav_map_query_req *q, size_t n, pfnav_map_query_result *out, void *stream);
/* pfnav_map_query with positions that may name resident entities: pos_uids[i] replaces (x, z) of query i and
 * dst_uids[i] replaces (dst_x, dst_z). Either array may be NULL; PFNAV_NULL_UID keeps the given value. The rules of
 * pfnav_pool_request_paths_resident apply. */
int  pfnav_map_query_resident(pfnav_ctx *ctx, const pfnav_map_query_req *q, const uint32_t *pos_uids,
                              const uint32_t *dst_uids, size_t n, pfnav_map_query_result *out, void *stream);

/* HOST array of n_agents records, uid == index. */
int  pfnav_agents_upload_movestate(pfnav_ctx *ctx, const pfnav_movestate *ms, size_t n);
/* After pfnav_agents_tick on the same stream: entity_compute_update for every work item, reading the
 * tick's new velocities and desired velocities. Needs pfnav_route_build for every layer the agents
 * use (global islands feed arrived(), movement.c:2170). Every movement state is accepted: MOVING / MOVING_IN_FORMATION
 * (formation inputs), SEEK_ENEMIES, ENTER_ENTITY_RANGE, TURNING, WAITING, ARRIVING_TO_CELL are decided on the device;
 * SURROUND_ENTITY with a live target is flagged PFNAV_TODO_SURROUND_QUERY (see there).
 * The map searches of arrived() run on the device, per used (flock, layer) pair, and so do ENTER_ENTITY_RANGE's
 * N_IsMaximallyClose searches around each target's position. With or without a movestate_ext table the call is
 * asynchronous on `stream` and waits for the device only when one of its buffers has to grow, or, when the arrival
 * constants are rebuilt, for the upload of the rebuild two rebuilds back (the request staging's pinned ring).
 * pfnav_route_build is checked on the host for every used (flock, layer) pair before anything is queued. One
 * configuration still waits: with a movestate_ext table, while some entity of this context stands on a layer without
 * pfnav_route_build, the call checks its ENTER_ENTITY_RANGE items with a target on the device and waits for that check;
 * PFNAV_ERR_ARG when one stands on such a layer. */
int  pfnav_agents_compute_updates(pfnav_ctx *ctx, void *stream);
/* Inspection / test entry: the (flock, layer) table of arrived()'s constants that the last pfnav_agents_compute_updates
 * built, one record per (flock, layer) pair some entity of the flock uses, in (flock, layer) order. Blocks until the
 * device is idle. out: up to maxout records; *out_n (may be NULL): the number of pairs. PFNAV_ERR_ARG when the table is
 * not current (not built yet, or the flocks, their layers or the committed map changed since). */
typedef struct pfnav_arrival_record {
    int32_t flock, layer;
    int32_t nearest_ok;                  /* N_ClosestPathable (nav.c:4126) from the flock target found a tile         */
    float   nearest[2];                  /* its (x, z): the target itself when its tile is free                       */
    int32_t mc_n;                        /* n_closest_island_tiles (nav.c:1226): the tile centres N_IsMaximallyClose   */
    float   mc[256][2];                  /* compares with, in the reference's order                                   */
} pfnav_arrival_record;
int  pfnav_agents_read_arrival_consts(pfnav_ctx *ctx, pfnav_arrival_record *out, size_t maxout, size_t *out_n);
/* Work-item order. Blocks until the update pass has finished. */
int  pfnav_agents_read_patches(pfnav_ctx *ctx, pfnav_patch *out, size_t maxout);
/* Device-side entity_apply_update for the movestate fields (movement.c:2693-2757: state, velocity +
 * velocity history, position, interpolation fields, next rotation), then refreshes the neighbour
 * records; follow with pfnav_agents_rebuild_index before the next tick. */
int  pfnav_agents_apply_updates(pfnav_ctx *ctx, void *stream);

/* Blockers of stopping and starting units on the device (opt-in). entity_apply_update's entity_finish_moving ->
 * entity_block (movement.c:580, 685) increfs the blockers under a unit that stops; SET_MOVING (:2750-2755) ->
 * entity_unblock (:560-600) releases them. pfnav_blocking is ms->blocking plus what entity_block recorded, one per entity,
 * kept on the device. 32 bytes. */
typedef struct pfnav_blocking {
    uint32_t blocking;               /* 0 / 1 */
    int32_t  faction_id;             /* the entity's faction (0..15); used for the ops it takes */
    float    stop_x, stop_z;         /* where its current block was taken (valid when blocking) */
    float    stop_radius;            /* the range that block was taken with */
    uint32_t _pad[3];
} pfnav_blocking;
/* HOST array, one record per entity (uid order). Describes blocks the caller has already counted (for example through
 * pfnav_blockers_* at load): it queues no op. blocking must be 0 or 1, faction_id 0..15. */
int  pfnav_agents_upload_blocking(pfnav_ctx *ctx, const pfnav_blocking *b, size_t n);
/* Read the device's blocking table back (waits for the device). */
int  pfnav_agents_read_blocking(pfnav_ctx *ctx, pfnav_blocking *out, size_t maxout);
#define PFNAV_APPLY_BLOCKERS (1u << 0)
/* flags == 0: pfnav_agents_apply_updates. PFNAV_APPLY_BLOCKERS: the same apply, and for every work item, in work order:
 *   block   - the patch has SET_STATE with next_block != 0, the entity is not GARRISONED and not blocking: incref a circle
 *             at its snapshot position (the position before this apply, G_Pos_GetXZFrom(gamestate.positions),
 *             movement.c:583) with range = its radius, its blocking record's faction_id and its flags; the record keeps
 *             stop_x / stop_z / stop_radius and blocking = 1;
 *   unblock - the patch has SET_MOVING and the entity is blocking: decref exactly the recorded circle (the entity's
 *             current flags pick the layers), blocking = 0.
 * The ops are decided and compacted in work order on the device into a context-owned op buffer that pfnav_map_commit
 * applies after the ops queued through pfnav_blockers_* (the result equals pfnav_blockers_batch with these ops appended).
 * Asynchronous on `stream`; it waits for the device only when the op buffer has to grow. Calls that use the blocking
 * table (this one, pfnav_agents_set_blocking, upload / read) are ordered by the caller, for example on one stream.
 * Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_ARG for an unknown flag or PFNAV_APPLY_BLOCKERS without
 * blocking records for the uploaded population; PFNAV_ERR_STATE (nothing changed) on a context in a multi-GPU job
 * (pfnav_mgpu_init / pfnav_group_create, or an own range that is not the whole population) that does not share
 * blockers: the map is replicated and a rank's ops would reach only its own copy. A job that shares blockers
 * (pfnav_mgpu_share_blockers / pfnav_group_share_blockers) exchanges them before the commit; its members' tables
 * cover their own ranges (see there). On a single context the own range is the whole population. */
int  pfnav_agents_apply_updates_ex(pfnav_ctx *ctx, uint32_t flags, void *stream);
/* What the tick decided, for the engine to act on: one record per work item whose patch the apply applies (the entity is
 * not GARRISONED) and that has SET_STATE, SET_MOVING or SET_DEST in its flags or a non-zero engine_todo. They drive
 * entity_finish_moving (ARRIVED / WAITING: events, combat stance), move_notify_motion_start (SET_MOVING), the re-issued
 * move order G_Move_SetDest (SET_DEST) and the surround decisions and field requests of engine_todo. 48 bytes. */
typedef struct pfnav_event {
    uint32_t uid;                     /* the work item's uid, numbered as at the collect call                           */
    uint32_t flags;                   /* the patch's flags, PFNAV_UPDATE_* (all of them)                                 */
    uint32_t todo;                    /* the patch's engine_todo, PFNAV_TODO_*                                          */
    int32_t  attack;                  /* the patch's next_attack (meaningful with SET_DEST)                              */
    uint32_t state_before;            /* agent.state before the apply                                                   */
    uint32_t state_after;             /* agent.state as the apply leaves it: SET_STATE writes next_state, then SET_MOVING
                                       * writes it again; neither: state_before                                         */
    float    dest[2];                 /* the patch's next_dest (meaningful with SET_DEST)                                */
    float    pos[2];                  /* agent.pos (x, z) as the apply leaves it: SET_POSITION ? next_pos x, z : agent.pos */
    uint32_t _pad[2];
} pfnav_event;
/* Collect the events of the last update pass, in work order, into a context-owned device list. Every field is a copy of
 * what pfnav_agents_read_patches and pfnav_agents_read_state would give (state_before and agent.pos read before the
 * apply), so the list equals the host filter of those two read-backs bit for bit.
 * - Call it after pfnav_agents_compute_updates and before the apply of that pass (pfnav_agents_apply_updates[_ex]), on
 *   the same stream: it reads the state and positions the apply overwrites.
 * - Asynchronous on `stream`: no host wait. The count stays on the device. The list is reserved for n_work records
 *   before the launch; it waits for the device only when it has to grow. An empty work list gives an empty list.
 * - Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_ARG when no update pass has run; PFNAV_ERR_STATE
 *   when the last update pass has already been applied. Nothing changes on an error.
 * Multi-GPU jobs: a member collects its own work items, with global uids; no collective is involved. When the members'
 * work lists come from pfnav_agents_set_work_dev, their lists joined in rank order equal the list of one context holding
 * the whole population. */
int  pfnav_agents_collect_events(pfnav_ctx *ctx, void *stream);
/* Read the list of the last collect: *out_n = its length, out[0 .. *out_n) the records. It waits for the collect
 * through an event recorded after it (not for later work on any stream) and copies through pinned memory.
 * - maxout < the length: PFNAV_ERR_NOMEM with *out_n set and out untouched; the list stays readable, so grow out and
 *   call again (maxout = 0 asks for the length only).
 * - The list stays readable, as often as wanted, until the next collect.
 * - Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_ARG for a NULL out_n, or a NULL out with maxout > 0;
 *   PFNAV_ERR_STATE when no collect has run, or when a call that renumbers the population has changed it since the
 *   collect (pfnav_agents_upload, pfnav_agents_upload_shard, pfnav_agents_change_population,
 *   pfnav_mgpu_change_population, pfnav_group_change_population): the uids would no longer name the same entities. */
int  pfnav_agents_read_events(pfnav_ctx *ctx, pfnav_event *out, size_t maxout, size_t *out_n);
/* The engine's own entity_block (block != 0) / entity_unblock (block == 0) for commands (stop, new move order) for n
 * uids, with the rules and the op buffer of PFNAV_APPLY_BLOCKERS: blocking at the entity's current position. Repeats
 * (within a call or across calls) change nothing. Errors as pfnav_agents_apply_updates_ex's, and PFNAV_ERR_ARG (nothing
 * changed) for a uid outside the context's own range (the population, on a single context). */
int  pfnav_agents_set_blocking(pfnav_ctx *ctx, const uint32_t *uids, size_t n, int block, void *stream);
/* Read the (updated) entity snapshot back: agents_out / ms_out may be NULL. */
int  pfnav_agents_read_state(pfnav_ctx *ctx, pfnav_agent *agents_out, pfnav_movestate *ms_out, size_t maxout);

/* Movement commands as deltas (SURVEY 7: the host pushes deltas, not whole-state re-uploads). One record is one entity's
 * change as move_process_cmds (movement.c:3246) leaves it in the engine's own tables; which state or flock an order gives
 * stays the engine's decision (make_flock, movement.c:855-862). Fields are written in the order of the mask bits. 64 bytes. */
#define PFNAV_DELTA_STATE        (1u << 0)   /* agent.state = state                                                      */
#define PFNAV_DELTA_FLOCK        (1u << 1)   /* agent.flock = flock (-1: none): an index into the flock table AFTER the call */
#define PFNAV_DELTA_AUX_DEST     (1u << 2)   /* agent.aux_dest1                                                          */
#define PFNAV_DELTA_FLAGS        (1u << 3)   /* agent.flags = flags & 0xFFFFFF (GARRISONED, COMBAT_HELD, WATER / AIR ...)  */
#define PFNAV_DELTA_SPEEDS       (1u << 4)   /* agent.max_speed, agent.speed                                             */
#define PFNAV_DELTA_RADIUS       (1u << 5)   /* agent.radius (may move the entity to another navigation layer)           */
#define PFNAV_DELTA_VELOCITY     (1u << 6)   /* agent.velocity (the velocity history is not touched)                     */
#define PFNAV_DELTA_POSITION     (1u << 7)   /* teleport (MOVE_CMD_UPDATE_POS): pos = prev_pos = position,
                                              * movestate.next_pos x and z = position, step = 0, left = 0                */
#define PFNAV_DELTA_CLEAR_HIST   (1u << 8)   /* move_notify_motion_start: zero movestate.vel_hist unless the entity is
                                              * COMBAT_HELD at that point -- pfnav_agents_apply_updates' SET_MOVING rule   */
#define PFNAV_DELTA_TARGET       (1u << 9)   /* movestate_ext.surround_target_uid = target_uid (PFNAV_NULL_UID: none),
                                              * movestate_ext.target_range = target_range                                */
typedef struct pfnav_agent_delta {
    uint32_t uid, mask;
    uint32_t state;
    int32_t  flock;
    uint32_t aux_dest1, flags;
    float    position[2], velocity[2], max_speed, speed, radius;
    uint32_t target_uid;
    float    target_range;
    uint32_t _pad;
} pfnav_agent_delta;
/* Apply n deltas (HOST array) to the device-resident population, and optionally replace the flock table.
 * - flocks == NULL: the flock table is unchanged (nflocks is ignored). Otherwise flocks[0 .. nflocks) is the whole new
 *   table: it may grow, shrink (when no entity keeps an index it drops) and entries may change.
 * - deltas and flocks are read before the call returns, whatever memory they are in: they can be reused at once.
 * - Deltas apply in array order; several deltas for one uid compose exactly as if applied one after the other.
 * - Everything is validated before anything changes: uid in the context's own range, no unknown mask bit, state within
 *   enum pfnav_move_state, -1 <= flock < the table's length after the call, finite floats, the entity's resulting
 *   navigation layer (Entity_NavLayerWithRadius of its flags and radius) created, POSITION / CLEAR_HIST only with an
 *   uploaded movestate table, TARGET only with an uploaded movestate_ext table and target_uid inside the population.
 *   Failure: PFNAV_ERR_ARG, device and host state untouched.
 * - Flock member lists (when a delta carried FLOCK or the table's length changed), neighbour records and the facts the
 *   tick keeps on the host (largest radius, any GARRISONED, arrival constants per (flock, layer) in use) are brought to
 *   what pfnav_agents_upload of the resulting population would leave. Member lists are rebuilt on the device.
 * - Asynchronous on `stream`, ordered like pfnav_agents_apply_updates_ex, except that it waits for the stream to read
 *   the new flock offsets (nflocks + 1 words) when the member lists were rebuilt and 8 bytes of population facts when a
 *   delta carried RADIUS or FLAGS. The device flock buffers and the call's scratch regrow (a device synchronisation)
 *   when the table or the batch outgrows them.
 * - Like pfnav_agents_apply_updates it leaves the spatial index stale: follow with pfnav_agents_rebuild_index. It does
 *   not touch the blocking table (pfnav_agents_set_blocking is the call for that) or the work list
 *   (pfnav_agents_set_work_dev).
 * - PFNAV_ERR_NO_DEVICE on a host-only context. PFNAV_ERR_STATE (nothing changed) on a context in a multi-GPU job
 *   (pfnav_mgpu_init / pfnav_group_create, or an own range that is not the whole population). */
int  pfnav_agents_commands(pfnav_ctx *ctx, const pfnav_agent_delta *deltas, size_t n,
                           const pfnav_flock *flocks, size_t nflocks, void *stream);
/* Units produced and units that die: remove entities from the device-resident population and append new ones.
 * - Numbering: a stable compaction followed by an append. remove_uids name entities of the population before the call
 *   (each < n_agents; a repeated uid is removed once). Survivor u gets the uid u - |{removed r < u}|, so survivors keep
 *   their order; appended entity k (add[k]) gets n_keep + k. There is no remap output: the engine updates its own
 *   uid -> index map with the same rule.
 * - Equivalence: afterwards every device table and host fact equals what reading the population back, deleting the
 *   removed rows, appending the new ones and uploading the result would leave (pfnav_agents_upload + _upload_movestate +
 *   _upload_movestate_ext + _upload_formation + _upload_blocking, for whichever tables exist): agents, neighbour records,
 *   movestate, movestate_ext, formation and blocking tables, the flock table and member lists, the largest radius, any
 *   GARRISONED, the (flock, layer) pairs in use and the arrival constants' invalidation. Beyond a re-upload:
 *     - every removed entity that holds a block (blocking record) queues the unblock op pfnav_agents_set_blocking(uid, 0)
 *       would queue, decided before the compaction; the next pfnav_map_commit applies it;
 *     - a survivor's movestate_ext.surround_target_uid is renumbered; a removed target becomes PFNAV_NULL_UID.
 * - Appended records: add_ms is required exactly when a movestate table was uploaded, add_blocking exactly when a
 *   blocking table covers the population (its records describe blocks already counted and queue no op: a new stationary
 *   unit takes its block with pfnav_agents_set_blocking after the call). add_ext and add_formation may be NULL where
 *   their table exists: defaults (ext zeroed with surround_target_uid = PFNAV_NULL_UID and rot = {0, 0, 0, 1}; formation
 *   zeroed: no formation). Appended ext targets name uids after the call. Records for a table that was never uploaded
 *   are refused.
 * - flocks == NULL keeps the flock table; otherwise flocks[0 .. nflocks) is the whole new table, as in
 *   pfnav_agents_commands; a table that would leave a surviving or appended entity with a dropped flock index is refused.
 * - Everything is validated before anything changes: remove uids in range, the upload's checks of appended agents
 *   (flock index within the table after the call, navigation layer created) and blocking records, finite floats,
 *   appended ext targets < the new population or PFNAV_NULL_UID. Failure: PFNAV_ERR_ARG, device and host state untouched.
 *   No removal, no addition and no table: nothing happens.
 * - The spatial index is rebuilt for the new population; the work list is emptied (follow with pfnav_agents_set_work_dev).
 * - Asynchronous on `stream`. It waits for the stream to read the new flock offsets and 8 bytes of population facts, and
 *   4 bytes more when removals may change whether any blocking record names a faction; it waits for the device when a
 *   per-entity buffer or the call's scratch regrows. Shares the scratch of pfnav_agents_commands and
 *   pfnav_agents_set_work_dev: order them on one stream. Input arrays are read before the call returns.
 * - PFNAV_ERR_NO_DEVICE on a host-only context. PFNAV_ERR_STATE (nothing changed) on a context in a multi-GPU job, as
 *   for pfnav_agents_commands: a job takes pfnav_mgpu_change_population / pfnav_group_change_population. */
int  pfnav_agents_change_population(pfnav_ctx *ctx, const uint32_t *remove_uids, size_t nremove,
                                    const pfnav_agent *add, const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext,
                                    const pfnav_formation_in *add_formation, const pfnav_blocking *add_blocking, size_t nadd,
                                    const pfnav_flock *flocks, size_t nflocks, void *stream);
/* pfnav_agents_commands for a whole multi-GPU job. Every rank calls the NCCL form with the same arguments, the job's
 * whole batch (uids global, in [0, n_total)); the group form is called once. Delta format, masks and the flock-table
 * rule are those of pfnav_agents_commands.
 * - Equivalence: after the call and the next pfnav_mgpu_gather / pfnav_group_gather, every member's snapshot is what
 *   one context holding the whole population would have after pfnav_agents_commands(same arguments): its own range's
 *   agent, movestate and movestate_ext records, the whole flock id column, the flock table, the member lists, largest
 *   radius and any GARRISONED, flock_layer_used of its own range (as pfnav_agents_upload_shard of the resulting range
 *   would leave it) and the arrival constants' invalidation.
 * - A member applies the deltas of the uids it owns as the solo call does. For every other uid it writes only what no
 *   tick step changes: the flock id, the neighbour record's radius and its low 24 flag bits (only uploads and command
 *   batches write those). Position, velocity and state of other members' entities arrive with the next gather, as
 *   always. From its complete flock column and records each member rebuilds the member lists and population facts on
 *   its device, so the next gather does not carry the flock column and rebuilds nothing on the host.
 * - All or nothing across the job: each member validates the deltas against the population (the checks of
 *   pfnav_agents_commands with [0, n_total) as the range) and its own entities' layers and flock indices, then the
 *   members exchange one verdict record {status, n_agents, n_flocks}: NCCL all-gathers it on `stream` and reads it, a
 *   group reads its members' host state. If any member refuses, every member returns that member's error and the text
 *   names it; members whose population or flock table sizes differ return PFNAV_ERR_ARG. Nothing changes anywhere.
 *   POSITION / CLEAR_HIST need every member's movestate table, TARGET every member's movestate_ext table.
 * - Streams: the NCCL form runs on `stream`, the group form on each member's context stream. Host waits as in the solo
 *   call (flock offsets, population facts), plus the verdict read of the NCCL form. It does not touch blocker ops or the
 *   work list: pfnav_agents_set_blocking for commands stays on the rank that owns the uids, before the exchange.
 * - Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_STATE (nothing changed) on a context in no job, for
 *   the NCCL form on a group member, and on every member when one of them has uploaded its range with
 *   pfnav_agents_upload_shard (without PFNAV_UPLOAD_SAME_FLOCKS) and not gathered since: its flock column is not
 *   complete. An empty batch without a table does nothing and exchanges nothing. */
int  pfnav_mgpu_commands(pfnav_ctx *ctx, const pfnav_agent_delta *deltas, size_t n,
                         const pfnav_flock *flocks, size_t nflocks, void *stream);
int  pfnav_group_commands(pfnav_group *g, const pfnav_agent_delta *deltas, size_t n,
                          const pfnav_flock *flocks, size_t nflocks);
/* pfnav_agents_change_population for a whole multi-GPU job. Every rank calls the NCCL form with the same arguments, the
 * job's whole batch (uids global, in [0, n_total)); the group form is called once. Arguments, their meaning and the
 * record rules are those of pfnav_agents_change_population.
 * - Numbering: the solo rule. Survivor u gets u - |{removed r < u}|, appended entity k gets n_keep + k. After the call
 *   every member owns pfnav_mgpu_shard_range(n_new, rank, world): its entity range moves with the population.
 * - Equivalence: after the call and the next pfnav_mgpu_gather / pfnav_group_gather, every member's snapshot is what one
 *   context holding the whole population would have after pfnav_agents_change_population(same arguments), restricted to
 *   the member's new range: the own range's agent, movestate, movestate_ext, formation and blocking records, the whole
 *   flock id column and neighbour records, the flock table and member lists, largest radius and any GARRISONED,
 *   flock_layer_used, blocking_n and blocking_any_fac of the own range (as pfnav_agents_upload_shard of the new range
 *   would leave them) and the arrival constants' invalidation.
 * - Moves: each member compacts its own survivors, and the flock id column and neighbour records of the whole population
 *   it holds; the survivors that cross a member boundary (at most nremove + nadd rows per boundary) move with all their
 *   records, NCCL broadcasts on `stream` for the NCCL form, peer copies on the members' context streams for the group.
 *   Each member writes the appended entities of its new range.
 * - Blocks and targets: a removed entity that holds a block queues its unblock op on its old owner, decided before any
 *   row moves; exchange the ops (pfnav_mgpu_exchange_blocker_ops / pfnav_group_exchange_blocker_ops) before
 *   pfnav_map_commit. Surround and enter-range targets are renumbered on every member; a removed target becomes
 *   PFNAV_NULL_UID.
 * - All or nothing across the job: each member validates the batch as the solo call does, its own survivors' flock
 *   indices against a shorter flock table included, then the members exchange one verdict record {status, n_agents,
 *   n_flocks, tables present}: NCCL all-gathers it on `stream` and reads it, a group reads its members' host state. If any
 *   member refuses, every member returns that member's error and the text names it; members whose population size, flock
 *   table size or set of uploaded tables differ return PFNAV_ERR_ARG. Nothing changes anywhere.
 * - After the call the work list is empty (follow with pfnav_agents_set_work_dev) and the spatial index is left to the
 *   gather that follows, which carries the neighbour records only: the member lists and population facts are rebuilt on
 *   each member's device. Host waits: the verdict read of the NCCL form, the received rows' flock ids and records (for the
 *   member's (flock, layer) facts), the flock offsets, population facts and, with a blocking table, one 4-byte fact;
 *   buffer regrowths wait for the device. Shares the scratch of pfnav_agents_commands and pfnav_agents_set_work_dev.
 * - Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_STATE (nothing changed) on a context in no job, for the
 *   NCCL form on a group member, and on every member when one of them has uploaded its range with
 *   pfnav_agents_upload_shard (without PFNAV_UPLOAD_SAME_FLOCKS) and not gathered since; for a group whose members sit
 *   on devices without peer access between them. An empty batch without a table does nothing and exchanges nothing. */
int  pfnav_mgpu_change_population(pfnav_ctx *ctx, const uint32_t *remove_uids, size_t nremove,
                                  const pfnav_agent *add, const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext,
                                  const pfnav_formation_in *add_formation, const pfnav_blocking *add_blocking, size_t nadd,
                                  const pfnav_flock *flocks, size_t nflocks, void *stream);
int  pfnav_group_change_population(pfnav_group *g, const uint32_t *remove_uids, size_t nremove,
                                   const pfnav_agent *add, const pfnav_movestate *add_ms, const pfnav_movestate_ext *add_ext,
                                   const pfnav_formation_in *add_formation, const pfnav_blocking *add_blocking, size_t nadd,
                                   const pfnav_flock *flocks, size_t nflocks);
/* Inputs beyond point seeking as deltas: the fields of pfnav_movestate_ext and the pfnav_formation_in records that the
 * engine decides, written for a subset of the population without reading or uploading the whole tables. The library
 * writes fields; which field an engine action sets stays the engine's decision (a turn order: TARGET_DIR, with the
 * TURNING state through pfnav_agents_commands; Entity_SetRot: ROT; a new surround or enter-range order: TARGET_PREV and
 * SURROUND_FIELD, with its target through PFNAV_DELTA_TARGET; a flock entering, moving in or leaving a formation:
 * FORMATION). surround_target_uid and target_range are PFNAV_DELTA_TARGET's; wait_prev and wait_ticks_left are decided
 * by the device. 128 bytes. */
#define PFNAV_INPUT_TARGET_PREV    (1u << 0)  /* movestate_ext.target_prev_pos                      */
#define PFNAV_INPUT_TARGET_DIR     (1u << 1)  /* movestate_ext.target_dir (STATE_TURNING)            */
#define PFNAV_INPUT_ROT            (1u << 2)  /* movestate_ext.rot (Entity_SetRot)                   */
#define PFNAV_INPUT_SURROUND_FIELD (1u << 3)  /* movestate_ext.using_surround_field, 0 or 1          */
#define PFNAV_INPUT_FORMATION      (1u << 4)  /* the whole pfnav_formation_in record                 */
typedef struct pfnav_input_delta {
    uint32_t uid, mask;
    float    target_prev_pos[2];
    float    target_dir[4];
    float    rot[4];
    uint32_t using_surround_field;
    uint32_t _pad[3];
    pfnav_formation_in formation;             /* offset 64 */
} pfnav_input_delta;                          /* 128 bytes */
/* Write n input deltas (HOST array) into the device-resident movestate_ext and formation tables.
 * - Order: records apply in array order; several records for one uid compose as if applied one after the other (per
 *   field, the last writer wins).
 * - Everything is validated before anything changes: uid in the context's own range, no unknown mask bit, every float
 *   the mask selects finite, using_surround_field 0 or 1, formation flags within the five PFNAV_FORM_* bits, the four
 *   movestate_ext bits only with an uploaded movestate_ext table. Failure: PFNAV_ERR_ARG, device and host state
 *   untouched. n == 0 does nothing.
 * - Formation table: when none exists, PFNAV_INPUT_FORMATION first creates one exactly as pfnav_agents_upload_formation
 *   of all-zero records would, then writes. A present table is not the same as no table (the velocity pass of
 *   ARRIVING_TO_CELL and MOVING_IN_FORMATION reads it), so a batch that creates it changes what the tick does for every
 *   entity in those states.
 * - Equivalence: afterwards both tables equal what reading them back (pfnav_agents_read_movestate_ext /
 *   pfnav_agents_read_formation), applying the records in order on the host and uploading them whole would leave.
 * - The call writes those two tables and nothing else: it leaves the spatial index, the arrival constants, the blocker
 *   ops and the work list as they are.
 * - Asynchronous on `stream`: the records go through the request staging and are read before the call returns, so the
 *   array can be reused at once. It waits for the device only when a table is created or the staging buffer grows.
 * - PFNAV_ERR_NO_DEVICE on a host-only context. PFNAV_ERR_STATE (nothing changed) on a context in a multi-GPU job, as
 *   for pfnav_agents_commands: a job takes pfnav_mgpu_input_deltas / pfnav_group_input_deltas. */
int  pfnav_agents_input_deltas(pfnav_ctx *ctx, const pfnav_input_delta *d, size_t n, void *stream);
/* pfnav_agents_input_deltas for a whole multi-GPU job. Every rank calls the NCCL form with the same arguments, the job's
 * whole batch (uids global, in [0, n_total)); the group form is called once. Record format and rules are the solo call's.
 * - Each member writes the records of the uids it owns. A batch with PFNAV_INPUT_FORMATION creates the formation table on
 *   every member that has none, so the members' sets of tables stay equal.
 * - All or nothing across the job: each member validates the whole batch (the solo checks with [0, n_total) as the
 *   range), then the members exchange one verdict record {status, n_agents, n_flocks, tables present}: NCCL all-gathers
 *   it on `stream` and reads it (the exchange of pfnav_mgpu_commands), a group reads its members' host state. If any
 *   member refuses, every member returns that member's error and the text names it; members whose population size or
 *   set of tables (movestate_ext, formation) differ return PFNAV_ERR_ARG. Nothing changes anywhere.
 * - Streams: the NCCL form runs on `stream` and waits for the verdict read, the group form on each member's context
 *   stream. n == 0 does nothing and exchanges nothing.
 * - Errors: PFNAV_ERR_NO_DEVICE on a host-only context; PFNAV_ERR_STATE (nothing changed) on a context in no job and
 *   for the NCCL form on a group member. */
int  pfnav_mgpu_input_deltas(pfnav_ctx *ctx, const pfnav_input_delta *d, size_t n, void *stream);
int  pfnav_group_input_deltas(pfnav_group *g, const pfnav_input_delta *d, size_t n);
/* pfnav_agents_set_work(ctx, NULL, 0) from the state resident on the device: the uids of the context's own range whose
 * state is neither ARRIVED nor WAITING, ascending, compacted on the device on `stream`. It waits for the stream once, to
 * read the 4-byte count that sizes the per-work-item buffers; it waits for the whole device only when the list outgrows
 * those buffers (they are then reallocated with room to spare) or the call's scratch has to grow. out_nwork may be NULL.
 * pfnav_agents_commands and this call share one device scratch buffer: order them on one stream (or with an event). */
int  pfnav_agents_set_work_dev(pfnav_ctx *ctx, void *stream, size_t *out_nwork);
/* Inspection and tests only, not for the tick loop: the current work list, in order. It waits for the whole device.
 * *out_n: the list's length; at most maxout uids are written (out may be NULL when maxout is 0). */
int  pfnav_agents_read_work(pfnav_ctx *ctx, uint32_t *out, size_t maxout, size_t *out_n);

/* Checkpoint / resume (G_Move_SaveState / G_Move_LoadState, SURVEY 5): the device-resident population as checkpoint
 * segments, and back. The format (csrc/pfnav_checkpoint_host.h): a 64-byte header (magic, format version, record sizes,
 * n_total, the segment's uid range [lo, hi), hz, nflocks, which of the movestate, movestate_ext, formation and blocking
 * tables exist), the whole flock table, then for each uid in [lo, hi), in uid order, its pfnav_agent, pfnav_movestate
 * and, where the tables exist, pfnav_movestate_ext, pfnav_formation_in and pfnav_blocking records. The map is not saved:
 * the engine rebuilds it. The field pool and its LRU state are not in these segments: pfnav_pool_save / pfnav_pool_restore
 * (below) save and restore them on their own, or the engine re-requests the fields after a restore.
 *
 * Save point: after the commit that follows the apply, the commands and the population change of a tick
 * (pfnav_agents_apply_updates[_ex] -> commands / pfnav_agents_set_blocking / population change -> exchange ->
 * pfnav_map_commit). There no device-decided blocker op is pending and the records are those the last apply left.
 * pfnav_agents_save writes one segment for the context's own range [shard_lo, shard_hi): on a single context the whole
 * population, in a multi-GPU job each member's range, and the members' segments together describe the population.
 * - out == NULL or cap < the segment's size: PFNAV_ERR_NOMEM with *out_size set, nothing written (as pfnav_ents_in_circles).
 * - The per-entity tables are packed on the device on `stream` into one staging buffer and copied to out in one copy; the
 *   call returns when out is filled.
 * - PFNAV_ERR_STATE (nothing written) when the last update pass is not applied, or when device blocker ops are not
 *   committed (in a job that shares blockers: not exchanged and committed). PFNAV_ERR_NO_DEVICE on a host-only context;
 *   PFNAV_ERR_ARG when no population was uploaded. */
int  pfnav_agents_save(pfnav_ctx *ctx, void *out, size_t cap, size_t *out_size, void *stream);
/* Restore from the nseg segments segs[i] (sizes[i] bytes each, host memory, any order) of one save, on a context whose map
 * is built (pfnav_map_build_nav, pfnav_route_build for every layer an entity of a flock stands on) and whose building
 * blockers the engine has already queued: a fresh map, whose blocker counts hold only those buildings. The restore does not
 * release the blocks of a population already on the context (blocking rows, or device ops not yet committed), so a load in
 * the middle of a session rebuilds the map first. A context outside any job takes the whole population; a member of a job
 * (pfnav_mgpu_init / pfnav_group_create) takes pfnav_mgpu_shard_range(n_total, rank, world) of its own job, whatever the
 * number of members that saved: segments of 3 members restore onto 1, 2 or 8.
 * - Everything is validated before anything changes: magic, version and record sizes; each segment's size; segments that
 *   overlap, leave a gap in [0, n_total) or disagree on n_total, hz, the flock table or the tables they hold; every record
 *   with the checks of the uploads and pfnav_agents_change_population and no others (flock index below the table's
 *   length, navigation layer created, finite floats, movestate_ext targets below n_total, blocking 0 / 1, faction_id
 *   0..15), so whatever the uploads accepted and pfnav_agents_save wrote restores.
 *   Failure: PFNAV_ERR_ARG. A layer without pfnav_route_build, or blocking records on a job member whose job does not
 *   share blockers: PFNAV_ERR_STATE. Either way nothing changes.
 * - Afterwards every table, the flock table, the member lists and the host facts are what pfnav_agents_upload_shard
 *   (flags 0) and pfnav_agents_upload_movestate / _movestate_ext / _formation / _blocking of the same records leave; a
 *   table the segments do not hold is dropped. The arrival constants are invalidated, the work list is empty and the
 *   event list is no longer readable.
 * - Beyond those uploads: for every restored record with blocking = 1, in uid order, the incref of its recorded circle
 *   (stop_x, stop_z, stop_radius, faction_id, on the layers of the entity's flags) is queued on the device on `stream`
 *   as a device-decided op; the next pfnav_map_commit applies it (in a job after pfnav_*_exchange_blocker_ops).
 * - Then, as after an upload: pfnav_map_commit, in a job pfnav_mgpu_gather / pfnav_group_gather, then
 *   pfnav_agents_set_work_dev, and the fields re-requested into the pool.
 * - The call waits for the device: the records go through the blocking copies of the uploads.
 * pfnav_group_restore: the same for every member of a group, in one call. The segments are validated once, then every
 * member's state; a refusal of either changes no member. The guarantee covers validation: a CUDA or allocation failure
 * while member i uploads (PFNAV_ERR_CUDA / PFNAV_ERR_NOMEM) leaves members 0 .. i-1 restored and the others as they were.
 * NCCL jobs: every rank calls pfnav_agents_restore with the same segments; no collective is involved. The verdict depends
 * on the segments and on the rank's map (layers created, pfnav_route_build of the layers in use), so every rank must
 * build the same layers for the ranks to agree. */
int  pfnav_agents_restore(pfnav_ctx *ctx, const void *const *segs, const size_t *sizes, size_t nseg, void *stream);
int  pfnav_group_restore(pfnav_group *g, const void *const *segs, const size_t *sizes, size_t nseg);

/* Field pool checkpoint (optional): the whole pool of one context as one segment, and back, so that a resumed game ticks
 * exactly like the game that was saved. Without it a restored context starts with a cold pool and fills it through the
 * miss path, which can build other fields than the saved pool held (a path field follows the route of the request that
 * built it, a LOS field its parent chunk's, repairs write fields in place, evictions follow the touch stamps), so the
 * continuation can differ from the saving game's. The format (csrc/pfnav_pool_host.h): a 64-byte header (magic "PFPL",
 * format version, record sizes, chunk_w, chunk_h, nlayers, ndests, max_fields, used, nzone, tick number, map digest, and
 * the counts of free-list entries, aux targets, their footprints and stored fields); the slot table, ff_ids, `has`
 * bytes, last requests, host touch stamps, owners and free list; the TARGET_ENTITY / TARGET_ENEMIES targets with their
 * footprints (what in-place repairs of those fields start from); the device touch stamps; then the flow and LOS bytes
 * (8192) of every slot with a `has` bit, in ascending slot order. Every section is 16-byte aligned.
 *
 * The map digest is a 64-bit value over the committed map: the cost, blocker counts, local islands and faction masks of
 * every tile of every layer, the enemy table (pfnav_set_enemy_factions), nlayers, chunk_w, chunk_h and the map position.
 * A segment restores only onto a context whose digest equals the saved one, so fields never land on a map they were not
 * built on.
 *
 * pfnav_pool_save: same sizing protocol as pfnav_agents_save.
 * - out == NULL or cap < the segment's size: PFNAV_ERR_NOMEM with *out_size set, nothing written.
 * - Ordered on `stream` (NULL: the context's stream) after forked field work and after a pending pfnav_pool_clear (a
 *   cleared pool saves as empty). The fields and the device touch stamps are packed on the device and come back in one
 *   copy; the call returns once out is filled.
 * - PFNAV_ERR_STATE (nothing written) while blocker ops are not committed: device-decided ops, pfnav_blockers_* calls or
 *   dirty chunks that the next pfnav_map_commit would apply, since that commit drops fields. PFNAV_ERR_NO_DEVICE on a
 *   host-only context; PFNAV_ERR_ARG when no pool was created.
 * pfnav_pool_restore: replaces the context's whole pool with the segment's: every slot-table entry, ff_id, `has` byte, last
 * request, host and device touch stamp, owner, the free-list order, `used`, the zone-held count, every aux target with its
 * footprints, the stored flow and LOS bytes, and the context's tick number (so that later evictions pick the same slots).
 * It invalidates the resident goal plan and changes nothing else: not the agents, the map, the work list or the events.
 * - Everything is validated before anything changes: PFNAV_ERR_ARG for a wrong magic, version or record size, a size that
 *   is not exact, a map geometry (chunk_w, chunk_h, nlayers) or pool geometry (ndests, max_fields) other than the
 *   context's, a map digest other than the context's committed map's, bookkeeping that breaks the pool's invariants (every
 *   slot below `used` is free, owned by the key that maps it, or zone-held; the zone-held count; free-list entries
 *   distinct, below `used`, unmapped and without fields; nothing at or above `used` mapped; a slot mapped by at most one
 *   key; ff_ids only on mapped keys; `has` bits within flow | LOS; no touch stamp above the tick number), a built flow
 *   field whose request names a layer that is not created, and an aux target with a bad kind or layer or a footprint
 *   that is not finite. PFNAV_ERR_STATE while blocker ops are not committed on the context (as on save); PFNAV_ERR_ARG
 *   when it has no pool. A refusal changes nothing.
 * - The call waits for the device before it writes the pool (a tick on any stream may read it) and returns once the pool
 *   is in place; the segment may be freed then.
 * Resume order: map built -> buildings queued -> pfnav_agents_restore -> (job: exchange) -> pfnav_map_commit ->
 * pfnav_pool_restore -> gather / index -> pfnav_agents_set_work_dev -> tick. Nothing needs to be re-requested.
 * Jobs: each member saves and restores its own pool, no collective is involved. A member's pool restored onto the member of
 * the same rank in a job with as many members gives the saving job's continuation. Any segment of the same map restores
 * onto any context with the same pool geometry, since it is a valid pool for that map; but with another member split the
 * work items whose misses a member serves change, and the continuation is not promised to equal the saving job's. */
int  pfnav_pool_save(pfnav_ctx *ctx, void *out, size_t cap, size_t *out_size, void *stream);
int  pfnav_pool_restore(pfnav_ctx *ctx, const void *seg, size_t size, void *stream);

/* State digest: 64-bit digests of the device-resident game state, computed on the device, so that a lockstep or replay
 * engine can compare a per-tick checksum between peers, or between a replay and its recording, without reading tables
 * back, and bisect to the first entity that differs. The definitions (csrc/pfnav_digest_host.h) are functions of the
 * bytes pfnav_agents_save / pfnav_pool_save write, so a digest can be recomputed on the host from saved segments:
 *   PFNAV_DIGEST_POPULATION  wrapping sum over the uids of the context's own range of a hash of the uid, the tables bits
 *                            and the row pfnav_agents_save writes for it (agent, movestate, movestate_ext, formation and
 *                            blocking records where the tables exist). With it, a block array: the same sum over the uids
 *                            [b << block_log2, (b + 1) << block_log2) for b < ceil(n_total >> block_log2), zero outside
 *                            the own range. Members' values and arrays add up (wrapping) to a single context's.
 *   PFNAV_DIGEST_FLOCKS      a chain over the flock table.
 *   PFNAV_DIGEST_RECORDS     wrapping sum over the whole population of a hash of (uid, 24-byte neighbour record): the
 *                            column every member of a job holds after a gather.
 *   PFNAV_DIGEST_MAP         the committed-map digest of the pool segment header.
 *   PFNAV_DIGEST_POOL        a digest of the segment pfnav_pool_save would write (its map digest word taken as zero).
 * A change confined to one 8-byte word of one row changes the population value and its block's entry for certain; other
 * changes change them except with probability about 2^-64.
 *
 * pfnav_state_digest queues the digest of the components in `what` on `stream` (NULL: the context's stream) and returns
 * without waiting for the device. It is ordered after the field work forked by the goal batches, as the pool's other
 * readers are, and hashes the state as it is at that point of `stream`; host-side parts (the flock table, the pool's
 * bookkeeping) are taken at the call. block_log2: 6..20 when POPULATION is selected, else ignored. One digest per context
 * is kept: a new call replaces the previous one (it is ordered after the previous one's copies).
 * Equality promise: at a point where pfnav_agents_save / pfnav_pool_save would succeed (after the commit that follows the
 * apply), the values equal the functions of csrc/pfnav_digest_host.h applied to the segments those calls would write;
 * RECORDS equals the sum over the segments of every member once the record column is current (a single context after
 * the apply; a job after the gather). Elsewhere the digest still hashes the state as it is.
 * - PFNAV_ERR_ARG, nothing queued: unknown `what` bits or none, block_log2 outside 6..20 with POPULATION, POPULATION,
 *   FLOCKS or RECORDS without an uploaded population, MAP without a map, POOL without a pool. PFNAV_ERR_NO_DEVICE on a
 *   host-only context.
 * pfnav_state_digest_read waits for that digest only (not for the stream) and writes the selected values into *out,
 * with n_total, the own range [lo, hi), the tables bits (1 movestate, 2 movestate_ext, 4 formation, 8 blocking) and hz.
 * blocks: NULL when the block array is not wanted; otherwise *nblocks is set to its length and, when cap is smaller,
 * PFNAV_ERR_NOMEM is returned with nothing else written (as pfnav_ents_in_circles). The digest stays readable until the
 * next pfnav_state_digest. PFNAV_ERR_STATE when no digest was queued. */
#define PFNAV_DIGEST_POPULATION (1u << 0)
#define PFNAV_DIGEST_FLOCKS     (1u << 1)
#define PFNAV_DIGEST_RECORDS    (1u << 2)
#define PFNAV_DIGEST_MAP        (1u << 3)
#define PFNAV_DIGEST_POOL       (1u << 4)
#define PFNAV_DIGEST_ALL        0x1Fu
typedef struct pfnav_digest {
    uint32_t what;                  /* the components held                                                   */
    int32_t  block_log2;
    uint32_t tables;                /* 1 movestate, 2 movestate_ext, 4 formation, 8 blocking                   */
    int32_t  hz;
    uint64_t n_total, lo, hi;       /* the population and the own range (a job's combined record: [0, n_total)) */
    uint64_t nblocks;
    uint64_t population, flocks, records, map, pool;
    /* job forms only (zero elsewhere): bit r set when member r's value differs from member 0's (ranks 63 and above
     * share bit 63) */
    uint64_t differ_flocks, differ_records, differ_map;
} pfnav_digest;
int  pfnav_state_digest(pfnav_ctx *ctx, uint32_t what, int block_log2, void *stream);
int  pfnav_state_digest_read(pfnav_ctx *ctx, pfnav_digest *out, uint64_t *blocks, size_t cap, size_t *nblocks);
/* The job forms. pfnav_group_state_digest digests every member (each on its context stream) and waits for them. out has
 * room for world + 1 records: out[0] is the job's, out[1 + r] member r's own as pfnav_state_digest_read gives it. In
 * out[0], population and blocks are the wrapping sums of the members' values (the single context's values), flocks,
 * records and map are member 0's with the differ_* masks, pool is zero: pools follow the member split, so each member's
 * is in its own record. blocks / cap / nblocks: the job's summed array, as for the read.
 * pfnav_mgpu_state_digest is the NCCL form: every rank calls it with the same arguments; it queues the rank's digest on
 * `stream` and all-gathers the ranks' fixed-size digest records in one collective on `stream`, without a host wait.
 * pfnav_state_digest_read then gives every rank the job's population (the sum), flocks, records and map (rank 0's) and
 * the differ_* masks, with its own pool, range and block array; the job's block array is the element-wise sum of the
 * ranks' arrays, which the engine forms only when it bisects.
 * Errors: those of pfnav_state_digest (members refused before any is queued); PFNAV_ERR_STATE for the NCCL form on a
 * context in no job or in an in-process group. */
int  pfnav_group_state_digest(pfnav_group *g, uint32_t what, int block_log2, pfnav_digest *out, uint64_t *blocks, size_t cap,
                              size_t *nblocks);
int  pfnav_mgpu_state_digest(pfnav_ctx *ctx, uint32_t what, int block_log2, void *stream);

/* N_FlowFieldUpdate with TARGET_ENEMIES / TARGET_ENTITY straight into the pool (what N_RequestAsyncEnemySeekField /
 * N_RequestAsyncSurroundField + N_AwaitAsyncFields leave in the field cache, nav.c:3769-3960): the fields of the listed
 * chunks become the flow fields of pool destination `dest`; entities name it through pfnav_agent::aux_dest1. The
 * footprints are remembered for the in-place repairs of N_DesiredEnemySeekVelocity / N_DesiredSurroundVelocity
 * (nav.c:3647-3675, 3729-3757), which pfnav_pool_repair runs for entities standing on a tile without direction. */
int  pfnav_pool_request_entity_fields(pfnav_ctx *ctx, int dest, int layer, int ref_layer, int target_kind,
                                      const pfnav_footprint *ents, size_t nents, const int32_t *chunks_rc, size_t n,
                                      void *stream);
/* One request of pfnav_pool_request_entity_fields_batch: the arguments of one pfnav_pool_request_entity_fields call,
 * with its footprints and chunks given as ranges of the batch's shared arrays. */
typedef struct pfnav_entity_field_req {   /* 32 bytes */
    int32_t  dest, layer, ref_layer, target_kind;   /* as pfnav_pool_request_entity_fields */
    uint32_t ent_off, ent_n;                        /* footprints ents[ent_off .. ent_off + ent_n) */
    uint32_t chunk_off, chunk_n;                    /* (r, c) pairs chunks_rc[2*chunk_off ..] */
} pfnav_entity_field_req;
/* N_RequestAsyncEnemySeekField / N_RequestAsyncSurroundField queued during a tick and built at once by
 * N_AwaitAsyncFields (nav.c:3769-3960): m requests against the device field pool in one call.
 * - Equivalence: the pool and the remembered footprints end exactly as pfnav_pool_request_entity_fields leaves them when
 *   called on requests 0 .. m-1 in order: flow bytes, `has` bytes, the ff_id pfnav_pool_get reports, LRU slot choices and
 *   evictions, and the footprints pfnav_pool_repair starts from. A later request wins: a repeated dest, or a repeated
 *   (dest, chunk), ends with the last request's field and footprints.
 * - Ranges of `ents` may overlap: several requests may name the same footprints (one enemy list for several factions).
 * - The whole batch is validated before anything changes: ranges, chunks, layers, target kinds, TARGET_ENTITY with
 *   ent_n == 1, the corners of every building footprint a field would use inside the map, and a map shape the padded
 *   chunk fields support (more than one chunk row and column, or 1 x 1). Failure: PFNAV_ERR_ARG, nothing changed.
 * - If the pool cannot hold request k's fields, requests 0 .. k-1 are done, *out_ndone = k (may be NULL) and
 *   PFNAV_ERR_NOMEM is returned; request k changed nothing.
 * - Launches are asynchronous on `stream` (NULL: the context's stream) and ordered after the field work forked by
 *   pfnav_pool_request_goals and after pfnav_pool_clear. The inputs are copied before the call returns, so the caller may
 *   reuse its buffers. The call does not wait for the device (except to evict under pool pressure). The seed frontiers
 *   are rasterised on the device.
 * - Host-only context: PFNAV_ERR_NO_DEVICE. */
int  pfnav_pool_request_entity_fields_batch(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m,
                                            const pfnav_footprint *ents, size_t nents,
                                            const int32_t *chunks_rc, size_t nchunks, void *stream, int *out_ndone);
/* pfnav_pool_request_entity_fields_batch for a whole job: every member with units of a faction seeking enemies needs
 * that faction's enemy fields. Each (dest, chunk) field is built on one member and copied to every member; the contract
 * is pfnav_mgpu_request_zones' (equivalence including the remembered footprints, owners, all or nothing with no
 * out_ndone, streams, errors). Every rank calls the NCCL form with the same arguments; the group form is called once. */
int  pfnav_mgpu_request_entity_fields_batch(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m,
                                            const pfnav_footprint *ents, size_t nents,
                                            const int32_t *chunks_rc, size_t nchunks, void *stream);
int  pfnav_group_request_entity_fields_batch(pfnav_group *g, const pfnav_entity_field_req *reqs, size_t m,
                                             const pfnav_footprint *ents, size_t nents,
                                             const int32_t *chunks_rc, size_t nchunks);
/* pfnav_pool_request_entity_fields_batch with the moving entities and the seekers named by uid, resolved on the device
 * from the resident records, so that the device-resident loop needs no positions on the host.
 * - Footprints: footprint k is ents[k] when ent_uids is NULL or ent_uids[k] == PFNAV_NULL_UID; otherwise it is the circle
 *   of resident entity ent_uids[k]: x, z = rec[uid].pos, sel_radius = rec[uid].radius, is_building = 0. ents may be NULL
 *   only when every entry names a uid. Buildings, and anything else outside the population, come in as footprints in
 *   the same array, so one enemy list can mix the two.
 * - Chunks: request i's chunk_off / chunk_n index seeker_uids, not chunks_rc. Its chunks are those of the tiles under
 *   those seekers' resident positions (M_Tile_DescForPoint2D, as the tick takes it), each once, in the order of its
 *   first seeker. A seeker whose position has no tile under it is PFNAV_ERR_ARG.
 * - Equivalence: the call leaves everything exactly as pfnav_pool_request_entity_fields_batch leaves it when given the
 *   footprints and chunk lists these rules resolve from the records as they are at the call: flow bytes, `has` bytes,
 *   the ff_id pfnav_pool_get reports, LRU slot choices and evictions, the footprints pfnav_pool_repair[_batch] starts
 *   from, *out_ndone and the NOMEM stop, and "a later request wins".
 * - Snapshot: as pfnav_ents_in_circles. Records written since the last index build (apply, commands, a job member's
 *   population change, pfnav_agents_upload_shard on a job member) give PFNAV_ERR_STATE and nothing changes. In the
 *   resident loop the call goes after pfnav_agents_rebuild_index / the gather and before pfnav_agents_set_work_dev and
 *   the tick.
 * - Validation before anything changes: everything the batch validates, applied to the resolved inputs; every uid below
 *   the whole population (global uids on a job member); nents, nseekers < 2^24; the NULL rules above. m == 0 is valid
 *   and resolves nothing. PFNAV_ERR_NO_DEVICE on a host-only context.
 * - Streams: queued on `stream` (NULL: the context's stream) after the forked field work, like the batch. One host wait
 *   reads the resolved values back (12 bytes per named footprint, 4 per seeker); after it, the batch's own behaviour.
 * The job forms relate to pfnav_mgpu_request_entity_fields_batch / pfnav_group_request_entity_fields_batch the same way
 * and keep their all or nothing: each member resolves from its own record column (equal on every member after a
 * gather), and a member that cannot resolve the batch (stale records, a seeker off the map) refuses it, so every
 * member returns that error and no pool changes. */
int  pfnav_pool_request_entity_fields_resident(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m,
                                               const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents,
                                               const uint32_t *seeker_uids, size_t nseekers, void *stream, int *out_ndone);
int  pfnav_mgpu_request_entity_fields_resident(pfnav_ctx *ctx, const pfnav_entity_field_req *reqs, size_t m,
                                               const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents,
                                               const uint32_t *seeker_uids, size_t nseekers, void *stream);
int  pfnav_group_request_entity_fields_resident(pfnav_group *g, const pfnav_entity_field_req *reqs, size_t m,
                                                const pfnav_footprint *ents, const uint32_t *ent_uids, size_t nents,
                                                const uint32_t *seeker_uids, size_t nseekers);

/* Test / tuning hook for pfnav_agents_tick: 0 = single-pass velocity kernel; 1 (default) = while LOS chains of
 * pfnav_pool_request_goals are still in flight, run the part of the update that does not depend on the
 * fields (neighbours, separation, velocity obstacles, admissible ray intersections) before joining them and
 * only the final choice after; 2 = always split. Results are identical in every mode. */
int  pfnav_set_two_phase(pfnav_ctx *ctx, int mode);

/* Test / tuning hook: cohesion pass (cohesion_force, movement.c:1653). 0 (default) = flocks of >= 20 000 members are summed
 * through the position index with an exp(-0.12 d) cut-off at 230 wu and a per-entity fall-back to the full member list
 * wherever the cut-off could matter beyond float rounding; 1 = always windowed; 2 = always the full member list. */
/* AStar_PortalGraphPath (a_star.c:429; SURVEY 8f-2) for a batch of n searches, one device thread per search. req: 8 ints
 * per search {start chunk index, start tile r, c, end chunk index, end tile r, c, finish chunk index, finish portal index};
 * out: (4 + 3 * max_hops) ints per search {status, nhops, cost (float bits), 0, then (chunk index, portal index, local
 * island) per hop from start to finish}; status 1 = path found, 0 = none, -1 = the search outgrew its device scratch or
 * max_hops. on_device == 0 runs the host planner's own routine instead (what pfnav_route_request_path uses), for
 * comparison. Needs pfnav_route_build(layer); blocker changes must be committed. */
int  pfnav_route_graph_paths(pfnav_ctx *ctx, int layer, const int32_t *req, int n, int32_t *out, int max_hops, int on_device);
int  pfnav_set_cohesion_mode(pfnav_ctx *ctx, int mode);
/* test / tuning hook: counters of G_ClearPath_NewVelocity's retry loop (clearpath.c:702-713) since the last reset:
 * out4 = {first solves without an admissible velocity, of those with both neighbour lists non-empty, entities that
 * replayed the loop literally (order-dependent tie), solves inside those replays} */
int  pfnav_agents_clearpath_stats(pfnav_ctx *ctx, uint64_t *out4, int reset);

/* flags for pfnav_agents_tick */
#define PFNAV_TICK_VDES_FROM_POOL   (1u << 0)  /* compute vdes + has_dest_los on device (nav.c:3468, 4026) */

/* navigation_tick_task's velocity phase (movement.c:4263-4287): desired velocity gather,
 * boids steering, neighbour search, ClearPath. Asynchronous on `stream`. */
int  pfnav_agents_tick(pfnav_ctx *ctx, uint32_t flags, void *stream);

/* R_GL_MoveReadNewVelocities (render.h:672): copy the nwork new velocities (xz, 8 bytes each,
 * in work-list order) to HOST memory; blocks until the tick has finished. */
int  pfnav_agents_read_velocities(pfnav_ctx *ctx, float *out_xz, size_t maxout);
/* Diagnostics: preferred velocity (vpref), vdes and has_dest_los of each work item. */
int  pfnav_agents_read_debug(pfnav_ctx *ctx, float *out_vpref_xz, float *out_vdes_xz,
                             uint8_t *out_has_los, size_t maxout);

/* G_Pos_EntsInCircleFrom (position.c:379): neighbour query through the device spatial index,
 * returning uids in the reference's order. One query of pfnav_ents_in_circles at a point (maxout > 0; range < 0
 * gives 0 uids); for parity tests of the index itself. */
int  pfnav_ents_in_circle(pfnav_ctx *ctx, float x, float z, float range, uint32_t *out,
                          int maxout, int *out_n);

/* G_Pos_EntsInCircle / G_Pos_EntsInCircleFrom (position.c:379) for a batch of n queries, answered on the device from the
 * position index. 24 bytes per query. */
typedef struct pfnav_ents_query {
    float    x, z;       /* centre, when uid == PFNAV_NULL_UID                                          */
    float    range;      /* G_Pos_EntsInCircleFrom's range                                              */
    uint32_t uid;        /* != PFNAV_NULL_UID: the centre is that entity's resident position instead   */
    int32_t  maxout;     /* the reference's maxout: the raw hits are cut here, before the garrison filter */
    uint32_t _pad;
} pfnav_ents_query;
/* - Answers: query i's uids are out_ids[out_offsets[i] .. out_offsets[i + 1]), *out_total = out_offsets[n]. Each is what
 *   pfnav_ents_in_circle(x, z, range, maxout) returns: the same uids in the same order, including the cut at maxout and
 *   filter_garrisoned's swap-remove when the population holds GARRISONED entities. range < 0, maxout == 0 or a centre
 *   off the grid give an empty answer.
 * - Uid centres: rec[uid].pos, the position the index was built from (G_Pos_EntsInCircle(G_Pos_GetXZ(uid), ...)).
 * - Snapshot: answers come from the index of the last rebuild (pfnav_agents_rebuild_index, a gather, an upload, a solo
 *   population change). pfnav_agents_apply_updates[_ex], the solo and job command calls, the job population change and
 *   pfnav_agents_upload_shard on a job member write records after it; until the next rebuild the call returns
 *   PFNAV_ERR_STATE and changes nothing, so that centres and hits always come from one snapshot.
 * - Validation, before anything runs (PFNAV_ERR_ARG, outputs untouched): q, out_offsets and out_total non-NULL when
 *   n > 0; out_ids non-NULL when cap > 0; x, z and range finite; maxout >= 0; uid == PFNAV_NULL_UID or uid < the whole
 *   population (global uids on a job member); the answers' bound (the sum of min(maxout, population)) below 2^32.
 *   n == 0 is valid (*out_total = 0). PFNAV_ERR_NO_DEVICE on a host-only context.
 * - Capacity: *out_total > cap returns PFNAV_ERR_NOMEM with out_offsets and *out_total written and out_ids untouched:
 *   grow the buffer and call again (cap = 0 asks for the sizes only). PFNAV_ERR_NOMEM with *out_total <= cap: the
 *   device could not hold the answers.
 * - Streams: queued on `stream` (NULL: the context's stream) after the rebuild and after the field work forked by
 *   pfnav_pool_request_goals; returns when the outputs are filled. One host wait (the totals) before the final copy;
 *   only the hits are copied back. */
int  pfnav_ents_in_circles(pfnav_ctx *ctx, const pfnav_ents_query *q, size_t n, uint32_t *out_offsets /* n + 1 */,
                           uint32_t *out_ids, size_t cap, size_t *out_total, void *stream);

/* Device-side hooks for zero-copy callers (bench `value` leg, multi-GPU all-gather):
 * raw device pointers to the resident 24-byte neighbour records (pos.xz, vel.xz, radius,
 * state << 24 | flags) in uid order, and to the velocity output (work-list order). */
int  pfnav_agents_device_ptrs(pfnav_ctx *ctx, void **d_records, void **d_velocities, size_t *n);
/* Re-build the spatial index from the (externally updated, e.g. all-gathered) record array. */
int  pfnav_agents_rebuild_index(pfnav_ctx *ctx, void *stream);

/* Optional per-kernel-group device timing (CUDA events on the launching stream) used by bench.py
 * for its roofline line. pfnav_profile_read drains the recorded intervals: ms_out / count_out have
 * 8 entries: 0 flow kernels, 1 LOS kernels, 2 spatial-index build, 3 desired velocity, 4 cohesion,
 * 5 agent velocity (ClearPath). */
int  pfnav_profile_enable(pfnav_ctx *ctx, int enable);
int  pfnav_profile_read(pfnav_ctx *ctx, float *ms_out, uint32_t *count_out);
/* Host wall-clock time of the cold goal-batch path, recorded while profiling is enabled, summed since the last
 * read and reset by it: ms_out / count_out have 8 entries: 0 pfnav_pool_clear, 1 waits on events and streams,
 * 2 goal planning, 3 merge and dependency sort, 4 pool slot reservation, 5 packing of the plan, 6 H2D enqueue,
 * 7 kernel launches (segments of pfnav_pool_request_goals_ex unless noted). */
int  pfnav_profile_read_host(pfnav_ctx *ctx, double *ms_out, uint32_t *count_out);

/* Number of kernels launched by this context since creation (bench `gpu_launches`). */
uint64_t pfnav_launch_count(const pfnav_ctx *ctx);

#ifdef __cplusplus
}
#endif
#endif /* PFNAV_H */
