"""ctypes binding of libpfnav.so (the C ABI in include/pfnav.h).  Host-side mirror of the
reference's field/movement interfaces for tests and bench.py: same names, same argument meaning.

There is no fallback: importing works without a GPU (symbol checks), but Nav() raises when the
library cannot create a context on an sm_90 (H100) device."""
import ctypes as C
import os
import numpy as np

from . import build as _build

FD_NONE, FD_NW, FD_N, FD_NE, FD_W, FD_E, FD_SW, FD_S, FD_SE = range(9)
TARGET_PORTAL, TARGET_TILE = 0, 1
FACTION_ID_NONE = 0xF
ISLAND_NONE = 0xFFFF
OK, ERR_ARG, ERR_CUDA, ERR_NO_DEVICE, ERR_STATE, ERR_NOMEM = 0, -1, -2, -3, -4, -5      # pfnav_status

FIELD_REQ = np.dtype([
    ("chunk_r", "<i4"), ("chunk_c", "<i4"), ("layer", "<i4"), ("faction_id", "<i4"),
    ("target_type", "<i4"), ("init", "<i4"), ("tile_r", "<i4"), ("tile_c", "<i4"),
    ("port_r0", "<i2"), ("port_c0", "<i2"), ("port_r1", "<i2"), ("port_c1", "<i2"),
    ("next_r0", "<i2"), ("next_c0", "<i2"), ("next_r1", "<i2"), ("next_c1", "<i2"),
    ("next_chunk_r", "<i4"), ("next_chunk_c", "<i4"), ("port_iid", "<u2"), ("next_iid", "<u2"),
    ("_pad", "<i4")])
assert FIELD_REQ.itemsize == 64

LOS_REQ = np.dtype([
    ("chunk_r", "<i4"), ("chunk_c", "<i4"), ("layer", "<i4"), ("faction_id", "<i4"),
    ("tgt_chunk_r", "<i4"), ("tgt_chunk_c", "<i4"), ("tgt_tile_r", "<i4"), ("tgt_tile_c", "<i4"),
    ("prev_index", "<i4"), ("prev_chunk_r", "<i4"), ("prev_chunk_c", "<i4"), ("_pad", "<i4")])
assert LOS_REQ.itemsize == 48

AGENT = np.dtype([
    ("pos", "<f4", 2), ("prev_pos", "<f4", 2), ("velocity", "<f4", 2), ("vdes", "<f4", 2),
    ("radius", "<f4"), ("max_speed", "<f4"), ("speed", "<f4"), ("state", "<u4"), ("flags", "<u4"),
    ("flock", "<i4"), ("has_dest_los", "<u4"), ("aux_dest1", "<u4")])
assert AGENT.itemsize == 64

FLOCK = np.dtype([("target", "<f4", 2), ("dest", "<i4"), ("layer", "<i4")])
assert FLOCK.itemsize == 16

MOVESTATE = np.dtype([
    ("next_pos", "<f4", 3), ("step", "<f4"), ("next_rot", "<f4", 4), ("combat_facing", "<f4", 4),
    ("vel_hist", "<f4", (14, 2)), ("left", "<i4"), ("vel_hist_idx", "<i4"), ("_pad", "<i4", 2)])
assert MOVESTATE.itemsize == 176

PATCH = np.dtype([
    ("flags", "<u4"), ("next_state", "<i4"), ("next_block", "<i4"), ("next_attack", "<i4"),
    ("next_velocity", "<f4", 2), ("next_pos", "<f4", 3), ("next_rot", "<f4", 4), ("next_ppos", "<f4", 3),
    ("next_npos", "<f4", 3), ("next_step", "<f4"), ("next_left", "<f4"), ("next_nrot", "<f4", 4),
    ("next_prot", "<f4", 4), ("wait_ticks_left", "<i4"), ("engine_todo", "<u4"), ("_padf", "<f4"),
    ("next_dest", "<f4", 2), ("next_target_prev", "<f4", 2), ("next_target_dir", "<f4", 4)])
assert PATCH.itemsize == 160

FORMATION_IN = np.dtype([
    ("cell_pos", "<f4", 2), ("cell_arrival_vdes", "<f4", 2), ("cohesion", "<f4", 2), ("align", "<f4", 2), ("drag", "<f4", 2),
    ("target_orientation", "<f4", 4), ("flags", "<u4"), ("_pad", "<u4")])
assert FORMATION_IN.itemsize == 64
FORM_HAS_FORMATION, FORM_ASSIGNMENT_READY, FORM_ASSIGNED_TO_CELL, FORM_IN_RANGE_OF_CELL, FORM_ARRIVED_AT_CELL = 1, 2, 4, 8, 16
MOVESTATE_EXT = np.dtype([
    ("wait_prev", "<i4"), ("wait_ticks_left", "<i4"), ("surround_target_uid", "<u4"), ("using_surround_field", "<u4"),
    ("target_range", "<f4"), ("target_prev_pos", "<f4", 2), ("_padf", "<f4"), ("target_dir", "<f4", 4), ("rot", "<f4", 4)])
assert MOVESTATE_EXT.itemsize == 64
NULL_UID = 0xFFFFFFFF
BLOCKING = np.dtype([("blocking", "<u4"), ("faction_id", "<i4"), ("stop_x", "<f4"), ("stop_z", "<f4"), ("stop_radius", "<f4"),
                     ("_pad", "<u4", 3)])
assert BLOCKING.itemsize == 32
APPLY_BLOCKERS = 1
AGENT_DELTA = np.dtype([
    ("uid", "<u4"), ("mask", "<u4"), ("state", "<u4"), ("flock", "<i4"), ("aux_dest1", "<u4"), ("flags", "<u4"),
    ("position", "<f4", 2), ("velocity", "<f4", 2), ("max_speed", "<f4"), ("speed", "<f4"), ("radius", "<f4"),
    ("target_uid", "<u4"), ("target_range", "<f4"), ("_pad", "<u4")])
assert AGENT_DELTA.itemsize == 64
(DELTA_STATE, DELTA_FLOCK, DELTA_AUX_DEST, DELTA_FLAGS, DELTA_SPEEDS, DELTA_RADIUS, DELTA_VELOCITY, DELTA_POSITION,
 DELTA_CLEAR_HIST, DELTA_TARGET) = (1 << i for i in range(10))
TODO_SURROUND_QUERY, TODO_USE_SURROUND_FIELD, TODO_DROP_SURROUND_FIELD = 1, 2, 4
INPUT_DELTA = np.dtype([
    ("uid", "<u4"), ("mask", "<u4"), ("target_prev_pos", "<f4", 2), ("target_dir", "<f4", 4), ("rot", "<f4", 4),
    ("using_surround_field", "<u4"), ("_pad", "<u4", 3), ("formation", FORMATION_IN)])
assert INPUT_DELTA.itemsize == 128 and INPUT_DELTA.fields["formation"][1] == 64
INPUT_TARGET_PREV, INPUT_TARGET_DIR, INPUT_ROT, INPUT_SURROUND_FIELD, INPUT_FORMATION = (1 << i for i in range(5))

REGION_REQ = np.dtype([
    ("layer", "<i4"), ("center_r", "<i4"), ("center_c", "<i4"), ("start_r", "<i4"), ("start_c", "<i4"),
    ("seed_off", "<i4"), ("seed_n", "<i4"), ("overlay_off", "<i4"), ("overlay_n", "<i4"),
    ("enemies", "<u2"), ("flags", "<u2")])
assert REGION_REQ.itemsize == 40
REGION_CREATE, REGION_FIXUP, REGION_CELL = 1, 2, 4

FOOTPRINT = np.dtype([("x", "<f4"), ("z", "<f4"), ("sel_radius", "<f4"), ("is_building", "<u4"), ("corners_xz", "<f4", 8)])
assert FOOTPRINT.itemsize == 48
TARGET_ENTITY, TARGET_ENEMIES = 0, 1
ENTITY_FIELD_REQ = np.dtype([("dest", "<i4"), ("layer", "<i4"), ("ref_layer", "<i4"), ("target_kind", "<i4"),
                             ("ent_off", "<u4"), ("ent_n", "<u4"), ("chunk_off", "<u4"), ("chunk_n", "<u4")])
assert ENTITY_FIELD_REQ.itemsize == 32
ZONE_REQ = np.dtype([("dest", "<i4"), ("layer", "<i4"), ("centre_x", "<f4"), ("centre_z", "<f4"), ("radius", "<i4"), ("_pad", "<i4")])
assert ZONE_REQ.itemsize == 24
QUERY_PATHABLE, QUERY_BLOCKED, QUERY_ADJACENT_IMPASSABLE, QUERY_CLOSEST_PATHABLE, QUERY_MAXIMALLY_CLOSE, QUERY_DEST_ID = range(6)
MAP_QUERY = np.dtype([("kind", "<i4"), ("layer", "<i4"), ("x", "<f4"), ("z", "<f4"), ("dst_x", "<f4"), ("dst_z", "<f4"),
                      ("tolerance", "<f4"), ("faction_id", "<i4")])
assert MAP_QUERY.itemsize == 32
MAP_QUERY_RESULT = np.dtype([("ok", "<i4"), ("dest_id", "<u4"), ("x", "<f4"), ("z", "<f4")])
assert MAP_QUERY_RESULT.itemsize == 16
ARRIVAL_RECORD = np.dtype([("flock", "<i4"), ("layer", "<i4"), ("nearest_ok", "<i4"), ("nearest", "<f4", 2), ("mc_n", "<i4"),
                           ("mc", "<f4", (256, 2))])
assert ARRIVAL_RECORD.itemsize == 2072
ENTS_QUERY = np.dtype([("x", "<f4"), ("z", "<f4"), ("range", "<f4"), ("uid", "<u4"), ("maxout", "<i4"), ("_pad", "<u4")])
assert ENTS_QUERY.itemsize == 24
EVENT = np.dtype([("uid", "<u4"), ("flags", "<u4"), ("todo", "<u4"), ("attack", "<i4"), ("state_before", "<u4"),
                  ("state_after", "<u4"), ("dest", "<f4", 2), ("pos", "<f4", 2), ("_pad", "<u4", 2)])
assert EVENT.itemsize == 48
# pfnav_digest (pfnav_state_digest_read) and its component bits
DIGEST = np.dtype([("what", "<u4"), ("block_log2", "<i4"), ("tables", "<u4"), ("hz", "<i4"), ("n_total", "<u8"),
                   ("lo", "<u8"), ("hi", "<u8"), ("nblocks", "<u8"), ("population", "<u8"), ("flocks", "<u8"),
                   ("records", "<u8"), ("map", "<u8"), ("pool", "<u8"), ("differ_flocks", "<u8"),
                   ("differ_records", "<u8"), ("differ_map", "<u8")])
assert DIGEST.itemsize == 112
DIGEST_POPULATION, DIGEST_FLOCKS, DIGEST_RECORDS, DIGEST_MAP, DIGEST_POOL = 1, 2, 4, 8, 16
DIGEST_ALL = 31

LOS_PREV_INPLACE = -3
TICK_VDES_FROM_POOL = 1
FLAG_MOVABLE, FLAG_WATER, FLAG_AIR, FLAG_GARRISONED, FLAG_COMBAT_HELD = 1 << 3, 1 << 14, 1 << 15, 1 << 18, 1 << 21

# every symbol include/pfnav.h declares
SYMBOLS = [
    "pfnav_last_error", "pfnav_version", "pfnav_create", "pfnav_destroy", "pfnav_map_create",
    "pfnav_map_upload_layer", "pfnav_map_update_chunk", "pfnav_map_build_nav", "pfnav_map_refresh_chunk",
    "pfnav_local_islands_get", "pfnav_portals_get", "pfnav_blockers_incref", "pfnav_blockers_decref", "pfnav_blockers_get",
    "pfnav_map_commit", "pfnav_plan_goal", "pfnav_route_build", "pfnav_route_islands_get",
    "pfnav_route_edges_get", "pfnav_route_request_path", "pfnav_create_hostonly", "pfnav_pool_request_path", "pfnav_pool_get", "pfnav_flow_fields_update",
    "pfnav_flow_fields_update_dev", "pfnav_los_fields_create", "pfnav_los_fields_create_dev",
    "pfnav_set_tma", "pfnav_pool_create", "pfnav_pool_put", "pfnav_pool_clear", "pfnav_pool_request_goal", "pfnav_pool_request_goals",
    "pfnav_agents_upload", "pfnav_agents_set_work", "pfnav_agents_tick",
    "pfnav_agents_read_velocities", "pfnav_agents_read_debug", "pfnav_ents_in_circle",
    "pfnav_agents_device_ptrs", "pfnav_agents_rebuild_index", "pfnav_launch_count", "pfnav_profile_enable",
    "pfnav_profile_read", "pfnav_map_cost_from_tiles", "pfnav_map_get_layer", "pfnav_fields_join", "pfnav_flow_fields_repair", "pfnav_pool_repair", "pfnav_pool_repair_batch", "pfnav_pool_repair_batch_stats", "pfnav_repair_seed_mask", "pfnav_set_enemy_factions", "pfnav_request_faction", "pfnav_set_two_phase", "pfnav_los_trace", "pfnav_set_los_variant", "pfnav_blockers_incref_obb", "pfnav_blockers_decref_obb",
    "pfnav_map_upload_factions", "pfnav_agents_upload_movestate", "pfnav_agents_compute_updates",
    "pfnav_agents_read_patches", "pfnav_agents_apply_updates", "pfnav_agents_read_state",
    "pfnav_region_fields", "pfnav_region_fields_dev", "pfnav_group_arrival_field", "pfnav_blockers_get_factions",
    "pfnav_route_arrival_consts", "pfnav_entity_seeds", "pfnav_entity_fields", "pfnav_pfmap_parse", "pfnav_map_load_pfmap", "pfnav_zone_seeds", "pfnav_zone_fields", "pfnav_pool_request_zone", "pfnav_group_arrival_velocity",
    "pfnav_mgpu_shard_range", "pfnav_mgpu_unique_id", "pfnav_mgpu_init", "pfnav_mgpu_finalize", "pfnav_mgpu_gather",
    "pfnav_group_create", "pfnav_group_gather", "pfnav_group_destroy", "pfnav_agents_upload_shard",
    "pfnav_pool_request_goals_ex", "pfnav_blockers_batch", "pfnav_map_set_pos",
    "pfnav_agents_upload_formation", "pfnav_agents_upload_movestate_ext", "pfnav_pool_request_entity_fields",
    "pfnav_pool_request_entity_fields_batch", "pfnav_pool_request_zones",
    "pfnav_set_cohesion_mode", "pfnav_agents_clearpath_stats", "pfnav_route_graph_paths", "pfnav_pool_request_paths",
    "pfnav_profile_read_host", "pfnav_map_query", "pfnav_agents_upload_blocking", "pfnav_agents_read_blocking",
    "pfnav_agents_apply_updates_ex", "pfnav_agents_set_blocking", "pfnav_mgpu_share_blockers", "pfnav_group_share_blockers",
    "pfnav_mgpu_exchange_blocker_ops", "pfnav_group_exchange_blocker_ops",
    "pfnav_mgpu_request_goals_ex", "pfnav_group_request_goals_ex", "pfnav_mgpu_fields_stats",
    "pfnav_mgpu_request_zones", "pfnav_group_request_zones", "pfnav_mgpu_request_entity_fields_batch",
    "pfnav_group_request_entity_fields_batch", "pfnav_pool_request_entity_fields_resident",
    "pfnav_mgpu_request_entity_fields_resident", "pfnav_group_request_entity_fields_resident",
    "pfnav_pool_request_paths_resident", "pfnav_map_query_resident", "pfnav_group_arrival_velocity_resident",
    "pfnav_agents_commands", "pfnav_agents_set_work_dev", "pfnav_agents_read_work",
    "pfnav_mgpu_commands", "pfnav_group_commands",
    "pfnav_agents_change_population", "pfnav_agents_read_movestate_ext", "pfnav_agents_read_arrival_consts",
    "pfnav_mgpu_change_population", "pfnav_group_change_population", "pfnav_ents_in_circles",
    "pfnav_agents_collect_events", "pfnav_agents_read_events",
    "pfnav_agents_input_deltas", "pfnav_mgpu_input_deltas", "pfnav_group_input_deltas", "pfnav_agents_read_formation",
    "pfnav_agents_save", "pfnav_agents_restore", "pfnav_group_restore", "pfnav_pool_save", "pfnav_pool_restore",
    "pfnav_state_digest", "pfnav_state_digest_read", "pfnav_group_state_digest", "pfnav_mgpu_state_digest",
]

_lib = None


def lib_path():
    return _build.LIB


def load():
    """dlopen libpfnav.so (building it first if the sources are newer). Raises if it cannot."""
    global _lib
    if _lib is not None:
        return _lib
    path = _build.LIB
    if not os.path.exists(path):
        path = _build.build()
    L = C.CDLL(path)
    L.pfnav_last_error.restype = C.c_char_p
    L.pfnav_launch_count.restype = C.c_uint64
    L.pfnav_launch_count.argtypes = [C.c_void_p]
    L.pfnav_create.argtypes = [C.c_int, C.POINTER(C.c_void_p)]
    L.pfnav_destroy.argtypes = [C.c_void_p]
    L.pfnav_map_create.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float]
    L.pfnav_map_upload_layer.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.pfnav_map_update_chunk.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.pfnav_map_build_nav.argtypes = [C.c_void_p, C.c_int]
    L.pfnav_fields_join.argtypes = [C.c_void_p, C.c_void_p]
    L.pfnav_set_enemy_factions.argtypes = [C.c_void_p, C.c_int, C.c_uint16]
    L.pfnav_request_faction.argtypes = [C.c_void_p, C.c_int]
    L.pfnav_set_two_phase.argtypes = [C.c_void_p, C.c_int]
    L.pfnav_set_los_variant.argtypes = [C.c_void_p, C.c_int]
    L.pfnav_blockers_incref_obb.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint32]
    L.pfnav_blockers_decref_obb.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_uint32]
    L.pfnav_los_trace.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfnav_map_upload_factions.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.pfnav_pool_repair.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pfnav_pool_repair_batch.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pfnav_pool_repair_batch_stats.argtypes = [C.c_void_p, C.c_void_p]
    L.pfnav_repair_seed_mask.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p]
    L.pfnav_flow_fields_repair.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_region_fields.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                      C.c_size_t, C.c_void_p]
    L.pfnav_region_fields_dev.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                          C.c_void_p]
    L.pfnav_pfmap_parse.argtypes = [C.c_char_p, C.c_size_t, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p, C.c_size_t]
    L.pfnav_map_load_pfmap.argtypes = [C.c_void_p, C.c_char_p, C.c_size_t, C.c_int, C.c_void_p, C.c_float, C.c_float]
    L.pfnav_route_arrival_consts.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.POINTER(C.c_int32), C.c_void_p, C.c_void_p,
                                             C.c_size_t, C.POINTER(C.c_int32)]
    L.pfnav_entity_seeds.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                     C.POINTER(C.c_size_t)]
    L.pfnav_entity_fields.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_zone_seeds.argtypes = [C.c_void_p] + [C.c_int] * 6 + [C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfnav_zone_fields.argtypes = [C.c_void_p] + [C.c_int] * 4 + [C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_pool_request_zone.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_int)]
    L.pfnav_pool_request_zones.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
    L.pfnav_map_query.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.pfnav_group_arrival_velocity.argtypes =[C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.pfnav_group_arrival_field.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_uint16, C.c_void_p, C.c_size_t, C.c_void_p,
                                            C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_agents_upload_movestate.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_compute_updates.argtypes = [C.c_void_p, C.c_void_p]
    L.pfnav_agents_read_patches.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_apply_updates.argtypes = [C.c_void_p, C.c_void_p]
    L.pfnav_agents_apply_updates_ex.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.pfnav_agents_collect_events.argtypes = [C.c_void_p, C.c_void_p]
    L.pfnav_agents_read_events.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfnav_agents_upload_blocking.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_read_blocking.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_set_blocking.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_void_p]
    L.pfnav_agents_read_state.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_commands.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_mgpu_commands.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_group_commands.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t]
    L.pfnav_agents_set_work_dev.argtypes = [C.c_void_p, C.c_void_p, C.POINTER(C.c_size_t)]
    L.pfnav_agents_read_work.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfnav_agents_change_population.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p,
                                                 C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_agents_read_movestate_ext.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_read_arrival_consts.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfnav_agents_read_formation.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_input_deltas.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_mgpu_input_deltas.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_group_input_deltas.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_mgpu_change_population.argtypes = L.pfnav_agents_change_population.argtypes
    L.pfnav_agents_save.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p]
    L.pfnav_agents_restore.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_group_restore.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_pool_save.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t), C.c_void_p]
    L.pfnav_pool_restore.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_state_digest.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]
    L.pfnav_state_digest_read.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.POINTER(C.c_size_t)]
    L.pfnav_group_state_digest.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t,
                                           C.POINTER(C.c_size_t)]
    L.pfnav_mgpu_state_digest.argtypes = [C.c_void_p, C.c_uint32, C.c_int, C.c_void_p]
    L.pfnav_group_change_population.argtypes = L.pfnav_agents_change_population.argtypes[:-1]
    L.pfnav_map_cost_from_tiles.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_size_t]
    L.pfnav_map_get_layer.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]
    L.pfnav_map_refresh_chunk.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int]
    L.pfnav_local_islands_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.pfnav_portals_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    L.pfnav_plan_goal.argtypes = [C.c_void_p] + [C.c_int] * 5 + [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                  C.POINTER(C.c_int), C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    L.pfnav_create_hostonly.argtypes = [C.POINTER(C.c_void_p)]
    L.pfnav_blockers_incref.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_int, C.c_uint32]
    L.pfnav_blockers_decref.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_int, C.c_uint32]
    L.pfnav_blockers_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.pfnav_blockers_get_factions.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.pfnav_map_commit.argtypes = [C.c_void_p, C.POINTER(C.c_int)]
    L.pfnav_pool_request_path.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p,
                                          C.POINTER(C.c_uint32), C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pfnav_pool_request_paths.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int)]
    L.pfnav_pool_get.argtypes =[C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    L.pfnav_route_build.argtypes = [C.c_void_p, C.c_int]
    L.pfnav_route_islands_get.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.pfnav_route_edges_get.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    L.pfnav_route_request_path.argtypes = [C.c_void_p, C.c_int, C.c_float, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int),
                                           C.c_void_p, C.c_void_p, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint32), C.POINTER(C.c_int)]
    L.pfnav_flow_fields_update.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_flow_fields_update_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.pfnav_flow_fields_update_general_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.pfnav_los_fields_create.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_los_fields_create_dev.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]
    L.pfnav_set_tma.argtypes = [C.c_void_p, C.c_int]
    L.pfnav_pool_create.argtypes = [C.c_void_p, C.c_int, C.c_int]
    L.pfnav_pool_put.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
    L.pfnav_pool_clear.argtypes = [C.c_void_p]
    L.pfnav_pool_request_goal.argtypes = [C.c_void_p] + [C.c_int] * 6 + [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pfnav_pool_request_goals.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p,
                                           C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pfnav_agents_upload.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
    L.pfnav_agents_set_work.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_pool_request_goals_ex.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p,
                                              C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pfnav_blockers_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_upload_formation.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_upload_movestate_ext.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_pool_request_entity_fields.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_size_t,
                                                   C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_pool_request_entity_fields_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                                         C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]
    L.pfnav_map_set_pos.argtypes = [C.c_void_p, C.c_float, C.c_float]
    L.pfnav_agents_upload_shard.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_size_t, C.c_size_t, C.c_void_p, C.c_size_t,
                                            C.c_int, C.c_uint32]
    L.pfnav_mgpu_shard_range.argtypes = [C.c_size_t, C.c_int, C.c_int, C.POINTER(C.c_size_t), C.POINTER(C.c_size_t)]
    L.pfnav_mgpu_unique_id.argtypes = [C.c_void_p]
    L.pfnav_mgpu_init.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.pfnav_mgpu_finalize.argtypes = [C.c_void_p]
    L.pfnav_mgpu_gather.argtypes = [C.c_void_p, C.c_void_p]
    L.pfnav_group_create.argtypes = [C.c_void_p, C.c_int, C.POINTER(C.c_void_p)]
    L.pfnav_group_gather.argtypes = [C.c_void_p]
    L.pfnav_group_destroy.argtypes = [C.c_void_p]
    L.pfnav_group_destroy.restype = None
    L.pfnav_mgpu_share_blockers.argtypes = [C.c_void_p]
    L.pfnav_group_share_blockers.argtypes = [C.c_void_p]
    L.pfnav_mgpu_exchange_blocker_ops.argtypes = [C.c_void_p, C.c_void_p]
    L.pfnav_group_exchange_blocker_ops.argtypes = [C.c_void_p]
    L.pfnav_mgpu_request_goals_ex.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p,
                                              C.POINTER(C.c_int), C.POINTER(C.c_int)]
    L.pfnav_group_request_goals_ex.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_uint32, C.c_void_p,
                                               C.c_void_p]
    L.pfnav_mgpu_fields_stats.argtypes = [C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int), C.c_void_p, C.c_int]
    L.pfnav_mgpu_request_zones.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.pfnav_group_request_zones.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_mgpu_request_entity_fields_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                                         C.c_size_t, C.c_void_p]
    L.pfnav_group_request_entity_fields_batch.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p,
                                                          C.c_size_t]
    L.pfnav_pool_request_entity_fields_resident.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                            C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p, C.POINTER(C.c_int)]
    L.pfnav_mgpu_request_entity_fields_resident.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                            C.c_size_t, C.c_void_p, C.c_size_t, C.c_void_p]
    L.pfnav_group_request_entity_fields_resident.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                                             C.c_size_t, C.c_void_p, C.c_size_t]
    L.pfnav_pool_request_paths_resident.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                                    C.POINTER(C.c_int)]
    L.pfnav_map_query_resident.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
    L.pfnav_group_arrival_velocity_resident.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_size_t,
                                                        C.c_void_p, C.c_void_p]
    L.pfnav_agents_tick.argtypes = [C.c_void_p, C.c_uint32, C.c_void_p]
    L.pfnav_agents_read_velocities.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_agents_read_debug.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t]
    L.pfnav_ents_in_circle.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_int, C.POINTER(C.c_int)]
    L.pfnav_ents_in_circles.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_size_t,
                                        C.POINTER(C.c_size_t), C.c_void_p]
    L.pfnav_agents_device_ptrs.argtypes = [C.c_void_p, C.POINTER(C.c_void_p), C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
    L.pfnav_agents_rebuild_index.argtypes = [C.c_void_p, C.c_void_p]
    L.pfnav_profile_enable.argtypes = [C.c_void_p, C.c_int]
    L.pfnav_profile_read.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    L.pfnav_profile_read_host.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
    _lib = L
    return L


class PfnavError(RuntimeError):
    pass


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def _population_args(remove, add, ms, ext, formation, blocking, flocks):
    """the arguments of pfnav_agents_change_population after ctx, without the stream; and the arrays they point into"""
    rm = np.ascontiguousarray(remove if remove is not None else [], np.uint32).reshape(-1)
    add = np.ascontiguousarray(add if add is not None else np.zeros(0, AGENT), AGENT).reshape(-1)
    recs = [None if r is None else np.ascontiguousarray(r, dt).reshape(-1)
            for r, dt in ((ms, MOVESTATE), (ext, MOVESTATE_EXT), (formation, FORMATION_IN), (blocking, BLOCKING))]
    for r in recs:
        assert r is None or len(r) == len(add)
    fl = None if flocks is None else np.ascontiguousarray(flocks, FLOCK).reshape(-1)
    ptr = lambda a: _p(a) if a is not None and len(a) else None
    args = (ptr(rm), len(rm), ptr(add), *[ptr(r) for r in recs], len(add), _p(fl) if fl is not None else None,
            0 if fl is None else len(fl))
    return args, (rm, add, recs, fl)


def _command_args(deltas, flocks):
    """(deltas, n, flocks, nflocks) of the command calls; flocks None: the table is unchanged (the pointers keep their
    arrays alive)"""
    d = np.ascontiguousarray(deltas, AGENT_DELTA).reshape(-1)
    fl = None if flocks is None else np.ascontiguousarray(flocks, FLOCK).reshape(-1)
    fp = None if fl is None else _p(fl if len(fl) else np.zeros(1, FLOCK))     # an empty table is still a table
    return _p(d) if len(d) else None, len(d), fp, 0 if fl is None else len(fl)


def _input_args(deltas):
    """(d, n) of the input-delta calls, and the array the pointer keeps alive"""
    d = np.ascontiguousarray(deltas, INPUT_DELTA).reshape(-1)
    return (_p(d) if len(d) else None, len(d)), d


def _resident_args(reqs, footprints, ent_uids, seekers):
    """the pointer arguments of the *_request_entity_fields_resident calls: (reqs, m, ents, ent_uids, nents, seekers,
    nseekers), with the arrays kept alive in the returned tuple's last item"""
    reqs = np.ascontiguousarray(reqs, ENTITY_FIELD_REQ)
    fp = None if footprints is None else np.ascontiguousarray(footprints, FOOTPRINT)
    uids = None if ent_uids is None else np.ascontiguousarray(ent_uids, np.uint32)
    sk = np.ascontiguousarray(seekers, np.uint32)
    nents = len(fp) if fp is not None else (0 if uids is None else len(uids))
    if fp is not None and uids is not None and len(uids) != len(fp):
        raise ValueError("footprints and ent_uids differ in length")
    ptr = lambda a: _p(a) if a is not None and len(a) else None
    return (ptr(reqs), len(reqs), ptr(fp), ptr(uids), nents, ptr(sk), len(sk), (reqs, fp, uids, sk))


def _named_points(n, uids, xz):
    """one endpoint array of pool_request_paths_resident: (uint32[n] or None, float32[n, 2] or None)"""
    u = None if uids is None else np.ascontiguousarray(uids, np.uint32).reshape(-1)
    p = None if xz is None else np.ascontiguousarray(xz, np.float32).reshape(-1, 2)
    if (u is not None and len(u) != n) or (p is not None and len(p) != n):
        raise ValueError("uids / points and dests differ in length")
    return u, p


def _chk(rc):
    if rc != 0:
        raise PfnavError("pfnav error %d: %s" % (rc, load().pfnav_last_error().decode()))


def tile_req(chunk, tile, layer=0, init=1):
    q = np.zeros(1, FIELD_REQ)
    q["chunk_r"], q["chunk_c"] = chunk
    q["layer"] = layer; q["faction_id"] = FACTION_ID_NONE
    q["target_type"] = TARGET_TILE; q["init"] = init
    q["tile_r"], q["tile_c"] = tile
    return q


def portal_req(chunk, port_ep, next_chunk, next_ep, port_iid, next_iid, layer=0, init=1):
    q = np.zeros(1, FIELD_REQ)
    q["chunk_r"], q["chunk_c"] = chunk
    q["layer"] = layer; q["faction_id"] = FACTION_ID_NONE
    q["target_type"] = TARGET_PORTAL; q["init"] = init
    q["port_r0"], q["port_c0"], q["port_r1"], q["port_c1"] = port_ep
    q["next_r0"], q["next_c0"], q["next_r1"], q["next_c1"] = next_ep
    q["next_chunk_r"], q["next_chunk_c"] = next_chunk
    q["port_iid"] = port_iid; q["next_iid"] = next_iid
    return q


def los_req(chunk, target_td, layer=0, prev_index=-1, prev_chunk=(0, 0)):
    q = np.zeros(1, LOS_REQ)
    q["chunk_r"], q["chunk_c"] = chunk
    q["layer"] = layer; q["faction_id"] = FACTION_ID_NONE
    q["tgt_chunk_r"], q["tgt_chunk_c"], q["tgt_tile_r"], q["tgt_tile_c"] = target_td
    q["prev_index"] = prev_index
    q["prev_chunk_r"], q["prev_chunk_c"] = prev_chunk
    return q


def pack_region_reqs(reqs, layer=0):
    """list of dicts {center, target | seeds, enemies, overlay, start, cell, no_create} -> (REGION_REQ[n], seeds int32[k, 2],
    overlay int32[m, 2]) as pfnav_region_fields takes them"""
    rec = np.zeros(len(reqs), REGION_REQ)
    seeds, ovs = [], []
    for i, q in enumerate(reqs):
        sd = np.asarray(q["seeds"] if q.get("seeds") is not None else [q["target"]], np.int32).reshape(-1, 2)
        ov = np.asarray(q["overlay"] if q.get("overlay") is not None else np.zeros((0, 2)), np.int32).reshape(-1, 2)
        flags = 0 if q.get("no_create") else REGION_CREATE
        if q.get("cell", q.get("seeds") is None):
            flags |= REGION_CELL
        if q.get("start") is not None:
            flags |= REGION_FIXUP
            rec["start_r"][i], rec["start_c"][i] = q["start"]
        rec["layer"][i] = layer
        rec["center_r"][i], rec["center_c"][i] = q["center"]
        rec["seed_off"][i], rec["seed_n"][i] = sum(len(s) for s in seeds), len(sd)
        rec["overlay_off"][i], rec["overlay_n"][i] = sum(len(o) for o in ovs), len(ov)
        rec["enemies"][i] = q.get("enemies", 0); rec["flags"][i] = flags
        seeds.append(sd); ovs.append(ov)
    sd = np.ascontiguousarray(np.concatenate(seeds) if seeds else np.zeros((0, 2), np.int32))
    ov = np.ascontiguousarray(np.concatenate(ovs) if ovs else np.zeros((0, 2), np.int32))
    return rec, sd, ov


def pfmap_parse(text):
    """PFMAP text (bytes) -> int32[H32][W32][4] = {pathable, type, base_height, ramp_height} (global row-major)"""
    L = load()
    rows, cols = C.c_int(0), C.c_int(0)
    _chk(L.pfnav_pfmap_parse(text, len(text), C.byref(rows), C.byref(cols), None, 0))
    rec = np.zeros((rows.value * cols.value, 32, 32, 4), np.int32)
    _chk(L.pfnav_pfmap_parse(text, len(text), C.byref(rows), C.byref(cols), _p(rec), rec.size // 4))
    return rec.reshape(rows.value, cols.value, 32, 32, 4).transpose(0, 2, 1, 3, 4).reshape(rows.value * 32, cols.value * 32, 4).copy()


def pfmap_write(tiles, materials=("Grass grass.png",), version="1.0", per_line=4):
    """the inverse (m_al_write_tile, map_asset_load.c:132) for test inputs: tiles int32[H32][W32][4]"""
    H, W = tiles.shape[0] // 32, tiles.shape[1] // 32
    out = ["version %s" % version, "num_materials %d" % len(materials)]
    if float(version) >= 1.1:
        out.append("num_splats 0")
    out += ["num_rows %d" % H, "num_cols %d" % W] + ["material " + m for m in materials]
    for cr in range(H):
        for cc in range(W):
            for r in range(32):
                row = []
                for c in range(32):
                    p, ty, bh, rh = [int(v) for v in tiles[cr * 32 + r, cc * 32 + c]]
                    row.append("%01X%c%02d%02d%03d%03d%01d0%01d%01d%01d%01d%01d%01d%01d000" % (
                        ty, "+" if bh >= 0 else "-", abs(bh), rh, 0, 0, 1 if p else 0, 1, 0, 0, 1, 1, 1, 1))
                for k in range(0, 32, per_line):
                    out.append(" ".join(row[k:k + per_line]))
    return ("\n".join(out) + "\n").encode()


class Nav:
    """One device navigation context (what `struct nav_private` is to the reference)."""

    def __init__(self, device=0, hostonly=False):
        """hostonly=True: a context with NO compute path, for the host-side structure code only"""
        self.L = load()
        h = C.c_void_p()
        if hostonly:
            _chk(self.L.pfnav_create_hostonly(C.byref(h)))
        else:
            _chk(self.L.pfnav_create(device, C.byref(h)))
        self.h = h
        self.nwork = 0

    def close(self):
        if self.h:
            self.L.pfnav_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- map ----
    def map_create(self, chunk_w, chunk_h, nlayers=1, map_x=0.0, map_z=0.0):
        self.cw, self.ch = chunk_w, chunk_h
        _chk(self.L.pfnav_map_create(self.h, chunk_w, chunk_h, nlayers, map_x, map_z))

    def map_load_pfmap(self, text, ref_layers, map_x=0.0, map_z=0.0):
        """parse a PFMAP image and build layer i under the reference layer ref_layers[i] (device cost pass + nav build)"""
        rl = np.ascontiguousarray(ref_layers, np.int32)
        rows, cols = C.c_int(0), C.c_int(0)
        _chk(self.L.pfnav_pfmap_parse(text, len(text), C.byref(rows), C.byref(cols), None, 0))
        _chk(self.L.pfnav_map_load_pfmap(self.h, text, len(text), len(rl), _p(rl), map_x, map_z))
        self.cw, self.ch = cols.value, rows.value

    def map_upload_layer(self, layer, cost_base, blockers=None, local_islands=None):
        cost_base = np.ascontiguousarray(cost_base, np.uint8)
        blockers = None if blockers is None else np.ascontiguousarray(blockers, np.uint16)
        local_islands = None if local_islands is None else np.ascontiguousarray(local_islands, np.uint16)
        _chk(self.L.pfnav_map_upload_layer(self.h, layer, _p(cost_base), _p(blockers), _p(local_islands)))

    def map_update_chunk(self, layer, chunk, cost_base=None, blockers=None, local_islands=None):
        a = None if cost_base is None else np.ascontiguousarray(cost_base, np.uint8)
        b = None if blockers is None else np.ascontiguousarray(blockers, np.uint16)
        c = None if local_islands is None else np.ascontiguousarray(local_islands, np.uint16)
        _chk(self.L.pfnav_map_update_chunk(self.h, layer, chunk[0], chunk[1], _p(a), _p(b), _p(c)))

    def map_cost_from_tiles(self, layer, ref_layer, tiles):
        """tiles: int32[H32][W32][4] = {pathable, type, base_height, ramp_height} (global row-major).
        Re-blocked here into per-chunk 16-byte records shaped like the head of the engine's
        `struct tile`, then passed as the engine would pass `chunk_tiles` (nav.c:2284)."""
        tiles = np.ascontiguousarray(tiles, np.int32)
        assert tiles.shape == (self.ch * 32, self.cw * 32, 4)
        rec = tiles.reshape(self.ch, 32, self.cw, 32, 4).transpose(0, 2, 1, 3, 4).copy()   # [cr][cc][32][32][4]
        rec[..., 0] = rec[..., 0] != 0         # `bool pathable` occupies byte 0 of the first word
        ptrs = (C.c_void_p * (self.cw * self.ch))()
        for i in range(self.cw * self.ch):
            ptrs[i] = rec[i // self.cw, i % self.cw].ctypes.data
        _chk(self.L.pfnav_map_cost_from_tiles(self.h, layer, ref_layer, ptrs, 16))

    def map_get_layer(self, layer=0):
        n = self.cw * self.ch
        cost = np.zeros((n, 64, 64), np.uint8)
        blk = np.zeros((n, 64, 64), np.uint16)
        liid = np.zeros((n, 64, 64), np.uint16)
        _chk(self.L.pfnav_map_get_layer(self.h, layer, _p(cost), _p(blk), _p(liid)))
        return cost, blk, liid

    def flow_fields_repair(self, targets, kinds, args, inout):
        """kinds: 0 nearest-pathable (arg = start_r << 8 | start_c), 1 island-to-nearest (arg = local island)"""
        targets = np.ascontiguousarray(targets, FIELD_REQ)
        kinds = np.ascontiguousarray(kinds, np.int32); args = np.ascontiguousarray(args, np.int32)
        buf = np.ascontiguousarray(inout, np.uint8).reshape(len(targets), 64, 64).copy()
        _chk(self.L.pfnav_flow_fields_repair(self.h, _p(targets), _p(kinds), _p(args), len(targets), _p(buf)))
        return buf

    def region_fields(self, dim, reqs, layer=0, inout=None):
        """reqs: list of dicts {center, target | seeds, enemies, overlay, start, cell} in absolute tile coordinates
        (the shape tests/cases.region_case builds) -> u8[n, dim, dim/2]. One pfnav_region_fields call."""
        rec, sd, ov = pack_region_reqs(reqs, layer)
        buf = (np.zeros((len(reqs), dim, dim // 2), np.uint8) if inout is None
               else np.ascontiguousarray(inout, np.uint8).reshape(len(reqs), dim, dim // 2).copy())
        _chk(self.L.pfnav_region_fields(self.h, dim, _p(rec), len(rec), _p(sd) if len(sd) else None, len(sd),
                                        _p(ov) if len(ov) else None, len(ov), _p(buf)))
        return buf

    def group_arrival_field(self, dim, targets_xz, center_xz, enemies=0, overlay=None, layer=0):
        """N_GroupArrivalFieldCreate (field.c:2525) with its world-space arguments"""
        t = np.ascontiguousarray(targets_xz, np.float32).reshape(-1, 2); c = np.ascontiguousarray(center_xz, np.float32)
        ov = np.ascontiguousarray(overlay if overlay is not None else np.zeros((0, 2)), np.int32).reshape(-1, 2)
        out = np.zeros((dim, dim // 2), np.uint8)
        _chk(self.L.pfnav_group_arrival_field(self.h, layer, dim, int(enemies), _p(t) if len(t) else None, len(t), _p(c),
                                              _p(ov) if len(ov) else None, len(ov), _p(out)))
        return out

    @staticmethod
    def footprints(pos_xz, sel_radius):
        """circle footprints (non-building entities) for entity_seeds / entity_fields"""
        pos = np.asarray(pos_xz, np.float32).reshape(-1, 2)
        fp = np.zeros(len(pos), FOOTPRINT)
        fp["x"], fp["z"] = pos[:, 0], pos[:, 1]
        fp["sel_radius"] = np.broadcast_to(np.asarray(sel_radius, np.float32), (len(pos),))
        return fp

    def entity_seeds(self, kind, ents, chunk, ref_layer=0):
        ents = np.ascontiguousarray(ents, FOOTPRINT)
        out = np.zeros((4 * 4096, 2), np.int32); n = C.c_size_t(0)
        _chk(self.L.pfnav_entity_seeds(self.h, ref_layer, kind, _p(ents) if len(ents) else None, len(ents), chunk[0], chunk[1],
                                       _p(out), len(out), C.byref(n)))
        return out[:n.value].copy()

    def entity_fields(self, kind, ents, chunks, layer=0, ref_layer=0):
        """N_FlowFieldInit + N_FlowFieldUpdate(TARGET_ENTITY | TARGET_ENEMIES) for the listed chunks -> u8[n, 64, 64]"""
        ents = np.ascontiguousarray(ents, FOOTPRINT)
        ch = np.ascontiguousarray(chunks, np.int32).reshape(-1, 2)
        out = np.zeros((len(ch), 64, 64), np.uint8)
        _chk(self.L.pfnav_entity_fields(self.h, layer, ref_layer, kind, _p(ents) if len(ents) else None, len(ents), _p(ch), len(ch), _p(out)))
        return out

    def route_arrival_consts(self, target_xz, layer=0):
        """-> (nearest_ok, nearest[2], mc[n, 2]): the constants of arrived() for one flock target"""
        ok, n = C.c_int32(0), C.c_int32(0)
        nearest = np.zeros(2, np.float32); mc = np.zeros((256, 2), np.float32)
        _chk(self.L.pfnav_route_arrival_consts(self.h, layer, float(target_xz[0]), float(target_xz[1]), C.byref(ok), _p(nearest), _p(mc), 256, C.byref(n)))
        return ok.value, nearest, mc[:n.value].copy()

    def map_query(self, queries, stream=0, out=None):
        """pfnav_map_query: MAP_QUERY records -> MAP_QUERY_RESULT records (answers from the committed map). `out`, when
        given, is the MAP_QUERY_RESULT array the call fills (left untouched when the call fails)."""
        q = np.ascontiguousarray(queries, MAP_QUERY)
        if out is None:
            out = np.zeros(len(q), MAP_QUERY_RESULT)
        assert out.dtype == MAP_QUERY_RESULT and out.flags.c_contiguous and len(out) >= len(q)
        _chk(self.L.pfnav_map_query(self.h, _p(q) if len(q) else None, len(q), _p(out) if len(q) else None, C.c_void_p(stream)))
        return out

    def zone_seeds(self, chunk, centre, radius, layer=0):
        out = np.zeros((4 * 4096, 2), np.int32); n = C.c_size_t(0)
        _chk(self.L.pfnav_zone_seeds(self.h, layer, chunk[0], chunk[1], int(centre[0]), int(centre[1]), int(radius), _p(out), len(out), C.byref(n)))
        return out[:n.value].copy()

    def zone_fields(self, centre, radius, chunks, layer=0):
        """N_FlowFieldInit + N_FlowFieldUpdate(TARGET_ZONE) for the listed chunks -> u8[n, 64, 64]"""
        ch = np.ascontiguousarray(chunks, np.int32).reshape(-1, 2)
        out = np.zeros((len(ch), 64, 64), np.uint8)
        _chk(self.L.pfnav_zone_fields(self.h, layer, int(centre[0]), int(centre[1]), int(radius), _p(ch), len(ch), _p(out)))
        return out

    def pool_request_zone(self, dest, centre_xz, radius, layer=0, stream=0):
        c = np.ascontiguousarray(centre_xz, np.float32); n = C.c_int(0)
        _chk(self.L.pfnav_pool_request_zone(self.h, dest, layer, _p(c), int(radius), C.c_void_p(stream), C.byref(n)))
        return n.value

    def pool_request_zones(self, reqs, stream=0):
        """pool_request_zone for every ZONE_REQ record of `reqs`, in order, in one asynchronous call -> (ndone, nfields
        int32[len(reqs)]). ndone < len(reqs): the pool could not hold request ndone's fields (PFNAV_ERR_NOMEM); requests
        before it are done."""
        reqs = np.ascontiguousarray(reqs, ZONE_REQ)
        nf = np.zeros(len(reqs), np.int32); ndone = C.c_int(0)
        rc = self.L.pfnav_pool_request_zones(self.h, _p(reqs) if len(reqs) else None, len(reqs), C.c_void_p(stream),
                                             _p(nf) if len(reqs) else None, C.byref(ndone))
        if rc != ERR_NOMEM:
            _chk(rc)
        return ndone.value, nf

    def group_arrival_velocity(self, dest, centre_xz, radius, pos_xz):
        c = np.ascontiguousarray(centre_xz, np.float32); pos = np.ascontiguousarray(pos_xz, np.float32).reshape(-1, 2)
        vel = np.zeros((len(pos), 2), np.float32); fl = np.zeros(len(pos), np.uint8)
        _chk(self.L.pfnav_group_arrival_velocity(self.h, dest, _p(c), int(radius), _p(pos), len(pos), _p(vel), _p(fl)))
        return vel, fl

    def pool_repair(self):
        a, b = C.c_int(0), C.c_int(0)
        _chk(self.L.pfnav_pool_repair(self.h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def pool_repair_batch(self, stream=None):
        """pool_repair in device rounds -> (nrequests, nrepairs, nrounds); the pool ends up exactly as pool_repair leaves it"""
        a, b, r = C.c_int(0), C.c_int(0), C.c_int(0)
        _chk(self.L.pfnav_pool_repair_batch(self.h, C.c_void_p(stream or 0), C.byref(a), C.byref(b), C.byref(r)))
        return a.value, b.value, r.value

    def pool_repair_batch_stats(self):
        """test / measurement hook: the last pool_repair_batch -> ((LOS, desired-velocity, enemy-field representatives),
        (rounds ended by rule (i), (ii), (iii)))"""
        out = np.zeros(6, np.int32)
        _chk(self.L.pfnav_pool_repair_batch_stats(self.h, _p(out)))
        return tuple(int(v) for v in out[:3]), tuple(int(v) for v in out[3:])

    def repair_seed_mask(self, chunk, kind, arg, layer=0):
        """the host's seeds of a repair of a TARGET_TILE field of `chunk` -> bool[64, 64]"""
        rows = np.zeros(64, np.uint64)
        _chk(self.L.pfnav_repair_seed_mask(self.h, layer, chunk[0], chunk[1], kind, arg, _p(rows)))
        return np.unpackbits(rows.view(np.uint8), bitorder="little").reshape(64, 64).astype(bool)

    def los_trace(self, enable=True, read_cap=0):
        """arm / read the per-field LOS trace -> uint64[n, 4] = taken, ready, done (ns), 1 + pops"""
        out = np.zeros((max(read_cap, 1), 4), np.uint64)
        n = C.c_size_t(0)
        _chk(self.L.pfnav_los_trace(self.h, int(enable), _p(out) if read_cap else None, read_cap, C.byref(n)))
        return out[:n.value]

    def set_los_variant(self, variant):
        _chk(self.L.pfnav_set_los_variant(self.h, variant))

    def set_two_phase(self, mode):
        _chk(self.L.pfnav_set_two_phase(self.h, mode))

    def request_faction(self, faction_id=FACTION_ID_NONE):
        _chk(self.L.pfnav_request_faction(self.h, faction_id))

    def set_enemy_factions(self, faction_id, mask):
        _chk(self.L.pfnav_set_enemy_factions(self.h, faction_id, int(mask)))

    def map_upload_factions(self, layer, factions):
        f = np.ascontiguousarray(factions, np.uint8)
        assert f.shape == (self.cw * self.ch, 15, 64, 64)
        _chk(self.L.pfnav_map_upload_factions(self.h, layer, _p(f)))

    def fields_join(self, stream=0):
        _chk(self.L.pfnav_fields_join(self.h, C.c_void_p(stream)))

    def map_build_nav(self, layer=0):
        _chk(self.L.pfnav_map_build_nav(self.h, layer))

    def map_refresh_chunk(self, layer, chunk):
        _chk(self.L.pfnav_map_refresh_chunk(self.h, layer, chunk[0], chunk[1]))

    def local_islands(self, layer=0):
        out = np.zeros((self.cw * self.ch, 64, 64), np.uint16)
        _chk(self.L.pfnav_local_islands_get(self.h, layer, _p(out)))
        return out

    def portals(self, layer=0):
        n = C.c_int(0)
        _chk(self.L.pfnav_portals_get(self.h, layer, None, 0, C.byref(n)))
        out = np.zeros((n.value, 10), np.int32)
        _chk(self.L.pfnav_portals_get(self.h, layer, _p(out), n.value, C.byref(n)))
        return out

    def plan_goal(self, target_td, layer=0):
        """-> (flow_reqs, flow_chunk, flow_wave, los_reqs, los_chunk)"""
        cap = self.cw * self.ch * 8 + 8
        fr = np.zeros(cap, FIELD_REQ); fc = np.zeros(cap, np.int32); fw = np.zeros(cap, np.int32)
        lr = np.zeros(cap, LOS_REQ); lc = np.zeros(cap, np.int32)
        nf, nl = C.c_int(0), C.c_int(0)
        _chk(self.L.pfnav_plan_goal(self.h, layer, target_td[0], target_td[1], target_td[2], target_td[3],
                                    _p(fr), _p(fc), _p(fw), cap, C.byref(nf), _p(lr), _p(lc), cap, C.byref(nl)))
        return fr[:nf.value].copy(), fc[:nf.value].copy(), fw[:nf.value].copy(), lr[:nl.value].copy(), lc[:nl.value].copy()

    def blockers_incref(self, x, z, radius, faction=0, flags=FLAG_MOVABLE):
        _chk(self.L.pfnav_blockers_incref(self.h, x, z, radius, faction, flags))

    def blockers_obb(self, corners_xz, incref=True, faction=0, flags=FLAG_MOVABLE):
        """corners_xz: (4, 2) bottom-face corners obb->corners[0], [1], [5], [4]"""
        c = np.ascontiguousarray(corners_xz, np.float32).reshape(8)
        f = self.L.pfnav_blockers_incref_obb if incref else self.L.pfnav_blockers_decref_obb
        _chk(f(self.h, _p(c), faction, flags))

    def blockers_decref(self, x, z, radius, faction=0, flags=FLAG_MOVABLE):
        _chk(self.L.pfnav_blockers_decref(self.h, x, z, radius, faction, flags))

    def blockers(self, layer=0):
        out = np.zeros((self.cw * self.ch, 64, 64), np.uint16)
        _chk(self.L.pfnav_blockers_get(self.h, layer, _p(out)))
        return out

    def faction_counts(self, layer=0):
        out = np.zeros((self.cw * self.ch, 15, 64, 64), np.uint8)
        _chk(self.L.pfnav_blockers_get_factions(self.h, layer, _p(out)))
        return out

    def map_commit(self):
        n = C.c_int(0)
        _chk(self.L.pfnav_map_commit(self.h, C.byref(n)))
        return n.value

    def route_build(self, layer=0):
        _chk(self.L.pfnav_route_build(self.h, layer))

    def route_islands(self, layer=0):
        out = np.zeros((self.cw * self.ch, 64, 64), np.uint16)
        _chk(self.L.pfnav_route_islands_get(self.h, layer, _p(out)))
        return out

    def route_edges(self, chunk_idx, portal_idx, layer=0):
        out = np.zeros((64, 3), np.uint32); n = C.c_int(0)
        _chk(self.L.pfnav_route_edges_get(self.h, layer, chunk_idx, portal_idx, _p(out), 64, C.byref(n)))
        return out[:n.value]

    def route_request_path(self, src, dst, layer=0, have_flow=None, have_los=None):
        """-> ok, dest_id, flow_reqs, flow_ffid, flow_chunk, los_reqs, los_chunk"""
        chunks = self.cw * self.ch
        hf = np.zeros(chunks, np.uint64) if have_flow is None else np.ascontiguousarray(have_flow, np.uint64)
        hl = np.zeros(chunks, np.uint8) if have_los is None else np.ascontiguousarray(have_los, np.uint8)
        cap = chunks * 4 + 8
        fr = np.zeros(cap, FIELD_REQ); fid = np.zeros(cap, np.uint64); fc = np.zeros(cap, np.int32)
        lr = np.zeros(cap, LOS_REQ); lc = np.zeros(cap, np.int32)
        nf, nl, ok, did = C.c_int(0), C.c_int(0), C.c_int(0), C.c_uint32(0)
        _chk(self.L.pfnav_route_request_path(self.h, layer, src[0], src[1], dst[0], dst[1], _p(hf), _p(hl), _p(fr), _p(fid), _p(fc),
                                             cap, C.byref(nf), _p(lr), _p(lc), cap, C.byref(nl), C.byref(did), C.byref(ok)))
        return bool(ok.value), did.value, fr[:nf.value].copy(), fid[:nf.value].copy(), fc[:nf.value].copy(), lr[:nl.value].copy(), lc[:nl.value].copy()

    def set_tma(self, enable):
        _chk(self.L.pfnav_set_tma(self.h, int(enable)))

    # ---- fields ----
    def flow_fields_update(self, reqs, inout=None):
        reqs = np.ascontiguousarray(reqs, FIELD_REQ)
        n = len(reqs)
        buf = np.zeros((n, 64, 64), np.uint8) if inout is None else np.ascontiguousarray(inout, np.uint8).reshape(n, 64, 64).copy()
        _chk(self.L.pfnav_flow_fields_update(self.h, _p(reqs), n, _p(buf)))
        return buf

    def flow_fields_update_dev(self, d_reqs_ptr, n, d_fields_ptr, stream=0, general=False):
        f = self.L.pfnav_flow_fields_update_general_dev if general else self.L.pfnav_flow_fields_update_dev
        _chk(f(self.h, C.c_void_p(d_reqs_ptr), n, C.c_void_p(d_fields_ptr), C.c_void_p(stream)))

    def region_fields_dev(self, dim, d_reqs_ptr, n, d_seeds_ptr, d_overlay_ptr, d_fields_ptr, stream=0):
        _chk(self.L.pfnav_region_fields_dev(self.h, dim, C.c_void_p(d_reqs_ptr), n, C.c_void_p(d_seeds_ptr),
                                            C.c_void_p(d_overlay_ptr), C.c_void_p(d_fields_ptr), C.c_void_p(stream)))

    def los_fields_create(self, reqs, prev_fields=None):
        """prev_fields: {request index: 64x64 previous LOS field} for requests with prev_index = LOS_PREV_INPLACE"""
        reqs = np.ascontiguousarray(reqs, LOS_REQ)
        n = len(reqs)
        out = np.zeros((n, 64, 64), np.uint8)
        for i, f in (prev_fields or {}).items():
            out[i] = f
        _chk(self.L.pfnav_los_fields_create(self.h, _p(reqs), n, _p(out)))
        return out

    def los_fields_create_dev(self, d_reqs_ptr, n, d_fields_ptr, wave_offsets, stream=0):
        wo = np.ascontiguousarray(wave_offsets, np.int32)
        _chk(self.L.pfnav_los_fields_create_dev(self.h, C.c_void_p(d_reqs_ptr), n, C.c_void_p(d_fields_ptr),
                                                len(wo) - 1, _p(wo), C.c_void_p(stream)))

    # ---- field pool ----
    def pool_create(self, ndests, max_fields):
        _chk(self.L.pfnav_pool_create(self.h, ndests, max_fields))

    def pool_put(self, dest, chunk, flow=None, los=None):
        f = None if flow is None else np.ascontiguousarray(flow, np.uint8)
        l = None if los is None else np.ascontiguousarray(los, np.uint8)
        _chk(self.L.pfnav_pool_put(self.h, dest, chunk[0], chunk[1], _p(f), _p(l)))

    def pool_clear(self):
        _chk(self.L.pfnav_pool_clear(self.h))

    def pool_save(self, stream=0):
        """pfnav_pool_save: the whole field pool of this context as one segment -> bytes (the size is asked first)"""
        size = C.c_size_t(0)
        rc = self.L.pfnav_pool_save(self.h, None, 0, C.byref(size), C.c_void_p(stream))
        if rc != ERR_NOMEM:
            _chk(rc)
        out = np.zeros(size.value, np.uint8)
        _chk(self.L.pfnav_pool_save(self.h, _p(out), size.value, C.byref(size), C.c_void_p(stream)))
        return out.tobytes()

    def pool_restore(self, segment, stream=0):
        """pfnav_pool_restore: replace this context's pool with a segment of pool_save (bytes-like), on the same map (after
        the map_commit that follows agents_restore); nothing needs to be re-requested"""
        buf = np.frombuffer(bytes(segment), np.uint8)
        _chk(self.L.pfnav_pool_restore(self.h, _p(buf), len(buf), C.c_void_p(stream)))

    def pool_request_goal(self, dest, target_td, layer=0, stream=0):
        nf, nl = C.c_int(0), C.c_int(0)
        _chk(self.L.pfnav_pool_request_goal(self.h, dest, layer, target_td[0], target_td[1], target_td[2],
                                            target_td[3], C.c_void_p(stream), C.byref(nf), C.byref(nl)))
        return nf.value, nl.value

    def pool_request_path(self, dest, src, dst, layer=0, stream=0):
        """-> ok, dest_id, n_flow, n_los"""
        did, ok, nf, nl = C.c_uint32(0), C.c_int(0), C.c_int(0), C.c_int(0)
        _chk(self.L.pfnav_pool_request_path(self.h, dest, layer, src[0], src[1], dst[0], dst[1], C.c_void_p(stream),
                                            C.byref(did), C.byref(ok), C.byref(nf), C.byref(nl)))
        return bool(ok.value), did.value, nf.value, nl.value

    def pool_request_paths(self, dests, src_xz, dst_xz, layer=0, stream=0):
        """a batch of pool_request_path calls, in order -> ok[n] (bool), dest_id[n], n_flow[n], n_los[n], ndone.
        ndone < n: the pool could not hold request ndone's fields (PFNAV_ERR_NOMEM); requests before it are done."""
        dests = np.ascontiguousarray(dests, np.int32).reshape(-1)
        src = np.ascontiguousarray(src_xz, np.float32).reshape(-1, 2)
        dst = np.ascontiguousarray(dst_xz, np.float32).reshape(-1, 2)
        n = len(dests)
        assert len(src) == n and len(dst) == n
        ok, nf, nl = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        did = np.zeros(n, np.uint32)
        ndone = C.c_int(0)
        rc = self.L.pfnav_pool_request_paths(self.h, n, _p(dests), layer, _p(src), _p(dst), C.c_void_p(stream), _p(did), _p(ok),
                                             _p(nf), _p(nl), C.byref(ndone))
        if rc != ERR_NOMEM:
            _chk(rc)
        return ok.astype(bool), did, nf, nl, ndone.value

    def pool_get(self, dest, chunk):
        """-> (flow or None, los or None, ffid)"""
        f = np.zeros((64, 64), np.uint8); l = np.zeros((64, 64), np.uint8)
        has, ffid = C.c_int(0), C.c_uint64(0)
        _chk(self.L.pfnav_pool_get(self.h, dest, chunk[0], chunk[1], _p(f), _p(l), C.byref(has), C.byref(ffid)))
        return (f if has.value & 1 else None), (l if has.value & 2 else None), ffid.value

    def pool_request_goals(self, dests, targets, layer=0, stream=0, flags=0):
        dests = np.ascontiguousarray(dests, np.int32)
        targets = np.ascontiguousarray(targets, np.int32).reshape(-1, 4)
        nf, nl = C.c_int(0), C.c_int(0)
        _chk(self.L.pfnav_pool_request_goals_ex(self.h, len(dests), _p(dests), layer, _p(targets), flags, C.c_void_p(stream),
                                                C.byref(nf), C.byref(nl)))
        return nf.value, nl.value

    def blockers_batch(self, ops):
        """ops: BLOCKER_OP records {x, z, range, faction_id, flags, delta}"""
        ops = np.ascontiguousarray(ops, BLOCKER_OP)
        _chk(self.L.pfnav_blockers_batch(self.h, _p(ops), len(ops)))

    # ---- agents ----
    def agents_upload(self, agents, flocks, hz=20):
        agents = np.ascontiguousarray(agents, AGENT)
        flocks = np.ascontiguousarray(flocks, FLOCK)
        self.nagents = len(agents)
        _chk(self.L.pfnav_agents_upload(self.h, _p(agents), len(agents), _p(flocks), len(flocks), hz))

    def agents_upload_shard(self, shard, lo, hi, n_total, flocks, hz=20, flags=0):
        """this context's own entity range [lo, hi) of a population of n_total (multi-GPU); shard[i] = entity lo + i"""
        shard = np.ascontiguousarray(shard, AGENT)
        flocks = np.ascontiguousarray(flocks, FLOCK)
        assert len(shard) == hi - lo
        self.nagents = n_total
        _chk(self.L.pfnav_agents_upload_shard(self.h, _p(shard), lo, hi, n_total, _p(flocks), len(flocks), hz, flags))

    def mgpu_init(self, rank, world, nccl_id):
        buf = (C.c_char * 128).from_buffer_copy(bytes(nccl_id))
        _chk(self.L.pfnav_mgpu_init(self.h, rank, world, buf))

    def mgpu_gather(self, stream=0):
        _chk(self.L.pfnav_mgpu_gather(self.h, C.c_void_p(stream)))

    def mgpu_finalize(self):
        _chk(self.L.pfnav_mgpu_finalize(self.h))

    def mgpu_share_blockers(self):
        """opt in: this rank takes its own entities' blockers on the device; call on every rank"""
        _chk(self.L.pfnav_mgpu_share_blockers(self.h))

    def mgpu_exchange_blocker_ops(self, stream=0):
        """collective: every rank ends up with every rank's pending device-decided blocker ops (before map_commit)"""
        _chk(self.L.pfnav_mgpu_exchange_blocker_ops(self.h, C.c_void_p(stream)))

    def mgpu_request_goals_ex(self, dests, targets, layer=0, flags=0, stream=0):
        """collective: pool_request_goals for the whole job, each field built on one rank -> this rank's solo (nf, nl)"""
        dests = np.ascontiguousarray(dests, np.int32)
        targets = np.ascontiguousarray(targets, np.int32).reshape(-1, 4)
        nf, nl = C.c_int(0), C.c_int(0)
        _chk(self.L.pfnav_mgpu_request_goals_ex(self.h, len(dests), _p(dests), layer, _p(targets), flags, C.c_void_p(stream),
                                                C.byref(nf), C.byref(nl)))
        return nf.value, nl.value

    def mgpu_request_zones(self, reqs, stream=0):
        """collective: pool_request_zones for the whole job, each field built on one rank -> nfields int32[len(reqs)];
        all or nothing across the ranks"""
        reqs = np.ascontiguousarray(reqs, ZONE_REQ)
        nf = np.zeros(len(reqs), np.int32)
        _chk(self.L.pfnav_mgpu_request_zones(self.h, _p(reqs) if len(reqs) else None, len(reqs), C.c_void_p(stream),
                                             _p(nf) if len(reqs) else None))
        return nf

    def mgpu_request_entity_fields_batch(self, reqs, footprints, chunks, stream=0):
        """collective: pool_request_entity_fields_batch for the whole job, each field built on one rank; all or nothing
        across the ranks"""
        reqs = np.ascontiguousarray(reqs, ENTITY_FIELD_REQ)
        fp = np.ascontiguousarray(footprints, FOOTPRINT)
        ch = np.ascontiguousarray(chunks, np.int32).reshape(-1, 2)
        _chk(self.L.pfnav_mgpu_request_entity_fields_batch(self.h, _p(reqs) if len(reqs) else None, len(reqs),
                                                           _p(fp) if len(fp) else None, len(fp), _p(ch) if len(ch) else None,
                                                           len(ch), C.c_void_p(stream)))

    def mgpu_request_entity_fields_resident(self, reqs, footprints, ent_uids, seekers, stream=0):
        """collective: pool_request_entity_fields_resident for the whole job, each member resolving the uids from its own
        records and each field built on one rank; all or nothing across the ranks"""
        a = _resident_args(reqs, footprints, ent_uids, seekers)
        _chk(self.L.pfnav_mgpu_request_entity_fields_resident(self.h, *a[:7], C.c_void_p(stream)))

    def mgpu_fields_stats(self, ngoals):
        """test hook: this member's last job batch -> (fields built: flow requests or zone / entity fields, LOS requests
        built, owner per goal or request)"""
        nf, nl = C.c_int(0), C.c_int(0)
        owner = np.zeros(ngoals, np.int32)
        _chk(self.L.pfnav_mgpu_fields_stats(self.h, C.byref(nf), C.byref(nl), _p(owner), ngoals))
        return nf.value, nl.value, owner

    def agents_set_work(self, uids=None):
        if uids is None:
            _chk(self.L.pfnav_agents_set_work(self.h, None, 0))
            self.nwork = -1
        else:
            uids = np.ascontiguousarray(uids, np.uint32)
            self.nwork = len(uids)
            _chk(self.L.pfnav_agents_set_work(self.h, _p(uids), len(uids)))

    def agents_tick(self, flags=0, stream=0):
        _chk(self.L.pfnav_agents_tick(self.h, flags, C.c_void_p(stream)))

    def agents_read_velocities(self, nwork):
        out = np.zeros((nwork, 2), np.float32)
        _chk(self.L.pfnav_agents_read_velocities(self.h, _p(out), nwork))
        return out

    def agents_upload_movestate(self, ms):
        ms = np.ascontiguousarray(ms, MOVESTATE)
        _chk(self.L.pfnav_agents_upload_movestate(self.h, _p(ms), len(ms)))

    def agents_upload_formation(self, f):
        f = np.ascontiguousarray(f, FORMATION_IN)
        _chk(self.L.pfnav_agents_upload_formation(self.h, _p(f), len(f)))

    def agents_upload_movestate_ext(self, ms):
        ms = np.ascontiguousarray(ms, MOVESTATE_EXT)
        _chk(self.L.pfnav_agents_upload_movestate_ext(self.h, _p(ms), len(ms)))

    def pool_request_entity_fields(self, dest, kind, footprints, chunks, layer=0, ref_layer=0, stream=0):
        fp = np.ascontiguousarray(footprints, FOOTPRINT)
        ch = np.ascontiguousarray(chunks, np.int32).reshape(-1, 2)
        _chk(self.L.pfnav_pool_request_entity_fields(self.h, dest, layer, ref_layer, kind, _p(fp), len(fp), _p(ch), len(ch),
                                                     C.c_void_p(stream)))

    def pool_request_entity_fields_batch(self, reqs, footprints, chunks, stream=0):
        """pool_request_entity_fields for every ENTITY_FIELD_REQ record of `reqs`, in order, in one call; their footprint
        and chunk ranges index `footprints` and `chunks` (int32[n, 2]) -> ndone. ndone < len(reqs): the pool could not hold
        request ndone's fields (PFNAV_ERR_NOMEM); requests before it are done."""
        reqs = np.ascontiguousarray(reqs, ENTITY_FIELD_REQ)
        fp = np.ascontiguousarray(footprints, FOOTPRINT)
        ch = np.ascontiguousarray(chunks, np.int32).reshape(-1, 2)
        ndone = C.c_int(0)
        rc = self.L.pfnav_pool_request_entity_fields_batch(self.h, _p(reqs) if len(reqs) else None, len(reqs), _p(fp) if len(fp) else None,
                                                           len(fp), _p(ch) if len(ch) else None, len(ch), C.c_void_p(stream),
                                                           C.byref(ndone))
        if rc != ERR_NOMEM:
            _chk(rc)
        return ndone.value

    def pool_request_paths_resident(self, dests, src_uids, src_xz, dst_uids, dst_xz, layer=0, stream=0):
        """pool_request_paths with endpoints that may name resident entities -> ok[n] (bool), dest_id[n], n_flow[n],
        n_los[n], ndone. `src_uids` / `dst_uids`: uint32 per request (NULL_UID: use the given point) or None (use the
        points as given); `src_xz` / `dst_xz`: float32 [n, 2] or None (every entry names a uid)."""
        dests = np.ascontiguousarray(dests, np.int32).reshape(-1)
        n = len(dests)
        su, sx = _named_points(n, src_uids, src_xz)
        du, dx = _named_points(n, dst_uids, dst_xz)
        ok, nf, nl = np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.int32)
        did = np.zeros(n, np.uint32)
        ndone = C.c_int(0)
        ptr = lambda a: _p(a) if a is not None and len(a) else None
        rc = self.L.pfnav_pool_request_paths_resident(self.h, n, ptr(dests), layer, ptr(su), ptr(sx), ptr(du), ptr(dx),
                                                      C.c_void_p(stream), ptr(did), ptr(ok), ptr(nf), ptr(nl), C.byref(ndone))
        if rc != ERR_NOMEM:
            _chk(rc)
        return ok.astype(bool), did, nf, nl, ndone.value

    def map_query_resident(self, queries, pos_uids=None, dst_uids=None, stream=0, out=None):
        """map_query with positions that may name resident entities: `pos_uids` / `dst_uids` (uint32 per query, NULL_UID
        keeps the given value, or None) replace (x, z) / (dst_x, dst_z). `out`, when given, is the MAP_QUERY_RESULT
        array the call fills (left untouched when the call fails)."""
        q = np.ascontiguousarray(queries, MAP_QUERY)
        pu = None if pos_uids is None else np.ascontiguousarray(pos_uids, np.uint32)
        du = None if dst_uids is None else np.ascontiguousarray(dst_uids, np.uint32)
        if (pu is not None and len(pu) != len(q)) or (du is not None and len(du) != len(q)):
            raise ValueError("pos_uids / dst_uids and queries differ in length")
        if out is None:
            out = np.zeros(len(q), MAP_QUERY_RESULT)
        assert out.dtype == MAP_QUERY_RESULT and out.flags.c_contiguous and len(out) >= len(q)
        ptr = lambda a: _p(a) if a is not None and len(a) else None
        _chk(self.L.pfnav_map_query_resident(self.h, ptr(q), ptr(pu), ptr(du), len(q), ptr(out) if len(q) else None,
                                             C.c_void_p(stream)))
        return out

    def group_arrival_velocity_resident(self, dest, centre_xz, radius, uids):
        """group_arrival_velocity for resident entities: position k is that of uids[k] -> (vel [n, 2], flags [n])"""
        c = np.ascontiguousarray(centre_xz, np.float32); u = np.ascontiguousarray(uids, np.uint32).reshape(-1)
        vel = np.zeros((len(u), 2), np.float32); fl = np.zeros(len(u), np.uint8)
        _chk(self.L.pfnav_group_arrival_velocity_resident(self.h, dest, _p(c), int(radius), _p(u) if len(u) else None, len(u),
                                                          _p(vel), _p(fl)))
        return vel, fl

    def pool_request_entity_fields_resident(self, reqs, footprints, ent_uids, seekers, stream=0):
        """pool_request_entity_fields_batch with footprints and seekers named by uid -> ndone. `footprints`: FOOTPRINT
        records or None (every entry names a uid); `ent_uids`: uint32 per footprint (NULL_UID: use footprints[k]) or None
        (use `footprints` as given); `seekers`: uint32 uids, which the requests' chunk ranges index. ndone < len(reqs): the
        pool could not hold request ndone's fields (PFNAV_ERR_NOMEM); requests before it are done."""
        a = _resident_args(reqs, footprints, ent_uids, seekers)
        ndone = C.c_int(0)
        rc = self.L.pfnav_pool_request_entity_fields_resident(self.h, *a[:7], C.c_void_p(stream), C.byref(ndone))
        if rc != ERR_NOMEM:
            _chk(rc)
        return ndone.value

    def route_graph_paths(self, req, max_hops=256, on_device=True, layer=0):
        """AStar_PortalGraphPath batch; req int32[n, 8]; -> status[n], cost[n], list of hop arrays [nhops, 3]"""
        req = np.ascontiguousarray(req, np.int32).reshape(-1, 8)
        n = len(req)
        out = np.zeros((n, 4 + 3 * max_hops), np.int32)
        _chk(self.L.pfnav_route_graph_paths(self.h, layer, _p(req), n, _p(out), max_hops, 1 if on_device else 0))
        cost = out[:, 2].copy().view(np.float32)
        hops = [out[i, 4:4 + 3 * max(out[i, 1], 0)].reshape(-1, 3).copy() if out[i, 0] == 1 else np.zeros((0, 3), np.int32) for i in range(n)]
        return out[:, 0].copy(), cost, hops

    def clearpath_stats(self, reset=True):
        out = np.zeros(4, np.uint64)
        _chk(self.L.pfnav_agents_clearpath_stats(self.h, _p(out), 1 if reset else 0))
        return dict(zip(("no_admissible", "loop_possible", "literal_replays", "replay_solves"), (int(v) for v in out)))

    def set_cohesion_mode(self, mode):
        _chk(self.L.pfnav_set_cohesion_mode(self.h, mode))

    def agents_compute_updates(self, stream=0):
        _chk(self.L.pfnav_agents_compute_updates(self.h, C.c_void_p(stream)))

    def agents_read_patches(self, nwork):
        out = np.zeros(nwork, PATCH)
        _chk(self.L.pfnav_agents_read_patches(self.h, _p(out), nwork))
        return out

    def agents_apply_updates(self, stream=0):
        _chk(self.L.pfnav_agents_apply_updates(self.h, C.c_void_p(stream)))

    def agents_apply_updates_ex(self, flags=APPLY_BLOCKERS, stream=0):
        """pfnav_agents_apply_updates_ex: flags = 0 is agents_apply_updates; APPLY_BLOCKERS also takes / releases the
        blockers of stopping / starting units on the device (applied by the next map_commit)"""
        _chk(self.L.pfnav_agents_apply_updates_ex(self.h, int(flags), C.c_void_p(stream)))

    def agents_collect_events(self, stream=0):
        """pfnav_agents_collect_events: the events of the last update pass, kept on the device (after
        agents_compute_updates, before the apply)"""
        _chk(self.L.pfnav_agents_collect_events(self.h, C.c_void_p(stream)))

    def agents_read_events(self, cap=None):
        """pfnav_agents_read_events -> EVENT records of the last collect, in work order. `cap`: the room of the first call
        (default: the length of the work list this object last set, which no list of it exceeds); a call that returns
        PFNAV_ERR_NOMEM is made once more with room for the length it reported."""
        cap = max(self.nwork, 0) if cap is None else cap
        n = C.c_size_t(0)
        out = np.zeros(max(cap, 1), EVENT)
        rc = self.L.pfnav_agents_read_events(self.h, _p(out), cap, C.byref(n))
        if rc == ERR_NOMEM:
            out = np.zeros(max(n.value, 1), EVENT)
            rc = self.L.pfnav_agents_read_events(self.h, _p(out), n.value, C.byref(n))
        _chk(rc)
        return out[:n.value].copy()

    def agents_upload_blocking(self, b):
        """BLOCKING records, one per entity (uid order); describes blocks already counted, queues no op"""
        b = np.ascontiguousarray(b, BLOCKING)
        _chk(self.L.pfnav_agents_upload_blocking(self.h, _p(b) if len(b) else None, len(b)))

    def agents_read_blocking(self, n):
        out = np.zeros(n, BLOCKING)
        _chk(self.L.pfnav_agents_read_blocking(self.h, _p(out) if n else None, n))
        return out

    def agents_set_blocking(self, uids, block=True, stream=0):
        """the engine's entity_block (block=True) / entity_unblock for the listed uids; repeats change nothing"""
        u = np.ascontiguousarray(uids, np.uint32).reshape(-1)
        _chk(self.L.pfnav_agents_set_blocking(self.h, _p(u) if len(u) else None, len(u), 1 if block else 0, C.c_void_p(stream)))

    def agents_commands(self, deltas, flocks=None, stream=0):
        """pfnav_agents_commands: AGENT_DELTA records applied in order; flocks (FLOCK records): the whole new flock
        table, None: unchanged. Follow with agents_rebuild_index."""
        _chk(self.L.pfnav_agents_commands(self.h, *_command_args(deltas, flocks), C.c_void_p(stream)))

    def mgpu_commands(self, deltas, flocks=None, stream=0):
        """collective: agents_commands for the whole job -- every rank passes the job's whole batch (global uids) and
        the same table; all or nothing across the ranks. Follow with mgpu_gather."""
        _chk(self.L.pfnav_mgpu_commands(self.h, *_command_args(deltas, flocks), C.c_void_p(stream)))

    def agents_change_population(self, remove, add, ms=None, ext=None, formation=None, blocking=None, flocks=None, stream=0):
        """pfnav_agents_change_population: remove the uids `remove` (numbering before the call; repeats removed once) and
        append the AGENT records `add`, with their MOVESTATE / MOVESTATE_EXT / FORMATION_IN / BLOCKING records (None: no
        records; ext and formation then take the defaults). Survivors keep their order and are renumbered densely, the
        appended entities follow. flocks (FLOCK records): the whole new flock table, None: unchanged. The work list is
        emptied: follow with agents_set_work_dev."""
        args, keep = _population_args(remove, add, ms, ext, formation, blocking, flocks)
        _chk(self.L.pfnav_agents_change_population(self.h, *args, C.c_void_p(stream)))
        self.nagents = getattr(self, "nagents", 0) - len(np.unique(keep[0])) + len(keep[1])
        self.nwork = 0

    def mgpu_change_population(self, remove, add, ms=None, ext=None, formation=None, blocking=None, flocks=None, stream=0):
        """collective: agents_change_population for the whole job -- every rank passes the job's whole batch (global
        uids) and the same table; all or nothing across the ranks. Afterwards the rank owns
        mgpu_shard_range(n_new, rank, world). Follow with mgpu_gather and agents_set_work_dev."""
        args, keep = _population_args(remove, add, ms, ext, formation, blocking, flocks)
        _chk(self.L.pfnav_mgpu_change_population(self.h, *args, C.c_void_p(stream)))
        self.nwork = 0

    def agents_read_movestate_ext(self, n):
        out = np.zeros(n, MOVESTATE_EXT)
        _chk(self.L.pfnav_agents_read_movestate_ext(self.h, _p(out) if n else None, n))
        return out

    def agents_read_arrival_consts(self):
        """pfnav_agents_read_arrival_consts: the (flock, layer) table of arrived()'s constants the last compute_updates
        built, as ARRIVAL_RECORD records in (flock, layer) order"""
        n = C.c_size_t(0)
        _chk(self.L.pfnav_agents_read_arrival_consts(self.h, None, 0, C.byref(n)))
        out = np.zeros(n.value, ARRIVAL_RECORD)
        if n.value:
            _chk(self.L.pfnav_agents_read_arrival_consts(self.h, _p(out), n.value, C.byref(n)))
        return out

    def agents_read_formation(self, n):
        out = np.zeros(n, FORMATION_IN)
        _chk(self.L.pfnav_agents_read_formation(self.h, _p(out) if n else None, n))
        return out

    def agents_input_deltas(self, deltas, stream=0):
        """pfnav_agents_input_deltas: INPUT_DELTA records written in order into the movestate_ext and formation
        tables (a FORMATION record creates a zeroed formation table when there is none)"""
        args, keep = _input_args(deltas)
        _chk(self.L.pfnav_agents_input_deltas(self.h, *args, C.c_void_p(stream)))

    def mgpu_input_deltas(self, deltas, stream=0):
        """collective: agents_input_deltas for the whole job -- every rank passes the job's whole batch (global uids);
        all or nothing across the ranks"""
        args, keep = _input_args(deltas)
        _chk(self.L.pfnav_mgpu_input_deltas(self.h, *args, C.c_void_p(stream)))

    def agents_set_work_dev(self, stream=0):
        """pfnav_agents_set_work_dev: agents_set_work(None) built on the device -> the number of work items"""
        n = C.c_size_t(0)
        _chk(self.L.pfnav_agents_set_work_dev(self.h, C.c_void_p(stream), C.byref(n)))
        self.nwork = n.value
        return n.value

    def agents_read_work(self):
        n = C.c_size_t(0)
        _chk(self.L.pfnav_agents_read_work(self.h, None, 0, C.byref(n)))
        out = np.zeros(n.value, np.uint32)
        _chk(self.L.pfnav_agents_read_work(self.h, _p(out) if n.value else None, n.value, C.byref(n)))
        return out

    def agents_save(self, stream=0):
        """pfnav_agents_save: the checkpoint segment of this context's own range -> bytes (the size is asked first)"""
        size = C.c_size_t(0)
        rc = self.L.pfnav_agents_save(self.h, None, 0, C.byref(size), C.c_void_p(stream))
        if rc != ERR_NOMEM:
            _chk(rc)
        out = np.zeros(size.value, np.uint8)
        _chk(self.L.pfnav_agents_save(self.h, _p(out), size.value, C.byref(size), C.c_void_p(stream)))
        return out.tobytes()

    def agents_restore(self, segments, stream=0):
        """pfnav_agents_restore from checkpoint segments (bytes-like, any order): this context takes the whole population,
        or its own shard range in a multi-GPU job. Follow with map_commit (the restored blocks), the gather in a job, and
        agents_set_work_dev."""
        args, keep = _segment_args(segments)
        _chk(self.L.pfnav_agents_restore(self.h, *args, C.c_void_p(stream)))
        self.nwork = 0

    def state_digest(self, what=DIGEST_ALL, block_log2=10, stream=0):
        """pfnav_state_digest: queue the digest of the components in `what` on `stream`; returns without waiting"""
        _chk(self.L.pfnav_state_digest(self.h, what, block_log2, C.c_void_p(stream)))

    def mgpu_state_digest(self, what=DIGEST_ALL, block_log2=10, stream=0):
        """collective: state_digest on every rank and one all-gather of the ranks' digest records; state_digest_read then
        gives the job's values and the differ_* masks"""
        _chk(self.L.pfnav_mgpu_state_digest(self.h, what, block_log2, C.c_void_p(stream)))

    def state_digest_read(self, blocks=True):
        """pfnav_state_digest_read -> (DIGEST record, uint64 block array or None); waits for the queued digest only"""
        d = np.zeros(1, DIGEST)
        n = C.c_size_t(0)
        if not blocks:
            _chk(self.L.pfnav_state_digest_read(self.h, _p(d), None, 0, C.byref(n)))
            return d[0], None
        rc = self.L.pfnav_state_digest_read(self.h, _p(d), _p(np.zeros(1, np.uint64)), 0, C.byref(n))
        if rc != ERR_NOMEM:                   # no block array: the read is done
            _chk(rc)
            return d[0], np.zeros(0, np.uint64)
        b = np.zeros(max(n.value, 1), np.uint64)
        _chk(self.L.pfnav_state_digest_read(self.h, _p(d), _p(b), n.value, C.byref(n)))
        return d[0], b[:n.value]

    def agents_read_state(self, n, movestate=True):
        a = np.zeros(n, AGENT)
        ms = np.zeros(n, MOVESTATE) if movestate else None
        _chk(self.L.pfnav_agents_read_state(self.h, _p(a), _p(ms), n))
        return a, ms

    def agents_read_debug(self, nwork):
        vpref = np.zeros((nwork, 2), np.float32)
        vdes = np.zeros((nwork, 2), np.float32)
        los = np.zeros(nwork, np.uint8)
        _chk(self.L.pfnav_agents_read_debug(self.h, _p(vpref), _p(vdes), _p(los), nwork))
        return vpref, vdes, los

    def ents_in_circle(self, x, z, r, maxout=512):
        out = np.zeros(maxout, np.uint32)
        n = C.c_int(0)
        _chk(self.L.pfnav_ents_in_circle(self.h, x, z, r, _p(out), maxout, C.byref(n)))
        return out[:n.value].copy()

    def ents_in_circles(self, queries, cap=None, stream=0):
        """pfnav_ents_in_circles: ENTS_QUERY records -> (offsets uint32[n + 1], ids uint32[offsets[n]]); query i's uids are
        ids[offsets[i]:offsets[i + 1]]. `cap`: the room of the first call (default 0: it only sizes the answers); a call
        that returns PFNAV_ERR_NOMEM is made again with room for the total it reported."""
        q = np.ascontiguousarray(queries, ENTS_QUERY)
        n = len(q)
        offsets = np.zeros(n + 1, np.uint32)
        total = C.c_size_t(0)
        qp, op = (_p(q), _p(offsets)) if n else (None, None)
        while True:
            ids = np.zeros(max(cap or 0, 1), np.uint32)
            rc = self.L.pfnav_ents_in_circles(self.h, qp, n, op, _p(ids), cap or 0, C.byref(total), C.c_void_p(stream))
            if rc != ERR_NOMEM or cap == total.value:
                break
            cap = total.value
        _chk(rc)
        return offsets, ids[:total.value].copy()

    def agents_device_ptrs(self):
        a, b, n = C.c_void_p(), C.c_void_p(), C.c_size_t()
        _chk(self.L.pfnav_agents_device_ptrs(self.h, C.byref(a), C.byref(b), C.byref(n)))
        return a.value, b.value, n.value

    def agents_rebuild_index(self, stream=0):
        _chk(self.L.pfnav_agents_rebuild_index(self.h, C.c_void_p(stream)))

    def profile_enable(self, on=True):
        _chk(self.L.pfnav_profile_enable(self.h, int(on)))

    def profile_read(self):
        """-> dict name -> (total_ms, launches_groups)"""
        ms = np.zeros(8, np.float32); cnt = np.zeros(8, np.uint32)
        _chk(self.L.pfnav_profile_read(self.h, _p(ms), _p(cnt)))
        names = ["flow", "los", "index", "vdes", "cohesion", "velocity", "update", "apply"]
        return {n: (float(ms[i]), int(cnt[i])) for i, n in enumerate(names)}

    HOST_SEGMENTS = ["clear", "wait", "plan", "merge", "reserve", "pack", "upload", "launch"]

    def profile_read_host(self):
        """host wall clock of pool_clear / pool_request_goals segments while profiling -> dict name -> (total_ms, count)"""
        ms = np.zeros(8, np.float64); cnt = np.zeros(8, np.uint32)
        _chk(self.L.pfnav_profile_read_host(self.h, _p(ms), _p(cnt)))
        return {n: (float(ms[i]), int(cnt[i])) for i, n in enumerate(self.HOST_SEGMENTS)}

    def launch_count(self):
        return int(self.L.pfnav_launch_count(self.h))


UPLOAD_SAME_FLOCKS = 1
REQUEST_MISSING_ONLY = 1
BLOCKER_OP = np.dtype([("x", np.float32), ("z", np.float32), ("range", np.float32), ("faction_id", np.int32),
                       ("flags", np.uint32), ("delta", np.int32)])


def mgpu_shard_range(n_total, rank, world):
    lo, hi = C.c_size_t(0), C.c_size_t(0)
    _chk(load().pfnav_mgpu_shard_range(n_total, rank, world, C.byref(lo), C.byref(hi)))
    return lo.value, hi.value


def mgpu_unique_id():
    buf = (C.c_char * 128)()
    _chk(load().pfnav_mgpu_unique_id(buf))
    return bytes(buf.raw)


class Group:
    """in-process multi-GPU group: several Nav contexts of this process, rank i = navs[i]"""

    def __init__(self, navs):
        self.navs = list(navs)
        arr = (C.c_void_p * len(navs))(*[n.h for n in navs])
        self.g = C.c_void_p(0)
        _chk(load().pfnav_group_create(arr, len(navs), C.byref(self.g)))

    def gather(self):
        _chk(load().pfnav_group_gather(self.g))

    def share_blockers(self):
        """opt in: the members take their own entities' blockers on the device"""
        _chk(load().pfnav_group_share_blockers(self.g))

    def exchange_blocker_ops(self):
        """every member ends up with every member's pending device-decided blocker ops (before map_commit)"""
        _chk(load().pfnav_group_exchange_blocker_ops(self.g))

    def request_goals_ex(self, dests, targets, layer=0, flags=0):
        """pool_request_goals for every member, each field built on one member -> per-member solo counts (nf[], nl[])"""
        dests = np.ascontiguousarray(dests, np.int32)
        targets = np.ascontiguousarray(targets, np.int32).reshape(-1, 4)
        nf, nl = np.zeros(len(self.navs), np.int32), np.zeros(len(self.navs), np.int32)
        _chk(load().pfnav_group_request_goals_ex(self.g, len(dests), _p(dests), layer, _p(targets), flags, _p(nf), _p(nl)))
        return nf, nl

    def request_zones(self, reqs):
        """pool_request_zones for every member, each field built on one member -> nfields int32[len(reqs)] (the same on
        every member); all or nothing across the members"""
        reqs = np.ascontiguousarray(reqs, ZONE_REQ)
        nf = np.zeros(len(reqs), np.int32)
        _chk(load().pfnav_group_request_zones(self.g, _p(reqs) if len(reqs) else None, len(reqs), _p(nf) if len(reqs) else None))
        return nf

    def request_entity_fields_batch(self, reqs, footprints, chunks):
        """pool_request_entity_fields_batch for every member, each field built on one member; all or nothing across the
        members"""
        reqs = np.ascontiguousarray(reqs, ENTITY_FIELD_REQ)
        fp = np.ascontiguousarray(footprints, FOOTPRINT)
        ch = np.ascontiguousarray(chunks, np.int32).reshape(-1, 2)
        _chk(load().pfnav_group_request_entity_fields_batch(self.g, _p(reqs) if len(reqs) else None, len(reqs),
                                                            _p(fp) if len(fp) else None, len(fp), _p(ch) if len(ch) else None,
                                                            len(ch)))

    def request_entity_fields_resident(self, reqs, footprints, ent_uids, seekers):
        """request_entity_fields_batch with footprints and seekers named by uid (Nav.pool_request_entity_fields_resident),
        each member resolving them from its own records; all or nothing across the members"""
        a = _resident_args(reqs, footprints, ent_uids, seekers)
        _chk(load().pfnav_group_request_entity_fields_resident(self.g, *a[:7]))

    def commands(self, deltas, flocks=None):
        """agents_commands for the whole group: the job's whole batch (global uids), each member applying its own
        entities' deltas; all or nothing across the members. Follow with gather."""
        _chk(load().pfnav_group_commands(self.g, *_command_args(deltas, flocks)))

    def input_deltas(self, deltas):
        """agents_input_deltas for the whole group: the job's whole batch (global uids), each member writing its own
        entities' records; all or nothing across the members"""
        args, keep = _input_args(deltas)
        _chk(load().pfnav_group_input_deltas(self.g, *args))

    def change_population(self, remove, add, ms=None, ext=None, formation=None, blocking=None, flocks=None):
        """agents_change_population for the whole group: the job's whole batch (global uids); member i then owns
        mgpu_shard_range(n_new, i, world). All or nothing across the members. Follow with gather and agents_set_work_dev."""
        args, keep = _population_args(remove, add, ms, ext, formation, blocking, flocks)
        _chk(load().pfnav_group_change_population(self.g, *args))
        for nv in self.navs:
            nv.nwork = 0

    def restore(self, segments):
        """agents_restore for every member in one call: each takes mgpu_shard_range(n_total, i, world) from the segments.
        Every member validates before any changes. Follow with map_commit, gather and agents_set_work_dev."""
        args, keep = _segment_args(segments)
        _chk(load().pfnav_group_restore(self.g, *args))
        for nv in self.navs:
            nv.nwork = 0

    def state_digest(self, what=DIGEST_ALL, block_log2=10):
        """pfnav_group_state_digest -> (DIGEST[world + 1]: the job's record, then each member's; the job's block array)"""
        out = np.zeros(len(self.navs) + 1, DIGEST)
        n = C.c_size_t(0)
        L = load()
        rc = L.pfnav_group_state_digest(self.g, what, block_log2, _p(out), _p(np.zeros(1, np.uint64)), 0, C.byref(n))
        if rc != ERR_NOMEM:                   # no block array: the call is done
            _chk(rc)
            return out, np.zeros(0, np.uint64)
        b = np.zeros(max(n.value, 1), np.uint64)
        _chk(L.pfnav_group_state_digest(self.g, what, block_log2, _p(out), _p(b), n.value, C.byref(n)))
        return out, b[:n.value]

    def close(self):
        if self.g:
            load().pfnav_group_destroy(self.g)
            self.g = None


def _segment_args(segments):
    """checkpoint segments -> ((const void *const *segs, const size_t *sizes, nseg), the buffers they point into)"""
    bufs = [np.frombuffer(bytes(sg), np.uint8) for sg in segments]
    ptrs = (C.c_void_p * max(len(bufs), 1))(*[b.ctypes.data for b in bufs])
    sizes = (C.c_size_t * max(len(bufs), 1))(*[len(b) for b in bufs])
    return (ptrs, sizes, len(bufs)), bufs


def pack_agents(a):
    """synth.make_agents() dict -> AGENT / FLOCK record arrays"""
    n = len(a["radius"])
    rec = np.zeros(n, AGENT)
    rec["pos"] = a["pos"]; rec["prev_pos"] = a["prev_pos"]; rec["velocity"] = a["vel"]
    rec["radius"] = a["radius"]; rec["max_speed"] = a["max_speed"]; rec["speed"] = a["speed"]
    rec["state"] = a["state"]; rec["flags"] = a["flags"]; rec["flock"] = a["flock_of"]
    if "vdes" in a:
        rec["vdes"] = a["vdes"]
    if "has_los" in a:
        rec["has_dest_los"] = a["has_los"]
    fl = np.zeros(len(a["flock_target"]), FLOCK)
    fl["target"] = a["flock_target"]
    fl["dest"] = np.arange(len(fl)) if "flock_dest_index" not in a else a["flock_dest_index"]
    fl["layer"] = 0
    return rec, fl
