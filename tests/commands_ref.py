"""The long way round that pfnav_agents_commands replaces, for the tests and tools/bench_agent_commands.py: the same
edits made in numpy on a read-back of the population, to be uploaded again in full."""
import numpy as np

import cases

capi = cases.capi


def apply_deltas_np(deltas, agents, ms, ext=None):
    """AGENT_DELTA records in array order on AGENT / MOVESTATE / MOVESTATE_EXT tables (in place)"""
    for x in np.ascontiguousarray(deltas, capi.AGENT_DELTA).reshape(-1):
        u, k = int(x["uid"]), int(x["mask"])
        if k & capi.DELTA_STATE: agents["state"][u] = x["state"]
        if k & capi.DELTA_FLOCK: agents["flock"][u] = x["flock"]
        if k & capi.DELTA_AUX_DEST: agents["aux_dest1"][u] = x["aux_dest1"]
        if k & capi.DELTA_FLAGS: agents["flags"][u] = x["flags"] & 0xFFFFFF
        if k & capi.DELTA_SPEEDS: agents["max_speed"][u], agents["speed"][u] = x["max_speed"], x["speed"]
        if k & capi.DELTA_RADIUS: agents["radius"][u] = x["radius"]
        if k & capi.DELTA_VELOCITY: agents["velocity"][u] = x["velocity"]
        if k & capi.DELTA_POSITION:
            agents["pos"][u] = agents["prev_pos"][u] = x["position"]
            ms["next_pos"][u, 0], ms["next_pos"][u, 2] = x["position"]
            ms["step"][u], ms["left"][u] = 0, 0
        if (k & capi.DELTA_CLEAR_HIST) and not (agents["flags"][u] & capi.FLAG_COMBAT_HELD): ms["vel_hist"][u] = 0
        if k & capi.DELTA_TARGET: ext["surround_target_uid"][u], ext["target_range"][u] = x["target_uid"], x["target_range"]


def deltas(uids, **fields):
    """one AGENT_DELTA per uid; the mask follows from the fields given (clear_hist=True, target=(uid, range))"""
    bits = dict(state=capi.DELTA_STATE, flock=capi.DELTA_FLOCK, aux_dest1=capi.DELTA_AUX_DEST, flags=capi.DELTA_FLAGS,
                radius=capi.DELTA_RADIUS, velocity=capi.DELTA_VELOCITY, position=capi.DELTA_POSITION)
    d = np.zeros(len(uids), capi.AGENT_DELTA)
    d["uid"] = uids
    for k, v in fields.items():
        if k == "clear_hist":
            d["mask"] |= capi.DELTA_CLEAR_HIST
        elif k == "speeds":
            d["mask"] |= capi.DELTA_SPEEDS; d["max_speed"], d["speed"] = v
        elif k == "target":
            d["mask"] |= capi.DELTA_TARGET; d["target_uid"], d["target_range"] = v
        else:
            d["mask"] |= bits[k]; d[k] = v
    return d
