"""The selection rule of pfnav_agents_collect_events restated in numpy: the events a tick's patches (read_patches) and the
population read before the apply (read_state) give, in work order."""
import numpy as np

import cases

capi = cases.capi
SET_STATE, SET_POSITION, SET_DEST, SET_MOVING = 1, 1 << 2, 1 << 10, 1 << 12


def expected_events(patches, agents, work):
    """patches: PATCH[len(work)]; agents: AGENT records indexed by uid (the state before the apply); work: the uids"""
    work = np.asarray(work, np.uint32)
    a = agents[work]
    f = patches["flags"]
    sel = (((f & (SET_STATE | SET_MOVING | SET_DEST)) != 0) | (patches["engine_todo"] != 0)) & \
          ((a["flags"] & capi.FLAG_GARRISONED) == 0)
    p, s = patches[sel], a[sel]
    ev = np.zeros(int(sel.sum()), capi.EVENT)
    ev["uid"] = work[sel]
    ev["flags"] = p["flags"]
    ev["todo"] = p["engine_todo"]
    ev["attack"] = p["next_attack"]
    ev["state_before"] = s["state"]
    ev["state_after"] = np.where((p["flags"] & (SET_STATE | SET_MOVING)) != 0, p["next_state"].astype(np.uint32), s["state"])
    ev["dest"] = p["next_dest"]
    ev["pos"] = np.where(((p["flags"] & SET_POSITION) != 0)[:, None], p["next_pos"][:, [0, 2]], s["pos"])
    return ev
