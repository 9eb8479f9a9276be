#!/usr/bin/env python
"""Blockers of stopping units, host path against device path, on an arriving crowd on the C2 map (bench.py's 16 x 16-chunk
map and 100 000-agent population, every flock's target moved to the flock's own centre so that the crowd arrives and the
adjacent-arrived cascade spreads).

Two contexts step the same ticks (agents_tick with a desired velocity towards the target, compute_updates). Per tick:
  host_ms:   read the patches and the snapshot positions back, apply_updates, build the entity_block / entity_unblock ops
             on the host from a host blocking table, blockers_batch, map_commit;
  device_ms: apply_updates_ex(APPLY_BLOCKERS), map_commit.
Each is a host clock from a device synchronise to the end of map_commit (which waits for the device). The two sides take
turns going first. After every tick the blocker counts, local islands and blocking tables of the two contexts must be
equal.
    python tools/bench_apply_blockers.py [--ticks 12] [--out FILE]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SET_STATE, SET_MOVING = 1, 1 << 12


def _crowd(bench, pf):
    capi = pf.capi
    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    a = W["agents"]
    for f in range(len(a["flock_target"])):
        a["flock_target"][f] = a["pos"][a["flock_of"] == f].mean(axis=0)
    d = a["flock_target"][a["flock_of"]] - a["pos"]
    a["vdes"] = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(np.float32)
    a["has_los"] = np.ones(len(d), np.uint32)
    a["state"][:] = 0
    rec, fl = capi.pack_agents(a)
    n = len(rec)
    ms = np.zeros(n, capi.MOVESTATE)
    ms["next_pos"][:, 0], ms["next_pos"][:, 2] = a["pos"][:, 0], a["pos"][:, 1]
    ms["step"] = 1.0
    ang = np.arctan2(a["vdes"][:, 1], a["vdes"][:, 0]) - np.pi / 2        # dir_quat_from_velocity, for the input only
    ms["next_rot"][:, 1], ms["next_rot"][:, 3] = np.sin(ang / 2), np.cos(ang / 2)
    ms["combat_facing"] = ms["next_rot"]
    return W, rec, fl, ms


def _context(capi, W, rec, fl, ms, device_blocking):
    nav = capi.Nav(0)
    nav.map_create(16, 16, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0); nav.route_build(0)
    nav.agents_upload(rec, fl, 20)
    nav.agents_upload_movestate(ms)
    if device_blocking:
        b = np.zeros(len(rec), capi.BLOCKING)
        b["faction_id"] = capi.FACTION_ID_NONE
        nav.agents_upload_blocking(b)
    return nav


def _host_side(capi, nav, work, tbl, n):
    """read back, apply, build the ops in work order, batch, commit -> number of ops"""
    p = nav.agents_read_patches(len(work))
    snap, _ = nav.agents_read_state(n, movestate=False)
    nav.agents_apply_updates()
    s = snap[work]
    blk = tbl["blocking"][work] != 0
    stop = ((p["flags"] & SET_STATE) != 0) & (p["next_block"] != 0) & ((s["flags"] & capi.FLAG_GARRISONED) == 0) & ~blk
    start = ((p["flags"] & SET_MOVING) != 0) & (blk | stop)
    u = work[stop]
    tbl["blocking"][u] = 1
    tbl["stop_x"][u], tbl["stop_z"][u], tbl["stop_radius"][u] = s["pos"][stop, 0], s["pos"][stop, 1], s["radius"][stop]
    idx = np.concatenate([np.nonzero(stop)[0], np.nonzero(start)[0]])
    delta = np.concatenate([np.ones(stop.sum(), np.int32), -np.ones(start.sum(), np.int32)])
    order = np.argsort(idx, kind="stable")
    uu = work[idx[order]]
    ops = np.zeros(len(uu), capi.BLOCKER_OP)
    ops["x"], ops["z"], ops["range"] = tbl["stop_x"][uu], tbl["stop_z"][uu], tbl["stop_radius"][uu]
    ops["faction_id"], ops["flags"], ops["delta"] = tbl["faction_id"][uu], snap["flags"][uu], delta[order]
    tbl["blocking"][work[start]] = 0
    if len(ops):
        nav.blockers_batch(ops)
    nav.map_commit()
    return len(ops)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--ticks", type=int, default=12)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    sys.path.insert(0, ROOT)
    pf = importlib.import_module("permafrost-engine_b200")
    bench = importlib.import_module("bench")
    capi = pf.capi
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu)
    W, rec, fl, ms = _crowd(bench, pf)
    n = len(rec)
    H, D = _context(capi, W, rec, fl, ms, False), _context(capi, W, rec, fl, ms, True)
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = capi.FACTION_ID_NONE
    out = open(args.out, "w") if args.out else None
    for t in range(args.ticks):
        st = H.agents_read_state(n, movestate=False)[0]["state"]
        work = np.nonzero((st != 2) & (st != 4))[0].astype(np.uint32)
        if not len(work):
            break
        for X in (H, D):
            X.agents_set_work(work)
            X.agents_tick(0)
            X.agents_compute_updates()
        times = {}
        for side in ((H, D) if t % 2 == 0 else (D, H)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            if side is H:
                nops = _host_side(capi, H, work, tbl, n)
            else:
                D.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
                D.map_commit()
            times["host" if side is H else "device"] = time.perf_counter() - t0
        identical = bool((H.blockers(0) == D.blockers(0)).all() and (H.local_islands(0) == D.local_islands(0)).all()
                         and D.agents_read_blocking(n).tobytes() == tbl.tobytes())
        assert identical, t
        row = {"map": "C2", "tick": t, "nwork": int(len(work)), "nops": int(nops), "blocking": int(tbl["blocking"].sum()),
               "host_ms": 1e3 * times["host"], "device_ms": 1e3 * times["device"], "identical": identical, "gpu": gpu}
        line = json.dumps(row)
        print(line, flush=True)
        if out:
            out.write(line + "\n"); out.flush()
    H.close(); D.close()


if __name__ == "__main__":
    main()
