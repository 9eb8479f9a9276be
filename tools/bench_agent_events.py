#!/usr/bin/env python
"""The tick's decisions back to the engine: the device event list against the patch read-back, on the C2 (100 000) and
C3 (1 000 000) populations of bench.py with every flock's target at the flock's own centre, so that a moving crowd
arrives over the ticks (the adjacent-arrived cascade spreads) while the rest keeps moving.

Two contexts step the same headless loop (set_work_dev, agents_tick with the desired velocity towards the target,
compute_updates, the side under test, rebuild_index). Per tick:
  events_ms:   collect_events, apply_updates, read_events;
  readback_ms: read_patches, apply_updates, the numpy filter of the patches (the selection of collect_events; the engine
               holds its own GARRISONED flags, taken once outside the timing). It cannot give state_before or the position
               the apply leaves: the apply overwrites both on the device.
Each is a host clock from a device synchronise to a device synchronise after the side's last call. The two sides take
turns going first. A run uploads the population afresh and steps --ticks ticks; the figures are the median and min / max
over --runs runs, per tick, with the number of work items and events. The first run checks that the two sides select the
same work items with the same uid, flags, todo, attack and dest.
    python tools/bench_agent_events.py [--workloads C2,C3] [--ticks 8] [--runs 7] [--out FILE]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SEL = 1 | (1 << 10) | (1 << 12)          # SET_STATE | SET_DEST | SET_MOVING


def _crowd(bench, pf, workload):
    capi = pf.capi
    bench.set_workload(workload)
    W = bench.build_workload(pf, 1, 0)
    a = W["agents"]
    for f in range(len(a["flock_target"])):
        a["flock_target"][f] = a["pos"][a["flock_of"] == f].mean(axis=0)
    d = a["flock_target"][a["flock_of"]] - a["pos"]
    a["vdes"] = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(np.float32)
    a["has_los"] = np.ones(len(d), np.uint32)
    a["state"][:] = 0
    rec, fl = capi.pack_agents(a)
    ms = np.zeros(len(rec), capi.MOVESTATE)
    ms["next_pos"][:, 0], ms["next_pos"][:, 2] = a["pos"][:, 0], a["pos"][:, 1]
    ms["step"] = 1.0
    ang = np.arctan2(a["vdes"][:, 1], a["vdes"][:, 0]) - np.pi / 2
    ms["next_rot"][:, 1], ms["next_rot"][:, 3] = np.sin(ang / 2), np.cos(ang / 2)
    ms["combat_facing"] = ms["next_rot"]
    return W, rec, fl, ms


def _filter(capi, p, work, garr):
    """the host's selection over the read-back patches"""
    sel = (((p["flags"] & SEL) != 0) | (p["engine_todo"] != 0)) & ~garr[work]
    q = p[sel]
    return work[sel], q["flags"], q["engine_todo"], q["next_attack"], q["next_dest"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workloads", default="C2,C3")
    ap.add_argument("--ticks", type=int, default=8)
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    sys.path.insert(0, ROOT)
    pf = importlib.import_module("permafrost-engine_b200")
    bench = importlib.import_module("bench")
    capi = pf.capi
    name, power = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                                 capture_output=True, text=True).stdout.strip().split(", ")
    out = open(args.out, "w") if args.out else None
    for wl in args.workloads.split(","):
        W, rec, fl, ms = _crowd(bench, pf, wl)
        n = len(rec)
        garr = (rec["flags"] & capi.FLAG_GARRISONED) != 0
        E, R = capi.Nav(0), capi.Nav(0)
        for X in (E, R):
            X.map_create(bench.CHUNKS, bench.CHUNKS, 1); X.map_upload_layer(0, W["cost"]); X.map_build_nav(0); X.route_build(0)
        times = {"events": np.zeros((args.runs, args.ticks)), "readback": np.zeros((args.runs, args.ticks))}
        nwork, nev = [0] * args.ticks, [0] * args.ticks
        for r in range(args.runs):
            for X in (E, R):
                X.agents_upload(rec, fl, 20)
                X.agents_upload_movestate(ms)
            for t in range(args.ticks):
                for X in (E, R):
                    nw = X.agents_set_work_dev()
                    X.agents_tick(0)
                    X.agents_compute_updates()
                work = R.agents_read_work()
                for side in (("events", "readback") if t % 2 == 0 else ("readback", "events")):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if side == "events":
                        E.agents_collect_events()
                        E.agents_apply_updates()
                        ev = E.agents_read_events()
                    else:
                        p = R.agents_read_patches(nw)
                        R.agents_apply_updates()
                        host = _filter(capi, p, work, garr)
                    torch.cuda.synchronize()
                    times[side][r, t] = 1e3 * (time.perf_counter() - t0)
                for X in (E, R):
                    X.agents_rebuild_index()
                nwork[t], nev[t] = int(nw), int(len(ev))
                if r == 0:
                    got = (ev["uid"], ev["flags"], ev["todo"], ev["attack"], ev["dest"])
                    assert all(np.array_equal(g, h) for g, h in zip(got, host)), (wl, t)
        for t in range(args.ticks):
            row = {"workload": wl, "entities": n, "tick": t, "work_items": nwork[t], "events": nev[t],
                   "event_bytes": 48 * nev[t], "patch_bytes": 160 * nwork[t], "runs": args.runs, "card": name,
                   "power_limit_w": float(power),
                   "what": "host-observed ms per tick from a device synchronise to a device synchronise"}
            for side in ("events", "readback"):
                v = times[side][:, t]
                row[side + "_ms"] = {"median": float(np.median(v)), "min": float(v.min()), "max": float(v.max())}
            line = json.dumps(row)
            print(line, flush=True)
            if out:
                out.write(line + "\n"); out.flush()
        E.close(); R.close()


if __name__ == "__main__":
    main()
