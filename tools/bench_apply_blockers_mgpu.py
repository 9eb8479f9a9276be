#!/usr/bin/env python
"""Blockers of stopping units in a sharded job, the host path against the shared device path, on tools/bench_apply_blockers.py's
arriving C2 crowd (bench.py's 16 x 16-chunk map and 100 000-agent population) split over an in-process group.

Two groups of `world` members step the same ticks (agents_tick with a desired velocity towards the target,
compute_updates, on every member's own range). Per tick:
  host_ms:   what a sharded engine does without the opt-in: read every member's patches and state back, apply_updates,
             build the entity_block / entity_unblock ops on the host from a host blocking table, then blockers_batch and
             map_commit on every member;
  device_ms: apply_updates_ex(APPLY_BLOCKERS) on every member, group_exchange_blocker_ops, map_commit on every member.
Each is a host clock from a synchronise of every member device to the end of the last map_commit (which waits for its
device). The two sides take turns going first; the pfnav_group_gather that follows is not timed. After every tick the
blocker counts and local islands of every member of both groups must be equal, and the device group's blocking tables
(own ranges, concatenated) must equal the host table.
With --devices 1 every member sits on device 0: such numbers say nothing about transfers between GPUs.
    python tools/bench_apply_blockers_mgpu.py [--worlds 2] [--devices N] [--ticks 12] [--out FILE]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench_apply_blockers as single      # noqa: E402

SET_STATE, SET_MOVING = single.SET_STATE, single.SET_MOVING


def _group(capi, W, rec, fl, ms, world, devices, device_blocking):
    n = len(rec)
    navs = []
    for r in range(world):
        nav = capi.Nav(r % devices)
        nav.map_create(16, 16, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0); nav.route_build(0)
        navs.append(nav)
    grp = capi.Group(navs)
    if device_blocking:
        grp.share_blockers()
    ranges = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
    for nav, (lo, hi) in zip(navs, ranges):
        nav.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, 20)
    grp.gather()
    for nav, (lo, hi) in zip(navs, ranges):
        nav.agents_upload_movestate(ms[lo:hi])
        if device_blocking:
            b = np.zeros(hi - lo, capi.BLOCKING)
            b["faction_id"] = capi.FACTION_ID_NONE
            nav.agents_upload_blocking(b)
    return grp, navs, ranges


def _host_ops(capi, work, p, snap, tbl):
    """the entity_block / entity_unblock ops of the tick in work order, from the patches and the snapshot; updates tbl"""
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
    return ops


def _own(work, lo, hi):
    return work[(work >= lo) & (work < hi)]


def run(pf, bench, world, devices, ticks, gpu, out):
    import torch
    capi = pf.capi
    W, rec, fl, ms = single._crowd(bench, pf)
    n = len(rec)
    gh, H, ranges = _group(capi, W, rec, fl, ms, world, devices, False)
    gd, D, _ = _group(capi, W, rec, fl, ms, world, devices, True)
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = capi.FACTION_ID_NONE

    def sync():
        for d in range(devices):
            torch.cuda.synchronize(d)

    def host_side(work):
        p = np.concatenate([nav.agents_read_patches(len(_own(work, lo, hi))) for nav, (lo, hi) in zip(H, ranges)])
        snap = np.concatenate([nav.agents_read_state(hi - lo, movestate=False)[0] for nav, (lo, hi) in zip(H, ranges)])
        for nav in H:
            nav.agents_apply_updates()
        ops = _host_ops(capi, work, p, snap, tbl)
        for nav in H:
            if len(ops):
                nav.blockers_batch(ops)
            nav.map_commit()
        return len(ops)

    def device_side():
        for nav in D:
            nav.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        gd.exchange_blocker_ops()
        for nav in D:
            nav.map_commit()

    rows = []
    for t in range(ticks):
        st = np.concatenate([nav.agents_read_state(hi - lo, movestate=False)[0]["state"] for nav, (lo, hi) in zip(H, ranges)])
        work = np.nonzero((st != 2) & (st != 4))[0].astype(np.uint32)
        if not len(work):
            break
        for g in (H, D):
            for nav, (lo, hi) in zip(g, ranges):
                nav.agents_set_work(_own(work, lo, hi))
                nav.agents_tick(0)
                nav.agents_compute_updates()
        times = {}
        for side in (("host", "device") if t % 2 == 0 else ("device", "host")):
            sync()
            t0 = time.perf_counter()
            if side == "host":
                nops = host_side(work)
            else:
                device_side()
            times[side] = time.perf_counter() - t0
        gh.gather(); gd.gather()
        b0, l0 = H[0].blockers(0), H[0].local_islands(0)
        identical = all((nav.blockers(0) == b0).all() and (nav.local_islands(0) == l0).all() for nav in H[1:] + D)
        got = np.concatenate([nav.agents_read_blocking(hi - lo) for nav, (lo, hi) in zip(D, ranges)])
        identical = bool(identical and got.tobytes() == tbl.tobytes())
        assert identical, (world, t)
        row = {"map": "C2", "world": world, "devices": min(devices, world), "tick": t, "nwork": int(len(work)),
               "nops": int(nops), "blocking": int(tbl["blocking"].sum()), "host_ms": 1e3 * times["host"],
               "device_ms": 1e3 * times["device"], "identical": identical, "gpu": gpu}
        line = json.dumps(row)
        print(line, flush=True)
        if out:
            out.write(line + "\n"); out.flush()
        rows.append(row)
    gh.close(); gd.close()
    for nav in H + D:
        nav.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="2", help="comma-separated group sizes")
    ap.add_argument("--devices", type=int, default=0, help="devices to spread the members over (0: all visible)")
    ap.add_argument("--ticks", type=int, default=12)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    sys.path.insert(0, ROOT)
    pf = importlib.import_module("permafrost-engine_b200")
    bench = importlib.import_module("bench")
    devices = args.devices or torch.cuda.device_count()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu, "devices:", devices)
    out = open(args.out, "w") if args.out else None
    for world in (int(w) for w in args.worlds.split(",")):
        rows = run(pf, bench, world, devices, args.ticks, gpu, out)
        h = np.median([r["host_ms"] for r in rows]); d = np.median([r["device_ms"] for r in rows])
        print("world %d on %d device(s): median host %.2f ms, device %.2f ms over %d ticks" % (world, min(devices, world), h, d, len(rows)),
              flush=True)


if __name__ == "__main__":
    main()
