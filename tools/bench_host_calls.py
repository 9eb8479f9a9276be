#!/usr/bin/env python
"""Per-call latency of the blocking host-array entry points on the C2 map (16 x 16 chunks): each call at the size the
engine's field.c drop-in (shim/field_pfnav.c) uses -- one field, one region, one chunk -- and at a batch of 1024.

    flow_fields_update   n requests (wave 0 of a goal's plan, repeated); flow_fields_update_inplace: the same, init = 0
    los_fields_create    n requests (the goal's LOS chain, repeated with its parents renumbered)
    region_fields        n group-arrival regions (dim 96); group_arrival_field: one field from n targets
    zone_fields / entity_fields (enemies)   n chunk fields
    group_arrival_velocity   n positions;  ents_in_circle: up to n ids;  pool_repair: the work list of 16384 agents

A goal batch is in the pool before the timings (the group-arrival velocities read it). Every call is timed with a host
clock around the call, which returns after its stream is synchronised; warm-up calls first, then the median and the
minimum of --reps. One JSON line per (call, n).
    python tools/bench_host_calls.py [--reps 50] [--sizes 1,1024] [--out FILE]"""
import argparse
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402

NGOALS, AGENTS = 16, 16384


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--sizes", default="1,1024")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    pf = importlib.import_module("permafrost-engine_b200")
    capi, synth = pf.capi, pf.synth
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    bench.set_workload("C2")
    cw = bench.CHUNKS
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, bench.MAP_SEED, rivers=True), cw, cw)
    nav = capi.Nav(0)
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.pool_create(NGOALS, 65536)
    a = synth.make_agents(cost, cw, cw, AGENTS, NGOALS, bench.MAP_SEED, radius=1.5, spacing=2.2)
    rec, fl = capi.pack_agents(a)
    nav.agents_upload(rec, fl, 20)
    nav.agents_set_work(np.arange(AGENTS, dtype=np.uint32))
    img = synth.blocked_to_image(cost, cw, cw)
    goals = []
    for tx, tz in fl["target"]:
        r, c = int(tz // 4), int(-tx // 4)
        goals.append([r // 64, c // 64, r % 64, c % 64])
    goals = np.array(goals, np.int32)
    assert all(img[g[0] * 64 + g[2], g[1] * 64 + g[3]] != 255 for g in goals)
    nav.pool_request_goals(np.arange(NGOALS, dtype=np.int32), goals)
    nav.fields_join()
    nav.agents_tick(capi.TICK_VDES_FROM_POOL)
    fr, _, fw, lr, _ = nav.plan_goal(tuple(goals[0]))
    fr = fr[fw == 0]
    pos = rec["pos"]
    centre = goals[0, :2] * 64 + goals[0, 2:]
    rng = np.random.default_rng(0)

    def los_batch(n):
        reps = -(-n // len(lr))
        big = np.concatenate([lr] * reps)
        for k in range(1, reps):
            sl = big[k * len(lr):(k + 1) * len(lr)]
            sl["prev_index"] = np.where(sl["prev_index"] >= 0, sl["prev_index"] + k * len(lr), sl["prev_index"])
        if n < len(lr):      # the destination chunk's request, which names no parent
            return big[lr["prev_index"] < 0][:n]
        return big[:n]

    def cases(n):
        H = cw * 64
        fq = fr[np.arange(n) % len(fr)]
        upd = fq.copy(); upd["init"] = 0
        base = nav.flow_fields_update(fq)
        lq = los_batch(n)
        cen = rng.integers(48, H - 48, (n, 2))
        regions = [dict(center=tuple(c), target=tuple(c + rng.integers(-20, 20, 2))) for c in cen]
        chunks = np.stack([np.arange(n) // cw % cw, np.arange(n) % cw], 1).astype(np.int32)
        fp = capi.Nav.footprints(pos[rng.integers(0, len(pos), n)], 1.5)
        p = pos[np.arange(n) % len(pos)]
        return [("flow_fields_update", lambda: nav.flow_fields_update(fq)),
                ("flow_fields_update_inplace", lambda: nav.flow_fields_update(upd, inout=base)),
                ("los_fields_create", lambda: nav.los_fields_create(lq)),
                ("region_fields", lambda: nav.region_fields(96, regions)),
                ("group_arrival_field", lambda: nav.group_arrival_field(96, p, p[0])),
                ("zone_fields", lambda: nav.zone_fields(centre, 16, chunks)),
                ("entity_fields", lambda: nav.entity_fields(capi.TARGET_ENEMIES, fp, chunks)),
                ("group_arrival_velocity", lambda: nav.group_arrival_velocity(0, p[0], 8, p)),
                ("ents_in_circle", lambda: nav.ents_in_circle(float(p[0, 0]), float(p[0, 1]), 60.0, n))]

    out = open(args.out, "w") if args.out else None

    def report(name, n, fn):
        for _ in range(3):
            fn()
        ts = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            ts.append(time.perf_counter() - t0)
        line = json.dumps({"call": name, "n": n, "median_ms": 1e3 * statistics.median(ts), "min_ms": 1e3 * min(ts),
                           "reps": args.reps, "gpu": gpu})
        print(line, flush=True)
        if out:
            out.write(line + "\n"); out.flush()

    for n in [int(s) for s in args.sizes.split(",")]:
        for name, fn in cases(n):
            report(name, n, fn)
    report("pool_repair", AGENTS, nav.pool_repair)
    nav.close()


if __name__ == "__main__":
    main()
