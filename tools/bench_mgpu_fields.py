#!/usr/bin/env python
"""A job's goal batch built once for the whole job (pfnav_group_request_goals_ex) against every member building its own
(pfnav_pool_request_goals_ex on each member), on bench.py's C2 map (16 x 16 chunks) with its 16 goals, every member of an
in-process group needing all of them.

Two sets of `world` contexts on the same map: the members of a group (job side) and plain contexts (solo side). Timed:
  cold:         pool_clear on every context (not timed), then the batch;
  missing_only: a commit of blockers at a few random points on every context (not timed, the same ops on both sides),
                then the batch with PFNAV_REQUEST_MISSING_ONLY -- bench.py's C5 loop.
Each time is a host clock from a synchronise of every member device to the synchronise of every member device after
the call: until every member's fields are ready. The sides alternate which goes first; median of --reps after --warmup.
At the end, every job member's pool must equal the solo side's context of the same rank for every (dest, chunk).
With every member on one device the members share its SMs, so the field work saved shows there too; transfers between
GPUs are not measured unless --devices > 1 on a box with that many.
    python tools/bench_mgpu_fields.py [--worlds 2,3] [--devices N] [--reps 5] [--warmup 2] [--out FILE]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _pool(nav, nd):
    out = []
    for d in range(nd):
        for c in range(nav.cw * nav.ch):
            f, l, ffid = nav.pool_get(d, divmod(c, nav.cw))
            out.append((int(f is not None) | int(l is not None) << 1, ffid, b"" if f is None else f.tobytes(),
                        b"" if l is None else l.tobytes()))
    return out


def run(pf, bench, world, devices, reps, warmup, gpu, out):
    import torch
    capi = pf.capi
    W = bench.build_workload(pf, 1, 0)
    cw, nd = bench.CHUNKS, W["g_hi"] - W["g_lo"]
    tg = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(W["g_lo"], W["g_hi"])], np.int32)
    dests = np.arange(nd, dtype=np.int32)
    devs = sorted({r % devices for r in range(world)})

    def ctx(dev):
        nav = capi.Nav(dev)
        nav.map_create(cw, cw, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0)
        nav.pool_create(nd, nd * cw * cw)
        return nav
    job = [ctx(r % devices) for r in range(world)]
    solo = [ctx(r % devices) for r in range(world)]
    grp = capi.Group(job)

    def sync():
        for d in devs:
            torch.cuda.synchronize(d)

    def timed(fn):
        sync()
        t0 = time.perf_counter()
        fn()
        sync()
        return (time.perf_counter() - t0) * 1e3

    def side_job(flags):
        return lambda: grp.request_goals_ex(dests, tg, 0, flags)

    def side_solo(flags):
        return lambda: [nav.pool_request_goals(dests, tg, flags=flags) for nav in solo]

    rng = np.random.default_rng(0xF1E1D5)
    rows = []
    for mode, flags in (("cold", 0), ("missing_only", capi.REQUEST_MISSING_ONLY)):
        if flags:       # start from full pools
            grp.request_goals_ex(dests, tg)
            for nav in solo:
                nav.pool_request_goals(dests, tg)
        for rep in range(warmup + reps):
            if flags:
                pts = [(float(rng.uniform(-cw * 256 + 64, -64)), float(rng.uniform(64, cw * 256 - 64))) for _ in range(4)]
                for nav in job + solo:
                    for x, z in pts:
                        nav.blockers_incref(x, z, 10.0)
                    nav.map_commit()
            else:
                for nav in job + solo:
                    nav.pool_clear()
            order = (("job", side_job(flags)), ("solo", side_solo(flags)))
            t = {}
            for name, fn in (order if rep % 2 == 0 else order[::-1]):
                t[name] = timed(fn)
            built = [nav.mgpu_fields_stats(nd)[:2] for nav in job]
            if rep >= warmup:
                rows.append(dict(world=world, devices=len(devs), mode=mode, rep=rep - warmup, job_ms=t["job"], solo_ms=t["solo"],
                                 job_built=[list(b) for b in built], gpu=gpu))
                if out:
                    out.write(json.dumps(rows[-1]) + "\n"); out.flush()
    same = all(_pool(a, nd) == _pool(b, nd) for a, b in zip(job, solo))
    grp.close()
    for nav in job + solo:
        nav.close()
    assert same, "job members' pools differ from the solo contexts'"
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="2,3", help="comma-separated group sizes")
    ap.add_argument("--devices", type=int, default=0, help="devices to spread the members over (0: all visible)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    pf = importlib.import_module("permafrost-engine_b200")
    bench = importlib.import_module("bench")
    bench.set_workload("C2")
    devices = args.devices or torch.cuda.device_count()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu, "devices:", devices, flush=True)
    out = open(args.out, "w") if args.out else None
    for world in (int(w) for w in args.worlds.split(",")):
        rows = run(pf, bench, world, devices, args.reps, args.warmup, gpu, out)
        for mode in ("cold", "missing_only"):
            rs = [r for r in rows if r["mode"] == mode]
            j, s = np.median([r["job_ms"] for r in rs]), np.median([r["solo_ms"] for r in rs])
            print("world %d on %d device(s), %s: median job %.2f ms, every member alone %.2f ms (%d reps); requests built per "
                  "member in the last job call: %s; pools identical" % (world, rs[0]["devices"], mode, j, s, len(rs),
                                                                       rs[-1]["job_built"]), flush=True)


if __name__ == "__main__":
    main()
