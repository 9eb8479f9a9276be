#!/usr/bin/env python
"""A job's zone and entity-field batches built once for the whole job (pfnav_group_request_zones,
pfnav_group_request_entity_fields_batch) against every member building its own (pfnav_pool_request_zones /
pfnav_pool_request_entity_fields_batch on each member), on the C2 map (16 x 16 chunks).

Workloads, cold (every pool cleared before each repetition, not timed):
  zones_M:  the M group-arrival zones of tools/bench_zone_fields.py (random open centres, radii from {4, 8, 16, 32, 80});
  entity_M: the front of tools/bench_entity_fields.py -- two factions of 4096 units, one TARGET_ENEMIES destination per
            faction over its units' chunks, plus M TARGET_ENTITY destinations over the 3 x 3 chunks around a target unit.
Two sets of `world` contexts: the members of a group (job side) and plain contexts (solo side). Each time is a host clock
from a synchronise of every member device to the synchronise after the call. The sides alternate which goes first; median
of --reps after --warmup. At the end every job member's pool must equal the solo context of the same rank for every
(dest, chunk). With every member on one device the members share its SMs; transfers between GPUs are not measured unless
--devices > 1 on a box with that many.
    python tools/bench_mgpu_aux_fields.py [--worlds 2,3] [--devices N] [--reps 5] [--warmup 2] [--out FILE]"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
import bench_zone_fields  # noqa: E402

CW = bench_zone_fields.CW
UNITS, RADIUS = 4096, 1.5


def zone_workload(capi, synth, cost, m):
    rows = bench_zone_fields._requests(synth, cost, m)
    reqs = np.zeros(m, capi.ZONE_REQ)
    for i, (d, xz, rad) in enumerate(rows):
        reqs[i]["dest"], reqs[i]["centre_x"], reqs[i]["centre_z"], reqs[i]["radius"] = d, xz[0], xz[1], rad
    return reqs


def entity_workload(capi, m):
    """the front of tools/bench_entity_fields.py -> (reqs, footprints, chunks)"""
    rng = np.random.default_rng(0x5EED)
    W = H = CW * 256.0
    pos = np.zeros((2, UNITS, 2), np.float32)
    for f in range(2):
        pos[f, :, 0] = -rng.uniform(0.0, W, UNITS)
        pos[f, :, 1] = H / 2 + (rng.uniform(-72.0, -6.0, UNITS) if f == 0 else rng.uniform(6.0, 72.0, UNITS))
    fp = capi.Nav.footprints(pos.reshape(-1, 2), RADIUS)
    chunks = []
    for f in range(2):
        r = (pos[f, :, 1] // 256).astype(int); c = (-pos[f, :, 0] // 256).astype(int)
        chunks.append(np.unique(np.stack([r, c], 1).clip(0, CW - 1), axis=0).astype(np.int32))
    reqs = [(0, capi.TARGET_ENEMIES, UNITS, UNITS), (1, capi.TARGET_ENEMIES, 0, UNITS)]
    for k, t in enumerate(rng.integers(0, 2 * UNITS, m)):
        tr, tc = int(fp["z"][t] // 256), int(-fp["x"][t] // 256)
        chunks.append(np.array([(r, c) for r in range(tr - 1, tr + 2) for c in range(tc - 1, tc + 2)
                                if 0 <= r < CW and 0 <= c < CW], np.int32))
        reqs.append((2 + k, capi.TARGET_ENTITY, int(t), 1))
    rec = np.zeros(len(reqs), capi.ENTITY_FIELD_REQ)
    coff = np.cumsum([0] + [len(c) for c in chunks])
    for i, (d, kind, e0, en) in enumerate(reqs):
        rec[i] = (d, 0, 0, kind, e0, en, coff[i], len(chunks[i]))
    return rec, fp, np.concatenate(chunks)


def _pool(nav, nd):
    out = []
    for d in range(nd):
        for c in range(CW * CW):
            f, _, ffid = nav.pool_get(d, divmod(c, CW))
            out.append((f is not None, ffid, b"" if f is None else f.tobytes()))
    return out


def run(pf, world, devices, reps, warmup, gpu, out, cases):
    import torch
    capi, synth = pf.capi, pf.synth
    cost = synth.cost_from_pathable(synth.make_map(CW, CW, bench_zone_fields.MAP_SEED, rivers=True), CW, CW)
    nd = 2 + max(m for _, m in cases)
    devs = sorted({r % devices for r in range(world)})

    def ctx(dev):
        nav = capi.Nav(dev)
        nav.map_create(CW, CW, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0)
        nav.pool_create(nd, 65536)
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

    rows = []
    for kind, m in cases:
        if kind == "zones":
            zr = zone_workload(capi, synth, cost, m)
            side_job = lambda: grp.request_zones(zr)
            side_solo = lambda: [nav.pool_request_zones(zr) for nav in solo]
            nfields = int(grp.request_zones(zr).sum())
        else:
            er, fp, ch = entity_workload(capi, m)
            side_job = lambda: grp.request_entity_fields_batch(er, fp, ch)
            side_solo = lambda: [nav.pool_request_entity_fields_batch(er, fp, ch) for nav in solo]
            nfields = len(ch)
        for rep in range(warmup + reps):
            for nav in job + solo:
                nav.pool_clear()
            order = (("job", side_job), ("solo", side_solo))
            t = {}
            for name, fn in (order if rep % 2 == 0 else order[::-1]):
                t[name] = timed(fn)
            built = [nav.mgpu_fields_stats(0)[0] for nav in job]
            if rep >= warmup:
                rows.append(dict(world=world, devices=len(devs), workload="%s_%d" % (kind, m), fields=nfields, rep=rep - warmup,
                                 job_ms=t["job"], solo_ms=t["solo"], job_built=built, gpu=gpu))
                if out:
                    out.write(json.dumps(rows[-1]) + "\n"); out.flush()
        same = all(_pool(a, nd) == _pool(b, nd) for a, b in zip(job, solo))
        assert same, "job members' pools differ from the solo contexts' (%s_%d)" % (kind, m)
    grp.close()
    for nav in job + solo:
        nav.close()
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--worlds", default="2,3", help="comma-separated group sizes")
    ap.add_argument("--devices", type=int, default=0, help="devices to spread the members over (0: all visible)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--cases", default="zones:16,zones:1024,entity:1024", help="kind:M,... (kind zones or entity)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    pf = importlib.import_module("permafrost-engine_b200")
    devices = args.devices or torch.cuda.device_count()
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu, "devices:", devices, flush=True)
    cases = [(k, int(m)) for k, m in (c.split(":") for c in args.cases.split(","))]
    out = open(args.out, "w") if args.out else None
    for world in (int(w) for w in args.worlds.split(",")):
        rows = run(pf, world, devices, args.reps, args.warmup, gpu, out, cases)
        for kind, m in cases:
            rs = [r for r in rows if r["workload"] == "%s_%d" % (kind, m)]
            j, s = np.median([r["job_ms"] for r in rs]), np.median([r["solo_ms"] for r in rs])
            print("world %d on %d device(s), %s_%d (%d fields): median job %.2f ms, every member alone %.2f ms (%d reps); "
                  "fields built per member: %s; pools identical" % (world, rs[0]["devices"], kind, m, rs[0]["fields"], j, s,
                                                                     len(rs), rs[-1]["job_built"]), flush=True)


if __name__ == "__main__":
    main()
