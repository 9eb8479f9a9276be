#!/usr/bin/env python
"""pfnav_map_query (one batch on the device) against the host routine called once per query, on the C2 map (16 x 16
chunks, bench.py's map seed) with 300 committed blockers.

A batch of n queries mixes the six kinds evenly, in turn from CLOSEST_PATHABLE (n = 1 is one CLOSEST_PATHABLE query).
Positions are random tiles of the map (any tile, so some searches start on impassable tiles); MAXIMALLY_CLOSE asks about a destination up to 16 tiles from the position with tolerance 1.5 x 3
wu. This mix is a choice made for the benchmark, not a distribution taken from the engine. The queries of each n are
drawn from their own seed.

batch_ms: host clock around one pfnav_map_query call (it ends in a stream synchronise), median of --reps after one
warm-up call. host_ms: pfnav_route_arrival_consts (the host routine the tick's arrived() constants use) called once per
CLOSEST_PATHABLE / MAXIMALLY_CLOSE query of the same batch, median of --reps; the probe kinds and DEST_ID have no host
routine in the library and are not in it. host_ms includes the Python side of each call (ctypes, the float32 tolerance
test in numpy); host_overhead_ms is the same loop with every point moved off the map, where the routine returns at once.
The host loop is timed up to --host-max queries; above that it is "not measured". Every host answer must equal the
batch's.
    python tools/bench_map_query.py [--reps 5] [--sizes 1,64,4096,65536] [--host-max 4096] [--out FILE]"""
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
MAP_SEED, CW = 0x5EED0001, 16


def _setup(capi, synth):
    cost = synth.cost_from_pathable(synth.make_map(CW, CW, MAP_SEED, rivers=True), CW, CW)
    nav = capi.Nav(0)
    nav.map_create(CW, CW, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    rng = np.random.default_rng(0x5EED)
    for _ in range(300):
        nav.blockers_incref(float(rng.uniform(-CW * 256, 0)), float(rng.uniform(0, CW * 256)), float(rng.uniform(1, 12)))
    nav.map_commit()
    return nav


def _queries(capi, synth, n):
    rng = np.random.default_rng([0x5EED, n])
    H = W = CW * 64
    r, c = rng.integers(0, H, n), rng.integers(0, W, n)
    dr, dc = np.clip(r + rng.integers(-16, 17, n), 0, H - 1), np.clip(c + rng.integers(-16, 17, n), 0, W - 1)
    q = np.zeros(n, capi.MAP_QUERY)
    q["kind"] = (capi.QUERY_CLOSEST_PATHABLE + np.arange(n)) % 6      # n = 1: one CLOSEST_PATHABLE query
    q["x"], q["z"] = -4.0 * c - 2.0, 4.0 * r + 2.0
    q["dst_x"], q["dst_z"] = -4.0 * dc - 2.0, 4.0 * dr + 2.0
    q["tolerance"] = 1.5 * 3.0
    q["faction_id"] = capi.FACTION_ID_NONE
    return q


def _host(nav, q):
    """the host routine per search query -> {index: (ok, x, z)}"""
    out = {}
    f = np.float32
    for i in np.nonzero((q["kind"] == 3) | (q["kind"] == 4))[0]:
        a = q[i]
        if a["kind"] == 3:
            ok, nearest, _ = nav.route_arrival_consts((a["x"], a["z"]))
            out[i] = (ok, nearest[0] if ok else 0.0, nearest[1] if ok else 0.0)
        else:
            _, _, mc = nav.route_arrival_consts((a["dst_x"], a["dst_z"]))
            dx, dz = mc[:, 0] - f(a["x"]), mc[:, 1] - f(a["z"])
            out[i] = (int((np.sqrt(dx * dx + dz * dz) <= f(a["tolerance"])).any()), 0.0, 0.0)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1,64,4096,65536")
    ap.add_argument("--host-max", type=int, default=4096)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    sys.path.insert(0, ROOT)
    pf = importlib.import_module("permafrost-engine_b200")
    capi, synth = pf.capi, pf.synth
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu)
    nav = _setup(capi, synth)
    out = open(args.out, "w") if args.out else None
    for n in [int(s) for s in args.sizes.split(",")]:
        q = _queries(capi, synth, n)
        res = nav.map_query(q)                       # warm-up
        tb = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            res = nav.map_query(q)
            tb.append(time.perf_counter() - t0)
        row = {"map": "C2", "n": n, "nsearch": int(((q["kind"] == 3) | (q["kind"] == 4)).sum()), "reps": args.reps,
               "batch_ms": 1e3 * statistics.median(tb)}
        if n <= args.host_max:
            th = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                h = _host(nav, q)
                th.append(time.perf_counter() - t0)
            off = q.copy()
            off["x"], off["dst_x"] = 1e6, 1e6
            to = []
            for _ in range(args.reps):
                t0 = time.perf_counter()
                _host(nav, off)
                to.append(time.perf_counter() - t0)
            for i, (ok, x, z) in h.items():
                assert res[i]["ok"] == ok and (q[i]["kind"] == 4 or (res[i]["x"] == x and res[i]["z"] == z)), i
            row.update(host_ms=1e3 * statistics.median(th), host_overhead_ms=1e3 * statistics.median(to), identical=True,
                       speedup=statistics.median(th) / statistics.median(tb))
        else:
            row.update(host_ms="not measured", host_overhead_ms="not measured", speedup="not measured")
        row["gpu"] = gpu
        line = json.dumps(row)
        print(line, flush=True)
        if out:
            out.write(line + "\n"); out.flush()
    nav.close()


if __name__ == "__main__":
    main()
