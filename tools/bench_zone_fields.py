#!/usr/bin/env python
"""pfnav_pool_request_zones (one batch) against pfnav_pool_request_zone in a loop, on the C2 map (16 x 16 chunks).

m flocks arrive at once, each requesting its group-arrival (TARGET_ZONE) fields into its own pool destination. Every zone
is centred on a random open tile; its radius is drawn from {4, 8, 16, 32, 80} tiles. This mix is a choice made for the
benchmark (small formations up to the radius whose seed budget reaches the dim x dim cap), not a distribution taken from
the engine. The requests of each m are drawn from their own seed, so every run and every tree times the same requests.
For each m, every repetition clears both pools (cold), then times the serial loop on one context and the batch on
another, each window ending in a device synchronise. One warm-up repetition, then the median of --reps. The two pools
must hold identical entries (flow bytes, has, ffid) for every (dest, chunk). `path` is where the batch flooded its seeds:
"host" when it made two launches (the pool-entry scatter and the integration), "device" when it made three
(k_zone_seed_bits in between).

--baseline DIR also times the serial loop of pfnav_pool_request_zone in another checkout (for example the commit before
the batch), built in place, in a subprocess on the same requests; its pool must equal the batch's.
    python tools/bench_zone_fields.py [--reps 5] [--sizes 1,2,4,8,16,64,256,1024] [--baseline DIR] [--out FILE]"""
import argparse
import hashlib
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RADII = (4, 8, 16, 32, 80)
MAP_SEED = 0x5EED0001            # bench.py's C2 map
CW = 16


def _setup(pf, ndests):
    capi, synth = pf.capi, pf.synth
    cost = synth.cost_from_pathable(synth.make_map(CW, CW, MAP_SEED, rivers=True), CW, CW)
    nav = capi.Nav(0)
    nav.map_create(CW, CW, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0)
    nav.pool_create(ndests, 65536)
    return nav, cost


def _requests(synth, cost, m):
    """m zones: (dest, world centre, radius)"""
    rng = np.random.default_rng([0x5EED, m])
    open_ = np.argwhere(synth.blocked_to_image(cost, CW, CW) != 0xFF)
    t = open_[rng.integers(0, len(open_), m)]
    rad = rng.choice(RADII, m)
    return [(i, synth.tile_center_xz(int(r) // 64, int(c) // 64, int(r) % 64, int(c) % 64), int(rad[i])) for i, (r, c) in enumerate(t)]


def _serial(nav, reqs):
    return [nav.pool_request_zone(d, xz, rad) for d, xz, rad in reqs]


def _digest(nav, m, nfields):
    h = hashlib.sha256(np.array(nfields, np.int64).tobytes())
    for d in range(m):
        for c in range(CW * CW):
            f, _, ffid = nav.pool_get(d, divmod(c, CW))
            h.update(np.array([f is not None, ffid], np.uint64).tobytes())
            if f is not None:
                h.update(f.tobytes())
    return h.hexdigest()


def serial_only(root, sizes, reps):
    """the serial loop alone, with the package of the checkout `root`: one JSON line per size"""
    sys.path.insert(0, root)
    import torch
    pf = importlib.import_module("permafrost-engine_b200")
    nav, cost = _setup(pf, max(sizes))
    for m in sizes:
        reqs = _requests(pf.synth, cost, m)
        ts = []
        for rep in range(reps + 1):
            nav.pool_clear(); torch.cuda.synchronize()
            t0 = time.perf_counter()
            nf = _serial(nav, reqs)
            torch.cuda.synchronize()
            if rep:
                ts.append(time.perf_counter() - t0)
        print(json.dumps({"m": m, "serial_ms": 1e3 * statistics.median(ts), "digest": _digest(nav, m, nf)}), flush=True)
    nav.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1,2,4,8,16,64,256,1024")
    ap.add_argument("--baseline", default=None, help="another checkout whose pfnav_pool_request_zone loop is timed too")
    ap.add_argument("--serial-only", default=None, help=argparse.SUPPRESS)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    sizes = [int(s) for s in args.sizes.split(",")]
    if args.serial_only:
        serial_only(args.serial_only, sizes, args.reps)
        return
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    sys.path.insert(0, ROOT)
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu)
    base = {}
    if args.baseline:
        r = subprocess.run([sys.executable, os.path.abspath(__file__), "--serial-only", os.path.abspath(args.baseline),
                            "--sizes", args.sizes, "--reps", str(args.reps)], capture_output=True, text=True, cwd=args.baseline)
        assert r.returncode == 0, r.stderr[-2000:]
        base = {b["m"]: b for b in (json.loads(l) for l in r.stdout.splitlines() if l.startswith("{"))}
    serial, cost = _setup(pf, max(sizes))
    batch, _ = _setup(pf, max(sizes))
    out = open(args.out, "w") if args.out else None
    for m in sizes:
        reqs = _requests(pf.synth, cost, m)
        rec = np.zeros(m, capi.ZONE_REQ)
        for i, (d, xz, rad) in enumerate(reqs):
            rec[i]["dest"], rec[i]["centre_x"], rec[i]["centre_z"], rec[i]["radius"] = d, xz[0], xz[1], rad
        ts, tb = [], []
        for rep in range(args.reps + 1):
            serial.pool_clear(); batch.pool_clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            nf_serial = _serial(serial, reqs)
            torch.cuda.synchronize()
            a = time.perf_counter() - t0
            l0 = batch.launch_count()
            t0 = time.perf_counter()
            done, nf_batch = batch.pool_request_zones(rec)
            torch.cuda.synchronize()
            b = time.perf_counter() - t0
            launches = batch.launch_count() - l0
            assert done == m and list(nf_batch) == nf_serial
            if rep:
                ts.append(a); tb.append(b)
        digest = _digest(batch, m, nf_serial)
        same = digest == _digest(serial, m, nf_serial)
        assert same, "the batch and the serial loop left different pools"
        row = {"map": "C2", "m": m, "fields": int(sum(nf_serial)), "radii": list(RADII), "reps": args.reps,
               "path": {2: "host", 3: "device"}.get(launches, "none"), "serial_ms": 1e3 * statistics.median(ts),
               "batch_ms": 1e3 * statistics.median(tb), "speedup": statistics.median(ts) / statistics.median(tb),
               "identical_pool": bool(same)}
        if m in base:
            assert base[m]["digest"] == digest, "the baseline's serial loop left a different pool"
            row.update(baseline_serial_ms=base[m]["serial_ms"], speedup_vs_baseline=base[m]["serial_ms"] / row["batch_ms"],
                       serial_vs_baseline=base[m]["serial_ms"] / row["serial_ms"], identical_to_baseline=True)
        row["gpu"] = gpu
        line = json.dumps(row)
        print(line, flush=True)
        if out:
            out.write(line + "\n"); out.flush()
    serial.close(); batch.close()


if __name__ == "__main__":
    main()
