#!/usr/bin/env python
"""pfnav_pool_request_entity_fields_batch (one batch) against pfnav_pool_request_entity_fields in a loop, on the C2 map
(16 x 16 chunks).

Two factions at war, 4096 units each (selection radius 1.5), stand in a front across the whole map. Every batch holds
one TARGET_ENEMIES (enemy-seek) destination per faction over the chunks its own units stand on -- the fields
N_RequestAsyncEnemySeekField asks for -- plus m TARGET_ENTITY (surround) destinations, each over the 3 x 3 chunks
around a target unit. For each m, every repetition clears both pools (cold), then times the serial loop on one context
and the batch on another, each window ending in a device synchronise. One warm-up repetition, then the median of --reps.
The two pools must hold identical entries (flow bytes, has, ffid) for every requested (dest, chunk).
    python tools/bench_entity_fields.py [--reps 5] [--sizes 1,4,16,64,256,1024] [--out FILE]"""
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

UNITS, RADIUS = 4096, 1.5


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1,4,16,64,256,1024")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    pf = importlib.import_module("permafrost-engine_b200")
    capi, synth = pf.capi, pf.synth
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu)
    bench.set_workload("C2")
    cw = bench.CHUNKS
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, bench.MAP_SEED, rivers=True), cw, cw)
    sizes = [int(s) for s in args.sizes.split(",")]
    navs = []
    for _ in range(2):
        nav = capi.Nav(0)
        nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0)
        nav.pool_create(2 + max(sizes), 65536)
        navs.append(nav)
    serial, batch = navs
    # the front: faction 0 in a band just above the map's middle row, faction 1 just below, across the full width
    rng = np.random.default_rng(0x5EED)
    W, H = cw * 256.0, cw * 256.0
    pos = np.zeros((2, UNITS, 2), np.float32)
    for f in range(2):
        pos[f, :, 0] = -rng.uniform(0.0, W, UNITS)
        pos[f, :, 1] = H / 2 + (rng.uniform(-72.0, -6.0, UNITS) if f == 0 else rng.uniform(6.0, 72.0, UNITS))
    fp = capi.Nav.footprints(pos.reshape(-1, 2), RADIUS)              # faction f = fp[f * UNITS:(f + 1) * UNITS]
    own_chunks = []
    for f in range(2):
        r = (pos[f, :, 1] // 256).astype(int); c = (-pos[f, :, 0] // 256).astype(int)
        own_chunks.append(np.unique(np.stack([r, c], 1).clip(0, cw - 1), axis=0).astype(np.int32))
    out = open(args.out, "w") if args.out else None
    for m in sizes:
        chunks = [own_chunks[0], own_chunks[1]]
        reqs = [(0, capi.TARGET_ENEMIES, UNITS, UNITS), (1, capi.TARGET_ENEMIES, 0, UNITS)]     # enemy seek: the other faction
        targets = rng.integers(0, 2 * UNITS, m)
        for k, t in enumerate(targets):
            tr, tc = int(fp["z"][t] // 256), int(-fp["x"][t] // 256)
            box = [(r, c) for r in range(tr - 1, tr + 2) for c in range(tc - 1, tc + 2) if 0 <= r < cw and 0 <= c < cw]
            chunks.append(np.array(box, np.int32))
            reqs.append((2 + k, capi.TARGET_ENTITY, int(t), 1))
        rec = np.zeros(len(reqs), capi.ENTITY_FIELD_REQ)
        coff = np.cumsum([0] + [len(c) for c in chunks])
        for i, (d, kind, e0, en) in enumerate(reqs):
            rec[i] = (d, 0, 0, kind, e0, en, coff[i], len(chunks[i]))
        allch = np.concatenate(chunks)
        ts, tb = [], []
        for rep in range(args.reps + 1):
            serial.pool_clear(); batch.pool_clear()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for i, (d, kind, e0, en) in enumerate(reqs):
                serial.pool_request_entity_fields(d, kind, fp[e0:e0 + en], chunks[i])
            torch.cuda.synchronize()
            a = time.perf_counter() - t0
            t0 = time.perf_counter()
            done = batch.pool_request_entity_fields_batch(rec, fp, allch)
            torch.cuda.synchronize()
            b = time.perf_counter() - t0
            assert done == len(reqs)
            if rep:
                ts.append(a); tb.append(b)
        keys = sorted({(d, int(r) * cw + int(c)) for i, (d, _, _, _) in enumerate(reqs) for r, c in chunks[i]})
        same = all(_entry(serial, d, c, cw) == _entry(batch, d, c, cw) for d, c in keys)
        assert same, "the batch and the serial loop left different pools"
        line = json.dumps({"map": "C2", "m_surround": m, "requests": len(reqs), "fields": int(len(allch)),
                           "footprints": int(len(fp)), "reps": args.reps, "serial_ms": 1e3 * statistics.median(ts),
                           "batch_ms": 1e3 * statistics.median(tb), "speedup": statistics.median(ts) / statistics.median(tb),
                           "identical_pool": bool(same), "pool_entries_compared": len(keys), "gpu": gpu})
        print(line, flush=True)
        if out:
            out.write(line + "\n"); out.flush()
    for nav in navs:
        nav.close()


def _entry(nav, d, c, cw):
    f, _, ffid = nav.pool_get(d, divmod(c, cw))
    return (ffid, None if f is None else f.tobytes())


if __name__ == "__main__":
    main()
