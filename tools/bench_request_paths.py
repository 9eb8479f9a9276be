#!/usr/bin/env python
"""pfnav_pool_request_paths (one batch) against pfnav_pool_request_path in a loop, on the C2 map (16 x 16 chunks).

For N seeded requests (sources on passable tiles) over 16, 64 or N distinct destinations, each repetition clears both
pools, then times the serial loop on one context and the batch on another, alternating, each window ending in a device
synchronise. One warm-up repetition, then the median of --reps. After the last repetition the per-request results must
be identical and the two pools identical: every (dest, chunk) entry when there are at most 64 destinations, a seeded
sample of 4096 entries otherwise.  python tools/bench_request_paths.py [--reps 5] [--sizes 1,4,...] [--out FILE]"""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--sizes", default="1,4,16,64,256,1024,4096")
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
    chunks = cw * cw
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, bench.MAP_SEED, rivers=True), cw, cw)
    sizes = [int(s) for s in args.sizes.split(",")]
    maxd = max(sizes)
    navs = []
    for _ in range(2):
        nav = capi.Nav(0)
        nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
        nav.pool_create(maxd, 65536)
        navs.append(nav)
    serial, batch = navs
    g = cost.reshape(cw, cw, 64, 64).transpose(0, 2, 1, 3).reshape(cw * 64, cw * 64)
    passable = np.argwhere(g != 255)
    world = lambda t: np.stack([-(t[:, 1] * 4.0 + 2.0), t[:, 0] * 4.0 + 2.0], 1).astype(np.float32)
    out = open(args.out, "w") if args.out else None

    def run_serial(d, s, t):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = [serial.pool_request_path(int(d[i]), tuple(s[i]), tuple(t[i])) for i in range(len(d))]
        torch.cuda.synchronize()
        return time.perf_counter() - t0, res

    def run_batch(d, s, t):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        res = batch.pool_request_paths(d, s, t)
        torch.cuda.synchronize()
        return time.perf_counter() - t0, res

    for n in sizes:
        for nd in sorted({min(16, n), min(64, n), n}):
            rng = np.random.default_rng(1000 * n + nd)
            targets = passable[rng.integers(0, len(passable), nd)]
            dests = (np.arange(n) if nd == n else rng.integers(0, nd, n)).astype(np.int32)
            src = world(passable[rng.integers(0, len(passable), n)])
            dst = world(targets[dests])
            ts, tb = [], []
            for rep in range(args.reps + 1):
                serial.pool_clear(); batch.pool_clear()
                a, rs = run_serial(dests, src, dst)
                b, rb = run_batch(dests, src, dst)
                if rep:
                    ts.append(a); tb.append(b)
            ok, did, nf, nl, done = rb
            same_req = done == n and all((bool(ok[i]), int(did[i]), int(nf[i]), int(nl[i])) == tuple(rs[i]) for i in range(n))
            keys = [(d, c) for d in range(nd) for c in range(chunks)] if nd <= 64 else \
                [(int(k) // chunks, int(k) % chunks) for k in np.random.default_rng(n).choice(nd * chunks, 4096, replace=False)]
            same_pool = all(_entry(serial, d, c, cw) == _entry(batch, d, c, cw) for d, c in keys)
            rec = {"map": "C2", "n": n, "dests": nd, "reps": args.reps, "serial_ms": 1e3 * statistics.median(ts),
                   "batch_ms": 1e3 * statistics.median(tb), "speedup": statistics.median(ts) / statistics.median(tb),
                   "fields": int(nf.sum()), "los": int(nl.sum()), "ok": int(ok.sum()), "identical_requests": bool(same_req),
                   "identical_pool": bool(same_pool), "pool_entries_compared": len(keys), "gpu": gpu}
            line = json.dumps(rec)
            print(line, flush=True)
            if out:
                out.write(line + "\n"); out.flush()
    for nav in navs:
        nav.close()


def _entry(nav, d, c, cw):
    f, l, ffid = nav.pool_get(d, divmod(c, cw))
    return (ffid, None if f is None else f.tobytes(), None if l is None else l.tobytes())


if __name__ == "__main__":
    main()
