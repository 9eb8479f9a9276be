#!/usr/bin/env python
"""Host-observed time of G_Pos_EntsInCircle queries answered by the device position index, on the bench's populations:

    batch   pfnav_ents_in_circles with n uid-centred queries (n in --sizes) on C2 (100 000 entities, 16 x 16 chunks), at
            each range of --ranges and each maxout of --maxouts; the centres are the first n entities of a seeded
            permutation
    loop    the same n queries as a loop of pfnav_ents_in_circle at the entities' positions (n <= --loop-max), whose
            answers are checked equal to the batch's
    c3      one batch of one query per entity of C3 (1 000 000 entities), r = 10, maxout 512

Each figure ends in the call's own stream synchronise. 2 warm-up calls, then --reps timed calls: median, min and max. The
card's name, power limit and maximum SM clock are read in the same run and written into every JSON line.
    python tools/bench_ents_query.py [--reps 7] [--out FILE]"""
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
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--sizes", default="1,64,4096,100000")
    ap.add_argument("--ranges", default="10,30,100")
    ap.add_argument("--maxouts", default="128,512")
    ap.add_argument("--loop-max", type=int, default=4096)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    out = open(args.out, "w") if args.out else None

    def timed(fn):
        for _ in range(2):
            fn()
        ts = []
        for _ in range(args.reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            ts.append(1e3 * (time.perf_counter() - t0))
        return statistics.median(ts), min(ts), max(ts)

    def report(**kw):
        line = json.dumps(dict(kw, reps=args.reps, gpu=gpu))
        print(line, flush=True)
        if out:
            out.write(line + "\n"); out.flush()

    def population(workload):
        bench.set_workload(workload)
        W = bench.build_workload(pf, 1, 0)
        bench.set_workload("C2")
        rec, fl = capi.pack_agents(W["agents"])
        nav = capi.Nav(0)
        nav.map_create(bench.CHUNKS, bench.CHUNKS, 1); nav.map_upload_layer(0, W["cost"])
        nav.agents_upload(rec, fl, 20)
        return nav, rec

    nav, rec = population("C2")
    order = np.random.default_rng(0).permutation(len(rec)).astype(np.uint32)
    for n in [int(s) for s in args.sizes.split(",")]:
        for r in [float(s) for s in args.ranges.split(",")]:
            for m in [int(s) for s in args.maxouts.split(",")]:
                q = np.zeros(n, capi.ENTS_QUERY)
                q["uid"], q["range"], q["maxout"] = order[:n], r, m
                off, ids = nav.ents_in_circles(q)
                cap = len(ids)
                med, lo, hi = timed(lambda: nav.ents_in_circles(q, cap=cap))
                report(workload="C2", kind="batch", n=n, range=r, maxout=m, hits=int(off[-1]), median_ms=med, min_ms=lo, max_ms=hi)
                if n <= args.loop_max:
                    pos = rec["pos"][order[:n]]
                    loop = lambda: [nav.ents_in_circle(float(x), float(z), r, m) for x, z in pos]
                    got = loop()
                    assert all(np.array_equal(got[i], ids[off[i]:off[i + 1]]) for i in range(n)), (n, r, m)
                    med, lo, hi = timed(loop)
                    report(workload="C2", kind="loop", n=n, range=r, maxout=m, hits=int(off[-1]), median_ms=med, min_ms=lo, max_ms=hi)
    nav.close()

    nav, rec = population("C3")
    q = np.zeros(len(rec), capi.ENTS_QUERY)
    q["uid"], q["range"], q["maxout"] = np.arange(len(rec), dtype=np.uint32), 10.0, 512
    off, ids = nav.ents_in_circles(q)
    cap = len(ids)
    med, lo, hi = timed(lambda: nav.ents_in_circles(q, cap=cap))
    report(workload="C3", kind="batch", n=len(q), range=10.0, maxout=512, hits=int(off[-1]), median_ms=med, min_ms=lo, max_ms=hi)
    nav.close()


if __name__ == "__main__":
    main()
