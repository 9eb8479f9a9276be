"""pfnav_pool_repair_batch against pfnav_pool_repair (the serial on-miss chain) on the C5 map and population of bench.py.

Two contexts are built identically (map, churned obstacles, goals, 62 500 agents). Every step moves the 1 000 obstacles on
both, commits, re-requests what the commit invalidated (REQUEST_MISSING_ONLY) and ticks; then the serial loop runs on one
context and the batch on the other, in alternating order, each timed by the host clock (both end in a device
synchronise). After every step the pools must be equal entry for entry. One warm-up step, then --reps timed steps.
Writes one JSON line per step, plus a summary line, to results/<card>/pool_repair_C5.jsonl.

    python tools/bench_pool_repair.py [--churn K] [--reps 5] [--out results]
"""
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


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0].split(",")
    return q[0].strip(), float(q[1])


def pool_equal(navs, ndests, chunks):
    for d in range(ndests):
        for c in range(chunks * chunks):
            a, b = (nav.pool_get(d, divmod(c, chunks)) for nav in navs)
            if a[2] != b[2] or (a[0] is None) != (b[0] is None) or (a[1] is None) != (b[1] is None):
                return False
            if a[0] is not None and not (a[0] == b[0]).all():
                return False
            if a[1] is not None and not (a[1] == b[1]).all():
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--churn", type=int, default=3, help="churn steps before the first measured step")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "results"))
    args = ap.parse_args()
    bench = importlib.import_module("bench")
    bench.set_workload("C5")
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    name, power = card()
    W = bench.build_workload(pf, 1, 0)
    C = bench.CHUNKS
    ngoals = W["g_hi"] - W["g_lo"]
    goals = np.array([[int(v) for v in W["agents"]["flock_target_tile"][f]] for f in range(W["g_lo"], W["g_hi"])], np.int32)
    dests = np.arange(ngoals, dtype=np.int32)
    navs, churns = [], []
    for _ in range(2):
        nav = capi.Nav(0)
        nav.map_create(C, C, 1)
        nav.map_upload_layer(0, W["cost"])
        nav.map_build_nav(0)
        nav.route_build(0)
        ch = bench.Churn(W["agents"], bench.WORKLOADS["C5"]["blockers"], C, bench.MAP_SEED + 77)
        ch.place(nav, capi)
        nav.map_commit()
        nav.pool_create(ngoals, ngoals * C * C)
        nav.agents_upload(W["rec"], W["flocks"], bench.HZ)
        nav.agents_set_work(np.arange(W["lo"], W["hi"], dtype=np.uint32))
        nav.pool_request_goals(dests, goals, 0)
        navs.append(nav); churns.append(ch)

    def churn_step():
        for nav, ch in zip(navs, churns):
            ch.move(nav, capi)
            nav.map_commit()
            nav.pool_request_goals(dests, goals, 0, 0, capi.REQUEST_MISSING_ONLY)
            nav.agents_tick(capi.TICK_VDES_FROM_POOL)

    for _ in range(args.churn):
        churn_step()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    path = os.path.join(args.out, cardname, "pool_repair_C5.jsonl")
    os.makedirs(os.path.dirname(path), exist_ok=True)
    rows, serial_ms, batch_ms, all_equal = [], [], [], True
    for rep in range(args.reps + 1):
        churn_step()
        order = (0, 1) if rep % 2 == 0 else (1, 0)
        res = {}
        for which in order:
            t0 = time.perf_counter()
            out = navs[0].pool_repair() if which == 0 else navs[1].pool_repair_batch()
            res[which] = (out, (time.perf_counter() - t0) * 1e3)
        equal = pool_equal(navs, ngoals, C) and res[0][0] == res[1][0][:2]
        all_equal &= equal
        row = dict(step=rep, warmup=rep == 0, card=name, power_limit_w=power, reps_per_phase=navs[1].pool_repair_batch_stats()[0], rounds_ended_by_rule=navs[1].pool_repair_batch_stats()[1],
                   nrequests=res[1][0][0], nrepairs=res[1][0][1], nrounds=res[1][0][2], serial_ms=res[0][1], batch_ms=res[1][1],
                   serial_counts=list(res[0][0]), pools_equal=bool(equal))
        rows.append(row)
        if rep > 0:
            serial_ms.append(res[0][1]); batch_ms.append(res[1][1])
        print(json.dumps(row), flush=True)
    summary = dict(summary=True, card=name, power_limit_w=power, workload="C5", churn_before=args.churn, reps=args.reps,
                   serial_ms_median=float(np.median(serial_ms)), batch_ms_median=float(np.median(batch_ms)),
                   pools_equal=bool(all_equal))
    print(json.dumps(summary), flush=True)
    with open(path, "w") as f:
        for r in rows + [summary]:
            f.write(json.dumps(r) + "\n")
    for nav in navs:
        nav.close()
    return 0 if all_equal else 1


if __name__ == "__main__":
    sys.exit(main())
