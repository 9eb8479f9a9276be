"""Host-observed time of saving and restoring the field pool (pfnav_pool_save / pfnav_pool_restore) at the benchmark's C2
workload (100 000 entities, 16 goals, a 16 x 16-chunk map, a pool of 16 x 256 fields), against the resume path without
it. The saving context runs a cold goal batch and --ticks ticks whose misses are served (pfnav_pool_repair_batch), then:

  save              pfnav_pool_save of the whole pool (map digest, device pack and one copy back; returns filled)
  restore           pfnav_pool_restore of that segment on a second context with the same map and population
  restore+tick      restore, then the first tick of the loop: agents_tick, the repair rounds, agents_tick
  rerequest+tick    the resume path without a pool restore: pfnav_pool_clear, the goals requested again
                    (pfnav_pool_request_goals), then the same first tick, whose repair rounds rebuild what the goal
                    batch does not (the path fields of misses)

A host clock around work that ends in a device synchronise; warm-up, then the median of --runs runs with min / max, the
restore and re-request arms alternated. These are end-to-end call times, not kernel shares of peak. The card's name and
power limit are read in the same process and written beside the numbers (default
results/h100_sxm_<power>w/pool_checkpoint.jsonl). There is no CPU arm: without a GPU the context cannot be created."""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_checkpoint import card, stats  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ticks", type=int, default=3, help="ticks with misses served before the save")
    ap.add_argument("--out", default=None, help="the .jsonl to append to (default results/h100_sxm_<power>w/pool_checkpoint.jsonl)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_pool_checkpoint.py needs a GPU: there is no CPU arm")
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench = importlib.import_module("bench")
    name, power = card()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    out = args.out or os.path.join(ROOT, "results", cardname, "pool_checkpoint.jsonl")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)

    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    rec, fl, n, cost = W["rec"], W["flocks"], W["n_total"], W["cost"]
    ng = W["g_hi"] - W["g_lo"]
    dests = np.arange(ng, dtype=np.int32)
    targets = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(W["g_lo"], W["g_hi"])], np.int32)
    work = np.arange(n, dtype=np.uint32)

    def ready():
        X = capi.Nav(0)
        X.map_create(bench.CHUNKS, bench.CHUNKS, 1)
        X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
        X.pool_create(ng, ng * bench.CHUNKS * bench.CHUNKS)
        X.agents_upload(rec, fl, bench.HZ)
        X.agents_rebuild_index()
        X.agents_set_work(work)
        return X

    def first_tick(X):
        X.agents_tick(capi.TICK_VDES_FROM_POOL)
        X.pool_repair_batch()
        X.agents_tick(capi.TICK_VDES_FROM_POOL)
        torch.cuda.synchronize()

    S = ready()
    S.pool_request_goals(dests, targets, 0)
    for _ in range(args.ticks):
        first_tick(S)
    seg = S.pool_save()
    h = np.frombuffer(seg[:64], np.uint32)
    used, nstored = int(h[6]), int(h[12])
    R = ready()
    t_save, t_rest, t_rt, t_rq = [], [], [], []
    for r in range(args.warmup + args.runs):
        t0 = time.perf_counter(); s2 = S.pool_save(); t1 = time.perf_counter()
        assert s2 == seg
        t2 = time.perf_counter(); R.pool_restore(seg); t3 = time.perf_counter()
        arms = [("restore", lambda: (R.pool_restore(seg), first_tick(R))),
                ("rerequest", lambda: (R.pool_clear(), R.pool_request_goals(dests, targets, 0), first_tick(R)))]
        if r % 2:
            arms.reverse()
        got = {}
        for arm, fn in arms:
            torch.cuda.synchronize()
            a = time.perf_counter(); fn(); b = time.perf_counter()
            got[arm] = (b - a) * 1e3
        if r >= args.warmup:
            t_save.append((t1 - t0) * 1e3); t_rest.append((t3 - t2) * 1e3)
            t_rt.append(got["restore"]); t_rq.append(got["rerequest"])
    S.close(); R.close()
    common = dict(workload="C2", n=n, goals=ng, max_fields=ng * bench.CHUNKS * bench.CHUNKS, used=used, stored=nstored,
                  bytes=len(seg), ticks_before_save=args.ticks)
    rows = [dict(arm="save", **common, **stats(t_save)),
            dict(arm="restore", **common, **stats(t_rest)),
            dict(arm="restore+first tick", **common, **stats(t_rt)),
            dict(arm="clear+request goals+first tick", **common, **stats(t_rq))]
    with open(out, "a") as f:
        for row in rows:
            row.update(card=name, power_limit_w=power, runs=args.runs)
            f.write(json.dumps(row) + "\n")
            print(json.dumps(row))


if __name__ == "__main__":
    main()
