"""Host-observed time of one tick's population change in an in-process multi-GPU group, two arms alternated:

  job       pfnav_group_change_population (k removals + k additions) + pfnav_group_gather
            + pfnav_agents_set_work_dev on every member
  reupload  pfnav_agents_read_state + pfnav_agents_read_blocking of every member's range + the same deletions and appends
            in numpy + pfnav_agents_upload_shard + pfnav_agents_upload_movestate + pfnav_agents_upload_blocking of every
            member's new range + pfnav_group_gather (flock column all-gather and host member rebuild)
            + pfnav_agents_set_work(NULL) on every member      (the only way in before the job call)

at the benchmark's C2 (100 000 entities) and C3 (1 000 000) populations, with 2 and 3 members on device 0 and
k = 1, 100 and 10 000 per tick: k random uids die and k copies of other entities are appended, so the population keeps
its size. Every member holds a movestate and a blocking table and the groups share blockers. A host clock around work
that ends in a device synchronise; warm-up, then the median of --runs runs with min / max. These are end-to-end call
times, not kernel shares of peak. Members on separate devices are not measured here. The card's name and power limit
are read in the same process and written beside the numbers: results/h100_sxm_<power>w/mgpu_population.jsonl. There is
no CPU arm: without a GPU the contexts cannot be created."""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_agent_population import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default="C2,C3")
    ap.add_argument("--worlds", default="2,3")
    ap.add_argument("--out", default=None, help="the .jsonl to append to (default results/h100_sxm_<power>w/mgpu_population.jsonl)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mgpu_population.py needs a GPU: there is no CPU arm")
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench = importlib.import_module("bench")
    name, power = card()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    out = args.out or os.path.join(ROOT, "results", cardname, "mgpu_population.jsonl")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    rows = []
    for wl in args.workloads.split(","):
        bench.set_workload(wl)
        W = bench.build_workload(pf, 1, 0)
        rec, fl, n = W["rec"], W["flocks"], W["n_total"]
        ms = np.zeros(n, capi.MOVESTATE)
        ms["next_rot"][:, 3] = 1.0
        blk = np.zeros(n, capi.BLOCKING)
        blk["faction_id"] = capi.FACTION_ID_NONE
        for world in [int(w) for w in args.worlds.split(",")]:
            arms = {}
            for arm in ("job", "reupload"):
                navs = [capi.Nav(0) for _ in range(world)]
                for X in navs:
                    X.map_create(bench.CHUNKS, bench.CHUNKS, 1); X.map_upload_layer(0, W["cost"])
                g = capi.Group(navs)
                g.share_blockers()
                for r, X in enumerate(navs):
                    lo, hi = capi.mgpu_shard_range(n, r, world)
                    X.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, bench.HZ)
                g.gather()
                for r, X in enumerate(navs):
                    lo, hi = capi.mgpu_shard_range(n, r, world)
                    X.agents_upload_movestate(ms[lo:hi]); X.agents_upload_blocking(blk[lo:hi])
                arms[arm] = (navs, g)
            rng = np.random.default_rng(1)

            def read(navs):
                parts = [X.agents_read_state(hi - lo) for X, (lo, hi) in
                         zip(navs, [capi.mgpu_shard_range(n, r, world) for r in range(world)])]
                return np.concatenate([p[0] for p in parts]), np.concatenate([p[1] for p in parts])

            for k in (1, 100, 10_000):
                t = {"job": [], "reupload": []}
                for it in range(args.warmup + args.runs):
                    rm = rng.choice(n, k, replace=False)
                    src = rng.choice(n, k, replace=False)
                    sa, sm = read(arms["job"][0])
                    add, add_ms, add_blk = sa[src].copy(), sm[src].copy(), blk[:k].copy()
                    for arm in ("job", "reupload"):
                        navs, g = arms[arm]
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        if arm == "job":
                            g.change_population(rm, add, ms=add_ms, blocking=add_blk)
                            g.gather()
                            for X in navs:
                                X.agents_set_work_dev()
                        else:
                            ranges = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
                            parts = [X.agents_read_state(hi - lo) for X, (lo, hi) in zip(navs, ranges)]
                            b = np.concatenate([X.agents_read_blocking(hi - lo) for X, (lo, hi) in zip(navs, ranges)])
                            a = np.concatenate([np.delete(np.concatenate([p[0] for p in parts]), rm), add])
                            m = np.concatenate([np.delete(np.concatenate([p[1] for p in parts]), rm), add_ms])
                            b = np.concatenate([np.delete(b, rm), add_blk])
                            for r, X in enumerate(navs):
                                lo, hi = capi.mgpu_shard_range(len(a), r, world)
                                X.agents_upload_shard(a[lo:hi], lo, hi, len(a), fl, bench.HZ)
                            g.gather()
                            for r, X in enumerate(navs):
                                lo, hi = capi.mgpu_shard_range(len(a), r, world)
                                X.agents_upload_movestate(m[lo:hi]); X.agents_upload_blocking(b[lo:hi])
                                X.agents_set_work(None)
                        torch.cuda.synchronize()
                        if it >= args.warmup:
                            t[arm].append((time.perf_counter() - t0) * 1e3)
                sj, sr = read(arms["job"][0]), read(arms["reupload"][0])
                assert sj[0].tobytes() == sr[0].tobytes() and sj[1].tobytes() == sr[1].tobytes()
                row = {"workload": wl, "entities": n, "members": world, "devices": 1, "removed_and_added_per_tick": k,
                       "runs": args.runs, "card": name, "power_limit_w": power,
                       "what": "host-observed ms per job population change + gather + work lists, ending in a device synchronise"}
                for arm in t:
                    row[arm + "_ms"] = {"median": float(np.median(t[arm])), "min": float(min(t[arm])), "max": float(max(t[arm]))}
                rows.append(row)
                print(json.dumps(row), flush=True)
            for navs, g in arms.values():
                g.close()
                for X in navs:
                    X.close()
    with open(out, "a") as f:
        for row in rows:
            f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
