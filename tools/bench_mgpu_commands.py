"""Host-observed time of one tick's command step in a multi-GPU job (an in-process group of 2 or 3 sharded contexts on
one GPU), two arms alternated:

  job       pfnav_group_commands (the job's whole batch of deltas) + pfnav_group_gather + pfnav_agents_set_work_dev on
            every member
  reupload  per member: pfnav_agents_read_state of its range + the same edits in numpy + pfnav_agents_upload_shard
            (without PFNAV_UPLOAD_SAME_FLOCKS) + pfnav_agents_upload_movestate; then pfnav_group_gather (which carries
            the flock column and rebuilds the member lists on the host) + pfnav_agents_set_work(NULL) on every member
            (the only way in before pfnav_group_commands)

at the benchmark's C2 (100 000 entities) and C3 (1 000 000) populations with 0, 100 and 10 000 orders per tick (half
stops, half move orders into another flock). A host clock around work that ends in a device synchronise; warm-up, then
the median of --runs runs with min / max. These are end-to-end call times on ONE GPU (the members share it), not
cross-device numbers and not kernel shares of peak. The card's name and power limit are read in the same process and
written beside the numbers: results/h100_sxm_<power>w/mgpu_commands.jsonl. There is no CPU arm: without a GPU the
contexts cannot be created."""
import argparse
import importlib
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_agent_commands import card


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default="C2,C3")
    ap.add_argument("--worlds", default="2,3")
    ap.add_argument("--out", default=None, help="the .jsonl to append to (default results/h100_sxm_<power>w/mgpu_commands.jsonl)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_mgpu_commands.py needs a GPU: there is no CPU arm")
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench = importlib.import_module("bench")
    import commands_ref as cr
    name, power = card()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    out = args.out or os.path.join(ROOT, "results", cardname, "mgpu_commands.jsonl")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    rows = []
    for wl in args.workloads.split(","):
        bench.set_workload(wl)
        W = bench.build_workload(pf, 1, 0)
        rec, fl, n = W["rec"], W["flocks"], W["n_total"]
        ms = np.zeros(n, capi.MOVESTATE)
        ms["next_rot"][:, 3] = 1.0
        for world in (int(w) for w in args.worlds.split(",")):
            ranges = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
            arms = {}
            for arm in ("job", "reupload"):
                navs = [capi.Nav(0) for _ in range(world)]
                for X in navs:
                    X.map_create(bench.CHUNKS, bench.CHUNKS, 1); X.map_upload_layer(0, W["cost"])
                grp = capi.Group(navs)
                for X, (lo, hi) in zip(navs, ranges):
                    X.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, bench.HZ)
                grp.gather()
                for X, (lo, hi) in zip(navs, ranges):
                    X.agents_upload_movestate(ms[lo:hi])
                arms[arm] = (grp, navs)
            rng = np.random.default_rng(1)
            for ncmd in (0, 100, 10_000):
                t = {"job": [], "reupload": []}
                nwork = {}
                for it in range(args.warmup + args.runs):
                    who = rng.choice(n, ncmd, replace=False)
                    d = np.concatenate([cr.deltas(who[:ncmd // 2], state=2, velocity=(0.0, 0.0)),
                                        cr.deltas(who[ncmd // 2:], state=0, flock=rng.integers(0, len(fl), ncmd - ncmd // 2), clear_hist=True)])
                    for arm in ("job", "reupload"):
                        grp, navs = arms[arm]
                        torch.cuda.synchronize()
                        t0 = time.perf_counter()
                        if arm == "job":
                            grp.commands(d)
                            grp.gather()
                            nwork[arm] = sum(X.agents_set_work_dev() for X in navs)
                        else:
                            for X, (lo, hi) in zip(navs, ranges):
                                sa, sm = X.agents_read_state(hi - lo)
                                sub = d[(d["uid"] >= lo) & (d["uid"] < hi)].copy()
                                sub["uid"] -= lo
                                cr.apply_deltas_np(sub, sa, sm)
                                X.agents_upload_shard(sa, lo, hi, n, fl, bench.HZ)
                                X.agents_upload_movestate(sm)
                            grp.gather()
                            for X in navs:
                                X.agents_set_work(None)
                        torch.cuda.synchronize()
                        if it >= args.warmup:
                            t[arm].append((time.perf_counter() - t0) * 1e3)
                        if arm == "reupload":
                            nwork[arm] = sum(len(X.agents_read_work()) for X in navs)     # outside the window: a check
                    assert nwork["job"] == nwork["reupload"], nwork
                row = {"workload": wl, "entities": n, "members": world, "devices": 1, "commands_per_tick": ncmd, "runs": args.runs,
                       "card": name, "power_limit_w": power,
                       "what": "host-observed ms per command step of the whole group on one GPU, ending in a device synchronise"}
                for arm in t:
                    row[arm + "_ms"] = {"median": float(np.median(t[arm])), "min": float(min(t[arm])), "max": float(max(t[arm]))}
                rows.append(row)
                print(json.dumps(row), flush=True)
            for grp, navs in arms.values():
                grp.close()
                for X in navs:
                    X.close()
    with open(out, "a") as f:
        for row in rows:
            f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
