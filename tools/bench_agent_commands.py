"""Host-observed time of one tick's command step on a device-resident population, two arms alternated:

  commands  pfnav_agents_commands (deltas) + pfnav_agents_rebuild_index + pfnav_agents_set_work_dev
  reupload  pfnav_agents_read_state + the same edits in numpy + pfnav_agents_upload + pfnav_agents_upload_movestate
            + pfnav_agents_set_work(NULL)          (the only way in before pfnav_agents_commands)

at the benchmark's C2 (100 000 entities) and C3 (1 000 000) populations with 0, 100 and 10 000 orders per tick (half
stops, half move orders into another flock). A host clock around work that ends in a device synchronise; warm-up, then
the median of --runs runs with min / max. These are end-to-end call times, not kernel shares of peak. The card's name
and power limit are read in the same process and written beside the numbers:
results/h100_sxm_<power>w/agent_commands.jsonl. There is no CPU arm: without a GPU the context cannot be created."""
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         check=True, capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, float(power)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default="C2,C3")
    ap.add_argument("--out", default=None, help="the .jsonl to append to (default results/h100_sxm_<power>w/agent_commands.jsonl)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_agent_commands.py needs a GPU: there is no CPU arm")
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench = importlib.import_module("bench")
    import commands_ref as cr
    name, power = card()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    out = args.out or os.path.join(ROOT, "results", cardname, "agent_commands.jsonl")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    rows = []
    for wl in args.workloads.split(","):
        bench.set_workload(wl)
        W = bench.build_workload(pf, 1, 0)
        rec, fl, n = W["rec"], W["flocks"], W["n_total"]
        ms = np.zeros(n, capi.MOVESTATE)
        ms["next_rot"][:, 3] = 1.0
        navs = {}
        for arm in ("commands", "reupload"):
            X = capi.Nav(0)
            X.map_create(bench.CHUNKS, bench.CHUNKS, 1); X.map_upload_layer(0, W["cost"])
            X.agents_upload(rec, fl, bench.HZ); X.agents_upload_movestate(ms)
            navs[arm] = X
        rng = np.random.default_rng(1)
        for ncmd in (0, 100, 10_000):
            t = {"commands": [], "reupload": []}
            nwork = {}
            for it in range(args.warmup + args.runs):
                who = rng.choice(n, ncmd, replace=False)
                d = np.concatenate([cr.deltas(who[:ncmd // 2], state=2, velocity=(0.0, 0.0)),
                                    cr.deltas(who[ncmd // 2:], state=0, flock=rng.integers(0, len(fl), ncmd - ncmd // 2), clear_hist=True)])
                for arm in ("commands", "reupload"):
                    X = navs[arm]
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if arm == "commands":
                        X.agents_commands(d)
                        X.agents_rebuild_index()
                        nwork[arm] = X.agents_set_work_dev()
                    else:
                        sa, sm = X.agents_read_state(n)
                        cr.apply_deltas_np(d, sa, sm)
                        X.agents_upload(sa, fl, bench.HZ)
                        X.agents_upload_movestate(sm)
                        X.agents_set_work(None)
                    torch.cuda.synchronize()
                    if it >= args.warmup:
                        t[arm].append((time.perf_counter() - t0) * 1e3)
                    if arm == "reupload":
                        nwork[arm] = len(X.agents_read_work())          # outside the window: a check, not part of the arm
                assert nwork["commands"] == nwork["reupload"], nwork
            row = {"workload": wl, "entities": n, "commands_per_tick": ncmd, "runs": args.runs, "card": name, "power_limit_w": power,
                   "what": "host-observed ms per command step, ending in a device synchronise"}
            for arm in t:
                row[arm + "_ms"] = {"median": float(np.median(t[arm])), "min": float(min(t[arm])), "max": float(max(t[arm]))}
            rows.append(row)
            print(json.dumps(row), flush=True)
        for X in navs.values():
            X.close()
    with open(out, "a") as f:
        for row in rows:
            f.write(json.dumps(row) + "\n")


if __name__ == "__main__":
    main()
