"""Host-observed time of one tick's population change on a device-resident population, two arms alternated:

  change    pfnav_agents_change_population (k removals + k additions) + pfnav_agents_set_work_dev
  reupload  pfnav_agents_read_state + pfnav_agents_read_blocking + the same deletions and appends in numpy
            + pfnav_agents_upload + pfnav_agents_upload_movestate + pfnav_agents_upload_blocking
            + pfnav_agents_set_work(NULL)          (the only way in before pfnav_agents_change_population)

at the benchmark's C2 (100 000 entities) and C3 (1 000 000) populations with k = 1, 100 and 10 000 per tick: k random
uids die and k copies of other entities are appended, so the population keeps its size. Both contexts hold a movestate
and a blocking table. A host clock around work that ends in a device synchronise; warm-up, then the median of --runs
runs with min / max. These are end-to-end call times, not kernel shares of peak. The card's name and power limit are
read in the same process and written beside the numbers: results/h100_sxm_<power>w/agent_population.jsonl. There is no
CPU arm: without a GPU the context cannot be created."""
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
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         check=True, capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, float(power)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--workloads", default="C2,C3")
    ap.add_argument("--out", default=None, help="the .jsonl to append to (default results/h100_sxm_<power>w/agent_population.jsonl)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_agent_population.py needs a GPU: there is no CPU arm")
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench = importlib.import_module("bench")
    name, power = card()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    out = args.out or os.path.join(ROOT, "results", cardname, "agent_population.jsonl")
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
        navs = {}
        for arm in ("change", "reupload"):
            X = capi.Nav(0)
            X.map_create(bench.CHUNKS, bench.CHUNKS, 1); X.map_upload_layer(0, W["cost"])
            X.agents_upload(rec, fl, bench.HZ); X.agents_upload_movestate(ms); X.agents_upload_blocking(blk)
            navs[arm] = X
        rng = np.random.default_rng(1)
        for k in (1, 100, 10_000):
            t = {"change": [], "reupload": []}
            nwork = {}
            for it in range(args.warmup + args.runs):
                rm = rng.choice(n, k, replace=False)
                src = rng.choice(n, k, replace=False)
                # the appended records are taken from the population before the call; both arms hold the same one
                sa, sm = navs["change"].agents_read_state(n)
                add, add_ms, add_blk = sa[src].copy(), sm[src].copy(), blk[:k].copy()
                for arm in ("change", "reupload"):
                    X = navs[arm]
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    if arm == "change":
                        X.agents_change_population(rm, add, ms=add_ms, blocking=add_blk)
                        nwork[arm] = X.agents_set_work_dev()
                    else:
                        a, m = X.agents_read_state(n)
                        b = X.agents_read_blocking(n)
                        X.agents_upload(np.concatenate([np.delete(a, rm), add]), fl, bench.HZ)
                        X.agents_upload_movestate(np.concatenate([np.delete(m, rm), add_ms]))
                        X.agents_upload_blocking(np.concatenate([np.delete(b, rm), add_blk]))
                        X.agents_set_work(None)
                    torch.cuda.synchronize()
                    if it >= args.warmup:
                        t[arm].append((time.perf_counter() - t0) * 1e3)
                    if arm == "reupload":
                        nwork[arm] = len(X.agents_read_work())          # outside the window: a check, not part of the arm
                assert nwork["change"] == nwork["reupload"], nwork
            sa = navs["change"].agents_read_state(n)[0]
            sb = navs["reupload"].agents_read_state(n)[0]
            assert sa.tobytes() == sb.tobytes()
            row = {"workload": wl, "entities": n, "removed_and_added_per_tick": k, "runs": args.runs, "card": name,
                   "power_limit_w": power, "what": "host-observed ms per population change, ending in a device synchronise"}
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
