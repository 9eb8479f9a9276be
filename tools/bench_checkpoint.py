"""Host-observed time of saving and restoring the device-resident population (pfnav_agents_save / pfnav_agents_restore /
pfnav_group_restore) at the benchmark's C2 population (100 000 entities, movestate, movestate_ext, formation and blocking
tables, every tenth unit holding a block):

  save             pfnav_agents_save of one context (the device pack and the one copy back; the call returns filled)
  restore          pfnav_agents_restore of the whole population on a fresh context with the map built, then
                   pfnav_map_commit (which applies the restored blocks): the time until the context can tick again
  group save       pfnav_agents_save on every member of a group of --members contexts on the same device
  group restore    pfnav_group_restore of those segments onto a fresh group, exchange, commit and gather

A host clock around work that ends in a device synchronise (every call above returns after one); warm-up, then the median
of --runs runs with min / max. These are end-to-end call times, not kernel shares of peak. The card's name and power limit
are read in the same process and written beside the numbers (default results/h100_sxm_<power>w/checkpoint.jsonl). There
is no CPU arm: without a GPU the context cannot be created."""
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


def stats(xs):
    xs = sorted(xs)
    return {"median_ms": xs[len(xs) // 2], "min_ms": xs[0], "max_ms": xs[-1]}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--members", type=int, default=2)
    ap.add_argument("--out", default=None, help="the .jsonl to append to (default results/h100_sxm_<power>w/checkpoint.jsonl)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_checkpoint.py needs a GPU: there is no CPU arm")
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench = importlib.import_module("bench")
    name, power = card()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    out = args.out or os.path.join(ROOT, "results", cardname, "checkpoint.jsonl")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)

    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    rec, fl, n, cost = W["rec"], W["flocks"], W["n_total"], W["cost"]
    ms = np.zeros(n, capi.MOVESTATE)
    ms["next_pos"][:, 0], ms["next_pos"][:, 2] = rec["pos"][:, 0], rec["pos"][:, 1]
    ms["step"] = 1.0; ms["next_rot"][:, 3] = 1.0; ms["combat_facing"][:, 3] = 1.0
    ext = np.zeros(n, capi.MOVESTATE_EXT); ext["surround_target_uid"] = capi.NULL_UID; ext["rot"][:, 3] = 1.0
    form = np.zeros(n, capi.FORMATION_IN); form["target_orientation"][:, 3] = 1.0
    blk = np.zeros(n, capi.BLOCKING); blk["faction_id"] = capi.FACTION_ID_NONE
    held = np.arange(0, n, 10)
    blk["blocking"][held] = 1
    blk["stop_x"][held], blk["stop_z"][held] = rec["pos"][held, 0], rec["pos"][held, 1]
    blk["stop_radius"][held] = rec["radius"][held]

    def ready(X):
        X.map_create(bench.CHUNKS, bench.CHUNKS, 1)
        X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)

    def tables(X, lo, hi):
        X.agents_upload_movestate(ms[lo:hi]); X.agents_upload_movestate_ext(ext[lo:hi])
        X.agents_upload_formation(form[lo:hi]); X.agents_upload_blocking(blk[lo:hi])

    rows = []
    # one context
    S = capi.Nav(0); ready(S); S.agents_upload(rec, fl, 20); tables(S, 0, n)
    seg = None
    t_save, t_rest = [], []
    for r in range(args.warmup + args.runs):
        t0 = time.perf_counter(); seg = S.agents_save(); t1 = time.perf_counter()
        R = capi.Nav(0); ready(R)
        t2 = time.perf_counter(); R.agents_restore([seg]); R.map_commit(); t3 = time.perf_counter()
        if r == args.warmup:
            assert R.agents_read_blocking(n).tobytes() == blk.tobytes()
        R.close()
        if r >= args.warmup:
            t_save.append((t1 - t0) * 1e3); t_rest.append((t3 - t2) * 1e3)
    S.close()
    rows.append(dict(arm="save", members=1, n=n, bytes=len(seg), **stats(t_save)))
    rows.append(dict(arm="restore+commit", members=1, n=n, bytes=len(seg), **stats(t_rest)))

    # a group of --members contexts on the same device
    w = args.members
    rg = [capi.mgpu_shard_range(n, r, w) for r in range(w)]
    navs = [capi.Nav(0) for _ in range(w)]
    for X in navs:
        ready(X)
    G = capi.Group(navs); G.share_blockers()
    for X, (lo, hi) in zip(navs, rg):
        X.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, 20)
    G.gather()
    for X, (lo, hi) in zip(navs, rg):
        tables(X, lo, hi)
    t_save, t_rest = [], []
    for r in range(args.warmup + args.runs):
        t0 = time.perf_counter(); segs = [X.agents_save() for X in navs]; t1 = time.perf_counter()
        rn = [capi.Nav(0) for _ in range(w)]
        for X in rn:
            ready(X)
        H = capi.Group(rn); H.share_blockers()
        t2 = time.perf_counter()
        H.restore(segs); H.exchange_blocker_ops()
        for X in rn:
            X.map_commit()
        H.gather()
        t3 = time.perf_counter()
        H.close()
        for X in rn:
            X.close()
        if r >= args.warmup:
            t_save.append((t1 - t0) * 1e3); t_rest.append((t3 - t2) * 1e3)
    G.close()
    for X in navs:
        X.close()
    rows.append(dict(arm="group save", members=w, n=n, bytes=sum(len(s) for s in segs), **stats(t_save)))
    rows.append(dict(arm="group restore+exchange+commit+gather", members=w, n=n, **stats(t_rest)))

    with open(out, "a") as f:
        for row in rows:
            row.update(card=name, power_limit_w=power, workload="C2", runs=args.runs)
            f.write(json.dumps(row) + "\n")
            print(json.dumps(row))


if __name__ == "__main__":
    main()
