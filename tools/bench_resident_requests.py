#!/usr/bin/env python
"""Path requests, map queries and group-arrival velocities for resident entities: pfnav_pool_request_paths_resident,
pfnav_map_query_resident and pfnav_group_arrival_velocity_resident against the path an engine without host positions
takes today -- pfnav_agents_read_state, the positions substituted in numpy, then the plain entry point -- on the C2 map
(16 x 16 chunks) with the C2 (100 000) and C3 (1 000 000) populations.

The entities stand on passable tiles. Per population, call kind and size (1, 64 and 4096 requests or queries; the
group arrival also takes a whole arriving flock of 10 000 uids), both arms run on two contexts holding the same
population and the same pool: path sources are random uids, destinations points next to 48 goals (the pool warms up
over the warm-up repetitions, identically on both); map queries mix CLOSEST_PATHABLE, DEST_ID and PATHABLE at uids;
arrival velocities are asked against a zone field. Each repetition times one arm and then the other, alternating which
goes first, each window a host clock around work that ends in a device synchronise. --warmup repetitions, then median,
min and max of --reps. The two arms' outputs must be identical. The card's name and power limit are read in the same
run and written with every line.
    python tools/bench_resident_requests.py [--reps 7] [--warmup 2] [--out FILE]
FILE defaults to results/<card>/resident_requests.jsonl."""
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
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import bench  # noqa: E402

NDESTS, ZONE_DEST, FLOCK = 48, 47, 10000
SIZES = (1, 64, 4096)


def card_dir(name, power):
    """results/<card>: h100_sxm_<W>w for an H100 SXM (HBM3), else the name in lower case"""
    watts = int(round(float(power.split()[0])))
    if "H100" in name and "HBM3" in name:
        return "h100_sxm_%dw" % watts
    return "%s_%dw" % ("".join(ch if ch.isalnum() else "_" for ch in name.lower()).strip("_"), watts)


def population(capi, synth, cost, cw, n, seed):
    rng = np.random.default_rng(seed)
    img = synth.blocked_to_image(cost, cw, cw)
    t = np.argwhere(img != 255)
    t = t[rng.integers(0, len(t), n)]
    pos = np.stack([-(t[:, 1] + rng.uniform(0.05, 0.95, n)) * 4.0, (t[:, 0] + rng.uniform(0.05, 0.95, n)) * 4.0], 1)
    rec = np.zeros(n, capi.AGENT)
    rec["pos"] = pos.astype(np.float32); rec["prev_pos"] = rec["pos"]
    rec["radius"] = 1.0; rec["max_speed"] = 20.0; rec["speed"] = 20.0; rec["flags"] = capi.FLAG_MOVABLE; rec["flock"] = -1
    fl = np.zeros(1, capi.FLOCK); fl["dest"] = -1
    return rec, fl, t


def substitute(nav, n, uids, given):
    pos = nav.agents_read_state(n, False)[0]["pos"]
    out = np.zeros((len(uids), 2), np.float32) if given is None else given.copy()
    named = uids != 0xFFFFFFFF
    out[named] = pos[uids[named]]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    ap.add_argument("--workloads", default="C2,C3")
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    pf = importlib.import_module("permafrost-engine_b200")
    capi, synth = pf.capi, pf.synth
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power = [s.strip() for s in gpu.split(",")]
    print("gpu:", gpu, flush=True)
    out_path = args.out or os.path.join(ROOT, "results", card_dir(name, power), "resident_requests.jsonl")
    os.makedirs(os.path.dirname(os.path.abspath(out_path)), exist_ok=True)
    lines = []
    bench.set_workload("C2")
    cw = bench.CHUNKS
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, bench.MAP_SEED, rivers=True), cw, cw)
    for wl in args.workloads.split(","):
        n = bench.WORKLOADS[wl]["agents"]
        rec, fl, tiles = population(capi, synth, cost, cw, n, 0x5EED + n)
        navs = []
        for _ in range(2):
            nav = capi.Nav(0)
            nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
            nav.pool_create(NDESTS, NDESTS * cw * cw)
            nav.agents_upload(rec, fl, 20)
            navs.append(nav)
        host, res = navs
        rng = np.random.default_rng(7)
        goals = tiles[rng.integers(0, len(tiles), NDESTS)]
        goal_xz = np.stack([-(goals[:, 1] + 0.5) * 4.0, (goals[:, 0] + 0.5) * 4.0], 1).astype(np.float32)
        centre = goal_xz[ZONE_DEST]
        for X in navs:
            X.pool_request_zone(ZONE_DEST, centre, 24)
        torch.cuda.synchronize()

        def arms(kind, k):
            uids = rng.choice(n, k, replace=False).astype(np.uint32)
            if kind == "paths":
                dests = rng.integers(0, NDESTS - 1, k).astype(np.int32)
                dst = goal_xz[dests]
                return (lambda: host.pool_request_paths(dests, substitute(host, n, uids, None), dst),
                        lambda: res.pool_request_paths_resident(dests, uids, None, None, dst))
            if kind == "map_query":
                q = np.zeros(k, capi.MAP_QUERY)
                q["kind"] = rng.choice([capi.QUERY_CLOSEST_PATHABLE, capi.QUERY_DEST_ID, capi.QUERY_PATHABLE], k)
                q["faction_id"] = capi.FACTION_ID_NONE

                def plain():
                    qa = q.copy()
                    xz = substitute(host, n, uids, None)
                    qa["x"], qa["z"] = xz[:, 0], xz[:, 1]
                    return host.map_query(qa)
                return plain, lambda: res.map_query_resident(q, uids, None)
            return (lambda: host.group_arrival_velocity(ZONE_DEST, centre, 24, substitute(host, n, uids, None)),
                    lambda: res.group_arrival_velocity_resident(ZONE_DEST, centre, 24, uids))

        cases = [(kind, k) for kind in ("paths", "map_query", "arrival") for k in SIZES] + [("arrival", FLOCK)]
        for kind, k in cases:
            a_plain, a_res = arms(kind, k)
            t = ([], [])
            for rep in range(args.warmup + args.reps):
                got = [None, None]
                for which in ((0, 1) if rep % 2 == 0 else (1, 0)):
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    got[which] = (a_plain, a_res)[which]()
                    torch.cuda.synchronize()
                    if rep >= args.warmup:
                        t[which].append(time.perf_counter() - t0)
                ga, gb = got
                if kind == "map_query":
                    assert ga.tobytes() == gb.tobytes(), (kind, k)
                else:
                    assert all(np.array_equal(x, y) for x, y in zip(ga, gb)), (kind, k)
            ms = lambda v: {"median": 1e3 * statistics.median(v), "min": 1e3 * min(v), "max": 1e3 * max(v)}
            line = json.dumps({"workload": wl, "entities": n, "call": kind, "n": k, "warmup": args.warmup,
                               "reps": args.reps, "read_back_numpy_plain_ms": ms(t[0]), "resident_ms": ms(t[1]),
                               "speedup_median": statistics.median(t[0]) / statistics.median(t[1]), "identical": True,
                               "gpu": name, "power_limit": power})
            print(line, flush=True)
            lines.append(line)
        for nav in navs:
            nav.close()
    with open(out_path, "w") as f:
        f.write("".join(s + "\n" for s in lines))


if __name__ == "__main__":
    main()
