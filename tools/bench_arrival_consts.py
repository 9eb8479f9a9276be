#!/usr/bin/env python
"""What arrived()'s map searches cost per tick, and pfnav_map_query's searches that leave the 128 x 128 window: this
tree against another build of the library (--base, e.g. the parent commit's tree with its libpfnav.so built), run
alternately in one invocation, each measurement in a fresh process.

loop: the C2 map (16 x 16 chunks, bench.py's map seed), --agents agents in F flocks (synth.make_agents), every agent a
work item. Each step toggles one committed blocker (pfnav_blockers_incref / decref + pfnav_map_commit, so the map epoch
moves every tick and the arrival constants are rebuilt), then pfnav_agents_tick, pfnav_agents_compute_updates,
pfnav_agents_apply_updates and pfnav_agents_rebuild_index. compute_ms: host clock around the compute_updates call
alone (what the engine's thread pays); step_ms: host clock around the whole step, ending in a device synchronise.
Medians over --steps after --warmup steps. "ext": a movestate_ext table is uploaded and E agents (each of
--enter-counts) are in ENTER_ENTITY_RANGE with a live target and range 0. The agents standing next to impassable terrain
are taken first, as units and as targets, so that the maximally-close search runs for them (an item is searched when its
new tile is next to an impassable or blocked tile); "enter_adjacent" counts those units at upload. Both builds must give
the same patches in the step after the timed ones ("patches_equal", a SHA-256 digest of the patch array).

query: the same map with a 200 x 200 impassable blob carved at its centre and one-tile islands in it; a batch of n
queries, half CLOSEST_PATHABLE from tiles at least 70 tiles inside the blob (they leave the 128 x 128 window) and half
MAXIMALLY_CLOSE towards the one-tile islands (empty lists: they leave every window). batch_ms: host clock around one
pfnav_map_query call (it ends in a stream synchronise), median of --reps after one warm-up call. Both builds must give
the same answers.

Every line also records the card's name and power limit, read in the same process.
    python tools/bench_arrival_consts.py --base DIR [--rounds 2] [--steps 10] [--out FILE]"""
import argparse
import hashlib
import importlib
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAP_SEED, AGENT_SEED, CW = 0x5EED0001, 0x5EED0001, 16


def _card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "unknown"


def _import(tree):
    sys.path.insert(0, tree)
    pf = importlib.import_module("permafrost-engine_b200")
    return pf.capi, pf.synth


def _loop(capi, synth, nflocks, n, enter, steps, warmup):
    import torch
    cost = synth.cost_from_pathable(synth.make_map(CW, CW, MAP_SEED, rivers=True), CW, CW)
    a = synth.make_agents(cost, CW, CW, n, nflocks, AGENT_SEED, radius=1.5, spacing=2.2, hz=20)
    rec, fl = capi.pack_agents(a)
    fl["dest"] = 0
    nav = capi.Nav(0)
    res = {}
    try:
        nav.map_create(CW, CW, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
        nav.agents_upload(rec, fl, 20)
        ms = np.zeros(n, capi.MOVESTATE)
        ms["next_pos"][:, 0] = rec["pos"][:, 0]; ms["next_pos"][:, 2] = rec["pos"][:, 1]
        ms["step"] = 1.0; ms["next_rot"][:, 3] = 1.0; ms["combat_facing"][:, 3] = 1.0
        nav.agents_upload_movestate(ms)
        if enter >= 0:                                          # ext: a movestate_ext table, even with no unit in range
            rng = np.random.default_rng(5)
            ext = np.zeros(n, capi.MOVESTATE_EXT)
            ext["surround_target_uid"] = 0xFFFFFFFF; ext["rot"][:, 3] = 1.0; ext["target_dir"][:, 3] = 1.0
            imp = synth.blocked_to_image(cost, CW, CW) == 0xFF
            near = np.zeros_like(imp)
            near[1:] |= imp[:-1]; near[:-1] |= imp[1:]; near[:, 1:] |= imp[:, :-1]; near[:, :-1] |= imp[:, 1:]
            r = np.clip((a["pos"][:, 1] / 4.0).astype(np.int64), 0, CW * 64 - 1)
            c = np.clip((-a["pos"][:, 0] / 4.0).astype(np.int64), 0, CW * 64 - 1)
            adj = rng.permutation(np.nonzero(near[r, c])[0])
            rest = rng.permutation(np.nonzero(~near[r, c])[0])
            who = np.concatenate([adj, rest])[:enter]
            ext["surround_target_uid"][who] = np.concatenate([adj, rest])[rng.integers(0, max(len(adj), 1), enter) % n]
            res["enter_adjacent"] = int(near[r, c][who].sum())
            ext["target_range"][who] = 0.0
            rec["state"][who] = 6                               # ENTER_ENTITY_RANGE
            nav.agents_upload(rec, fl, 20)
            nav.agents_upload_movestate(ms)
            nav.agents_upload_movestate_ext(ext)
        nav.agents_set_work(np.arange(n, dtype=np.uint32))
        bx, bz = float(a["pos"][0][0]) - 40.0, float(a["pos"][0][1]) + 40.0
        on = [False]
        comp, step = [], []

        def one():
            (nav.blockers_decref if on[0] else nav.blockers_incref)(bx, bz, 6.0)
            on[0] = not on[0]
            nav.map_commit()
            nav.agents_tick(0)
            t = time.perf_counter()
            nav.agents_compute_updates()
            c = time.perf_counter() - t
            nav.agents_apply_updates()
            nav.agents_rebuild_index()
            return c
        for _ in range(warmup):
            one()
        torch.cuda.synchronize()
        for _ in range(steps):
            t0 = time.perf_counter()
            c = one()
            torch.cuda.synchronize()
            step.append((time.perf_counter() - t0) * 1e3); comp.append(c * 1e3)
        res.update({"compute_ms": statistics.median(comp), "step_ms": statistics.median(step)})
        nav.agents_tick(0)
        nav.agents_compute_updates()
        res["patches"] = hashlib.sha256(nav.agents_read_patches(n).tobytes()).hexdigest()
        return res
    finally:
        nav.close()


def _query(capi, synth, n, reps):
    cost = synth.cost_from_pathable(synth.make_map(CW, CW, MAP_SEED, rivers=True), CW, CW)
    img = synth.blocked_to_image(cost, CW, CW).copy()
    img[412:612, 412:612] = 0xFF
    islands = [(430 + 12 * k, 430) for k in range(8)]
    for r, c in islands:
        img[r, c] = 1
    cost = synth.image_to_blocked(img, CW, CW)
    rng = np.random.default_rng(11)
    q = np.zeros(n, capi.MAP_QUERY)
    for i in range(n):
        if i % 2 == 0:
            r, c = (int(v) for v in rng.integers(482, 542, 2))
            x, z = synth.tile_center_xz(r // 64, c // 64, r % 64, c % 64, 0.0, 0.0)
            q[i] = (capi.QUERY_CLOSEST_PATHABLE, 0, x, z, 0, 0, 0, 0)
        else:
            r, c = islands[i % len(islands)]
            x, z = synth.tile_center_xz(r // 64, c // 64, r % 64, c % 64, 0.0, 0.0)
            q[i] = (capi.QUERY_MAXIMALLY_CLOSE, 0, x + 4.0, z, x, z, 8.0, 0)
    nav = capi.Nav(0)
    try:
        nav.map_create(CW, CW, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
        out = nav.map_query(q)
        ts = []
        for _ in range(reps):
            t = time.perf_counter()
            out = nav.map_query(q)
            ts.append((time.perf_counter() - t) * 1e3)
        return {"batch_ms": statistics.median(ts), "answers": out.tobytes().hex()}
    finally:
        nav.close()


def worker(args):
    capi, synth = _import(args.tree)
    if args.job == "query":
        r = _query(capi, synth, args.n, args.reps)
    else:
        r = _loop(capi, synth, args.flocks, args.agents, args.enter if args.job == "ext" else -1, args.steps, args.warmup)
    print(json.dumps(r))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", help="tree of the build to compare with (its libpfnav.so built)")
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--agents", type=int, default=100_000)
    ap.add_argument("--enter", type=int, default=64)
    ap.add_argument("--enter-counts", default="0,64,1000,10000")
    ap.add_argument("--flock-counts", default="16,2500")
    ap.add_argument("--query-sizes", default="2,64,512")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--out")
    ap.add_argument("--worker", action="store_true")
    ap.add_argument("--tree", default=ROOT)
    ap.add_argument("--job", default="loop")
    ap.add_argument("--flocks", type=int, default=16)
    ap.add_argument("--n", type=int, default=2)
    args = ap.parse_args()
    if args.worker:
        return worker(args)
    card = _card()
    trees = [("new", ROOT)] + ([("base", os.path.abspath(args.base))] if args.base else [])
    jobs = [("loop", f, 0) for f in map(int, args.flock_counts.split(","))] + \
           [("ext", f, e) for f in map(int, args.flock_counts.split(",")) for e in map(int, args.enter_counts.split(","))] + \
           [("query", 0, int(s)) for s in args.query_sizes.split(",")]
    lines = []
    for job, f, n in jobs:
        answers, digests = {}, {}
        for rnd in range(args.rounds):
            for name, tree in (trees if rnd % 2 == 0 else trees[::-1]):
                cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--tree", tree, "--job", job, "--flocks", str(f),
                       "--n", str(n), "--agents", str(args.agents), "--enter", str(n if job == "ext" else args.enter),
                       "--steps", str(args.steps),
                       "--warmup", str(args.warmup), "--reps", str(args.reps)]
                r = subprocess.run(cmd, capture_output=True, text=True)
                if r.returncode != 0:
                    res = {"error": r.stderr.strip().splitlines()[-1] if r.stderr.strip() else "exit %d" % r.returncode}
                else:
                    res = json.loads(r.stdout.strip().splitlines()[-1])
                if "answers" in res:
                    answers.setdefault(name, res.pop("answers"))
                if "patches" in res:
                    digests.setdefault(name, set()).add(res.pop("patches"))
                line = {"card": card, "build": name, "round": rnd, "job": job, "map": "C2", "agents": args.agents if job != "query" else 0,
                        "flocks": f, "enter_units": n if job == "ext" else 0, "queries": n if job == "query" else 0, **res}
                print(json.dumps(line), flush=True)
                lines.append(line)
        if job == "query" and len(answers) == 2:
            same = answers["new"] == answers["base"]
            print(json.dumps({"job": job, "queries": n, "answers_equal": same}), flush=True)
            lines.append({"card": card, "job": job, "queries": n, "answers_equal": same})
        if job != "query" and len(digests) == 2:
            same = len(digests["new"] | digests["base"]) == 1
            line = {"card": card, "job": job, "flocks": f, "enter_units": n if job == "ext" else 0, "patches_equal": same}
            print(json.dumps(line), flush=True)
            lines.append(line)
    if args.out:
        with open(args.out, "a") as fh:
            for line in lines:
                fh.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
