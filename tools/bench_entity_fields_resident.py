#!/usr/bin/env python
"""Enemy-seek fields for a resident population: pfnav_pool_request_entity_fields_resident against the path an engine
without host positions takes today -- pfnav_agents_read_state, footprints and seeker chunks in numpy, then
pfnav_pool_request_entity_fields_batch -- on the C2 map (16 x 16 chunks).

100 000 entities stand on passable tiles. One seek-enemies tick of four factions: each faction's request names an enemy
list of 75 000 uids and 2 500 seekers (10 000 in all), on reference layer f. Both paths run on contexts holding the same
population; each repetition clears both pools (cold), then times one path and then the other, alternating which goes
first, each window ending in a device synchronise. --warmup repetitions, then median, min and max of --reps. The two
pools must hold identical entries (flow bytes, has, ffid) for every (dest, chunk).
    python tools/bench_entity_fields_resident.py [--reps 7] [--warmup 2] [--out FILE]"""
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

N, ENEMIES, SEEKERS, FACTIONS = 100000, 75000, 10000, 4


def chunk_of(pos, cw, ch):
    """M_Tile_DescForPoint2D's chunk (map at the origin) in the tick's arithmetic; -1 off the map"""
    px, pz = pos[:, 0].astype(np.float32), pos[:, 1].astype(np.float32)
    on = ~((px > 0) | (px < -np.float32(cw * 256)) | (pz < 0) | (pz > np.float32(ch * 256)))
    r = np.clip((np.abs(pz.astype(np.float64)) / 256.0).astype(np.int64), 0, ch - 1)
    c = np.clip((np.abs(px.astype(np.float64)) / 256.0).astype(np.int64), 0, cw - 1)
    return np.where(on, r * cw + c, -1)


def today(nav, capi, reqs, uids, seekers, cw):
    """the host path: read the population back, build the batch's inputs, make the batch"""
    a, _ = nav.agents_read_state(N, False)
    fp = np.zeros(len(uids), capi.FOOTPRINT)
    fp["x"], fp["z"], fp["sel_radius"] = a["pos"][uids, 0], a["pos"][uids, 1], a["radius"][uids]
    sc = chunk_of(a["pos"][seekers], cw, cw)
    assert (sc >= 0).all()
    out, chunks, nch = reqs.copy(), [], 0
    for i, q in enumerate(reqs):
        s = sc[int(q["chunk_off"]):int(q["chunk_off"]) + int(q["chunk_n"])]
        _, first = np.unique(s, return_index=True)
        seen = s[np.sort(first)]
        out["chunk_off"][i], out["chunk_n"][i] = nch, len(seen)
        chunks.append(np.stack([seen // cw, seen % cw], 1))
        nch += len(seen)
    return nav.pool_request_entity_fields_batch(out, fp, np.concatenate(chunks).astype(np.int32))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    pf = importlib.import_module("permafrost-engine_b200")
    capi, synth = pf.capi, pf.synth
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu)
    bench.set_workload("C2")
    cw = bench.CHUNKS
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, bench.MAP_SEED, rivers=True), cw, cw)
    rng = np.random.default_rng(0x5EED)
    img = synth.blocked_to_image(cost, cw, cw)
    t = np.argwhere(img != 255)
    t = t[rng.integers(0, len(t), N)]
    pos = np.stack([-(t[:, 1] + rng.uniform(0.05, 0.95, N)) * 4.0, (t[:, 0] + rng.uniform(0.05, 0.95, N)) * 4.0], 1)
    rec = np.zeros(N, capi.AGENT)
    rec["pos"] = pos.astype(np.float32); rec["prev_pos"] = rec["pos"]
    rec["radius"] = rng.choice(np.array([1.0, 1.5, 3.0, 4.5], np.float32), N)
    rec["max_speed"] = 20.0; rec["speed"] = 20.0; rec["flags"] = capi.FLAG_MOVABLE; rec["flock"] = -1
    fl = np.zeros(1, capi.FLOCK); fl["dest"] = -1
    navs = []
    for _ in range(2):
        nav = capi.Nav(0)
        nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0)
        nav.pool_create(FACTIONS, FACTIONS * cw * cw)
        nav.agents_upload(rec, fl, 20)
        navs.append(nav)
    host, res = navs
    uids = np.concatenate([rng.choice(N, ENEMIES, replace=False) for _ in range(FACTIONS)]).astype(np.uint32)
    seekers = rng.choice(N, SEEKERS, replace=False).astype(np.uint32)
    per = SEEKERS // FACTIONS
    reqs = np.zeros(FACTIONS, capi.ENTITY_FIELD_REQ)
    for f in range(FACTIONS):
        reqs[f] = (f, 0, f, capi.TARGET_ENEMIES, f * ENEMIES, ENEMIES, f * per, per)
    th, tr = [], []
    for rep in range(args.warmup + args.reps):
        host.pool_clear(); res.pool_clear()
        torch.cuda.synchronize()
        order = [0, 1] if rep % 2 == 0 else [1, 0]
        for which in order:
            t0 = time.perf_counter()
            if which == 0:
                done = today(host, capi, reqs, uids, seekers, cw)
            else:
                done = res.pool_request_entity_fields_resident(reqs, None, uids, seekers)
            torch.cuda.synchronize()
            dt = time.perf_counter() - t0
            assert done == FACTIONS
            if rep >= args.warmup:
                (th if which == 0 else tr).append(dt)
    same = all(_entry(host, d, c, cw) == _entry(res, d, c, cw) for d in range(FACTIONS) for c in range(cw * cw))
    assert same, "the two paths left different pools"
    fields = sum(1 for d in range(FACTIONS) for c in range(cw * cw) if _entry(res, d, c, cw)[1] is not None)
    ms = lambda v: {"median": 1e3 * statistics.median(v), "min": 1e3 * min(v), "max": 1e3 * max(v)}
    line = json.dumps({"map": "C2", "entities": N, "factions": FACTIONS, "enemy_uids_per_faction": ENEMIES,
                       "seekers": SEEKERS, "fields": fields, "warmup": args.warmup, "reps": args.reps,
                       "read_back_numpy_batch_ms": ms(th), "resident_ms": ms(tr),
                       "speedup_median": statistics.median(th) / statistics.median(tr), "identical_pool": bool(same),
                       "gpu": gpu})
    print(line, flush=True)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")
    for nav in navs:
        nav.close()


def _entry(nav, d, c, cw):
    f, _, ffid = nav.pool_get(d, divmod(c, cw))
    return (ffid, None if f is None else f.tobytes())


if __name__ == "__main__":
    main()
