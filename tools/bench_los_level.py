#!/usr/bin/env python3
"""The LOS phase of the C2 cold goal batch (pfnav_pool_request_goals: 16 goals x 256 chunks), LOS variant 1 (k_los_b, the
byte-state heap replay) against variant 2 (k_los_level, level-parallel with the replay as fallback). Per variant, one JSON
line: the LOS makespan from the per-field trace (first take to last finish, median and spread over --reps batches), the
fields the level kernel replayed, and the critical dependency chain (walked back from the last finisher): its length, the
non-empty and replayed fields on it, and the most replayed fields on any one chain."""
import argparse, importlib, json, os, sys
import numpy as np
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch
import bench

REPLAYED = 1 << 31


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    nav = capi.Nav(0)
    C = bench.CHUNKS
    nav.map_create(C, C, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0)
    goals = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(W["g_lo"], W["g_hi"])], np.int32)
    nav.pool_create(len(goals), len(goals) * C * C)
    st = torch.cuda.Stream(); torch.cuda.set_stream(st)
    dests = np.arange(len(goals), dtype=np.int32)
    prop = torch.cuda.get_device_properties(0)
    for variant in (1, 2, 1, 2):
        nav.set_los_variant(variant)
        for _ in range(3):
            nav.pool_clear(); nav.pool_request_goals(dests, goals, 0, st.cuda_stream); nav.fields_join(st.cuda_stream)
        torch.cuda.synchronize()
        spans, traces = [], []
        for _ in range(args.reps):
            nav.los_trace(True)
            nav.pool_clear(); nav.pool_request_goals(dests, goals, 0, st.cuda_stream); nav.fields_join(st.cuda_stream)
            torch.cuda.synchronize()
            tr = nav.los_trace(False, read_cap=len(goals) * C * C).astype(np.int64)
            spans.append((tr[:, 2].max() - tr[:, 0].min()) / 1e6)
            traces.append(tr)
        tr = traces[int(np.argsort(spans)[len(spans) // 2])]
        prev = (tr[:, 3] >> 32) - 1
        word = tr[:, 3] & 0xFFFFFFFF
        rep = (word & REPLAYED) != 0
        pops = (word & 0x7FFFFFFF)
        # replayed fields on every root-to-field chain, and the critical chain back from the last finisher
        on_chain = np.zeros(len(tr), np.int64)
        for i in range(len(tr)):          # requests are dependency-sorted: a field's prev comes first
            on_chain[i] = (on_chain[prev[i]] if prev[i] >= 0 else 0) + int(rep[i])
        i, chain = int(np.argmax(tr[:, 2])), []
        while i >= 0:
            chain.append(i); i = int(prev[i])
        print(json.dumps({
            "gpu": prop.name, "los_variant": variant, "fields": int(len(tr)), "nonempty_fields": int((pops > 0).sum()),
            "replayed_fields": int(rep.sum()), "los_ms_median": round(float(np.median(spans)), 4),
            "los_ms_min": round(float(np.min(spans)), 4), "los_ms_max": round(float(np.max(spans)), 4),
            "critical_chain_fields": len(chain), "critical_chain_nonempty": int(sum(pops[k] > 0 for k in chain)),
            "critical_chain_pops": int(sum(max(int(pops[k]) - 1, 0) for k in chain)),
            "critical_chain_replayed": int(sum(rep[k] for k in chain)), "max_replayed_on_any_chain": int(on_chain.max())}),
            flush=True)
    nav.close()


if __name__ == "__main__":
    main()
