#!/usr/bin/env python
"""Where the host time of bench.py's cold C2 step goes: pfnav_pool_clear + pfnav_pool_request_goals on the C2 workload.

Prints, with the card's name and power limit read in the same run:
  * the host wall-clock segments of pool_clear / pool_request_goals (pfnav_profile_read_host: waits, planning, merge,
    slot reservation, packing, H2D enqueue, launches), per cold batch, over --steps back-to-back cold steps
    (pool_clear + pool_request_goals + index rebuild + tick on one stream, no host synchronisation in between);
  * the device time per step of those cold steps and of the same steps with the plan resident on the device
    (same kernels, no host planning): their difference is time the GPU spends waiting for the host;
  * one isolated cold batch between two synchronisations: its device span (event before pool_clear -> event after the
    fields are joined), its flow and LOS kernel-group times, and the idle gap = span - max(flow, LOS) (the flow waves
    and the LOS chains run concurrently on two streams).
    python tools/bench_cold_request.py [--steps 20] [--warmup 5] [--out FILE]"""
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
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--isolated", type=int, default=7, help="isolated cold batches (median)")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "needs the GPU"
    gpu = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    print("gpu:", gpu, "| host cpus:", os.cpu_count(), flush=True)
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    cw = bench.CHUNKS
    nav = capi.Nav(0)
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0)
    ngoals = W["g_hi"] - W["g_lo"]
    nav.pool_create(ngoals, ngoals * cw * cw)
    nwork = W["hi"] - W["lo"]
    nav.agents_upload_shard(W["rec"][W["lo"]:W["hi"]], W["lo"], W["hi"], W["n_total"], W["flocks"], bench.HZ, 0)
    nav.agents_set_work(np.arange(W["lo"], W["hi"], dtype=np.uint32))
    dests = np.arange(ngoals, dtype=np.int32)
    targets = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(W["g_lo"], W["g_hi"])], np.int32)
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    sp = stream.cuda_stream
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")

    def step(cold):
        if cold:
            nav.pool_clear()
        nav.pool_request_goals(dests, targets, 0, sp)
        nav.agents_rebuild_index(sp)
        nav.agents_tick(capi.TICK_VDES_FROM_POOL, sp)

    def loop(cold, steps):
        """back-to-back steps like bench.py's timed(): events around every step, L2 flushed outside them"""
        ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        for k in range(steps):
            flush.zero_()
            ev[k][0].record(stream)
            step(cold)
            ev[k][1].record(stream)
        torch.cuda.synchronize()
        wall = time.perf_counter() - t0
        return sum(a.elapsed_time(b) for a, b in ev) / steps, 1e3 * wall / steps

    for _ in range(max(args.warmup, 3)):
        step(True)
    cold_ms, cold_wall = loop(True, args.steps)
    step(False)
    res_ms, res_wall = loop(False, args.steps)
    # host segments of the same back-to-back cold loop, profiling on (a separate run: the timers and events cost a little)
    nav.profile_enable(True)
    nav.profile_read(); nav.profile_read_host()
    loop(True, args.steps)
    seg = nav.profile_read_host()
    nav.profile_read()
    seg_loop = {k: v[0] / args.steps for k, v in seg.items()}
    # isolated cold batches
    spans, flows, loss, walls, segs = [], [], [], [], []
    for _ in range(args.isolated):
        flush.zero_()
        torch.cuda.synchronize()
        nav.profile_read(); nav.profile_read_host()
        a_, b_ = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0 = time.perf_counter()
        a_.record(stream)
        nav.pool_clear()
        nav.pool_request_goals(dests, targets, 0, sp)
        nav.fields_join(sp)
        b_.record(stream)
        torch.cuda.synchronize()
        walls.append(1e3 * (time.perf_counter() - t0))
        spans.append(a_.elapsed_time(b_))
        p = nav.profile_read()
        flows.append(p["flow"][0]); loss.append(p["los"][0])
        segs.append(nav.profile_read_host())
        nav.agents_rebuild_index(sp); nav.agents_tick(capi.TICK_VDES_FROM_POOL, sp)
    nav.profile_enable(False)
    torch.cuda.synchronize()
    med = statistics.median
    seg_iso = {k: med([s[k][0] for s in segs]) for k in segs[0]}
    span, fl, lo = med(spans), med(flows), med(loss)
    rec = {"map": "C2", "goals": ngoals, "agents": nwork, "gpu": gpu, "host_cpus": os.cpu_count(), "steps": args.steps,
           "cold_ms_per_step": cold_ms, "cold_wall_ms_per_step": cold_wall,
           "resident_plan_ms_per_step": res_ms, "resident_plan_wall_ms_per_step": res_wall,
           "gpu_waits_for_host_ms_per_step": cold_ms - res_ms,
           "host_ms_per_cold_step": seg_loop, "host_total_ms_per_cold_step": sum(seg_loop.values()),
           "isolated": {"host_ms": seg_iso, "host_total_ms": sum(seg_iso.values()), "call_wall_ms": med(walls),
                        "device_span_ms": span, "flow_ms": fl, "los_ms": lo, "idle_gap_ms": span - max(fl, lo)}}
    print("%-34s %9s %9s" % ("host segment (ms)", "in loop", "isolated"))
    for k in capi.Nav.HOST_SEGMENTS:
        print("%-34s %9.3f %9.3f" % (k, seg_loop[k], seg_iso[k]))
    print("%-34s %9.3f %9.3f" % ("total", rec["host_total_ms_per_cold_step"], rec["isolated"]["host_total_ms"]))
    print("cold step %.3f ms (wall %.3f), resident-plan step %.3f ms (wall %.3f): GPU waits %.3f ms/step for the host"
          % (cold_ms, cold_wall, res_ms, res_wall, cold_ms - res_ms))
    print("isolated cold batch: device span %.3f ms, flow %.3f ms, LOS %.3f ms, idle gap %.3f ms, call wall %.3f ms"
          % (span, fl, lo, span - max(fl, lo), med(walls)))
    line = json.dumps(rec)
    print(line, flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(line + "\n")
    nav.close()


if __name__ == "__main__":
    main()
