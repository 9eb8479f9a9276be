"""Host-observed time of checking the game state by digest (pfnav_state_digest + pfnav_state_digest_read) against reading
the state back and hashing it on the host (pfnav_agents_save + pfnav_pool_save + the same digests computed from the
segments by csrc/pfnav_digest_host.h), at the benchmark's C2 (100 000 entities) and C3 (1 000 000 entities) workloads
with every optional table (movestate, movestate_ext, formation, blocking), a pool filled by a cold goal batch and
--ticks ticks whose misses are served, and every digest component.

  digest+read   pfnav_state_digest(ALL, block_log2) then pfnav_state_digest_read with the block array
  save+hash     pfnav_agents_save + pfnav_pool_save, then pf_digest_agents_segment and pf_digest_pool_segment on the
                host (the values are checked equal to the device's)

A host clock around work that ends in a device synchronise; warm-up, then the median of --runs runs with min / max, the
two arms alternated. Separately, in a torch.profiler run of its own, the device time of k_digest_rows (the population
pass) over --prof launches: the bytes it must read (n x row bytes) over that time, as a share of the H100 SXM's 3.35 TB/s
HBM3 data-sheet bandwidth. The card's name and power limit are read in the same process and written beside the numbers
(default results/h100_sxm_<power>w/state_digest.jsonl). There is no CPU arm: without a GPU the context cannot be created."""
import argparse
import ctypes as C
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench_checkpoint import card, stats  # noqa: E402

HBM_PEAK = 3.35e12                  # bytes / s, H100 SXM data sheet
ROW_BYTES = 64 + 176 + 64 + 64 + 32  # agent, movestate, movestate_ext, formation, blocking


def host_oracle(tmp):
    so = os.path.join(tmp, "libdigest_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", os.path.join(ROOT, "tests", "emu", "digest_emu.cpp"),
                    "-o", so], check=True)
    D = C.CDLL(so)
    D.emu_dg_nblocks.restype = C.c_size_t
    D.emu_dg_nblocks.argtypes = [C.c_size_t, C.c_int]
    D.emu_dg_agents.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_char_p]
    D.emu_dg_pool.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p]
    return D


def host_digest(D, aseg, pseg, n, k):
    blocks = np.zeros(max(D.emu_dg_nblocks(n, k), 1), np.uint64)
    out, pool = np.zeros(3, np.uint64), np.zeros(1, np.uint64)
    err = C.create_string_buffer(256)
    a, p = np.frombuffer(aseg, np.uint8), np.frombuffer(pseg, np.uint8)
    assert D.emu_dg_agents(a.ctypes.data, len(a), k, blocks.ctypes.data, out.ctypes.data, err) == 0, err.value
    assert D.emu_dg_pool(p.ctypes.data, len(p), pool.ctypes.data, err) == 0, err.value
    return int(out[0]), int(out[1]), int(out[2]), int(pool[0]), blocks[:D.emu_dg_nblocks(n, k)]


def one_workload(wl, args, pf, bench, D, torch):
    capi = pf.capi
    bench.set_workload(wl)
    W = bench.build_workload(pf, 1, 0)
    rec, fl, n, cost = W["rec"], W["flocks"], W["n_total"], W["cost"]
    ng = W["g_hi"] - W["g_lo"]
    dests = np.arange(ng, dtype=np.int32)
    targets = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(W["g_lo"], W["g_hi"])], np.int32)
    X = capi.Nav(0)
    X.map_create(bench.CHUNKS, bench.CHUNKS, 1)
    X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
    X.pool_create(ng, ng * bench.CHUNKS * bench.CHUNKS)
    X.agents_upload(rec, fl, bench.HZ)
    X.agents_upload_movestate(np.zeros(n, capi.MOVESTATE))
    ext = np.zeros(n, capi.MOVESTATE_EXT); ext["surround_target_uid"] = capi.NULL_UID; ext["rot"][:, 3] = 1.0
    X.agents_upload_movestate_ext(ext)
    form = np.zeros(n, capi.FORMATION_IN); form["target_orientation"][:, 3] = 1.0
    X.agents_upload_formation(form)
    blk = np.zeros(n, capi.BLOCKING); blk["faction_id"] = capi.FACTION_ID_NONE
    X.agents_upload_blocking(blk)
    X.map_commit()
    X.agents_rebuild_index()
    X.agents_set_work(np.arange(n, dtype=np.uint32))
    X.pool_request_goals(dests, targets, 0)
    for _ in range(args.ticks):
        X.agents_tick(capi.TICK_VDES_FROM_POOL); X.pool_repair_batch(); X.agents_tick(capi.TICK_VDES_FROM_POOL)
    torch.cuda.synchronize()
    k = args.block_log2

    def digest_arm():
        X.state_digest(capi.DIGEST_ALL, k)
        return X.state_digest_read()

    def save_arm():
        aseg, pseg = X.agents_save(), X.pool_save()
        return host_digest(D, aseg, pseg, n, k), len(aseg) + len(pseg)

    d, blocks = digest_arm()
    (pop, flocks, records, pool, hblocks), nbytes = save_arm()
    assert (int(d["population"]), int(d["flocks"]), int(d["records"]), int(d["pool"])) == (pop, flocks, records, pool)
    assert (blocks == hblocks).all()
    t = {"digest+read": [], "save+hash": []}
    for r in range(args.warmup + args.runs):
        arms = [("digest+read", digest_arm), ("save+hash", save_arm)]
        if r % 2:
            arms.reverse()
        for arm, fn in arms:
            torch.cuda.synchronize()
            a = time.perf_counter(); fn(); b = time.perf_counter()
            if r >= args.warmup:
                t[arm].append((b - a) * 1e3)
    # the population pass on its own, in a profiled run
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(args.prof):
            X.state_digest(capi.DIGEST_POPULATION, k)
        torch.cuda.synchronize()
    X.state_digest_read()
    rows_us = [e.device_time_total / max(e.count, 1) for e in prof.key_averages() if e.key.startswith("k_digest_rows")
               or "k_digest_rows" in e.key]
    X.close()
    common = dict(workload=wl, n=n, tables="movestate+movestate_ext+formation+blocking", block_log2=k, nblocks=len(blocks),
                  goals=ng, ticks_before=args.ticks, saved_bytes=nbytes)
    out = [dict(arm="digest+read", **common, **stats(t["digest+read"])),
           dict(arm="agents_save+pool_save+host hash", **common, **stats(t["save+hash"]))]
    if rows_us:
        us = rows_us[0]
        out.append(dict(arm="k_digest_rows", **common, kernel_us=us, bytes_read=n * ROW_BYTES,
                        hbm_share=n * ROW_BYTES / (us * 1e-6) / HBM_PEAK, launches=args.prof))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--ticks", type=int, default=3, help="ticks with misses served before the measurements")
    ap.add_argument("--block-log2", type=int, default=10)
    ap.add_argument("--prof", type=int, default=20, help="profiled population passes")
    ap.add_argument("--workloads", default="C2,C3")
    ap.add_argument("--out", default=None, help="the .jsonl to append to (default results/h100_sxm_<power>w/state_digest.jsonl)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_state_digest.py needs a GPU: there is no CPU arm")
    pf = importlib.import_module("permafrost-engine_b200")
    bench = importlib.import_module("bench")
    name, power = card()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    out = args.out or os.path.join(ROOT, "results", cardname, "state_digest.jsonl")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    with tempfile.TemporaryDirectory() as tmp:
        D = host_oracle(tmp)
        rows = []
        for wl in args.workloads.split(","):
            rows += one_workload(wl, args, pf, bench, D, torch)
    with open(out, "a") as f:
        for row in rows:
            row.update(card=name, power_limit_w=power, runs=args.runs)
            f.write(json.dumps(row) + "\n")
            print(json.dumps(row), flush=True)


if __name__ == "__main__":
    main()
