"""Host-observed time of writing inputs beyond point seeking into a device-resident population, two arms alternated:

  deltas     pfnav_agents_input_deltas (the records)
  reupload   pfnav_agents_read_movestate_ext + pfnav_agents_read_formation + the same writes in numpy +
             pfnav_agents_upload_movestate_ext + pfnav_agents_upload_formation   (the only way in before the call)

at the benchmark's C2 population (100 000 entities, both tables uploaded) with batches of 1, 1 000 and 10 000 records of
every mask over distinct uids. A host clock around work that ends in a device synchronise; warm-up, then the median of
--runs runs with min / max. These are end-to-end call times, not kernel shares of peak. The card's name and power limit
are read in the same process and written beside the numbers: results/h100_sxm_<power>w/input_deltas.jsonl. There is no
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
sys.path.insert(0, os.path.join(ROOT, "tests"))


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader,nounits", "-i", "0"],
                         check=True, capture_output=True, text=True).stdout.strip().splitlines()[0]
    name, power = [x.strip() for x in out.split(",")]
    return name, float(power)


def apply_vectorised(capi, ext, form, d):
    """the records' writes on the host copies, one fancy assignment per field (the uids of a batch are distinct)"""
    for bit, name in ((capi.INPUT_TARGET_PREV, "target_prev_pos"), (capi.INPUT_TARGET_DIR, "target_dir"),
                      (capi.INPUT_ROT, "rot"), (capi.INPUT_SURROUND_FIELD, "using_surround_field")):
        sel = (d["mask"] & bit) != 0
        ext[name][d["uid"][sel]] = d[name][sel]
    sel = (d["mask"] & capi.INPUT_FORMATION) != 0
    form[d["uid"][sel]] = d["formation"][sel]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--runs", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=None, help="the .jsonl to append to (default results/h100_sxm_<power>w/input_deltas.jsonl)")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bench_input_deltas.py needs a GPU: there is no CPU arm")
    pf = importlib.import_module("permafrost-engine_b200")
    capi = pf.capi
    bench = importlib.import_module("bench")
    import inputs_ref as ir
    name, power = card()
    cardname = ("h100_sxm_%dw" % round(power)) if "H100" in name else name.replace(" ", "_").lower()
    out = args.out or os.path.join(ROOT, "results", cardname, "input_deltas.jsonl")
    os.makedirs(os.path.dirname(os.path.abspath(out)), exist_ok=True)
    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    rec, fl, n = W["rec"], W["flocks"], W["n_total"]
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID; ext["rot"][:, 3] = 1.0
    form = np.zeros(n, capi.FORMATION_IN)
    navs = {}
    for arm in ("deltas", "reupload"):
        X = capi.Nav(0)
        X.map_create(bench.CHUNKS, bench.CHUNKS, 1); X.map_upload_layer(0, W["cost"])
        X.agents_upload(rec, fl, bench.HZ)
        X.agents_upload_movestate_ext(ext); X.agents_upload_formation(form)
        navs[arm] = X
    rng = np.random.default_rng(1)
    rows = []
    for k in (1, 1_000, 10_000):
        t = {"deltas": [], "reupload": []}
        for it in range(args.warmup + args.runs):
            d = ir.random_inputs(rng, k, np.arange(n))
            d["uid"] = rng.choice(n, k, replace=False)
            for arm in ("deltas", "reupload"):
                X = navs[arm]
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                if arm == "deltas":
                    X.agents_input_deltas(d)
                else:
                    e, f = X.agents_read_movestate_ext(n), X.agents_read_formation(n)
                    apply_vectorised(capi, e, f, d)
                    X.agents_upload_movestate_ext(e); X.agents_upload_formation(f)
                torch.cuda.synchronize()
                if it >= args.warmup:
                    t[arm].append((time.perf_counter() - t0) * 1e3)
        for a, b in ((navs["deltas"].agents_read_movestate_ext(n), navs["reupload"].agents_read_movestate_ext(n)),
                     (navs["deltas"].agents_read_formation(n), navs["reupload"].agents_read_formation(n))):
            assert a.tobytes() == b.tobytes()                    # outside the window: a check, not part of an arm
        row = {"workload": "C2", "entities": n, "records": k, "runs": args.runs, "card": name, "power_limit_w": power,
               "what": "host-observed ms per batch of input deltas, ending in a device synchronise"}
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
