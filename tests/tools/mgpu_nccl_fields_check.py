"""NCCL transport of a job's goal batches (pfnav_mgpu_request_goals_ex), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29513 tests/tools/mgpu_nccl_fields_check.py
Every rank holds a job member and a single context built from the same seeds that gets the same calls, with
pfnav_pool_request_goals_ex in place of the job's batch. A cold batch, then (after rank-specific earlier batches and
commits that dirty chunks, so that the ranks hold different fields) PFNAV_REQUEST_MISSING_ONLY batches: every member's
pool must equal its single context's for every (dest, chunk) -- has bits, ff_id, flow and LOS bytes -- with its solo
counts; every rank must report the same owners, and the ranks' built requests must add up to the union of the lacked
fields. World 1 runs on one GPU; world >= 2 needs as many GPUs (NCCL puts no two ranks on one GPU).
Prints "mgpu_nccl_fields_check PASS world=N" on rank 0. torch.distributed is used only to hand the NCCL id around and
to collect the results for the comparison."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases
from test_gpu_mgpu_fields import _has, _nav, _pool, _targets, synth_cost

capi = cases.capi


def run(rank, world, local):
    cw, nd = 4, 6
    cost = synth_cost(cw, 505)
    ids = [capi.mgpu_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    nav = _nav(local, cost, cw, nd, nd * cw * cw)
    one = _nav(local, cost, cw, nd, nd * cw * cw)
    nav.mgpu_init(rank, world, ids[0])
    rng = np.random.default_rng(11)
    tg = _targets(nav, nd, rng)
    ok = True

    def job(dests, flags, label):
        nonlocal ok
        dests = np.asarray(dests, np.int32)
        t = tg[dests]
        has = _has(nav, nd)
        lack = {k: (3 if not flags else (~h & 3)) for k, h in has.items()}
        lacks = [None] * world
        dist.all_gather_object(lacks, lack)
        per = []
        for d, tt in zip(dests, t):
            _, fc, _, _, lc = nav.plan_goal(tuple(int(v) for v in tt))
            per.append((sum(any(L[(int(d), int(c))] & 1 for L in lacks) for c in fc),
                        sum(any(L[(int(d), int(c))] & 2 for L in lacks) for c in lc)))
        got = nav.mgpu_request_goals_ex(dests, t, flags=flags)
        want = one.pool_request_goals(dests, t, flags=flags)
        same = got == want and _pool(nav, nd) == _pool(one, nd)
        bf, bl, owner = nav.mgpu_fields_stats(len(dests))
        parts = [None] * world
        dist.all_gather_object(parts, (same, bf, bl, owner.tolist()))
        good = (all(q[0] for q in parts) and all(q[3] == parts[0][3] for q in parts)
                and sum(q[1] for q in parts) == sum(p[0] for p in per) and sum(q[2] for q in parts) == sum(p[1] for p in per)
                and all((parts[0][3][g] >= 0) == (sum(per[g]) > 0) for g in range(len(per))))
        if rank == 0:
            print("%s: union %d flow / %d LOS requests, built per rank %s, identical=%s" % (
                label, sum(p[0] for p in per), sum(p[1] for p in per), [(q[1], q[2]) for q in parts], good), flush=True)
        ok &= good

    job(range(nd), 0, "cold")
    for X in (nav, one):                        # rank-specific earlier batches: the ranks hold different fields
        X.pool_clear()
        held = [rank % nd, (rank + 2) % nd]
        X.pool_request_goals(held, tg[held])
    job(range(nd), capi.REQUEST_MISSING_ONLY, "missing-only, diverged")
    for step in range(3):
        x, z = float(rng.uniform(-cw * 256 + 40, -40)), float(rng.uniform(40, cw * 256 - 40))
        for X in (nav, one):
            X.blockers_incref(x, z, 6.0 + 4 * step)
            X.map_commit()
        job(range(nd), capi.REQUEST_MISSING_ONLY, "missing-only after commit %d" % step)
    nav.mgpu_finalize(); nav.close(); one.close()
    return ok


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    ok = run(rank, world, local)
    if rank == 0:
        print("mgpu_nccl_fields_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
