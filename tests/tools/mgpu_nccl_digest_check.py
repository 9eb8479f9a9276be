"""NCCL jobs and state digests (pfnav_mgpu_state_digest), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29517 tests/tools/mgpu_nccl_digest_check.py
Every rank uploads its own range with movestate, movestate_ext and blocking tables, and rank 0 also runs ONE context with
the whole population. For 4 steps of the same movement command batches (pfnav_mgpu_commands on the job, followed by the
gather; pfnav_agents_commands on the single context), every rank queues the NCCL digest and reads it: the job's
population, flocks, records and map equal the single context's digest, the differ masks are empty, each rank's own range
is its shard, and the ranks' block arrays summed element-wise equal the single context's. Then
rank 0 moves one of its entities without a gather: its records value differs from the others' and every rank's read
shows rank 0's value with the other ranks in the records mask. Runs at any world size, world 1 included (one H100).
Prints "mgpu_nccl_digest_check PASS world=N" on rank 0. torch.distributed is used only to hand the NCCL id around and to
collect the results."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases

capi = cases.capi
KEYS = ("population", "flocks", "records", "map")
WHAT = capi.DIGEST_POPULATION | capi.DIGEST_FLOCKS | capi.DIGEST_RECORDS | capi.DIGEST_MAP
K = 6


def run(rank, world, local):
    hz, cw = 20, 3
    p, cost, a, ms = cases.update_case(4242, hz)
    n = len(a["radius"])
    nf = len(a["flock_target"])
    a["flock_dest_index"] = np.arange(nf, dtype=np.int32)
    rec, fl = capi.pack_agents(a)
    perm = np.random.default_rng(5).permutation(n)
    rec, ms = rec[perm].copy(), ms[perm].copy()
    ext = np.zeros(n, capi.MOVESTATE_EXT); ext["surround_target_uid"] = capi.NULL_UID; ext["rot"][:, 3] = 1.0
    blk = np.zeros(n, capi.BLOCKING); blk["faction_id"] = capi.FACTION_ID_NONE
    lo, hi = capi.mgpu_shard_range(n, rank, world)

    def make(X):
        X.map_create(cw, cw, 1); X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
        X.pool_create(nf + 2, (nf + 2) * cw * cw)

    def batch(t, m=40):
        r = np.random.default_rng(100 + t)
        c = np.zeros(m, capi.AGENT_DELTA)
        c["uid"] = r.choice(n, m, replace=False)
        c["mask"] = (1 << 4) | (1 << 6)               # PFNAV_DELTA_SPEEDS | PFNAV_DELTA_VELOCITY
        c["velocity"] = r.standard_normal((m, 2)).astype(np.float32)
        c["max_speed"] = rec["max_speed"][c["uid"]]
        c["speed"] = r.random(m).astype(np.float32) * c["max_speed"]
        return c

    ids = [capi.mgpu_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    X = capi.Nav(local)
    make(X)
    X.mgpu_init(rank, world, ids[0])
    X.mgpu_share_blockers()
    X.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, hz)
    X.mgpu_gather()
    X.agents_upload_movestate(ms[lo:hi]); X.agents_upload_movestate_ext(ext[lo:hi]); X.agents_upload_blocking(blk[lo:hi])
    X.map_commit(); X.mgpu_gather(); X.agents_set_work_dev()
    one = None
    if rank == 0:
        one = capi.Nav(local)
        make(one)
        one.agents_upload(rec, fl, hz)
        one.agents_upload_movestate(ms); one.agents_upload_movestate_ext(ext); one.agents_upload_blocking(blk)
        one.map_commit(); one.agents_rebuild_index(); one.agents_set_work_dev()

    ok = True
    for t in range(5):
        if t:
            X.mgpu_commands(batch(t)); X.mgpu_gather()
            if one is not None:
                one.agents_commands(batch(t)); one.agents_rebuild_index()
        X.mgpu_state_digest(WHAT, K)
        d, blocks = X.state_digest_read()
        ok &= (int(d["lo"]), int(d["hi"])) == (lo, hi)
        ok &= int(d["differ_flocks"]) == int(d["differ_records"]) == int(d["differ_map"]) == 0
        mine = [int(d[k]) for k in KEYS]
        all_blocks = [None] * world
        dist.all_gather_object(all_blocks, blocks)
        ref = [None, None]
        if one is not None:
            one.state_digest(WHAT, K)
            od, ob = one.state_digest_read()
            with np.errstate(over="ignore"):
                summed = np.sum(all_blocks, axis=0, dtype=np.uint64)
            ref = [[int(od[k]) for k in KEYS], bool((summed == ob).all())]
        dist.broadcast_object_list(ref, src=0)
        ok &= mine == ref[0] and ref[1]
    # rank 0's record column differs from the others': every rank sees the other ranks in the records mask
    if rank == 0 and hi > lo:
        moved = rec[lo:hi].copy()
        moved["pos"][0] += 1.0
        X.agents_upload_shard(moved, lo, hi, n, fl, hz)
    X.mgpu_state_digest(capi.DIGEST_RECORDS, K)
    d, _ = X.state_digest_read(blocks=False)
    want = 0 if world == 1 else ((1 << world) - 2)
    ok &= int(d["differ_records"]) == want
    res = [None] * world
    dist.all_gather_object(res, ok)
    if one is not None:
        one.close()
    X.mgpu_finalize(); X.close()
    return all(res)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    ok = run(rank, world, local)
    if rank == 0:
        print("mgpu_nccl_digest_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
