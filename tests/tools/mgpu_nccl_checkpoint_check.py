"""NCCL jobs and checkpoints (pfnav_agents_save / pfnav_agents_restore), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29516 tests/tools/mgpu_nccl_checkpoint_check.py
Every rank uploads its own range with movestate, movestate_ext and blocking tables (the job shares blockers), stops a
few units (their blocks are taken on the device and exchanged), runs resident ticks, and saves its range at the save
point. Rank 0 restores every rank's segment on ONE context; a second job (a fresh NCCL communicator on fresh contexts)
restores the same segments, each rank taking its own range, exchanges and commits the restored blocks and gathers. Then:
the second job's segments joined equal the first job's byte for byte, the single context's segment equals them too, and
on every rank the second job's next ticks (velocities, patches, own entity state) equal, bit for bit, the first job's own
ticks after its save with its pool cleared (the same member split: each member serves its own work items' field misses).
Runs at any world size, world 1 included (one H100). Prints "mgpu_nccl_checkpoint_check PASS world=N" on rank 0.
torch.distributed is used only to hand the NCCL ids and segments around and to collect the results."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases

capi = cases.capi
ST_ARRIVED = 2
HDR = 64


def rows(seg, nflocks):
    return seg[HDR + 16 * nflocks:]


def run(rank, world, local):
    hz, cw = 20, 3
    p, cost, a, ms = cases.update_case(4242, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(5)
    nf = len(a["flock_target"])
    a["flock_dest_index"] = np.arange(nf, dtype=np.int32)
    rec, fl = capi.pack_agents(a)
    perm = rng.permutation(n)                         # every flock on every rank
    rec, ms = rec[perm].copy(), ms[perm].copy()
    ext = np.zeros(n, capi.MOVESTATE_EXT); ext["surround_target_uid"] = capi.NULL_UID; ext["rot"][:, 3] = 1.0
    blk = np.zeros(n, capi.BLOCKING); blk["faction_id"] = capi.FACTION_ID_NONE
    stop = np.nonzero((rec["state"] == ST_ARRIVED) & ((rec["flags"] & capi.FLAG_GARRISONED) == 0))[0].astype(np.uint32)
    lo, hi = capi.mgpu_shard_range(n, rank, world)

    def make(X):
        X.map_create(cw, cw, 1); X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
        X.pool_create(nf + 2, (nf + 2) * cw * cw)

    def job(restore_from=None):
        ids = [capi.mgpu_unique_id() if rank == 0 else None]
        dist.broadcast_object_list(ids, src=0)
        X = capi.Nav(local)
        make(X)
        X.mgpu_init(rank, world, ids[0])
        X.mgpu_share_blockers()
        if restore_from is None:
            X.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, hz)
            X.mgpu_gather()
            X.agents_upload_movestate(ms[lo:hi]); X.agents_upload_movestate_ext(ext[lo:hi]); X.agents_upload_blocking(blk[lo:hi])
            X.agents_set_blocking(stop[(stop >= lo) & (stop < hi)], True)
        else:
            X.agents_restore(restore_from)
        X.mgpu_exchange_blocker_ops()
        X.map_commit()
        X.mgpu_gather()
        X.agents_set_work_dev()
        return X

    def tick(X):
        nw = len(X.agents_read_work())
        out = b""
        if nw:
            for _ in range(2):
                X.agents_tick(capi.TICK_VDES_FROM_POOL); X.pool_repair()
            X.agents_tick(capi.TICK_VDES_FROM_POOL)
            X.agents_compute_updates()
            out = X.agents_read_velocities(nw).tobytes() + X.agents_read_patches(nw).tobytes()
            X.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        X.mgpu_exchange_blocker_ops()
        X.map_commit()
        X.mgpu_gather()
        X.agents_set_work_dev()
        st, mst = X.agents_read_state(hi - lo)
        return out + st.tobytes() + mst.tobytes()

    J1 = job()
    for _ in range(3):
        tick(J1)
    seg = J1.agents_save()
    segs = [None] * world
    dist.all_gather_object(segs, seg)
    J1.pool_clear()
    cont = [tick(J1) for _ in range(3)]
    J1.mgpu_finalize(); J1.close()

    ok = True
    one = None
    if rank == 0:
        one = capi.Nav(local)
        make(one)
        one.agents_restore(segs)
        one.map_commit(); one.agents_rebuild_index(); one.agents_set_work_dev()
        ok &= rows(one.agents_save(), nf) == b"".join(rows(s, nf) for s in segs)
    J2 = job(restore_from=segs)
    seg2 = J2.agents_save()
    back = [None] * world
    dist.all_gather_object(back, seg2)
    ok &= b"".join(rows(s, nf) for s in back) == b"".join(rows(s, nf) for s in segs)
    ok &= [tick(J2) for _ in range(3)] == cont
    if rank == 0:
        one.close()
    res = [None] * world
    dist.all_gather_object(res, ok)
    J2.mgpu_finalize(); J2.close()
    return all(res)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    ok = run(rank, world, local)
    if rank == 0:
        print("mgpu_nccl_checkpoint_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
