"""NCCL transport of shared device blockers (pfnav_mgpu_share_blockers, pfnav_mgpu_exchange_blocker_ops), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29512 tests/tools/mgpu_nccl_blockers_check.py
Every rank uploads only its own entity range and its own range of the blocking table; three device-resident ticks
(tick -> compute_updates -> apply_updates_ex(APPLY_BLOCKERS) -> pfnav_mgpu_exchange_blocker_ops -> map_commit ->
pfnav_mgpu_gather) must give, bit for bit, what ONE context holding the whole population gives on the single-context
device path (computed on rank 0): velocities, patches, entity state, blocker counts, local islands, the blocking tables
(own ranges, concatenated) and every rank's ndirty. Needs >= 2 GPUs (NCCL puts no two ranks on one GPU).
Prints "mgpu_nccl_blockers_check PASS world=N" on rank 0. torch.distributed is used only to hand the NCCL id around and
to collect the results for the comparison."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases

capi = cases.capi


def run(rank, world, local):
    hz, cw = 20, 3
    p, cost, a, ms = cases.update_case(4242, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(5)
    a["vdes"] = rng.normal(size=(n, 2)).astype(np.float32)
    a["vdes"] /= np.linalg.norm(a["vdes"], axis=1, keepdims=True)
    a["has_los"] = (rng.random(n) < 0.2).astype(np.uint32)
    rec, fl = capi.pack_agents(a)
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = np.where(rng.random(n) < 0.5, capi.FACTION_ID_NONE, rng.integers(0, 15, n)).astype(np.int32)
    ids = [capi.mgpu_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    nav = capi.Nav(local)
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.mgpu_init(rank, world, ids[0])
    nav.mgpu_share_blockers()
    lo, hi = capi.mgpu_shard_range(n, rank, world)
    nav.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, hz)
    nav.mgpu_gather()
    nav.agents_upload_movestate(ms[lo:hi])
    nav.agents_upload_blocking(tbl[lo:hi])
    one = None
    if rank == 0:
        one = capi.Nav(local)
        one.map_create(cw, cw, 1); one.map_upload_layer(0, cost); one.map_build_nav(0); one.route_build(0)
        one.agents_upload(rec, fl, hz); one.agents_upload_movestate(ms)
        one.agents_upload_blocking(tbl)
    moving = (a["state"] != 2) & (a["state"] != 4)
    ok = True
    for tick in range(3):
        work = np.nonzero(moving)[0].astype(np.uint32)
        w = work[(work >= lo) & (work < hi)]
        nav.agents_set_work(w); nav.agents_tick(0)
        v = nav.agents_read_velocities(len(w))
        nav.agents_compute_updates(); pt = nav.agents_read_patches(len(w))
        nav.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        nav.mgpu_exchange_blocker_ops()
        nd = nav.map_commit()
        nav.mgpu_gather()
        st = nav.agents_read_state(hi - lo)[0]
        maps = (nav.blockers(0).tobytes(), nav.local_islands(0).tobytes(), nav.agents_read_blocking(hi - lo).tobytes())
        parts = [None] * world
        dist.all_gather_object(parts, (v.tobytes(), pt.tobytes(), st.tobytes(), nd, maps))
        state_all = np.frombuffer(b"".join(q[2] for q in parts), capi.AGENT)
        if rank == 0:
            one.agents_set_work(work); one.agents_tick(0)
            v1 = one.agents_read_velocities(len(work))
            one.agents_compute_updates(); p1 = one.agents_read_patches(len(work))
            one.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
            nd1 = one.map_commit()
            one.agents_rebuild_index()
            a1 = one.agents_read_state(n)[0]
            b1, l1 = one.blockers(0).tobytes(), one.local_islands(0).tobytes()
            good = (b"".join(q[0] for q in parts) == v1.tobytes() and b"".join(q[1] for q in parts) == p1.tobytes()
                    and state_all.tobytes() == a1.tobytes()
                    and all(q[3] == nd1 and q[4][0] == b1 and q[4][1] == l1 for q in parts)
                    and b"".join(q[4][2] for q in parts) == one.agents_read_blocking(n).tobytes())
            print("tick %d: %d work items, ndirty %d, identical=%s" % (tick, len(work), nd1, good), flush=True)
            ok &= good
        moving = (state_all["state"] != 2) & (state_all["state"] != 4)
    nav.mgpu_finalize(); nav.close()
    if rank == 0:
        one.close()
    return ok


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    ok = run(rank, world, local)
    if rank == 0:
        print("mgpu_nccl_blockers_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
