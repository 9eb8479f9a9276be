"""NCCL transport of job command batches (pfnav_mgpu_commands), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29513 tests/tools/mgpu_nccl_commands_check.py
Every rank uploads only its own entity range and takes the job's whole batch of deltas each round (stops, regrouping
move orders with CLEAR_HIST, a flock appended to the table), then pfnav_mgpu_gather -> agents_set_work_dev -> tick ->
compute_updates -> apply_updates -> pfnav_mgpu_gather. That must give, bit for bit, what ONE context holding the whole
population gives with pfnav_agents_commands (computed on rank 0): work lists, velocities, patches and entity state
(own ranges, concatenated). One batch that only the last rank can refuse (it keeps members of a flock the new table
drops) must fail on every rank and change nothing. Runs at any world size, world 1 included (one H100).
Prints "mgpu_nccl_commands_check PASS world=N" on rank 0. torch.distributed is used only to hand the NCCL id around and
to collect the results for the comparison."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases
import commands_ref as cr

capi = cases.capi
ST_MOVING, ST_ARRIVED = 0, 2


def run(rank, world, local):
    hz, cw = 20, 3
    p, cost, a, ms = cases.update_case(4242, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(5)
    a["vdes"] = rng.normal(size=(n, 2)).astype(np.float32)
    a["vdes"] /= np.linalg.norm(a["vdes"], axis=1, keepdims=True)
    rec, fl = capi.pack_agents(a)
    perm = rng.permutation(n)                         # every flock on every rank
    rec, ms = rec[perm].copy(), ms[perm].copy()
    ids = [capi.mgpu_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    nav = capi.Nav(local)
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.mgpu_init(rank, world, ids[0])
    lo, hi = capi.mgpu_shard_range(n, rank, world)
    nav.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, hz)
    nav.mgpu_gather()
    nav.agents_upload_movestate(ms[lo:hi])
    one = None
    if rank == 0:
        one = capi.Nav(local)
        one.map_create(cw, cw, 1); one.map_upload_layer(0, cost); one.map_build_nav(0); one.route_build(0)
        one.agents_upload(rec, fl, hz); one.agents_upload_movestate(ms)
    ok = True
    state = rec
    for rnd in range(4):
        moving = np.nonzero(state["state"] == ST_MOVING)[0]
        stop = rng.choice(moving, 60, replace=False)
        go = rng.choice(np.setdiff1d(np.arange(n), stop), 90, replace=False)
        d = np.concatenate([cr.deltas(stop, state=ST_ARRIVED, velocity=(0.0, 0.0)),
                            cr.deltas(go, state=ST_MOVING, flock=rng.integers(0, len(fl), len(go)), clear_hist=True)])
        if rnd == 1:
            grown = np.zeros(len(fl) + 1, capi.FLOCK)
            grown[:-1] = fl
            grown["target"][-1], grown["dest"][-1] = state["pos"][go].mean(axis=0), len(fl)
            fl = grown
            d = np.concatenate([d, cr.deltas(go[::2], flock=len(fl) - 1)])
        if rnd == 2:
            # the last rank keeps members of the last flock, which the table drops: every rank refuses
            last = np.nonzero(state["flock"] == len(fl) - 1)[0]
            llo, lhi = capi.mgpu_shard_range(n, world - 1, world)
            if len(last[(last >= llo) & (last < lhi)]):
                try:
                    nav.mgpu_commands(cr.deltas(last[(last < llo) | (last >= lhi)], flock=0), fl[:-1].copy())
                    refused = False
                except capi.PfnavError as e:
                    refused = "error -1" in str(e) and "rank %d" % (world - 1) in str(e)
                parts = [None] * world
                dist.all_gather_object(parts, refused)
                if rank == 0:
                    print("round %d: the stranded-flock batch refused on every rank=%s" % (rnd, all(parts)), flush=True)
                ok &= all(parts)
        nav.mgpu_commands(d, fl if rnd == 1 else None)
        nav.mgpu_gather()
        nw = nav.agents_set_work_dev()
        w = nav.agents_read_work()
        nav.agents_tick(0)
        v = nav.agents_read_velocities(nw)
        nav.agents_compute_updates(); pt = nav.agents_read_patches(nw)
        nav.agents_apply_updates()
        nav.mgpu_gather()
        st = nav.agents_read_state(hi - lo)[0]
        parts = [None] * world
        dist.all_gather_object(parts, (w.tobytes(), v.tobytes(), pt.tobytes(), st.tobytes()))
        state = np.frombuffer(b"".join(q[3] for q in parts), capi.AGENT).copy()
        if rank == 0:
            one.agents_commands(d, fl if rnd == 1 else None)
            one.agents_rebuild_index()
            nw1 = one.agents_set_work_dev()
            w1 = one.agents_read_work()
            one.agents_tick(0)
            v1 = one.agents_read_velocities(nw1)
            one.agents_compute_updates(); p1 = one.agents_read_patches(nw1)
            one.agents_apply_updates()
            one.agents_rebuild_index()
            a1 = one.agents_read_state(n)[0]
            good = (b"".join(q[0] for q in parts) == w1.tobytes() and b"".join(q[1] for q in parts) == v1.tobytes()
                    and b"".join(q[2] for q in parts) == p1.tobytes() and state.tobytes() == a1.tobytes())
            print("round %d: %d deltas, %d work items, identical=%s" % (rnd, len(d), nw1, good), flush=True)
            ok &= good
    res = [None] * world
    dist.all_gather_object(res, ok)
    nav.mgpu_finalize(); nav.close()
    if rank == 0:
        one.close()
    return all(res)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    ok = run(rank, world, local)
    if rank == 0:
        print("mgpu_nccl_commands_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
