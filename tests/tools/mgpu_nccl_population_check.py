"""NCCL transport of job population changes (pfnav_mgpu_change_population), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29514 tests/tools/mgpu_nccl_population_check.py
Every rank uploads only its own entity range and takes the job's whole population change each round (removals spread
over the population, appended entities copied from survivors, a flock appended to the table), then pfnav_mgpu_gather ->
agents_set_work_dev -> tick -> compute_updates -> apply_updates -> pfnav_mgpu_gather. That must give, bit for bit, what
ONE context holding the whole population gives with pfnav_agents_change_population (computed on rank 0): work lists,
velocities, patches and entity state (own ranges, concatenated; every rank owns the balanced range of the new
population). One change that only the last rank can refuse (it keeps members of a flock the new table drops) must fail on
every rank and change nothing. Runs at any world size, world 1 included (one H100).
Prints "mgpu_nccl_population_check PASS world=N" on rank 0. torch.distributed is used only to hand the NCCL id around
and to collect the results for the comparison."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases

capi = cases.capi
ST_MOVING = 0


def run(rank, world, local):
    hz, cw = 20, 3
    p, cost, a, ms = cases.update_case(4242, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(5)
    nf0 = len(a["flock_target"])
    a["flock_dest_index"] = np.arange(nf0, dtype=np.int32)
    rec, fl = capi.pack_agents(a)
    perm = rng.permutation(n)                         # every flock on every rank
    rec, ms = rec[perm].copy(), ms[perm].copy()
    ids = [capi.mgpu_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    ndests = nf0 + 3

    def make(X):
        X.map_create(cw, cw, 1); X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
        X.pool_create(ndests, ndests * cw * cw)

    nav = capi.Nav(local)
    make(nav)
    nav.mgpu_init(rank, world, ids[0])
    lo, hi = capi.mgpu_shard_range(n, rank, world)
    nav.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, hz)
    nav.mgpu_gather()
    nav.agents_upload_movestate(ms[lo:hi])
    one = None
    if rank == 0:
        one = capi.Nav(local)
        make(one)
        one.agents_upload(rec, fl, hz); one.agents_upload_movestate(ms)
    ok = True
    state, mstate = rec, ms
    for rnd in range(4):
        k = 40 + 20 * rnd
        rm = rng.choice(n, k, replace=False)
        who = rng.choice(np.nonzero(state["state"] == ST_MOVING)[0], k // 2, replace=False)
        add = state[who].copy(); add["pos"] += np.float32(0.5); add["prev_pos"] += np.float32(0.5)
        add_ms = mstate[who].copy(); add_ms["next_pos"][:, 0] += np.float32(0.5); add_ms["next_pos"][:, 2] += np.float32(0.5)
        newfl = None
        if rnd == 1:
            newfl = np.zeros(len(fl) + 1, capi.FLOCK)
            newfl[:-1] = fl
            newfl["target"][-1], newfl["dest"][-1] = state["pos"][who].mean(axis=0), len(fl)
            fl = newfl
            add["flock"][::2] = len(fl) - 1
        if rnd == 2:
            # the last rank keeps members of the last flock, which the table drops: every rank refuses
            last = np.nonzero(state["flock"] == len(fl) - 1)[0]
            llo, lhi = capi.mgpu_shard_range(n, world - 1, world)
            if len(last[(last >= llo) & (last < lhi)]):
                try:
                    nav.mgpu_change_population(last[(last < llo) | (last >= lhi)], np.zeros(0, capi.AGENT),
                                               ms=np.zeros(0, capi.MOVESTATE), flocks=fl[:-1].copy())
                    refused = False
                except capi.PfnavError as e:
                    refused = "error -1" in str(e) and "rank %d" % (world - 1) in str(e)
                parts = [None] * world
                dist.all_gather_object(parts, refused)
                if rank == 0:
                    print("round %d: the stranded-flock change refused on every rank=%s" % (rnd, all(parts)), flush=True)
                ok &= all(parts)
        nav.mgpu_change_population(rm, add, ms=add_ms, flocks=newfl)
        n = n - len(rm) + len(add)
        lo, hi = capi.mgpu_shard_range(n, rank, world)
        nav.mgpu_gather()
        nw = nav.agents_set_work_dev()
        w = nav.agents_read_work()
        nav.agents_tick(capi.TICK_VDES_FROM_POOL); nav.pool_repair(); nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        v = nav.agents_read_velocities(nw)
        nav.agents_compute_updates(); pt = nav.agents_read_patches(nw)
        nav.agents_apply_updates()
        nav.mgpu_gather()
        st, mst = nav.agents_read_state(hi - lo)
        parts = [None] * world
        dist.all_gather_object(parts, (w.tobytes(), v.tobytes(), pt.tobytes(), st.tobytes(), mst.tobytes()))
        state = np.frombuffer(b"".join(q[3] for q in parts), capi.AGENT).copy()
        mstate = np.frombuffer(b"".join(q[4] for q in parts), capi.MOVESTATE).copy()
        if rank == 0:
            one.agents_change_population(rm, add, ms=add_ms, flocks=newfl)
            nw1 = one.agents_set_work_dev()
            w1 = one.agents_read_work()
            one.agents_tick(capi.TICK_VDES_FROM_POOL); one.pool_repair(); one.agents_tick(capi.TICK_VDES_FROM_POOL)
            v1 = one.agents_read_velocities(nw1)
            one.agents_compute_updates(); p1 = one.agents_read_patches(nw1)
            one.agents_apply_updates()
            one.agents_rebuild_index()
            a1, m1 = one.agents_read_state(n)
            good = (b"".join(q[0] for q in parts) == w1.tobytes() and b"".join(q[1] for q in parts) == v1.tobytes()
                    and b"".join(q[2] for q in parts) == p1.tobytes() and state.tobytes() == a1.tobytes()
                    and mstate.tobytes() == m1.tobytes())
            print("round %d: -%d +%d entities, n=%d, %d work items, identical=%s" % (rnd, len(rm), len(add), n, nw1, good), flush=True)
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
        print("mgpu_nccl_population_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
