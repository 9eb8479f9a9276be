"""NCCL transport of job input-delta batches (pfnav_mgpu_input_deltas), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29514 tests/tools/mgpu_nccl_input_deltas_check.py
Every rank uploads only its own entity range with its movestate_ext table and no formation table, and takes the job's
whole batch each round: turn orders (TURNING through pfnav_mgpu_commands, TARGET_DIR), rot writes, formation records
(the first round creates the table on every rank) and random records of every mask; then pfnav_mgpu_gather ->
agents_set_work_dev -> tick -> compute_updates -> apply_updates -> pfnav_mgpu_gather. That must give, bit for bit, what
ONE context holding the whole population gives with pfnav_agents_input_deltas (computed on rank 0): work lists,
velocities, patches, entity state and both tables (own ranges, concatenated). One batch with a record every rank refuses
must fail on every rank and change nothing. Runs at any world size, world 1 included (one H100).
Prints "mgpu_nccl_input_deltas_check PASS world=N" on rank 0. torch.distributed is used only to hand the NCCL id around
and to collect the results for the comparison."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases
import commands_ref as cr
import inputs_ref as ir

capi = cases.capi
ST_MOVING, ST_TURNING, ST_CELL = 0, 7, 8


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
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID; ext["rot"] = ms["next_rot"]; ext["target_dir"] = ms["next_rot"]
    ids = [capi.mgpu_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    nav = capi.Nav(local)
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.mgpu_init(rank, world, ids[0])
    lo, hi = capi.mgpu_shard_range(n, rank, world)
    nav.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, hz)
    nav.mgpu_gather()
    nav.agents_upload_movestate(ms[lo:hi])
    nav.agents_upload_movestate_ext(ext[lo:hi])
    one = None
    if rank == 0:
        one = capi.Nav(local)
        one.map_create(cw, cw, 1); one.map_upload_layer(0, cost); one.map_build_nav(0); one.route_build(0)
        one.agents_upload(rec, fl, hz); one.agents_upload_movestate(ms); one.agents_upload_movestate_ext(ext)
    ok = True
    state = rec
    for rnd in range(4):
        moving = np.nonzero((state["state"] == ST_MOVING) & ((state["flags"] & capi.FLAG_GARRISONED) == 0))[0]
        who = rng.choice(moving, 160, replace=False)
        turn, rot, form = who[:40], who[40:80], who[80:]
        c = np.concatenate([cr.deltas(turn, state=ST_TURNING), cr.deltas(form[::2], state=ST_CELL)])
        f = np.zeros(len(form), capi.FORMATION_IN)
        f["cell_pos"] = state["pos"][form] + rng.normal(scale=5.0, size=(len(form), 2)).astype(np.float32)
        v = rng.normal(size=(len(form), 2)); f["cell_arrival_vdes"] = v / np.linalg.norm(v, axis=1, keepdims=True)
        f["flags"] = capi.FORM_HAS_FORMATION | capi.FORM_ASSIGNMENT_READY | capi.FORM_ASSIGNED_TO_CELL
        d = np.concatenate([ir.inputs(turn, target_dir=cases.dir_quat(rng.normal(size=(len(turn), 2)))),
                            ir.inputs(rot, rot=cases.dir_quat(-state["velocity"][rot])),
                            ir.inputs(form, formation=f), ir.random_inputs(rng, 200, who)])
        if rnd == 2:
            bad = d.copy()
            bad["mask"][-1] = capi.INPUT_SURROUND_FIELD; bad["using_surround_field"][-1] = 2
            try:
                nav.mgpu_input_deltas(bad)
                refused = False
            except capi.PfnavError as e:
                refused = "error -1" in str(e)
            parts = [None] * world
            dist.all_gather_object(parts, refused)
            if rank == 0:
                print("round %d: the bad batch refused on every rank=%s" % (rnd, all(parts)), flush=True)
            ok &= all(parts)
        nav.mgpu_commands(c)
        nav.mgpu_input_deltas(d)
        nav.mgpu_gather()
        tabs = (nav.agents_read_movestate_ext(hi - lo).tobytes(), nav.agents_read_formation(hi - lo).tobytes())
        nw = nav.agents_set_work_dev()
        w = nav.agents_read_work()
        nav.agents_tick(0)
        v = nav.agents_read_velocities(nw)
        nav.agents_compute_updates(); pt = nav.agents_read_patches(nw)
        nav.agents_apply_updates()
        nav.mgpu_gather()
        st = nav.agents_read_state(hi - lo)[0]
        parts = [None] * world
        dist.all_gather_object(parts, (w.tobytes(), v.tobytes(), pt.tobytes(), st.tobytes()) + tabs)
        state = np.frombuffer(b"".join(q[3] for q in parts), capi.AGENT).copy()
        if rank == 0:
            one.agents_commands(c)
            one.agents_input_deltas(d)
            one.agents_rebuild_index()
            t1 = (one.agents_read_movestate_ext(n).tobytes(), one.agents_read_formation(n).tobytes())
            nw1 = one.agents_set_work_dev()
            w1 = one.agents_read_work()
            one.agents_tick(0)
            v1 = one.agents_read_velocities(nw1)
            one.agents_compute_updates(); p1 = one.agents_read_patches(nw1)
            one.agents_apply_updates()
            one.agents_rebuild_index()
            a1 = one.agents_read_state(n)[0]
            good = (b"".join(q[0] for q in parts) == w1.tobytes() and b"".join(q[1] for q in parts) == v1.tobytes()
                    and b"".join(q[2] for q in parts) == p1.tobytes() and state.tobytes() == a1.tobytes()
                    and b"".join(q[4] for q in parts) == t1[0] and b"".join(q[5] for q in parts) == t1[1])
            print("round %d: %d records, %d work items, identical=%s" % (rnd, len(d), nw1, good), flush=True)
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
        print("mgpu_nccl_input_deltas_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
