"""NCCL form of the entity-field batch named by uid (pfnav_mgpu_request_entity_fields_resident), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29515 tests/tools/mgpu_nccl_entity_fields_resident_check.py
Every rank holds a job member (its shard of one population, gathered) and a single context with the map and pool only,
which takes pfnav_pool_request_entity_fields_batch on the footprints and seeker chunks built in numpy from the records
read back. Every member's pool must equal its single context's for every (dest, chunk) -- has bits, ff_id, flow bytes.
Then rank 0 uploads its shard again without a gather: every rank must return PFNAV_ERR_STATE with no pool changed, and
after the gather the call succeeds again. World 1 runs on one GPU; world >= 2 needs as many GPUs.
Prints "mgpu_nccl_entity_fields_resident_check PASS world=N" on rank 0. torch.distributed is used only to hand the NCCL
id around and to collect the results."""
import ctypes as C
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases
from test_gpu_entity_field_batch import _pool
from test_gpu_entity_fields_resident import batch_case, resolve
from test_gpu_mgpu_commands import _population

capi = cases.capi


def _ctx(local, cost, nd):
    X = capi.Nav(local)
    X.map_create(3, 3, 1)
    X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
    X.pool_create(nd, nd * 9)
    return X


def run(rank, world, local):
    cost, rec, fl, _ = _population(4242, 20)
    n, nd = len(rec), len(fl) + 10
    ids = [capi.mgpu_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    nav, one = _ctx(local, cost, nd), _ctx(local, cost, nd)
    nav.mgpu_init(rank, world, ids[0])
    lo, hi = capi.mgpu_shard_range(n, rank, world)
    nav.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, 20)
    nav.mgpu_gather()
    one.agents_upload(rec, fl, 20)                      # read back for twin A's inputs only
    reqs, fp, uids, seekers = batch_case(3, 3, n, 24, nd, 13)
    ra, fa, ca = resolve(one, n, reqs, fp, uids, seekers, 3, 3)
    nav.mgpu_request_entity_fields_resident(reqs, fp, uids, seekers)
    same = one.pool_request_entity_fields_batch(ra, fa, ca) == len(reqs) and _pool(nav, nd, 3, 3) == _pool(one, nd, 3, 3)
    if rank == 0:
        nav.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, 20, capi.UPLOAD_SAME_FLOCKS)
    before = _pool(nav, nd, 3, 3)
    a = capi._resident_args(reqs, fp, uids, seekers)
    rc = nav.L.pfnav_mgpu_request_entity_fields_resident(nav.h, *a[:7], C.c_void_p(0))
    refused = rc == capi.ERR_STATE and _pool(nav, nd, 3, 3) == before
    nav.mgpu_gather()
    nav.mgpu_request_entity_fields_resident(reqs, fp, uids, seekers)
    again = _pool(nav, nd, 3, 3) == before
    parts = [None] * world
    dist.all_gather_object(parts, (same, refused, again))
    if rank == 0:
        print("per rank (equal, stale refused, equal again): %s" % parts, flush=True)
    nav.mgpu_finalize(); nav.close(); one.close()
    return all(all(p) for p in parts)


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    ok = run(rank, world, local)
    if rank == 0:
        print("mgpu_nccl_entity_fields_resident_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
