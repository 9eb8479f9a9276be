"""NCCL transport of a job's zone and entity-field batches (pfnav_mgpu_request_zones,
pfnav_mgpu_request_entity_fields_batch), one process per GPU:
    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29514 tests/tools/mgpu_nccl_aux_fields_check.py
Every rank holds a job member and a single context built from the same seeds that gets the same calls, with the solo
batch in place of the job's. Zone batches (a few large zones with a repeated dest and one centred off the map, then 80
small ones) and entity-field batches (mixed TARGET_ENEMIES / TARGET_ENTITY requests with shared footprint ranges and
repeated keys), after rank-specific earlier batches so that the ranks' pools differ: every member's pool must equal its
single context's for every (dest, chunk) -- has bits, ff_id, flow bytes -- with the same field counts; every rank must
report the same owners, and the ranks' built fields must add up to the distinct keys written. World 1 runs on one GPU;
world >= 2 needs as many GPUs (NCCL puts no two ranks on one GPU).
Prints "mgpu_nccl_aux_fields_check PASS world=N" on rank 0. torch.distributed is used only to hand the NCCL id around
and to collect the results for the comparison."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import torch
import torch.distributed as dist
import cases
from test_gpu_entity_field_batch import _mixed
from test_gpu_mgpu_aux_fields import _entity_keys, _nav, _pool, _zone_case, _zone_keys
from test_gpu_zone_batch import _reqs, _xz

capi = cases.capi


def run(rank, world, local):
    cw, nd = 4, 90
    rng = np.random.default_rng(21)
    cost, tiles, radii = _zone_case(cw, 0x5EED0A07, 84, [3, 6, 10, 16], rng)
    ids = [capi.mgpu_unique_id() if rank == 0 else None]
    dist.broadcast_object_list(ids, src=0)
    nav = _nav(local, cost, cw, nd, nd * cw * cw)
    one = _nav(local, cost, cw, nd, nd * cw * cw)
    nav.mgpu_init(rank, world, ids[0])
    fp, ereqs, chunks = _mixed(cw, cw, 200, 120, 80, 7)
    ok = True

    def check(label, keys, m, same):
        nonlocal ok
        last = {}
        for i, ks in enumerate(keys):
            for k in ks:
                last[k] = i
        built, _, owner = nav.mgpu_fields_stats(m)
        parts = [None] * world
        dist.all_gather_object(parts, (same, built, owner.tolist()))
        good = (all(q[0] for q in parts) and all(q[2] == parts[0][2] for q in parts)
                and sum(q[1] for q in parts) == len(last)
                and all((parts[0][2][i] >= 0) == (i in set(last.values())) for i in range(m)))
        if rank == 0:
            print("%s: %d keys, built per rank %s, identical=%s" % (label, len(last), [q[1] for q in parts], good), flush=True)
        ok &= good

    def zones(reqs, t, label):
        got = nav.mgpu_request_zones(reqs)
        nd_, want = one.pool_request_zones(reqs)
        check(label, _zone_keys(reqs, t, cw), len(reqs),
              nd_ == len(reqs) and np.array_equal(got, want) and _pool(nav, nd) == _pool(one, nd))

    def entity(reqs, label):
        nav.mgpu_request_entity_fields_batch(reqs, fp, chunks)
        n = one.pool_request_entity_fields_batch(reqs, fp, chunks)
        check(label, _entity_keys(reqs, chunks, cw), len(reqs), n == len(reqs) and _pool(nav, nd) == _pool(one, nd))

    for X in (nav, one):                        # rank-specific earlier batches: the ranks hold different fields
        X.pool_request_entity_fields_batch(ereqs[rank % 5 * 10:rank % 5 * 10 + 10], fp, chunks)
    big = tiles[:3] + [None] + tiles[3:4]
    xz = [(1000.0, -1000.0) if t is None else _xz(t) for t in big]
    zones(_reqs([(d, p, r) for d, p, r in zip([80, 81, 81, 82, 83], xz, [40, 60, 90, 30, 80])]), big, "large zones")
    small = tiles[4:]
    zones(_reqs([(i, _xz(t), r) for i, (t, r) in enumerate(zip(small, radii[4:]))]), small, "80 small zones")
    entity(ereqs, "entity fields")
    entity(ereqs[:40], "entity fields again")
    nav.mgpu_finalize(); nav.close(); one.close()
    return ok


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("gloo")
    ok = run(rank, world, local)
    if rank == 0:
        print("mgpu_nccl_aux_fields_check %s world=%d" % ("PASS" if ok else "FAIL", world), flush=True)
    dist.destroy_process_group()
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
