"""The cold goal request (pfnav_pool_clear + pfnav_pool_request_goals) on the C2 workload: pool_clear only marks the
device pool stale and the batch queues without host waits, so these check what that must not change.

  * back-to-back cold steps on one stream with no host synchronisation compute what the same steps compute with a
    device synchronisation after each;
  * a pool_clear directly followed by a tick, a pool_get or a pool_repair sees an empty pool;
  * the pool after one cold batch of the C2 goals is byte-identical to what the implementation with the blocking
    clear and the synchronous upload produced (digest in tests/golden/cold_batch_c2.sha256).

python tests/test_gpu_cold_request.py prints the digest of the tree it runs in. tests/golden/cold_batch_c2.sha256 was
recorded that way on an H100, in the tree of the implementation before the non-blocking cold request (blocking
pool_clear, host waits and a pageable, synchronised upload in the goal batch). It is a regression baseline of the
CUDA path, not a reference output: a sha256 over the flow / LOS request counts and every (destination, chunk) entry of
the pool read back with pfnav_pool_get (has bits, ffid, flow and LOS bytes). Slot numbers are not visible through the
ABI; they enter the digest only through what each entry reads back."""
import hashlib
import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(ROOT, "tests", "golden", "cold_batch_c2.sha256")


def _setup(pf, agents=True):
    """a fresh context on the bench's C2 workload: map, pool, population, work list -> (nav, W, dests, targets)"""
    bench = importlib.import_module("bench")
    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    capi, cw = pf.capi, bench.CHUNKS
    nav = capi.Nav(0)
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0)
    ngoals = W["g_hi"] - W["g_lo"]
    nav.pool_create(ngoals, ngoals * cw * cw)
    if agents:
        nav.agents_upload_shard(W["rec"][W["lo"]:W["hi"]], W["lo"], W["hi"], W["n_total"], W["flocks"], bench.HZ, 0)
        nav.agents_set_work(np.arange(W["lo"], W["hi"], dtype=np.uint32))
    dests = np.arange(ngoals, dtype=np.int32)
    targets = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(W["g_lo"], W["g_hi"])], np.int32)
    return nav, W, dests, targets


def _pool_bytes(nav, ndests, nchunks):
    """every (dest, chunk) entry read back: has bits, ffid, flow and LOS bytes"""
    out = []
    for d in range(ndests):
        for c in range(nchunks):
            f, l, ffid = nav.pool_get(d, divmod(c, nav.cw))
            out.append((int(f is not None) | int(l is not None) << 1, ffid,
                        b"" if f is None else f.tobytes(), b"" if l is None else l.tobytes()))
    return out


def cold_batch_digest(pf):
    """sha256 over the field counts and the whole pool after one cold batch of the C2 goals"""
    nav, W, dests, targets = _setup(pf, agents=False)
    try:
        nav.pool_clear()
        nf, nl = nav.pool_request_goals(dests, targets, 0)
        h = hashlib.sha256(np.array([nf, nl], np.int64).tobytes())
        for has, ffid, f, l in _pool_bytes(nav, len(dests), nav.cw * nav.cw):
            h.update(np.array([has, ffid], np.uint64).tobytes()); h.update(f); h.update(l)
        return h.hexdigest()
    finally:
        nav.close()


def test_cold_batch_pool_golden(pf):
    with open(GOLDEN) as f:
        want = f.read().split()[0]
    assert cold_batch_digest(pf) == want


def test_back_to_back_cold_steps_match_synchronised(pf):
    """K cold steps (pool_clear + pool_request_goals + index + tick) queued on one stream without a host wait, against
    the same K steps with torch.cuda.synchronize() after each: pool bytes, desired velocities, LOS flags and velocities
    of the last tick are identical. Both runs split the velocity update the same way (two-phase forced), so that the
    comparison does not depend on how far the host runs ahead."""
    import torch
    capi = pf.capi
    results = []
    for sync in (False, True):
        nav, W, dests, targets = _setup(pf)
        try:
            nav.set_two_phase(2)
            stream = torch.cuda.Stream()
            sp = stream.cuda_stream
            for _ in range(4):
                nav.pool_clear()
                nav.pool_request_goals(dests, targets, 0, sp)
                nav.agents_rebuild_index(sp)
                nav.agents_tick(capi.TICK_VDES_FROM_POOL, sp)
                if sync:
                    torch.cuda.synchronize()
            torch.cuda.synchronize()
            nwork = W["hi"] - W["lo"]
            vpref, vdes, los = nav.agents_read_debug(nwork)
            results.append((_pool_bytes(nav, len(dests), nav.cw * nav.cw), vdes, los, nav.agents_read_velocities(nwork)))
        finally:
            nav.close()
    (pa, da, la, va), (pb, db, lb, vb) = results
    assert pa == pb
    assert np.array_equal(da, db) and np.array_equal(la, lb) and np.array_equal(va, vb)
    assert (np.abs(da).sum(axis=1) > 0).mean() > 0.99        # the ticks did read the fields


def test_clear_then_tick_get_repair_see_empty_pool(pf):
    """pool_clear marks the device pool stale; the next entry point brings it up to date on its own stream. A tick, a
    pool_get and a pool_repair right after a clear see an empty pool: no desired velocity, no LOS flag, no entry, and
    the same misses as a context whose pool was never filled."""
    import torch
    capi = pf.capi
    nav, W, dests, targets = _setup(pf)
    fresh, _, _, _ = _setup(pf)
    try:
        nwork = W["hi"] - W["lo"]
        nav.pool_request_goals(dests, targets, 0)
        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        torch.cuda.synchronize()
        assert (np.abs(nav.agents_read_debug(nwork)[1]).sum(axis=1) > 0).mean() > 0.99
        nav.pool_clear()
        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        _, vdes, los = nav.agents_read_debug(nwork)
        assert not vdes.any() and not los.any()
        nav.pool_request_goals(dests, targets, 0)
        nav.pool_clear()
        assert all(e == (0, 0, b"", b"") for e in _pool_bytes(nav, len(dests), nav.cw * nav.cw))
        # the on-miss chain on a sample of the population (N_RequestPath per miss needs the portal graph)
        work = np.sort(np.random.default_rng(5).choice(np.arange(W["lo"], W["hi"]), 2000, replace=False)).astype(np.uint32)
        for n in (nav, fresh):
            n.route_build(0)
            n.agents_set_work(work)
        nav.pool_request_goals(dests, targets, 0)
        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        nav.pool_clear()
        assert nav.pool_repair() == fresh.pool_repair()
        assert _pool_bytes(nav, len(dests), nav.cw * nav.cw) == _pool_bytes(fresh, len(dests), nav.cw * nav.cw)
    finally:
        fresh.close()
        nav.close()


def test_resident_plan_only_on_an_unchanged_pool(pf):
    """A repeated identical goal batch relaunches its resident plan without planning again. A pool_put, a pool_clear, a
    map_commit that drops fields, a zone batch or an entity-field batch changes the pool under the plan: the next
    identical batch plans again."""
    capi = pf.capi
    nav, W, dests, targets = _setup(pf, agents=False)
    try:
        nav.profile_enable(True)
        x, z = -(100 * 4 + 2.0), 100 * 4 + 2.0              # world position of tile (100, 100), in chunk (1, 1)
        zone = np.zeros(1, capi.ZONE_REQ)
        zone["dest"], zone["centre_x"], zone["centre_z"], zone["radius"] = 0, x, z, 6
        ent = np.zeros(1, capi.ENTITY_FIELD_REQ)
        ent["dest"], ent["target_kind"], ent["ent_n"], ent["chunk_n"] = 1, capi.TARGET_ENTITY, 1, 1
        fp = np.zeros(1, capi.FOOTPRINT)
        fp["x"], fp["z"], fp["sel_radius"] = x, z, 3.0

        def commit():
            nav.blockers_incref(x, z, 3.0)
            assert nav.map_commit() > 0

        changes = {"put": lambda: nav.pool_put(0, (0, 0), flow=np.zeros(4096, np.uint8)),
                   "clear": nav.pool_clear,
                   "commit": commit,
                   "zones": lambda: nav.pool_request_zones(zone),
                   "entity": lambda: nav.pool_request_entity_fields_batch(ent, fp, np.array([[1, 1]], np.int32))}

        def plans():            # planning passes of one goal batch (profile_read_host returns the counts since its last call)
            nav.pool_request_goals(dests, targets, 0)
            return nav.profile_read_host()["plan"][1]

        assert plans() == 1
        assert plans() == 0, "the repeated batch planned again"
        for name, change in changes.items():
            change()
            assert plans() == 1, "the batch after %s reused the resident plan" % name
            assert plans() == 0, "the repeated batch after %s planned again" % name
    finally:
        nav.close()


if __name__ == "__main__":
    print(cold_batch_digest(importlib.import_module("permafrost-engine_b200")))
