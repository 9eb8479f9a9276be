"""pfnav_ents_in_circles on the device: batches of G_Pos_EntsInCircle[From] queries against the plain-C port's
pfo_ents_in_circle (oracle/pf_oracle.c, pinned to the reference by tests/test_oracle.py) and against the single-query
pfnav_ents_in_circle, uid for uid and in order. The populations: a 1 500-entity world with and without GARRISONED
entities (every walk, the cut at maxout, filter_garrisoned's swap-remove), a query centred on every entity of the bench's
C2 population at the tick's two ranges, and a sample of C3 with the whole million present. Then the call's contract:
n == 0, the capacity retry, every argument error, the stale-index refusal, and groups of 2 and 3 members answering every
query exactly as one context holding the whole population."""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import pytest

import cases
from test_gpu_mgpu_commands import Job, _population

pytestmark = pytest.mark.gpu
capi = cases.capi
NULL = capi.NULL_UID
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def bench():
    return importlib.import_module("bench")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def queries(rows):
    q = np.zeros(len(rows), capi.ENTS_QUERY)
    for i, (x, z, r, uid, maxout) in enumerate(rows):
        q[i] = (x, z, r, uid, maxout, 0)
    return q


def raw_call(nav, q, cap, offsets=None, ids=None, total=None, stream=0):
    """pfnav_ents_in_circles itself -> (rc, offsets, ids, total)"""
    q = np.ascontiguousarray(q, capi.ENTS_QUERY)
    offsets = np.full(len(q) + 1, 0xDEAD, np.uint32) if offsets is None else offsets
    ids = np.full(max(cap, 1), 0xBEEF, np.uint32) if ids is None else ids
    t = C.c_size_t(12345 if total is None else total)
    rc = nav.L.pfnav_ents_in_circles(nav.h, _p(q) if len(q) else None, len(q), _p(offsets), _p(ids), cap, C.byref(t),
                                     C.c_void_p(stream))
    return rc, offsets, ids, t.value


def expected(port, pos, q):
    out = []
    for r in q:
        x, z = (float(r["x"]), float(r["z"])) if r["uid"] == NULL else (float(pos[r["uid"], 0]), float(pos[r["uid"], 1]))
        out.append(port.ents_in_circle(x, z, float(r["range"]), int(r["maxout"])))
    return out


def check(nav, port, pos, q, singles=True):
    """the batch equals the port and, query by query, pfnav_ents_in_circle at the same centre"""
    off, ids = nav.ents_in_circles(q)
    assert off[0] == 0 and len(ids) == off[-1] and (np.diff(off.astype(np.int64)) >= 0).all()
    want = expected(port, pos, q)
    bad = [i for i in range(len(q)) if not np.array_equal(ids[off[i]:off[i + 1]], want[i])]
    assert not bad, (len(bad), [(int(i), tuple(q[i]), ids[off[i]:off[i + 1]][:6], want[i][:6]) for i in bad[:3]])
    if singles:
        for i, r in enumerate(q):
            if r["maxout"] == 0:
                continue
            x, z = (float(r["x"]), float(r["z"])) if r["uid"] == NULL else (float(pos[r["uid"], 0]), float(pos[r["uid"], 1]))
            assert np.array_equal(nav.ents_in_circle(x, z, float(r["range"]), int(r["maxout"])), want[i]), i
    return off, ids


class Small:
    """a 1 500-entity population on a 3 x 3-chunk map, in the port and on the device"""

    def __init__(self, pforacle, nav, seed, garrisoned):
        _, cost, a = cases.agent_case(3, 1500, 3, seed, 0.03, 2.6)
        if garrisoned:
            g = np.random.default_rng(seed + 17).random(len(a["radius"])) < garrisoned
            a["flags"] = a["flags"] | np.where(g, capi.FLAG_GARRISONED, 0).astype(a["flags"].dtype)
        self.rec, fl = capi.pack_agents(a)
        self.pos = self.rec["pos"]
        self.port = pforacle.OracleWorld(pforacle.OracleMap(3, 3, cost), self.rec, fl, 20)
        nav.map_create(3, 3, 1); nav.map_upload_layer(0, cost)
        nav.agents_upload(self.rec, fl, 20)

    def case_queries(self, rng):
        n, span = len(self.rec), 3 * 256.0
        rows = []
        for u in rng.choice(n, 40, replace=False):
            for r in (0.0, 1.5, 10.0, 30.0, 46.875, 46.875 + 1.0 / 256, 60.0):
                for m in (1, 32, 512):
                    rows.append((float(self.pos[u, 0]), float(self.pos[u, 1]), r, NULL, m))
                    rows.append((0.0, 0.0, r, int(u), m))
        rows += [(-span / 2, span / 2, r, NULL, m) for r in (0.45 * span, 2 * span) for m in (32, 512, 5000)]
        rows += [(300.0, 300.0, 10.0, NULL, 512), (-span / 2, -200.0, 30.0, NULL, 512), (20.0, float(self.pos[0, 1]), 30.0, NULL, 512),
                 (0.0, 0.0, -1.0, 5, 512), (0.0, 0.0, 30.0, 5, 0), (float(self.pos[1, 0]), float(self.pos[1, 1]), 30.0, NULL, 0)]
        return queries(rows)


@pytest.mark.parametrize("garrisoned", [0.0, 0.15])
def test_case_batches(pforacle, nav, garrisoned):
    W = Small(pforacle, nav, 3131, garrisoned)
    try:
        q = W.case_queries(np.random.default_rng(5))
        off, ids = check(nav, W.port, W.pos, q)
        lens = np.diff(off.astype(np.int64))
        assert (lens[q["maxout"] == 1] <= 1).all()
        assert lens.max() >= 512 and (lens == 0).sum() >= 5
        if garrisoned:        # the cut holds GARRISONED entities, and the swap-remove reorders the survivors
            garr = (W.rec["flags"] & capi.FLAG_GARRISONED) != 0
            moved = 0
            for i, r in enumerate(q):
                if r["uid"] == NULL or r["range"] < 10.0:
                    continue
                x, z = float(W.pos[r["uid"], 0]), float(W.pos[r["uid"], 1])
                cut = W.port.ents_in_circle(x, z, float(r["range"]), 1 << 20)[:int(r["maxout"])]
                moved += not np.array_equal(ids[off[i]:off[i + 1]], cut[~garr[cut]])
            assert moved > 20
        # the same batch split across calls, on a stream of the caller's
        import torch
        s = torch.cuda.Stream()
        h = len(q) // 3
        o2, i2 = nav.ents_in_circles(q[h:], stream=s.cuda_stream)
        assert np.array_equal(i2, ids[off[h]:]) and np.array_equal(o2.astype(np.int64), off[h:].astype(np.int64) - off[h])
    finally:
        W.port.close()


def _bench_population(pf, bench, workload):
    bench.set_workload(workload)
    try:
        W = bench.build_workload(pf, 1, 0)
    finally:
        bench.set_workload("C2")
    rec, fl = capi.pack_agents(W["agents"])
    return W, rec, fl


def test_c2_every_entity(pf, pforacle, nav, bench):
    """a query centred on every entity of the bench's C2 population at 10 wu (maxout 512) and 30 wu (maxout 128)"""
    W, rec, fl = _bench_population(pf, bench, "C2")
    port = pforacle.OracleWorld(pforacle.OracleMap(bench.CHUNKS, bench.CHUNKS, W["cost"]), rec, fl, 20)
    try:
        nav.map_create(bench.CHUNKS, bench.CHUNKS, 1); nav.map_upload_layer(0, W["cost"])
        nav.agents_upload(rec, fl, 20)
        n = len(rec)
        q = np.zeros(2 * n, capi.ENTS_QUERY)
        q["uid"] = np.tile(np.arange(n, dtype=np.uint32), 2)
        q["range"][:n], q["maxout"][:n], q["range"][n:], q["maxout"][n:] = 10.0, 512, 30.0, 128
        off, ids = check(nav, port, rec["pos"], q, singles=False)
        for k in range(len(q)):
            i = int(q["uid"][k])
            got = nav.ents_in_circle(float(rec["pos"][i, 0]), float(rec["pos"][i, 1]), float(q["range"][k]), int(q["maxout"][k]))
            assert np.array_equal(got, ids[off[k]:off[k + 1]]), k
        assert np.diff(off.astype(np.int64))[n:].max() == 128
    finally:
        port.close()


def test_c3_sample_whole_population(pf, pforacle, nav, bench):
    """20 000 uid-centred and point queries on C3 with the whole million entities in the index"""
    W, rec, fl = _bench_population(pf, bench, "C3")
    port = pforacle.OracleWorld(pforacle.OracleMap(bench.CHUNKS, bench.CHUNKS, W["cost"]), rec, fl, 20)
    try:
        nav.map_create(bench.CHUNKS, bench.CHUNKS, 1); nav.map_upload_layer(0, W["cost"])
        nav.agents_upload(rec, fl, 20)
        rng = np.random.default_rng(21)
        u = rng.choice(len(rec), 5000, replace=False)
        rows = [(0.0, 0.0, r, int(i), m) for i in u for r, m in ((10.0, 512), (30.0, 128))]
        rows += [(float(rec["pos"][i, 0]) + 0.5, float(rec["pos"][i, 1]) - 0.5, r, NULL, m) for i in u for r, m in ((10.0, 512), (30.0, 128))]
        q = queries(rows)
        off, ids = check(nav, port, rec["pos"], q, singles=False)
        for k in range(0, len(q), 10):
            r = q[k]
            x, z = (float(r["x"]), float(r["z"])) if r["uid"] == NULL else map(float, rec["pos"][r["uid"]])
            assert np.array_equal(nav.ents_in_circle(x, z, float(r["range"]), int(r["maxout"])), ids[off[k]:off[k + 1]]), k
    finally:
        port.close()


def test_contract(pforacle, nav):
    """n == 0, the capacity retry, every argument error (outputs untouched) and a host-only context"""
    W = Small(pforacle, nav, 77, 0.0)
    try:
        q = W.case_queries(np.random.default_rng(3))
        off_full, ids_full = nav.ents_in_circles(q)
        total = len(ids_full)
        # n == 0
        rc, o, _, t = raw_call(nav, q[:0], 0)
        assert rc == capi.OK and t == 0 and o[0] == 0
        # capacity: PFNAV_ERR_NOMEM with the offsets and the total written, ids untouched; then success after growing
        rc, o, ids, t = raw_call(nav, q, total - 1)
        assert rc == capi.ERR_NOMEM and t == total and np.array_equal(o, off_full) and (ids == 0xBEEF).all()
        rc, o, ids, t = raw_call(nav, q, 0, ids=np.full(1, 0xBEEF, np.uint32))
        assert rc == capi.ERR_NOMEM and t == total and (ids == 0xBEEF).all()
        rc, o, ids, t = raw_call(nav, q, total)
        assert rc == capi.OK and t == total and np.array_equal(o, off_full) and np.array_equal(ids[:total], ids_full)
        # argument errors: nothing written
        n = len(W.rec)
        bad = [("x", np.nan), ("z", np.inf), ("range", np.nan), ("range", -np.inf), ("maxout", -1), ("uid", n),
               ("uid", NULL - 1)]
        for field, v in bad:
            qb = q.copy()
            qb[len(qb) // 2][field] = v
            rc, o, ids, t = raw_call(nav, qb, total)
            assert rc == capi.ERR_ARG and t == 12345 and (o == 0xDEAD).all() and (ids == 0xBEEF).all(), (field, v)
        # answers that could pass 2^32 uids: 2 863 312 queries that may each hold all 1 500 entities
        big = np.zeros(2_863_312, capi.ENTS_QUERY)
        big["range"], big["uid"], big["maxout"] = 10.0, 0, 1500
        assert n == 1500 and raw_call(nav, big, 0)[0] == capi.ERR_ARG
        assert raw_call(nav, big[:-1], 0)[0] == capi.ERR_NOMEM
        nav2 = capi.Nav(0)
        try:
            ok = raw_call(nav2, q[:1], 8)[0]
            assert ok == capi.ERR_ARG                                           # no population uploaded
        finally:
            nav2.close()
        L, h = nav.L, nav.h
        t = C.c_size_t(7)
        o = np.zeros(len(q) + 1, np.uint32)
        assert L.pfnav_ents_in_circles(h, None, 3, _p(o), None, 0, C.byref(t), None) == capi.ERR_ARG
        assert L.pfnav_ents_in_circles(h, _p(q), 3, None, None, 0, C.byref(t), None) == capi.ERR_ARG
        assert L.pfnav_ents_in_circles(h, _p(q), 3, _p(o), None, 0, None, None) == capi.ERR_ARG
        assert L.pfnav_ents_in_circles(h, _p(q), 3, _p(o), None, 8, C.byref(t), None) == capi.ERR_ARG
        assert t.value == 7
        ho = capi.Nav(hostonly=True)
        try:
            assert L.pfnav_ents_in_circles(ho.h, _p(q), 3, _p(o), None, 0, C.byref(t), None) == capi.ERR_NO_DEVICE
        finally:
            ho.close()
    finally:
        W.port.close()


def test_stale_index_refused(pforacle):
    """records written by apply_updates or agents_commands leave the index stale: PFNAV_ERR_STATE, nothing written, until
    agents_rebuild_index"""
    cost, rec, fl, ms = _population(4242, 20)
    J = Job(3, cost, rec, fl, ms, 20, 2)
    try:
        one = J.one
        q = queries([(0.0, 0.0, r, int(u), 512) for u in range(0, J.n, 13) for r in (10.0, 30.0)])
        before = one.ents_in_circles(q)
        nw = len(one.agents_read_work())
        assert nw > 0
        J._tick_one(one, nw, 1)                                  # ... compute_updates, apply_updates
        rc, o, ids, t = raw_call(one, q, 1 << 20)
        assert rc == capi.ERR_STATE and t == 12345 and (o == 0xDEAD).all() and (ids == 0xBEEF).all()
        one.agents_rebuild_index()
        after = one.ents_in_circles(q)
        assert not np.array_equal(after[1], before[1]), "the entities moved"
        one.agents_commands(cases_deltas(rec))
        one.ents_in_circle(0.0, 0.0, 10.0, 8)                   # the single query keeps its behaviour: it never refuses
        assert raw_call(one, q, 1 << 20)[0] == capi.ERR_STATE
        one.agents_rebuild_index()
        assert raw_call(one, q, 1 << 20)[0] == capi.OK
    finally:
        J.close()


def cases_deltas(rec):
    import commands_ref as cr
    u = np.arange(0, len(rec), 97, dtype=np.uint32)
    return cr.deltas(u, velocity=(rec["velocity"][u] * np.float32(0.5)).astype(np.float32))


@pytest.mark.parametrize("world", [2, 3])
def test_group_members_answer_every_query(pforacle, world):
    """after a gather every member holds the whole index: each answers every query, with uid centres from any member's
    range, exactly as one context holding the whole population; between a job's writes and the gather they refuse"""
    cost, rec, fl, ms = _population(4242, 20)
    J = Job(3, cost, rec, fl, ms, 20, world)
    try:
        rng = np.random.default_rng(world)
        u = rng.choice(J.n, 400, replace=False)
        pos = J.one.agents_read_state(J.n, False)[0]["pos"]
        q = queries([(0.0, 0.0, r, int(i), m) for i in u for r, m in ((10.0, 512), (30.0, 128), (60.0, 16))] +
                    [(float(pos[i, 0]), float(pos[i, 1]), 30.0, NULL, 64) for i in u[:50]])
        for step in range(2):
            want = J.one.ents_in_circles(q)
            for nv in J.navs:
                got = nv.ents_in_circles(q)
                assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
            J.one.agents_commands(cases_deltas(rec))
            J.grp.commands(cases_deltas(rec))
            for nv in J.navs:
                assert raw_call(nv, q, 1 << 20)[0] == capi.ERR_STATE
            J.one.agents_rebuild_index()
            J.grp.gather()
        for nv, (lo, hi) in zip(J.navs, J.ranges):                # a shard upload leaves the member stale until the gather
            nv.agents_upload_shard(J.one.agents_read_state(J.n, False)[0][lo:hi], lo, hi, J.n, J.fl, 20, capi.UPLOAD_SAME_FLOCKS)
            assert raw_call(nv, q, 1 << 20)[0] == capi.ERR_STATE
        J.grp.gather()
        want = J.one.ents_in_circles(q)
        for nv in J.navs:
            got = nv.ents_in_circles(q)
            assert np.array_equal(got[1], want[1])
    finally:
        J.close()
