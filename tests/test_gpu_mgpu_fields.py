"""Goal batches of a multi-GPU job (pfnav_group_request_goals_ex): each (dest, chunk) field is built on one member and
copied to the members that lack it. Every member is compared with a single context built from the same seeds that gets
the same calls, with pfnav_pool_request_goals_ex in place of the job's batch: for every (dest, chunk), identical has
bits, ff_id, flow and LOS bytes, and the member's solo request counts. The compute counts of the test hook
pfnav_mgpu_fields_stats show each goal's union of lacked fields built on exactly one member.

Groups of 2 and 3 members on device 0, and on further devices where the box has them. The NCCL transport is checked by
tests/tools/mgpu_nccl_fields_check.py under torchrun."""
import ctypes as C
import importlib
import os
import sys

import numpy as np
import pytest

import cases

capi = cases.capi
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _devices(world):
    import torch
    n = torch.cuda.device_count()
    return [i % n for i in range(world)]


def _nav(dev, cost, cw, ndests, max_fields):
    nv = capi.Nav(dev)
    nv.map_create(cw, cw, 1)
    nv.map_upload_layer(0, cost)
    nv.map_build_nav(0)
    nv.pool_create(ndests, max_fields)
    return nv


def _pool(nav, ndests):
    """every (dest, chunk) entry: has bits, ffid, flow and LOS bytes"""
    out = []
    for d in range(ndests):
        for c in range(nav.cw * nav.ch):
            f, l, ffid = nav.pool_get(d, divmod(c, nav.cw))
            out.append((int(f is not None) | int(l is not None) << 1, ffid,
                        b"" if f is None else f.tobytes(), b"" if l is None else l.tobytes()))
    return out


def _has(nav, ndests):
    n = nav.cw * nav.ch
    return {divmod(i, n): e[0] for i, e in enumerate(_pool(nav, ndests))}


class Twins:
    """`world` members of an in-process group, and for member r a single context `solo[r]` that gets every call member r
    gets, with the solo goal batch in place of the job's"""

    def __init__(self, cost, cw, ndests, max_fields, world):
        self.cw, self.ndests, self.world = cw, ndests, world
        self.navs = [_nav(d, cost, cw, ndests, max_fields) for d in _devices(world)]
        self.solo = [_nav(0, cost, cw, ndests, max_fields) for _ in range(world)]
        self.grp = capi.Group(self.navs)

    def pairs(self):
        return list(zip(self.navs, self.solo))

    def close(self):
        self.grp.close()
        for X in self.navs + self.solo:
            X.close()

    def each(self, fn):
        """the same call on every member and every single context"""
        for X in self.navs + self.solo:
            fn(X)

    def solo_request(self, r, dests, targets, flags=0):
        """an ordinary solo batch on member r and its twin (how members come to hold different fields)"""
        a = self.navs[r].pool_request_goals(dests, targets, flags=flags)
        assert self.solo[r].pool_request_goals(dests, targets, flags=flags) == a

    def union_counts(self, dests, targets, flags):
        """flow / LOS requests of the union of the members' lacked fields, goal by goal"""
        mo = flags & capi.REQUEST_MISSING_ONLY
        has = [_has(nv, self.ndests) for nv in self.navs] if mo else None
        per = []
        for d, t in zip(dests, targets):
            _, fc, _, _, lc = self.navs[0].plan_goal(tuple(int(v) for v in t))
            lack = lambda c, bit: not mo or any(not (h[(int(d), int(c))] & bit) for h in has)
            per.append((sum(lack(c, 1) for c in fc), sum(lack(c, 2) for c in lc)))
        return per

    def job(self, dests, targets, flags=0):
        dests = np.asarray(dests, np.int32)
        targets = np.asarray(targets, np.int32).reshape(-1, 4)
        per = self.union_counts(dests, targets, flags)
        nf, nl = self.grp.request_goals_ex(dests, targets, 0, flags)
        for r, S in enumerate(self.solo):
            assert (int(nf[r]), int(nl[r])) == S.pool_request_goals(dests, targets, flags=flags), "solo counts differ"
        self.compare()
        # each goal's union fields were built on its owner alone, and the members' counts add up to the union
        stats = [nv.mgpu_fields_stats(len(dests)) for nv in self.navs]
        owner = stats[0][2]
        for s in stats:
            assert np.array_equal(s[2], owner), "members disagree on the owners"
        for g, (uf, ul) in enumerate(per):
            assert (owner[g] >= 0) == (uf + ul > 0), (g, owner[g], uf, ul)
        for r, (bf, bl, _) in enumerate(stats):
            assert (bf, bl) == (sum(per[g][0] for g in range(len(per)) if owner[g] == r),
                                sum(per[g][1] for g in range(len(per)) if owner[g] == r)), r
        assert sum(s[0] for s in stats) == sum(p[0] for p in per)
        assert sum(s[1] for s in stats) == sum(p[1] for p in per)
        return owner, per

    def compare(self):
        for r, (nv, S) in enumerate(self.pairs()):
            a, b = _pool(nv, self.ndests), _pool(S, self.ndests)
            bad = [i for i in range(len(a)) if a[i] != b[i]]
            assert not bad, "member %d: %d entries differ, first (dest, chunk) %s" % (r, len(bad), divmod(bad[0], nv.cw * nv.ch))


def synth_cost(cw, seed):
    p = cases.noise_map(cw, cw, seed, 0.0)
    return cases.synth.cost_from_pathable(p, cw, cw)


def _targets(nav, n, rng):
    """n goals on passable tiles: int32[n, 4] {chunk_r, chunk_c, tile_r, tile_c}"""
    cost = nav.map_get_layer(0)[0]
    out = []
    while len(out) < n:
        cr, cc, tr, tc = int(rng.integers(nav.ch)), int(rng.integers(nav.cw)), int(rng.integers(64)), int(rng.integers(64))
        if cost[cr * nav.cw + cc, tr, tc] != 0xFF:
            out.append((cr, cc, tr, tc))
    return np.array(out, np.int32)


def _c2():
    """the bench's C2 map and its 16 goals -> (cost, cw, targets)"""
    sys.path.insert(0, ROOT)
    bench = importlib.import_module("bench")
    bench.set_workload("C2")
    W = bench.build_workload(cases.pf, 1, 0)
    targets = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(W["g_lo"], W["g_hi"])], np.int32)
    return W["cost"], bench.CHUNKS, targets


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_cold_small(pf, world):
    """a cold batch of 6 goals on a 4 x 4-chunk map: every member builds some, all end with every field"""
    cost = synth_cost(4, 101)
    T = Twins(cost, 4, 6, 6 * 16, world)
    try:
        tg = _targets(T.navs[0], 6, np.random.default_rng(7))
        owner, per = T.job(np.arange(6), tg)
        assert len(set(owner.tolist())) == world, owner          # 6 goals spread over every member
        T.job(np.arange(6), tg)                                  # again on a full pool: everything rebuilt once more
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_c2_cold(pf, world):
    """the C2 map with its 16 goals, every member needing all of them"""
    cost, cw, tg = _c2()
    T = Twins(cost, cw, 16, 16 * cw * cw, world)
    try:
        T.job(np.arange(16), tg)
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_repeated_dests(pf, world):
    """a destination named twice in one batch (with its one target), cold and missing-only"""
    cost = synth_cost(3, 202)
    T = Twins(cost, 3, 4, 4 * 9, world)
    try:
        tg = _targets(T.navs[0], 3, np.random.default_rng(3))
        dests = [0, 1, 0, 2, 1]
        T.job(dests, tg[[0, 1, 0, 2, 1]])
        T.job(dests, tg[[0, 1, 0, 2, 1]], capi.REQUEST_MISSING_ONLY)
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_fewer_goals_than_members(pf, world):
    cost = synth_cost(3, 303)
    T = Twins(cost, 3, 2, 2 * 9, world)
    try:
        tg = _targets(T.navs[0], 1, np.random.default_rng(5))
        owner, _ = T.job([1], tg)
        assert owner.tolist() == [0]
    finally:
        T.close()


@pytest.mark.gpu
def test_attacking_faction(pf):
    """a faction at war and a path-request faction set on every context (the flow kernels take the general path)"""
    cost = synth_cost(3, 404)
    T = Twins(cost, 3, 4, 4 * 9, 2)
    try:
        T.each(lambda X: X.set_enemy_factions(2, 1 << 5))
        T.each(lambda X: X.request_faction(2))
        tg = _targets(T.navs[0], 4, np.random.default_rng(9))
        T.job(np.arange(4), tg)
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_missing_only_diverged(pf, world):
    """members that hold different fields -- different earlier batches, then commits that dirty chunks -- rebuild with
    PFNAV_REQUEST_MISSING_ONLY: a member writes only what it lacks, the union is built once; rebuilt LOS fields read
    parents that every member kept"""
    cw, nd = 4, 6
    cost = synth_cost(cw, 505)
    T = Twins(cost, cw, nd, nd * cw * cw, world)
    try:
        rng = np.random.default_rng(11)
        tg = _targets(T.navs[0], nd, rng)
        for r in range(world):                  # member r holds goals r, r + 1 (and r + 3 on the last member)
            held = [r, r + 1] + ([r + 3] if r == world - 1 else [])
            T.solo_request(r, held, tg[held])
        T.job(np.arange(nd), tg, capi.REQUEST_MISSING_ONLY)
        for step in range(3):                   # blockers dirty a few chunks on every context; rebuild what was dropped
            x, z = float(rng.uniform(-cw * 256 + 40, -40)), float(rng.uniform(40, cw * 256 - 40))     # map_x = map_z = 0
            T.each(lambda X: X.blockers_incref(x, z, 6.0 + 4 * step))
            nds = []
            T.each(lambda X: nds.append(X.map_commit()))
            assert len(set(nds)) == 1 and nds[0] > 0, nds
            T.job(np.arange(nd), tg, capi.REQUEST_MISSING_ONLY)
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_small_pool_evictions_diverge(pf, world):
    """a pool too small for every goal: earlier batches evict different fields on different members, and the job's
    batch then evicts by each member's own LRU order"""
    cw, nd = 3, 6
    cost = synth_cost(cw, 606)
    T = Twins(cost, cw, nd, 3 * 9 + 4, world)
    try:
        tg = _targets(T.navs[0], nd, np.random.default_rng(13))
        for r in range(world):
            T.solo_request(r, [r], tg[[r]])
            T.solo_request(r, [3, 4, 5][:r + 1], tg[[3, 4, 5][:r + 1]])
            T.solo_request(r, [(r + 1) % 3, 5], tg[[(r + 1) % 3, 5]])
        T.compare()
        T.job([0, 1, 2], tg[:3])
        T.job([3, 4], tg[3:5])
    finally:
        T.close()


@pytest.mark.gpu
def test_errors(pf):
    """bad dest, bad layer and a pool too small on one member: every member refuses and no pool changes; a context in no
    job and the NCCL form on a group member -> PFNAV_ERR_STATE"""
    L = capi.load()
    cost = synth_cost(3, 707)
    T = Twins(cost, 3, 4, 4 * 9, 2)
    small = None
    try:
        tg = _targets(T.navs[0], 4, np.random.default_rng(17))
        T.job([0, 1], tg[:2])
        before = [_pool(nv, 4) for nv in T.navs]
        nf = np.zeros(2, np.int32)
        nl = np.zeros(2, np.int32)

        def call(g, dests, t, layer=0):
            d = np.ascontiguousarray(dests, np.int32)
            t = np.ascontiguousarray(t, np.int32)
            return L.pfnav_group_request_goals_ex(g, len(d), d.ctypes.data_as(C.c_void_p), layer, t.ctypes.data_as(C.c_void_p), 0,
                                                  nf.ctypes.data_as(C.c_void_p), nl.ctypes.data_as(C.c_void_p))
        assert call(T.grp.g, [2, 4], tg[2:4]) == capi.ERR_ARG
        assert call(T.grp.g, [2, 3], tg[2:4], layer=1) == capi.ERR_ARG
        assert call(None, [2], tg[2:3]) == capi.ERR_ARG
        assert [_pool(nv, 4) for nv in T.navs] == before
        # a context outside any job; the NCCL form on a group member
        d = np.zeros(1, np.int32)
        for h in (T.solo[0].h, T.navs[0].h):
            assert L.pfnav_mgpu_request_goals_ex(h, 1, d.ctypes.data_as(C.c_void_p), 0, tg.ctypes.data_as(C.c_void_p), 0,
                                                 None, None, None) == capi.ERR_STATE
        T.compare()
    finally:
        T.close()
    # NOMEM on one member: a group whose second member's pool holds only 9 fields
    navs = [_nav(0, cost, 3, 4, 4 * 9), _nav(0, cost, 3, 4, 9)]
    grp = capi.Group(navs)
    try:
        tg = _targets(navs[0], 2, np.random.default_rng(19))
        navs[1].pool_request_goals([0], tg[:1])
        navs[0].pool_request_goals([0], tg[:1])
        before = [_pool(nv, 4) for nv in navs]
        d = np.array([0, 1], np.int32)
        rc = L.pfnav_group_request_goals_ex(grp.g, 2, d.ctypes.data_as(C.c_void_p), 0, tg.ctypes.data_as(C.c_void_p), 0,
                                            None, None)
        assert rc == capi.ERR_NOMEM
        assert [_pool(nv, 4) for nv in navs] == before
    finally:
        grp.close()
        for nv in navs:
            nv.close()


@pytest.mark.gpu
def test_unexchanged_blocker_ops(pf):
    """device blocker ops decided on one member and not yet exchanged: PFNAV_ERR_STATE on the job's batch, no pool
    changed; after the exchange and the commit the batch goes through"""
    from test_gpu_mgpu_blockers import Job, _case
    L = capi.load()
    cost, a, ms = _case(12, 20)
    J = Job(cost, a, ms, 20, 2)
    try:
        lo0 = J.ranges[0][0]
        tg = _targets(J.navs[0], 1, np.random.default_rng(23))
        J.navs[0].agents_set_blocking(np.arange(lo0, lo0 + 40, dtype=np.uint32), True)
        before = [_pool(nv, J.nflocks) for nv in J.navs]
        d = np.zeros(1, np.int32)
        rc = L.pfnav_group_request_goals_ex(J.grp.g, 1, d.ctypes.data_as(C.c_void_p), 0, tg.ctypes.data_as(C.c_void_p), 0,
                                            None, None)
        assert rc == capi.ERR_STATE
        assert [_pool(nv, J.nflocks) for nv in J.navs] == before
        J.grp.exchange_blocker_ops()
        for nv in J.navs:
            nv.map_commit()
        J.grp.request_goals_ex(d, tg)
    finally:
        J.close()


def test_errors_host_only(pf):
    """a host-only context has no device: PFNAV_ERR_NO_DEVICE"""
    L = capi.load()
    nav = capi.Nav(hostonly=True)
    try:
        d, t = np.zeros(1, np.int32), np.zeros(4, np.int32)
        assert L.pfnav_mgpu_request_goals_ex(nav.h, 1, d.ctypes.data_as(C.c_void_p), 0, t.ctypes.data_as(C.c_void_p), 0,
                                             None, None, None) == capi.ERR_NO_DEVICE
    finally:
        nav.close()
