"""Blockers of stopping and starting units taken on the device by the members of a multi-GPU job that shares them
(pfnav_group_share_blockers, pfnav_group_exchange_blocker_ops) against one context holding the whole population on the
single-context device path (pfnav_agents_apply_updates_ex with PFNAV_APPLY_BLOCKERS, pfnav_agents_set_blocking).

Every scenario builds the single context and a group of 2 or 3 sharded members (on device 0, and on further devices
where the box has them) from the same seeds. Per tick the members run compute_updates -> apply_updates_ex ->
[set_blocking] -> exchange_blocker_ops -> map_commit -> gather. After every tick, on every member: identical blocker and
faction counts on every layer, local islands, portal edges and pool entries (has bits, ff_ids, bytes) to the single
context's; the members' blocking tables (own ranges, concatenated) and entity state equal the single context's; the
next tick's velocities and patches are identical and every member's map_commit reports the single context's ndirty.
The NCCL transport is checked by tests/tools/mgpu_nccl_blockers_check.py under torchrun (needs >= 2 GPUs)."""
import ctypes as C

import numpy as np
import pytest

import cases
from test_gpu_apply_blockers import _factions

capi = cases.capi
ST_ARRIVED, ST_WAITING = 2, 4


def _devices(world):
    import torch
    n = torch.cuda.device_count()
    return [i % n for i in range(world)]


class Job:
    """ONE: a single context on the device path; navs: `world` sharded members of a group that shares blockers"""

    def __init__(self, cost, a, ms, hz, world, nlayers=1, tbl=None, cw=3):
        self.cw, self.nlayers, self.n, self.world = cw, nlayers, len(a["radius"]), world
        self.nflocks = len(a["flock_target"])
        rec, fl = capi.pack_agents(a)
        self.rec = rec
        if tbl is None:
            tbl = np.zeros(self.n, capi.BLOCKING)
            tbl["faction_id"] = capi.FACTION_ID_NONE
        self.ranges = [capi.mgpu_shard_range(self.n, r, world) for r in range(world)]
        self.one = capi.Nav(0)
        self.navs = [capi.Nav(d) for d in _devices(world)]
        self.grp = None
        for X in self.all():
            X.map_create(cw, cw, nlayers)
            for l in range(nlayers):
                X.map_upload_layer(l, cost); X.map_build_nav(l); X.route_build(l)
            X.pool_create(self.nflocks, self.nflocks * cw * cw)
        self.grp = capi.Group(self.navs)
        self.grp.share_blockers()
        self.one.agents_upload(rec, fl, hz)
        self.one.agents_upload_movestate(ms)
        for nv, (lo, hi) in zip(self.navs, self.ranges):
            nv.agents_upload_shard(rec[lo:hi], lo, hi, self.n, fl, hz)
        self.grp.gather()
        for nv, (lo, hi) in zip(self.navs, self.ranges):
            nv.agents_upload_movestate(ms[lo:hi])
        pre = tbl["blocking"] != 0
        for X in self.all():
            if pre.any():           # blocks counted at load go to every rank through pfnav_blockers_*
                ops = np.zeros(int(pre.sum()), capi.BLOCKER_OP)
                ops["x"], ops["z"], ops["range"] = tbl["stop_x"][pre], tbl["stop_z"][pre], tbl["stop_radius"][pre]
                ops["faction_id"], ops["flags"], ops["delta"] = tbl["faction_id"][pre], rec["flags"][pre], 1
                X.blockers_batch(ops)
                X.map_commit()
            # the same pool entries everywhere, for the commits to invalidate: one path per flock to its target
            for f in range(self.nflocks):
                src, dst = a["pos"][np.nonzero(a["flock_of"] == f)[0][0]], a["flock_target"][f]
                X.pool_request_path(f, (float(src[0]), float(src[1])), (float(dst[0]), float(dst[1])))
        self.one.agents_upload_blocking(tbl)
        for nv, (lo, hi) in zip(self.navs, self.ranges):
            nv.agents_upload_blocking(tbl[lo:hi])

    def all(self):
        return [self.one] + self.navs

    def close(self):
        if self.grp is not None:
            self.grp.close()
        for X in self.all():
            X.close()

    def own(self, r, uids):
        lo, hi = self.ranges[r]
        uids = np.asarray(uids, np.uint32)
        return uids[(uids >= lo) & (uids < hi)]

    def commit_all(self, nd1):
        """exchange, then commit every member: each reports the single context's ndirty"""
        self.grp.exchange_blocker_ops()
        nds = [nv.map_commit() for nv in self.navs]
        assert nds == [nd1] * self.world, (nds, nd1)

    def tick(self, work):
        """one tick on both sides -> blocks taken by the single context in this tick"""
        one = self.one
        before = one.agents_read_blocking(self.n)["blocking"]
        one.agents_set_work(work)
        if len(work):
            one.agents_tick(0)
        v1 = one.agents_read_velocities(len(work))
        one.agents_compute_updates()
        p1 = one.agents_read_patches(len(work))
        one.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        nd1 = one.map_commit()
        one.agents_rebuild_index()
        vs, ps = [], []
        for r, nv in enumerate(self.navs):
            w = self.own(r, work)
            nv.agents_set_work(w)
            if len(w):
                nv.agents_tick(0)
        for r, nv in enumerate(self.navs):
            w = self.own(r, work)
            if not len(w):          # a member without work decides no op, and still takes part in the exchange
                vs.append(np.zeros((0, 2), np.float32)); ps.append(np.zeros(0, capi.PATCH))
                continue
            vs.append(nv.agents_read_velocities(len(w)))
            nv.agents_compute_updates()
            ps.append(nv.agents_read_patches(len(w)))
            nv.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        self.commit_all(nd1)
        self.grp.gather()
        assert np.concatenate(vs).tobytes() == v1.tobytes(), "velocities differ"
        assert np.concatenate(ps).tobytes() == p1.tobytes(), "patches differ"
        self.compare()
        return int(((one.agents_read_blocking(self.n)["blocking"] != 0) & (before == 0)).sum())

    def set_blocking(self, per_rank, block):
        """set_blocking of per_rank[r] (uids of rank r's own range) on the members, of all of them on the single context"""
        self.one.agents_set_blocking(np.concatenate([np.asarray(u, np.uint32) for u in per_rank]), block)
        nd1 = self.one.map_commit()
        for nv, u in zip(self.navs, per_rank):
            if len(u):
                nv.agents_set_blocking(u, block)
        self.commit_all(nd1)
        self.compare()
        return nd1

    def compare(self):
        one, cw = self.one, self.cw
        ref = [(one.blockers(l), one.faction_counts(l), one.local_islands(l), one.portals(l)) for l in range(self.nlayers)]
        pool = [[one.pool_get(d, divmod(c, cw)) for c in range(cw * cw)] for d in range(self.nflocks)]
        for r, nv in enumerate(self.navs):
            for l, (blk, fac, liid, portals) in enumerate(ref):
                assert (nv.blockers(l) == blk).all(), ("blockers", r, l)
                assert (nv.faction_counts(l) == fac).all(), ("faction counts", r, l)
                assert (nv.local_islands(l) == liid).all(), ("local islands", r, l)
                for pr in portals:
                    ci, pi = int(pr[0]) * cw + int(pr[1]), int(pr[2])
                    assert (nv.route_edges(ci, pi, l) == one.route_edges(ci, pi, l)).all(), ("route edges", r, l, ci, pi)
            for d in range(self.nflocks):
                for c in range(cw * cw):
                    fa, la, ia = pool[d][c]
                    fb, lb, ib = nv.pool_get(d, divmod(c, cw))
                    assert ia == ib and (fa is None) == (fb is None) and (la is None) == (lb is None), ("pool entry", r, d, c)
                    assert (fa is None or (fa == fb).all()) and (la is None or (la == lb).all()), ("pool bytes", r, d, c)
        got = np.concatenate([nv.agents_read_blocking(hi - lo) for nv, (lo, hi) in zip(self.navs, self.ranges)])
        exp = one.agents_read_blocking(self.n)
        assert got.tobytes() == exp.tobytes(), np.nonzero(got != exp)[0][:10]
        a1, m1 = one.agents_read_state(self.n)
        parts = [nv.agents_read_state(hi - lo) for nv, (lo, hi) in zip(self.navs, self.ranges)]
        assert np.concatenate([p[0] for p in parts]).tobytes() == a1.tobytes(), "entity state differs"
        assert np.concatenate([p[1] for p in parts]).tobytes() == m1.tobytes(), "movestate differs"

    def still_work(self):
        st = self.one.agents_read_state(self.n, movestate=False)[0]["state"]
        return np.nonzero((st != ST_ARRIVED) & (st != ST_WAITING))[0].astype(np.uint32)


def _case(seed, hz):
    p, cost, a, ms = cases.update_case(seed, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(seed + 5)
    a["vdes"] = rng.normal(size=(n, 2)).astype(np.float32)
    a["vdes"] /= np.linalg.norm(a["vdes"], axis=1, keepdims=True)
    a["has_los"] = (rng.random(n) < 0.2).astype(np.uint32)
    return cost, a, ms


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
@pytest.mark.parametrize("hz", [20, 10, 5, 1])
def test_update_case_ticks(pf, hz, world):
    """the arriving crowd of cases.update_case over three ticks: faction-tagged records, a few units already blocking
    at load, and radii wider than the bit window, two of them on the last rank"""
    cost, a, ms = _case(4242, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(hz)
    lo, hi = capi.mgpu_shard_range(n, world - 1, world)
    a["radius"][np.concatenate([rng.choice(n, 2, replace=False), rng.choice(np.arange(lo, hi), 2, replace=False)])] = 50.0
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = _factions(n, hz)
    pre = rng.random(n) < 0.03
    tbl["blocking"][pre] = 1
    tbl["stop_x"][pre], tbl["stop_z"][pre] = a["pos"][pre, 0], a["pos"][pre, 1]
    tbl["stop_radius"][pre] = a["radius"][pre]
    J = Job(cost, a, ms, hz, world, nlayers=4, tbl=tbl)     # a radius of 50 takes the 7 x 7 ground layer
    try:
        J.compare()
        nblock = sum(J.tick(J.still_work()) for _ in range(3))
        assert nblock > 0, nblock
    finally:
        J.close()


@pytest.mark.gpu
def test_one_rank_then_none(pf):
    """ticks whose work lies in the middle rank's range only (the other members decide no op but still receive), then
    a tick with no work anywhere (an exchange of nothing), then the whole work list"""
    cost, a, ms = _case(4242, 20)
    n = len(a["radius"])
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = _factions(n, 3)
    J = Job(cost, a, ms, 20, 3, tbl=tbl)
    try:
        taken = 0
        for _ in range(3):
            taken += J.tick(J.own(1, J.still_work()))
            if taken:
                break
        assert taken > 0, "no unit of the middle rank stopped"
        assert J.tick(np.zeros(0, np.uint32)) == 0
        J.tick(J.still_work())
    finally:
        J.close()


@pytest.mark.gpu
def test_faction_ops_on_one_rank(pf):
    """only rank 1's entities carry a faction: its faction-tagged ops must make the faction counts appear on rank 0,
    which decided none"""
    cost, a, ms = _case(4243, 20)
    n = len(a["radius"])
    rng = np.random.default_rng(2)
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = capi.FACTION_ID_NONE
    lo, hi = capi.mgpu_shard_range(n, 1, 2)
    tbl["faction_id"][lo:hi] = rng.integers(0, 4, hi - lo)
    J = Job(cost, a, ms, 20, 2, tbl=tbl)
    try:
        sel = rng.choice(np.arange(lo, hi), 200, replace=False).astype(np.uint32)
        J.set_blocking([np.zeros(0, np.uint32), sel], True)
        assert J.one.faction_counts(0).any()
        J.tick(J.still_work())
        J.set_blocking([np.zeros(0, np.uint32), sel[::2]], False)
    finally:
        J.close()


@pytest.mark.gpu
def test_air_and_ground_twelve_layers(pf):
    """AIR and non-air units on a 12-layer map: two ticks, then set_blocking block / unblock on every rank"""
    cost, a, ms = _case(31, 20)
    n = len(a["radius"])
    rng = np.random.default_rng(31)
    air = rng.random(n) < 0.3
    a["flags"][air] |= capi.FLAG_AIR
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = _factions(n, 31)
    J = Job(cost, a, ms, 20, 2, nlayers=12, tbl=tbl)
    try:
        for _ in range(2):
            J.tick(J.still_work())
        sel = rng.choice(n, 300, replace=False).astype(np.uint32)
        J.set_blocking([J.own(r, sel) for r in range(2)], True)
        assert J.one.blockers(8).any() and J.one.blockers(0).any()
        J.set_blocking([J.own(r, sel[:150]) for r in range(2)], False)
    finally:
        J.close()


@pytest.mark.gpu
def test_set_blocking_each_rank(pf):
    """set_blocking on every rank's own uids: repeats within a call and repeated calls change nothing, GARRISONED
    entities take no op, radii beyond the bit window on a non-zero rank are rasterised on the host by every member
    after the exchange"""
    cost, a, ms = _case(4243, 20)
    n = len(a["radius"])
    world = 3
    rng = np.random.default_rng(1)
    lo, hi = capi.mgpu_shard_range(n, 1, world)
    wide = rng.choice(np.arange(lo, hi), 6, replace=False)
    a["radius"][wide] = rng.uniform(49.0, 90.0, 6).astype(np.float32)
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = rng.integers(0, 4, n)
    J = Job(cost, a, ms, 20, world, nlayers=4, tbl=tbl)
    try:
        garr = np.nonzero(a["flags"] & capi.FLAG_GARRISONED)[0]
        assert len(garr)
        sel = np.concatenate([rng.choice(n, 300, replace=False), wide, garr]).astype(np.uint32)
        per = [J.own(r, sel) for r in range(world)]
        per = [np.concatenate([u, u[:20]]) for u in per]          # repeats inside one call
        J.set_blocking(per, True)
        b = J.one.agents_read_blocking(n)
        assert not b["blocking"][garr].any()
        assert (b["stop_radius"][b["blocking"] != 0] > 48).sum() == int(((a["flags"][wide] & capi.FLAG_GARRISONED) == 0).sum()) > 0
        assert J.set_blocking(per, True) == 0                      # nothing left to block
        J.tick(J.still_work())
        J.set_blocking([u[::2] for u in per], False)
        J.set_blocking([u[::2] for u in per], False)
    finally:
        J.close()


@pytest.mark.gpu
def test_receive_buffer_grows(pf):
    """a small exchange, then rank 0 holds a few pending ops of its own when rank 1 sends hundreds: rank 0's op buffers
    grow and keep its own ops. Then a second exchange before the commit sends only what was decided after the first."""
    cost, a, ms = _case(4244, 20)
    n = len(a["radius"])
    rng = np.random.default_rng(4)
    J = Job(cost, a, ms, 20, 2)
    try:
        (lo0, hi0), (lo1, hi1) = J.ranges
        r0 = rng.choice(np.arange(lo0, hi0), 6, replace=False).astype(np.uint32)
        r1 = rng.choice(np.arange(lo1, hi1), 400, replace=False).astype(np.uint32)
        J.set_blocking([r0[:3], np.zeros(0, np.uint32)], True)
        J.set_blocking([r0[3:], r1], True)
        # rank 0 releases, is exchanged; rank 1 releases after that exchange: a second exchange carries rank 1's ops only
        J.one.agents_set_blocking(np.concatenate([r0[:2], r1[:100]]), False)
        nd1 = J.one.map_commit()
        J.navs[0].agents_set_blocking(r0[:2], False)
        J.grp.exchange_blocker_ops()
        J.navs[1].agents_set_blocking(r1[:100], False)
        J.commit_all(nd1)
        J.compare()
    finally:
        J.close()


@pytest.mark.gpu
def test_errors(pf):
    """a commit or a count read with unexchanged ops -> PFNAV_ERR_STATE and nothing applied; a set_blocking uid outside
    the own range -> PFNAV_ERR_ARG and nothing changed; the NCCL calls on a group member -> PFNAV_ERR_ARG"""
    L = capi.load()
    cost, a, ms = _case(12, 20)
    n = len(a["radius"])
    J = Job(cost, a, ms, 20, 2)
    try:
        (lo0, hi0), (lo1, hi1) = J.ranges
        u0 = np.arange(lo0, lo0 + 40, dtype=np.uint32)
        J.navs[0].agents_set_blocking(u0, True)
        cw = J.cw
        blk = np.zeros((cw * cw, 64, 64), np.uint16)
        fac = np.zeros((cw * cw, 15, 64, 64), np.uint8)
        nd = C.c_int(-1)
        assert L.pfnav_map_commit(J.navs[0].h, C.byref(nd)) == capi.ERR_STATE
        assert L.pfnav_blockers_get(J.navs[0].h, 0, blk.ctypes.data_as(C.c_void_p)) == capi.ERR_STATE
        assert L.pfnav_blockers_get_factions(J.navs[0].h, 0, fac.ctypes.data_as(C.c_void_p)) == capi.ERR_STATE
        J.one.agents_set_blocking(u0, True)
        nd1 = J.one.map_commit()
        assert nd1 > 0
        J.commit_all(nd1)          # applied once, after the exchange
        J.compare()
        # outside the own range: rejected, nothing changes
        for nv, bad in ((J.navs[0], hi0), (J.navs[1], lo1 - 1), (J.navs[1], n)):
            u = np.array([lo1 if nv is J.navs[1] else lo0, bad], np.uint32)
            assert L.pfnav_agents_set_blocking(nv.h, u.ctypes.data_as(C.c_void_p), 2, 0, None) == capi.ERR_ARG
        J.commit_all(0)
        J.compare()
        # the NCCL transport's calls on a member of an in-process group
        for nv in J.navs:
            assert L.pfnav_mgpu_share_blockers(nv.h) == capi.ERR_ARG
            assert L.pfnav_mgpu_exchange_blocker_ops(nv.h, None) == capi.ERR_ARG
    finally:
        J.close()


@pytest.mark.gpu
def test_errors_not_shared(pf):
    """a context outside any job and a group that did not opt in -> PFNAV_ERR_STATE; members holding populations of
    different sizes -> PFNAV_ERR_ARG; pfnav_group_destroy clears the opt-in"""
    L = capi.load()
    cost, a, ms = _case(12, 20)
    n = len(a["radius"])
    rec, fl = capi.pack_agents(a)
    nav = capi.Nav(0)
    try:
        nav.map_create(3, 3, 1); nav.map_upload_layer(0, cost)
        assert L.pfnav_mgpu_share_blockers(nav.h) == capi.ERR_STATE
        assert L.pfnav_mgpu_exchange_blocker_ops(nav.h, None) == capi.ERR_STATE
    finally:
        nav.close()
    assert L.pfnav_group_share_blockers(None) == capi.ERR_ARG
    assert L.pfnav_group_exchange_blocker_ops(None) == capi.ERR_ARG
    navs = [capi.Nav(0), capi.Nav(0)]
    grp = capi.Group(navs)
    try:
        for nv in navs:
            nv.map_create(3, 3, 1); nv.map_upload_layer(0, cost)
        lo, hi = capi.mgpu_shard_range(n, 0, 2)
        navs[0].agents_upload_shard(rec[lo:hi], lo, hi, n, fl, 20)
        lo1, hi1 = capi.mgpu_shard_range(n - 1, 1, 2)
        navs[1].agents_upload_shard(rec[lo1:hi1], lo1, hi1, n - 1, fl, 20)
        assert L.pfnav_group_share_blockers(grp.g) == capi.ERR_ARG
        assert L.pfnav_group_exchange_blocker_ops(grp.g) == capi.ERR_STATE
        lo1, hi1 = capi.mgpu_shard_range(n, 1, 2)
        navs[1].agents_upload_shard(rec[lo1:hi1], lo1, hi1, n, fl, 20)
        grp.share_blockers()
        blk = np.zeros(n, capi.BLOCKING)
        navs[0].agents_upload_blocking(blk[lo:hi])
        grp.exchange_blocker_ops()
    finally:
        grp.close()
    try:
        # no longer in a job: the own range is half the population again, as without the opt-in
        assert L.pfnav_agents_upload_blocking(navs[0].h, blk[lo:hi].ctypes.data_as(C.c_void_p), hi - lo) == capi.ERR_STATE
    finally:
        for nv in navs:
            nv.close()


def test_errors_host_only(pf):
    """a host-only context has no device: PFNAV_ERR_NO_DEVICE"""
    L = capi.load()
    nav = capi.Nav(hostonly=True)
    try:
        assert L.pfnav_mgpu_share_blockers(nav.h) == capi.ERR_NO_DEVICE
        assert L.pfnav_mgpu_exchange_blocker_ops(nav.h, None) == capi.ERR_NO_DEVICE
    finally:
        nav.close()
