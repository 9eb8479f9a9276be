"""Blockers of stopping and starting units taken on the device (pfnav_agents_apply_updates_ex with PFNAV_APPLY_BLOCKERS,
pfnav_agents_set_blocking) against the host path the engine takes without it: read the patches back, build the
entity_block / entity_unblock ops (movement.c:560-600, 685) in work order from a blocking table kept on the host,
pfnav_blockers_batch, pfnav_map_commit.

Every scenario builds two contexts from the same seeds, A (host path) and B (device path), and requires after every
tick: identical blocker and faction counts on every layer, local islands, portal edges, pool entries (has bits, ff_ids,
bytes), blocking tables, entity state, and the next tick's velocities and patches."""
import ctypes as C

import numpy as np
import pytest

import cases

capi, synth = cases.capi, cases.synth
SET_STATE, SET_MOVING = 1, 1 << 12
ST_ARRIVED, ST_WAITING = 2, 4


def _host_ops(work, patches, agents, tbl):
    """the ops of PFNAV_APPLY_BLOCKERS in work order; agents: the snapshot before the apply; updates tbl"""
    ops = []
    for w, u in enumerate(work):
        p, a = patches[w], agents[u]
        if (p["flags"] & SET_STATE) and p["next_block"] != 0 and not (a["flags"] & capi.FLAG_GARRISONED) and not tbl["blocking"][u]:
            tbl["blocking"][u] = 1
            tbl["stop_x"][u], tbl["stop_z"][u] = a["pos"]
            tbl["stop_radius"][u] = a["radius"]
            ops.append((tbl["stop_x"][u], tbl["stop_z"][u], tbl["stop_radius"][u], tbl["faction_id"][u], a["flags"], 1))
        if (p["flags"] & SET_MOVING) and tbl["blocking"][u]:
            tbl["blocking"][u] = 0
            ops.append((tbl["stop_x"][u], tbl["stop_z"][u], tbl["stop_radius"][u], tbl["faction_id"][u], a["flags"], -1))
    return np.array(ops, capi.BLOCKER_OP)


def _host_set_blocking(uids, block, agents, tbl):
    """pfnav_agents_set_blocking's rules on the host table: first occurrence of a uid only"""
    ops = []
    for u in dict.fromkeys(int(x) for x in uids):
        a = agents[u]
        if block and not (a["flags"] & capi.FLAG_GARRISONED) and not tbl["blocking"][u]:
            tbl["blocking"][u] = 1
            tbl["stop_x"][u], tbl["stop_z"][u] = a["pos"]
            tbl["stop_radius"][u] = a["radius"]
            ops.append((tbl["stop_x"][u], tbl["stop_z"][u], tbl["stop_radius"][u], tbl["faction_id"][u], a["flags"], 1))
        elif not block and tbl["blocking"][u]:
            tbl["blocking"][u] = 0
            ops.append((tbl["stop_x"][u], tbl["stop_z"][u], tbl["stop_radius"][u], tbl["faction_id"][u], a["flags"], -1))
    return np.array(ops, capi.BLOCKER_OP)


class Pair:
    """contexts A (host path) and B (device path) built from the same inputs"""

    def __init__(self, cw, cost, a, ms, hz, nlayers=1, ext=None, tbl=None):
        self.cw, self.nlayers, self.n = cw, nlayers, len(a["radius"])
        self.nflocks = len(a["flock_target"])
        aa = dict(a); aa["flock_dest_index"] = np.arange(self.nflocks, dtype=np.int32)
        rec, fl = capi.pack_agents(aa)
        self.tbl = np.zeros(self.n, capi.BLOCKING) if tbl is None else tbl.copy()
        if tbl is None:
            self.tbl["faction_id"] = capi.FACTION_ID_NONE
        self.A, self.B = capi.Nav(0), capi.Nav(0)
        for X in (self.A, self.B):
            X.map_create(cw, cw, nlayers)
            for l in range(nlayers):
                X.map_upload_layer(l, cost); X.map_build_nav(l); X.route_build(l)
            X.pool_create(self.nflocks, self.nflocks * cw * cw)
            X.agents_upload(rec, fl, hz)
            X.agents_upload_movestate(ms)
            if ext is not None:
                X.agents_upload_movestate_ext(ext)
            pre = self.tbl[self.tbl["blocking"] != 0]
            if len(pre):            # blocks counted at load, which the uploaded records then describe
                ops = np.zeros(len(pre), capi.BLOCKER_OP)
                ops["x"], ops["z"], ops["range"], ops["faction_id"] = pre["stop_x"], pre["stop_z"], pre["stop_radius"], pre["faction_id"]
                ops["flags"] = rec["flags"][self.tbl["blocking"] != 0]; ops["delta"] = 1
                X.blockers_batch(ops)
                X.map_commit()
        self.B.agents_upload_blocking(self.tbl)

    def close(self):
        self.A.close(); self.B.close()

    def state(self, X):
        return X.agents_read_state(self.n)

    def tick(self, work):
        """one tick on both sides -> (blocks, unblocks) taken by A's host ops"""
        out = []
        for X in (self.A, self.B):
            X.agents_set_work(work)
            if len(work):
                cases.settle_pool(X, pool=(self.nflocks, self.cw * self.cw))
            X.agents_compute_updates()
            out.append((X.agents_read_velocities(len(work)), X.agents_read_patches(len(work))))
        (va, pa), (vb, pb) = out
        assert va.tobytes() == vb.tobytes(), "velocities differ"
        assert pa.tobytes() == pb.tobytes(), "patches differ"
        snap, _ = self.state(self.A)
        self.A.agents_apply_updates()
        ops = _host_ops(work, pa, snap, self.tbl)
        if len(ops):
            self.A.blockers_batch(ops)
        nda = self.A.map_commit()
        self.B.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        ndb = self.B.map_commit()
        assert nda == ndb
        self.compare()
        return int((ops["delta"] > 0).sum()) if len(ops) else 0, int((ops["delta"] < 0).sum()) if len(ops) else 0

    def set_blocking(self, uids, block):
        snap, _ = self.state(self.A)
        ops = _host_set_blocking(uids, block, snap, self.tbl)
        if len(ops):
            self.A.blockers_batch(ops)
        self.A.map_commit()
        self.B.agents_set_blocking(uids, block)
        self.B.map_commit()
        self.compare()
        return ops

    def compare(self):
        A, B = self.A, self.B
        for l in range(self.nlayers):
            assert (A.blockers(l) == B.blockers(l)).all(), ("blockers", l)
            assert (A.faction_counts(l) == B.faction_counts(l)).all(), ("faction counts", l)
            assert (A.local_islands(l) == B.local_islands(l)).all(), ("local islands", l)
            for pr in A.portals(l):
                ci, pi = int(pr[0]) * self.cw + int(pr[1]), int(pr[2])
                assert (A.route_edges(ci, pi, l) == B.route_edges(ci, pi, l)).all(), ("route edges", l, ci, pi)
        for d in range(self.nflocks):
            for c in range(self.cw * self.cw):
                fa, la, ia = A.pool_get(d, divmod(c, self.cw))
                fb, lb, ib = B.pool_get(d, divmod(c, self.cw))
                assert ia == ib and (fa is None) == (fb is None) and (la is None) == (lb is None), ("pool entry", d, c)
                assert (fa is None or (fa == fb).all()) and (la is None or (la == lb).all()), ("pool bytes", d, c)
        got = B.agents_read_blocking(self.n)
        assert got.tobytes() == self.tbl.tobytes(), np.nonzero(got != self.tbl)[0][:10]
        sa, ma = self.state(A)
        sb, mb = self.state(B)
        assert sa.tobytes() == sb.tobytes() and ma.tobytes() == mb.tobytes(), "entity state differs"

    def still_work(self):
        st = self.state(self.A)[0]["state"]
        return np.nonzero((st != ST_ARRIVED) & (st != ST_WAITING))[0].astype(np.uint32)


def _factions(n, seed):
    rng = np.random.default_rng(seed)
    return np.where(rng.random(n) < 0.5, capi.FACTION_ID_NONE, rng.integers(0, 15, n)).astype(np.int32)


@pytest.mark.gpu
@pytest.mark.parametrize("hz", [20, 10, 5, 1])
def test_update_case_ticks(pf, hz):
    """the arriving crowd of cases.update_case (arrivals, adjacent-arrived cascade, WAITING, GARRISONED units), three
    ticks; faction-tagged records, a few units already blocking at load and four radii wider than the bit window"""
    p, cost, a, ms = cases.update_case(4242, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(hz)
    a["radius"][rng.choice(n, 4, replace=False)] = 50.0
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = _factions(n, hz)
    pre = rng.random(n) < 0.03
    tbl["blocking"][pre] = 1
    tbl["stop_x"][pre], tbl["stop_z"][pre] = a["pos"][pre, 0], a["pos"][pre, 1]
    tbl["stop_radius"][pre] = a["radius"][pre]
    P = Pair(3, cost, a, ms, hz, nlayers=4, tbl=tbl)     # a radius of 50 takes the 7 x 7 ground layer
    try:
        P.compare()
        nblock = 0
        for _ in range(3):
            b, _u = P.tick(P.still_work())
            nblock += b
        assert nblock > 20, nblock
    finally:
        P.close()


@pytest.mark.gpu
def test_waiting_expiry_unblocks(pf):
    """WAITING units with a short wait_ticks_left block through set_blocking, then expire into SET_MOVING one tick at a
    time: each releases exactly its recorded circle, and the counts end where they were before the block"""
    p, cost, a, ms = cases.update_case(77, 20)
    n = len(a["radius"])
    rng = np.random.default_rng(5)
    waiting = np.sort(rng.choice(np.nonzero(a["state"] == 0)[0], 80, replace=False)).astype(np.uint32)
    a["state"][waiting] = ST_WAITING
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID
    ext["wait_prev"][waiting] = 0
    ext["wait_ticks_left"][waiting] = rng.integers(1, 4, len(waiting))
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = _factions(n, 9)
    P = Pair(3, cost, a, ms, 20, ext=ext, tbl=tbl)
    try:
        before = [(P.B.blockers(0), P.B.faction_counts(0))]
        ops = P.set_blocking(waiting, True)
        assert len(ops) == len(waiting) - int(((a["flags"][waiting] & capi.FLAG_GARRISONED) != 0).sum())
        assert not (P.B.blockers(0) == before[0][0]).all()
        released = 0
        for _ in range(4):
            st = P.state(P.A)[0]["state"]
            work = waiting[st[waiting] == ST_WAITING]
            if not len(work):
                break
            _b, u = P.tick(work)
            released += u
        # every expiry released its block; a unit that left WAITING another way keeps it until a command releases it
        still = waiting[P.B.agents_read_blocking(n)["blocking"][waiting] != 0]
        assert released + len(still) == len(ops) and released >= 0.9 * len(ops), (released, len(still), len(ops))
        P.set_blocking(still, False)
        assert not P.B.agents_read_blocking(n)["blocking"].any()
        assert (P.B.blockers(0) == before[0][0]).all() and (P.B.faction_counts(0) == before[0][1]).all()
    finally:
        P.close()


@pytest.mark.gpu
def test_air_and_ground_twelve_layers(pf):
    """AIR and non-air units on a 12-layer map: non-air ops count on the ground and water layers, AIR ops on the air
    layers; two ticks, then set_blocking block / unblock"""
    p, cost, a, ms = cases.update_case(31, 20)
    n = len(a["radius"])
    rng = np.random.default_rng(31)
    air = rng.random(n) < 0.3
    a["flags"][air] |= capi.FLAG_AIR
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = _factions(n, 31)
    P = Pair(3, cost, a, ms, 20, nlayers=12, tbl=tbl)
    try:
        for _ in range(2):
            P.tick(P.still_work())
        sel = rng.choice(n, 300, replace=False)
        P.set_blocking(sel, True)
        assert P.B.agents_read_blocking(n)["blocking"][sel[air[sel]]].any()
        assert P.B.blockers(8).any() and P.B.blockers(0).any()
        P.set_blocking(sel[:150], False)
    finally:
        P.close()


@pytest.mark.gpu
def test_set_blocking_repeats_garrisoned_wide(pf):
    """set_blocking by uid: repeated uids within a call and repeated calls change nothing, GARRISONED entities take no
    op, radii beyond the bit window go through the host rasteriser; then faction-tagged blocks and an attacking
    pool_request_path"""
    p, cost, a, ms = cases.update_case(4243, 20)
    n = len(a["radius"])
    rng = np.random.default_rng(1)
    wide = rng.choice(n, 6, replace=False)
    a["radius"][wide] = rng.uniform(49.0, 90.0, 6).astype(np.float32)
    tbl = np.zeros(n, capi.BLOCKING)
    tbl["faction_id"] = rng.integers(0, 4, n)
    P = Pair(3, cost, a, ms, 20, nlayers=4, tbl=tbl)
    try:
        garr = np.nonzero(a["flags"] & capi.FLAG_GARRISONED)[0]
        assert len(garr)
        sel = np.concatenate([rng.choice(n, 200, replace=False), wide, garr])
        sel = np.concatenate([sel, sel[:50]])           # repeats inside one call
        ops = P.set_blocking(sel, True)
        assert (ops["range"] > 48).sum() == int(((a["flags"][wide] & capi.FLAG_GARRISONED) == 0).sum()) > 0
        assert not P.B.agents_read_blocking(n)["blocking"][garr].any()
        blk = P.B.blockers(0)
        assert len(P.set_blocking(sel, True)) == 0 and (P.B.blockers(0) == blk).all()
        # an attacking request: faction 3 is at war with 0 and 1, whose blocks it may cross
        for X in (P.A, P.B):
            X.set_enemy_factions(3, 0b11)
            X.request_faction(3)
        src, dst = a["pos"][int(sel[0])], a["flock_target"][1]
        ra = P.A.pool_request_path(0, (float(src[0]), float(src[1])), (float(dst[0]), float(dst[1])))
        rb = P.B.pool_request_path(0, (float(src[0]), float(src[1])), (float(dst[0]), float(dst[1])))
        assert ra == rb
        for X in (P.A, P.B):
            X.request_faction(capi.FACTION_ID_NONE)
        P.compare()
        ops = P.set_blocking(sel[::2], False)
        assert len(ops) > 0
        assert len(P.set_blocking(sel[::2], False)) == 0
    finally:
        P.close()


@pytest.mark.gpu
def test_empty_work_list(pf):
    p, cost, a, ms = cases.update_case(11, 20)
    P = Pair(3, cost, a, ms, 20)
    try:
        P.tick(P.still_work())
        assert P.tick(np.zeros(0, np.uint32)) == (0, 0)
    finally:
        P.close()


@pytest.mark.gpu
def test_errors_on_device(pf):
    """no blocking records -> PFNAV_ERR_ARG; contexts that uploaded halves of a population as shards -> PFNAV_ERR_STATE,
    and nothing changes"""
    L = capi.load()
    p, cost, a, ms = cases.update_case(12, 20)
    n = len(a["radius"])
    aa = dict(a); aa["flock_dest_index"] = np.arange(len(a["flock_target"]), dtype=np.int32)
    rec, fl = capi.pack_agents(aa)
    uids = np.arange(10, dtype=np.uint32)
    nav = capi.Nav(0)
    try:
        nav.map_create(3, 3, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
        nav.agents_upload(rec, fl, 20); nav.agents_upload_movestate(ms)
        nav.agents_set_work(np.arange(n, dtype=np.uint32))
        nav.agents_tick(0); nav.agents_compute_updates()
        assert L.pfnav_agents_apply_updates_ex(nav.h, capi.APPLY_BLOCKERS, None) == capi.ERR_ARG
        assert L.pfnav_agents_apply_updates_ex(nav.h, 2, None) == capi.ERR_ARG
        assert L.pfnav_agents_set_blocking(nav.h, uids.ctypes.data_as(C.c_void_p), 10, 1, None) == capi.ERR_ARG
        bad = np.zeros(n, capi.BLOCKING); bad["faction_id"] = 16
        assert L.pfnav_agents_upload_blocking(nav.h, bad.ctypes.data_as(C.c_void_p), n) == capi.ERR_ARG
        good = np.zeros(n, capi.BLOCKING)
        nav.agents_upload_blocking(good)
        big = np.array([n], np.uint32)
        assert L.pfnav_agents_set_blocking(nav.h, big.ctypes.data_as(C.c_void_p), 1, 1, None) == capi.ERR_ARG
    finally:
        nav.close()
    navs = [capi.Nav(0), capi.Nav(0)]
    grp = capi.Group(navs)
    try:
        blk = np.zeros(n, capi.BLOCKING)
        for r, nv in enumerate(navs):
            lo, hi = capi.mgpu_shard_range(n, r, 2)
            nv.map_create(3, 3, 1); nv.map_upload_layer(0, cost)
            nv.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, 20)
            assert L.pfnav_agents_upload_blocking(nv.h, blk[lo:hi].ctypes.data_as(C.c_void_p), hi - lo) == capi.ERR_STATE
            assert L.pfnav_agents_upload_blocking(nv.h, blk.ctypes.data_as(C.c_void_p), n) == capi.ERR_STATE
            assert L.pfnav_agents_set_blocking(nv.h, uids.ctypes.data_as(C.c_void_p), 10, 1, None) == capi.ERR_STATE
            assert L.pfnav_agents_apply_updates_ex(nv.h, capi.APPLY_BLOCKERS, None) == capi.ERR_STATE
            assert nv.map_commit() == 0 and not nv.blockers(0).any()
    finally:
        grp.close()
        for nv in navs:
            nv.close()


def test_errors_host_only(pf):
    """a host-only context has no device to decide ops on: PFNAV_ERR_NO_DEVICE"""
    L = capi.load()
    nav = capi.Nav(hostonly=True)
    try:
        b = np.zeros(4, capi.BLOCKING)
        u = np.arange(4, dtype=np.uint32)
        assert L.pfnav_agents_upload_blocking(nav.h, b.ctypes.data_as(C.c_void_p), 4) == capi.ERR_NO_DEVICE
        assert L.pfnav_agents_read_blocking(nav.h, b.ctypes.data_as(C.c_void_p), 4) == capi.ERR_NO_DEVICE
        assert L.pfnav_agents_set_blocking(nav.h, u.ctypes.data_as(C.c_void_p), 4, 1, None) == capi.ERR_NO_DEVICE
        assert L.pfnav_agents_apply_updates_ex(nav.h, capi.APPLY_BLOCKERS, None) == capi.ERR_NO_DEVICE
    finally:
        nav.close()


class _DeviceBlockingNav:
    """a Nav whose apply takes the blocks of stopping units on the device: cases.run_trajectory's own incref of every
    stopped unit is then the device's, and only the host-only mirror still takes it by hand"""

    def __init__(self, nav):
        self._nav = nav

    def __getattr__(self, name):
        return getattr(self._nav, name)

    def agents_upload(self, rec, fl, hz):
        self._nav.agents_upload(rec, fl, hz)
        b = np.zeros(len(rec), capi.BLOCKING)
        b["faction_id"] = 0                     # the faction cases.run_trajectory increfs with
        self._nav.agents_upload_blocking(b)

    def agents_apply_updates(self, stream=0):
        self._nav.agents_apply_updates_ex(capi.APPLY_BLOCKERS, stream)

    def blockers_incref(self, *args):
        pass


@pytest.mark.gpu
@pytest.mark.parametrize("hz", [20, 10, 5, 1])
def test_trajectory_with_device_blocking(pf, nav, pforacle, pfref_or_golden, hz):
    """test_gpu_scale's device-resident trajectories (a marching crowd for eight ticks, an arriving crowd for one) with
    the blocks taken by pfnav_agents_apply_updates_ex: positions, states, velocities and patches against the plain-C port
    re-seeded every tick (or the compiled reference), blocker counts against a host-only mirror (or the reference), and
    local islands, exactly as the host-side blocking run checks them"""
    cw = 3
    dnav = _DeviceBlockingNav(nav)
    p, cost, a = cases.agent_case(cw, 1500, 3, 3131, 0.03, 2.6)
    a["state"][:] = 0
    n = len(a["radius"])
    ms = np.zeros(n, capi.MOVESTATE)
    ms["next_pos"][:, 0] = a["pos"][:, 0]; ms["next_pos"][:, 2] = a["pos"][:, 1]
    ms["step"] = 1.0 / (20 // hz)
    ms["next_rot"] = cases.dir_quat(a["vel"] + 1e-6)
    ms["combat_facing"] = ms["next_rot"]
    ms["vel_hist"] = np.repeat(a["vel"][:, None, :], 14, axis=1)
    ref = pfref_or_golden.RefMap(cw, cw, p) if pfref_or_golden else None
    try:
        out = cases.run_trajectory(dnav, ref, pforacle, a, ms, cw, cost, hz, 8, with_blockers=True, follow=True)
        assert len(out) == 8 and out[-1][0] > 1000, out
    finally:
        if ref is not None:
            ref.close()
    p, cost, a, ms = cases.update_case(4242, hz)
    ref = pfref_or_golden.RefMap(cw, cw, p) if pfref_or_golden else None
    try:
        out = cases.run_trajectory(dnav, ref, pforacle, a, ms, cw, cost, hz, 1, with_blockers=True)
        assert len(out) == 1 and out[0][0] > 1000, out
        assert nav.agents_read_blocking(len(a["radius"]))["blocking"].sum() > 50
    finally:
        if ref is not None:
            ref.close()
