"""pfnav_group_commands: a job's command batch given whole to every member of an in-process group of 2 or 3 sharded
contexts (3: unequal ranges), against one context holding the whole population that takes the same batch through
pfnav_agents_commands.

Every scenario builds the single context and the group (on device 0, and on further devices where the box has them) from
the same seeds. After each batch and the gather: every member's entity state and movestate (own ranges, concatenated)
equal the single context's byte for byte, and agents_set_work_dev gives the single context's work list split by range.
Then resident ticks (tick, compute_updates, apply_updates, gather, work list): velocities, preferred / desired
velocities, LOS bits, patches and state bit for bit on every member. Cohesion over flocks whose members sit on every
rank is what pins each member's device-built member lists, and the neighbour queries pin the population facts (largest
radius, any GARRISONED) a member refreshes from the radii and flag bits it wrote for the other members' entities.
The NCCL form is checked by tests/tools/mgpu_nccl_commands_check.py under torchrun."""
import numpy as np
import pytest

import cases
import commands_ref as cr

capi, synth = cases.capi, cases.synth
ST_MOVING, ST_ARRIVED, ST_SEEK, ST_WAITING, ST_SURROUND = 0, 2, 3, 4, 5
GARR = capi.FLAG_GARRISONED


def _devices(world):
    import torch
    n = torch.cuda.device_count()
    return [i % n for i in range(world)]


class Job:
    """one: a single context taking agents_commands; navs: `world` sharded members of a group taking Group.commands"""

    def __init__(self, cw, cost, rec, fl, ms, hz, world, nlayers=1, ext=None, ndests=None, blocking=False, ms_upload=None):
        self.n, self.world, self.hz = len(rec), world, hz
        self.fl = np.ascontiguousarray(fl, capi.FLOCK).copy()
        ndests = ndests or len(fl)
        self.blocking = blocking
        self.ranges = [capi.mgpu_shard_range(self.n, r, world) for r in range(world)]
        self.one = capi.Nav(0)
        self.navs = [capi.Nav(d) for d in _devices(world)]
        self.grp = None
        for X in self.all():
            X.map_create(cw, cw, nlayers)
            for l in range(nlayers):
                X.map_upload_layer(l, cost); X.map_build_nav(l); X.route_build(l)
            X.pool_create(ndests, ndests * cw * cw)
        self.grp = capi.Group(self.navs)
        if blocking:
            self.grp.share_blockers()
        tbl = np.zeros(self.n, capi.BLOCKING); tbl["faction_id"] = capi.FACTION_ID_NONE
        self.one.agents_upload(rec, self.fl, hz)
        self.one.agents_upload_movestate(ms)
        for nv, (lo, hi) in zip(self.navs, self.ranges):
            nv.agents_upload_shard(rec[lo:hi], lo, hi, self.n, self.fl, hz)
        self.grp.gather()
        for r, (X, lo, hi) in enumerate([(self.one, 0, self.n)] + [(nv, lo, hi) for nv, (lo, hi) in zip(self.navs, self.ranges)]):
            if X is not self.one and (ms_upload is None or ms_upload[r - 1]):
                X.agents_upload_movestate(ms[lo:hi])
            if ext is not None:
                X.agents_upload_movestate_ext(ext[lo:hi])
            if blocking:
                X.agents_upload_blocking(tbl[lo:hi])
        self.work_lists()

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

    def commands(self, d, flocks=None, block=None):
        """the batch on both sides, then gather, work lists and state; block: (uids to unblock, uids to block) through
        agents_set_blocking on the owning members, exchange and map_commit"""
        self.one.agents_commands(d, flocks)
        self.grp.commands(d, flocks)
        if flocks is not None:
            self.fl = np.ascontiguousarray(flocks, capi.FLOCK).copy()
        if block is not None:
            self.one.agents_set_blocking(block[0], False); self.one.agents_set_blocking(block[1], True)
            nd1 = self.one.map_commit()
            for r, nv in enumerate(self.navs):
                nv.agents_set_blocking(self.own(r, block[0]), False); nv.agents_set_blocking(self.own(r, block[1]), True)
            self.grp.exchange_blocker_ops()
            assert [nv.map_commit() for nv in self.navs] == [nd1] * self.world
        self.one.agents_rebuild_index()
        self.grp.gather()
        self.work_lists()
        return self.compare()

    def work_lists(self):
        n1 = self.one.agents_set_work_dev()
        w1 = self.one.agents_read_work()
        assert n1 == len(w1)
        for r, nv in enumerate(self.navs):
            nw = nv.agents_set_work_dev()
            w = nv.agents_read_work()
            assert nw == len(w) and np.array_equal(w, self.own(r, w1)), ("work list", r)
        return w1

    def compare(self, movestate=True):
        a1, m1 = self.one.agents_read_state(self.n, movestate)
        parts = [nv.agents_read_state(hi - lo, movestate) for nv, (lo, hi) in zip(self.navs, self.ranges)]
        aN = np.concatenate([p[0] for p in parts])
        assert aN.tobytes() == a1.tobytes(), np.nonzero(aN != a1)[0][:10]
        if movestate:
            assert np.concatenate([p[1] for p in parts]).tobytes() == m1.tobytes(), "movestate differs"
        if self.blocking:
            got = np.concatenate([nv.agents_read_blocking(hi - lo) for nv, (lo, hi) in zip(self.navs, self.ranges)])
            assert got.tobytes() == self.one.agents_read_blocking(self.n).tobytes()
            for nv in self.navs:
                assert (nv.blockers(0) == self.one.blockers(0)).all()
        return a1

    def _tick_one(self, X, nw, passes):
        for _ in range(passes):              # serve the pool misses of the new orders; the same calls on every context
            X.agents_tick(capi.TICK_VDES_FROM_POOL)
            X.pool_repair()
        X.agents_tick(capi.TICK_VDES_FROM_POOL)
        X.agents_compute_updates()
        out = (X.agents_read_velocities(nw),) + X.agents_read_debug(nw) + (X.agents_read_patches(nw),)
        if self.blocking:
            X.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        else:
            X.agents_apply_updates()
        return out

    def tick(self, passes=2):
        """one resident tick on every context, compared at every output"""
        one = self.one
        nw1 = len(one.agents_read_work())
        ref = self._tick_one(one, nw1, passes) if nw1 else None
        if self.blocking:
            nd1 = one.map_commit()
        one.agents_rebuild_index()
        outs = []
        for nv in self.navs:
            nw = len(nv.agents_read_work())
            if nw:
                outs.append(self._tick_one(nv, nw, passes))
        if self.blocking:
            self.grp.exchange_blocker_ops()
            assert [nv.map_commit() for nv in self.navs] == [nd1] * self.world
        self.grp.gather()
        if ref is not None:
            for k, name in enumerate(("velocities", "vpref", "vdes", "los", "patches")):
                got = np.concatenate([o[k] for o in outs])
                assert got.tobytes() == ref[k].tobytes(), (name, np.nonzero(got != ref[k])[0][:10])
        self.work_lists()
        return self.compare()

    def ticks(self, k=8):
        for _ in range(k):
            s = self.tick()
        return s


def _population(seed, hz):
    """cases.update_case with the entities shuffled: its flocks are contiguous uid blocks, and here every flock must have
    members on every rank"""
    p, cost, a, ms = cases.update_case(seed, hz)
    nf = len(a["flock_target"])
    aa = dict(a); aa["flock_dest_index"] = np.arange(nf, dtype=np.int32)
    rec, fl = capi.pack_agents(aa)
    perm = np.random.default_rng(seed).permutation(len(rec))
    return cost, rec[perm].copy(), fl, ms[perm].copy()


def _case(world, seed=4242, hz=20, extra_flocks=1, ext=False, **kw):
    cost, rec, fl, ms = _population(seed, hz)
    nf = len(fl)
    e = None
    if ext:
        e = np.zeros(len(rec), capi.MOVESTATE_EXT); e["surround_target_uid"] = capi.NULL_UID
    return Job(3, cost, rec, fl, ms, hz, world, ext=e, ndests=nf + extra_flocks + 2, **kw), rec, fl


def _grown(fl, target, dest):
    out = np.zeros(len(fl) + 1, capi.FLOCK)
    out[:-1] = fl
    out["target"][-1], out["dest"][-1], out["layer"][-1] = target, dest, 0
    return out


def _on_every_rank(J, uids):
    """the listed uids hold members of every rank"""
    return all(len(J.own(r, uids)) for r in range(J.world))


WORLDS = pytest.mark.parametrize("world", [2, 3])


@pytest.mark.gpu
def test_symbols(pf):
    assert "pfnav_mgpu_commands" in capi.SYMBOLS and "pfnav_group_commands" in capi.SYMBOLS


@pytest.mark.gpu
@WORLDS
def test_new_flock_with_several_deltas_per_uid(pf, world):
    """ARRIVED units and part of a moving flock, from every rank, get a move order to a flock appended to the table; the
    order of one unit arrives as several deltas"""
    J, rec, fl = _case(world)
    try:
        J.ticks(2)
        s = J.compare()
        spread = lambda u, k: np.unique(u[np.linspace(0, len(u) - 1, min(k, len(u))).astype(int)])
        who = np.concatenate([spread(np.nonzero(s["state"] == ST_ARRIVED)[0], 60), spread(np.nonzero((s["state"] == ST_MOVING) & (s["flock"] == 1))[0], 90)])
        assert _on_every_rank(J, who)
        new = _grown(J.fl, s["pos"][who].mean(axis=0) + 30.0, len(fl))
        d = np.concatenate([cr.deltas(who[:10], flock=0), cr.deltas(who, state=ST_MOVING, clear_hist=True), cr.deltas(who, flock=len(fl))])
        J.commands(d, new)
        s = J.ticks(8)
        assert (s["flock"][who] == len(fl)).all()
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_flock_emptied_stop_and_teleport(pf, world):
    J, rec, fl = _case(world, seed=77)
    try:
        J.tick()
        s = J.compare()
        f2 = np.nonzero(s["flock"] == 2)[0]
        J.commands(cr.deltas(f2, flock=1))
        s = J.ticks(3)
        assert not (s["flock"] == 2).any()
        moving = np.nonzero(s["state"] == ST_MOVING)[0]
        J.commands(cr.deltas(moving[::7], state=ST_ARRIVED, velocity=(0.0, 0.0)))
        s = J.ticks(2)
        moving = np.nonzero(s["state"] == ST_MOVING)[0][::11]
        donors = np.nonzero(s["state"] == ST_ARRIVED)[0][:len(moving)]
        moving = moving[:len(donors)]
        J.commands(cr.deltas(moving, position=s["pos"][donors] + np.float32(0.75)))
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_flock_emptied_and_dropped_in_one_batch(pf, world):
    J, rec, fl = _case(world, seed=31)
    try:
        J.tick()
        s = J.compare()
        last = len(fl) - 1
        J.commands(cr.deltas(np.nonzero(s["flock"] == last)[0], flock=0), J.fl[:last].copy())
        s = J.ticks(4)
        assert s["flock"].max() == last - 1
        who = np.nonzero(s["state"] == ST_MOVING)[0][::6]
        J.commands(cr.deltas(who, flock=last), _grown(J.fl, s["pos"][who].mean(axis=0), last))
        J.ticks(4)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_layer_change_and_garrison_flips(pf, world):
    J, rec, fl = _case(world, seed=99, nlayers=2)
    try:
        J.tick()
        s = J.compare()
        grow = np.nonzero(s["state"] == ST_MOVING)[0][::9]
        J.commands(cr.deltas(grow, radius=6.0))
        s = J.ticks(2)
        g = np.nonzero(s["flags"] & GARR)[0]
        assert len(g)
        J.commands(cr.deltas(g, flags=s["flags"][g] & ~np.uint32(GARR)))
        s = J.ticks(3)
        g = np.nonzero(s["state"] == ST_MOVING)[0][5::13]
        J.commands(cr.deltas(g, flags=s["flags"][g] | np.uint32(GARR)))
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_seek_and_surround_targets(pf, world):
    """TARGET writes go into the owners' movestate_ext tables; batches precede the first tick, as in the single-context
    suite"""
    J, rec, fl = _case(world, seed=5, ext=True)
    try:
        nf = len(fl)
        allchunks = [(c // 3, c % 3) for c in range(9)]
        foes = np.arange(0, 40, 8)
        for X in J.all():
            fp = X.footprints(rec["pos"], rec["radius"])
            X.pool_request_entity_fields(nf + 1, capi.TARGET_ENEMIES, fp[foes], allchunks)
            X.pool_request_entity_fields(nf + 2, capi.TARGET_ENTITY, fp[3:4], allchunks)
        mv = np.nonzero(rec["state"] == ST_MOVING)[0]
        seek, sur = mv[100:160], mv[::9][:40]
        d = np.concatenate([cr.deltas(seek, state=ST_SEEK, flock=-1, aux_dest1=nf + 2),
                            cr.deltas(sur, state=ST_SURROUND, aux_dest1=nf + 3, target=(3, 0.0)),
                            cr.deltas(sur[:5], target=(capi.NULL_UID, 2.5))])
        J.commands(d)
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_foreign_radius_and_garrison_set_the_facts(pf, world):
    """one entity of rank 0 next to rank 1's units grows to the population's largest radius (every member's neighbour
    query widens); later one entity of the last rank is GARRISONED in a population with none (the query starts
    filtering on every member)"""
    J, rec, fl = _case(world, seed=12)
    try:
        s = J.compare()
        if (s["flags"] & GARR).any():
            g = np.nonzero(s["flags"] & GARR)[0]
            J.commands(cr.deltas(g, flags=s["flags"][g] & ~np.uint32(GARR)))
        s = J.tick()
        lo1, hi1 = J.ranges[1]
        near = s["pos"][lo1:hi1].mean(axis=0)
        own0 = np.arange(*J.ranges[0])
        big = int(own0[np.argmin(np.linalg.norm(s["pos"][own0] - near, axis=1))])
        assert s["radius"].max() < 4.99
        J.commands(cr.deltas([big], radius=4.99))
        s = J.ticks(3)
        lo, hi = J.ranges[-1]
        moving = np.nonzero(s["state"][lo:hi] == ST_MOVING)[0] + lo
        J.commands(cr.deltas(moving[:1], flags=s["flags"][moving[:1]] | np.uint32(GARR)))
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_batch_on_one_range_only(pf, world):
    """every delta names a uid of the middle / last rank: the others apply no own record, only flock ids"""
    J, rec, fl = _case(world, seed=13)
    try:
        s = J.tick()
        lo, hi = J.ranges[1]
        who = np.nonzero(s["state"][lo:hi] == ST_MOVING)[0][::4] + lo
        J.commands(np.concatenate([cr.deltas(who, flock=0), cr.deltas(who[::2], state=ST_ARRIVED, velocity=(0.0, 0.0))]))
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_c2_order_waves(pf, world):
    """the benchmark's C2 population (100 000 agents, 16 goals) with device blockers shared by the group: every tick a
    wave of stops and regrouping move orders from every rank, their blockers taken through agents_set_blocking on the
    owners and the exchange"""
    import importlib, os, sys
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    bench = importlib.import_module("bench")
    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    rec, fl, n = W["rec"], W["flocks"], W["n_total"]
    ms = np.zeros(n, capi.MOVESTATE)
    ms["next_pos"][:, 0], ms["next_pos"][:, 2] = rec["pos"][:, 0], rec["pos"][:, 1]
    face = fl["target"][rec["flock"]] - rec["pos"]
    ms["step"] = 1.0; ms["next_rot"] = cases.dir_quat(face); ms["combat_facing"] = ms["next_rot"]
    ms["vel_hist"] = rec["velocity"][:, None, :]
    goals = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(len(fl))], np.int32)
    J = Job(bench.CHUNKS, W["cost"], rec, fl, ms, 20, world, blocking=True)
    rng = np.random.default_rng(8)
    try:
        for X in J.all():
            X.pool_request_goals(np.arange(len(fl), dtype=np.int32), goals, 0)
        for t in range(4):
            s = J.tick(passes=0)
            moving = np.nonzero(s["state"] == ST_MOVING)[0]
            stop = rng.choice(moving, min(200, len(moving)), replace=False)
            rest = np.setdiff1d(np.arange(n), stop)
            go = rng.choice(rest, 300, replace=False)
            d = np.concatenate([cr.deltas(stop, state=ST_ARRIVED, velocity=(0.0, 0.0)),
                                cr.deltas(go, state=ST_MOVING, flock=rng.integers(0, len(fl), len(go)), clear_hist=True)])
            J.commands(d, block=(go.astype(np.uint32), stop.astype(np.uint32)))
        J.tick(passes=0)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_more_flocks_than_one_scan_pass(pf, world):
    """2 500 flocks (three passes of the scan over the flocks), a third of the population regrouped: preferred velocities
    (cohesion over the member lists) and velocities bit for bit"""
    rng = np.random.default_rng(4)
    n, nf = 20_000, 2_500
    cost = synth.cost_from_pathable(synth.make_map(4, 4, 0x5EED0000), 4, 4)
    a = synth.make_agents(cost, 4, 4, n, 2, 0x5EED0000, radius=1.0, spacing=2.2)
    rec, _ = capi.pack_agents(a)
    rec["flock"] = rng.integers(-1, nf - 100, n)
    fl = np.zeros(nf, capi.FLOCK)
    fl["target"] = rng.uniform(-900, -100, (nf, 2)) * [1, -1]; fl["dest"] = -1
    d = cr.deltas(rng.choice(n, n // 3, replace=False), flock=rng.integers(-1, nf, n // 3))
    ranges = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
    one, navs = capi.Nav(0), [capi.Nav(dv) for dv in _devices(world)]
    grp = None
    try:
        for X in [one] + navs:
            X.map_create(4, 4, 1); X.map_upload_layer(0, cost)
            X.set_cohesion_mode(2)                            # the member lists, not the windowed pass
        grp = capi.Group(navs)
        one.agents_upload(rec, fl, 20)
        for nv, (lo, hi) in zip(navs, ranges):
            nv.agents_upload_shard(rec[lo:hi], lo, hi, n, fl, 20)
        grp.gather()
        one.agents_commands(d)
        one.agents_rebuild_index()
        grp.commands(d)
        grp.gather()
        nw = one.agents_set_work_dev()
        one.agents_tick(0)
        vp1, v1 = one.agents_read_debug(nw)[0], one.agents_read_velocities(nw)
        vps, vs = [], []
        for nv in navs:
            k = nv.agents_set_work_dev()
            nv.agents_tick(0)
            vps.append(nv.agents_read_debug(k)[0]); vs.append(nv.agents_read_velocities(k))
        assert np.concatenate(vps).tobytes() == vp1.tobytes() and np.concatenate(vs).tobytes() == v1.tobytes()
    finally:
        if grp is not None:
            grp.close()
        for X in [one] + navs:
            X.close()


@pytest.mark.gpu
@WORLDS
def test_refusals_change_nothing_anywhere(pf, world):
    """batches that only one member can refuse fail on every member and change nothing: a stranded flock index on one
    rank, and POSITION for a uid of the member without a movestate table; a following valid batch and ticks still equal
    the single context that never saw them. Then the state errors: a member whose range was uploaded in full and not
    gathered since, the NCCL form on a group member, a context in no job, a host-only context."""
    cost, rec, fl, ms = _population(21, 20)
    nf = len(fl)
    J = Job(3, cost, rec, fl, ms, 20, world, ndests=nf + 2, ms_upload=[True] * (world - 1) + [False])
    try:
        before = J.compare(movestate=False)
        last = nf - 1
        keep = np.nonzero(rec["flock"] == last)[0]
        lo, hi = J.ranges[-1]
        assert len(J.own(world - 1, keep)) and len(keep) > len(J.own(world - 1, keep))
        stranded = cr.deltas(keep[(keep < lo) | (keep >= hi)], flock=0)      # the last rank keeps members of the dropped flock
        with pytest.raises(capi.PfnavError, match="error -1.*member %d" % (world - 1)):
            J.grp.commands(stranded, J.fl[:last].copy())
        with pytest.raises(capi.PfnavError, match="error -1.*member %d" % (world - 1)):
            J.grp.commands(np.concatenate([cr.deltas(np.arange(10), state=ST_ARRIVED), cr.deltas([hi - 1], position=(1.0, 1.0))]))
        J.grp.gather()
        J.work_lists()
        assert J.compare(movestate=False).tobytes() == before.tobytes()
        J.navs[-1].agents_upload_movestate(ms[lo:hi])
        s = J.tick()
        who = np.nonzero(s["state"] == ST_MOVING)[0][::5]
        J.commands(cr.deltas(who, flock=last, state=ST_MOVING))
        J.ticks(8)
        # state errors
        with pytest.raises(capi.PfnavError, match="error -4"):
            J.navs[0].mgpu_commands(cr.deltas([0], state=0))
        lone = capi.Nav(0)
        host = capi.Nav(0, hostonly=True)
        try:
            with pytest.raises(capi.PfnavError, match="error -4"):
                lone.mgpu_commands(cr.deltas([0], state=0))
            with pytest.raises(capi.PfnavError, match="error -3"):
                host.mgpu_commands(cr.deltas([0], state=0))
        finally:
            lone.close(); host.close()
        s = J.compare()
        lo0, hi0 = J.ranges[0]
        J.navs[0].agents_upload_shard(J.navs[0].agents_read_state(hi0 - lo0, movestate=False)[0], lo0, hi0, J.n, J.fl, 20)
        with pytest.raises(capi.PfnavError, match="error -4"):
            J.grp.commands(cr.deltas([lo0], state=ST_ARRIVED))
        J.grp.gather()
        J.grp.commands(cr.deltas([lo0], state=ST_ARRIVED))
        assert J.navs[0].agents_read_state(1, movestate=False)[0]["state"][0] == ST_ARRIVED
    finally:
        J.close()
