"""pfnav_group_change_population: a job's population change given whole to an in-process group of 2 or 3 sharded
contexts (3: unequal ranges), against one context holding the whole population that takes the same batch through
pfnav_agents_change_population.

After each change, exchange of the blocker ops, commit and gather: every member owns the balanced range of the new
population; its own-range agents, movestate, movestate_ext and blocking records (concatenated over the members) equal the
single context's byte for byte, blocker grids are equal on every member, and agents_set_work_dev gives the single
context's work list split by range. Then resident ticks agree bit for bit (velocities, preferred / desired velocities,
LOS bits, patches, state): cohesion pins each member's device-built member lists, the neighbour queries its population
facts, and the formation inputs enter through the tick. The NCCL form is checked by
tests/tools/mgpu_nccl_population_check.py under torchrun."""
import numpy as np
import pytest

import cases
import commands_ref as cr
from test_gpu_mgpu_commands import Job, _devices, _population

capi, synth = cases.capi, cases.synth
ST_MOVING, ST_ARRIVED, ST_SURROUND = 0, 2, 5
WORLDS = pytest.mark.parametrize("world", [2, 3])


def _ext_default(n):
    e = np.zeros(n, capi.MOVESTATE_EXT)
    e["surround_target_uid"] = capi.NULL_UID
    e["rot"][:, 3] = 1.0
    return e


class PopJob(Job):
    def __init__(self, *a, form=None, **kw):
        super().__init__(*a, **kw)
        self.has_ext = kw.get("ext") is not None
        if form is not None:
            for X, (lo, hi) in [(self.one, (0, self.n))] + list(zip(self.navs, self.ranges)):
                X.agents_upload_formation(form[lo:hi])

    def change(self, rm, add, ms, ext=None, form=None, blk=None, flocks=None):
        rm = np.asarray(rm, np.int64).reshape(-1)
        add = np.ascontiguousarray(add, capi.AGENT)
        self.one.agents_change_population(rm, add, ms=ms, ext=ext, formation=form, blocking=blk, flocks=flocks)
        self.grp.change_population(rm, add, ms=ms, ext=ext, formation=form, blocking=blk, flocks=flocks)
        self.n = self.n - len(np.unique(rm)) + len(add)
        self.ranges = [capi.mgpu_shard_range(self.n, r, self.world) for r in range(self.world)]
        if flocks is not None:
            self.fl = np.ascontiguousarray(flocks, capi.FLOCK).copy()
        if self.blocking:
            nd1 = self.one.map_commit()
            self.grp.exchange_blocker_ops()
            assert [nv.map_commit() for nv in self.navs] == [nd1] * self.world
        assert len(self.one.agents_read_work()) == 0 and all(len(nv.agents_read_work()) == 0 for nv in self.navs)
        self.grp.gather()
        for nv in self.navs:
            assert nv.agents_device_ptrs()[2] == self.n
        self.work_lists()
        return self.compare()

    def compare(self, movestate=True):
        a1 = super().compare(movestate)
        if self.has_ext:
            got = np.concatenate([nv.agents_read_movestate_ext(hi - lo) for nv, (lo, hi) in zip(self.navs, self.ranges)])
            assert got.tobytes() == self.one.agents_read_movestate_ext(self.n).tobytes(), "movestate_ext differs"
        return a1


def _case(world, seed=4242, hz=20, ext=False, form=False, blocking=False, nlayers=1, extra_flocks=1):
    cost, rec, fl, ms = _population(seed, hz)
    n, nf = len(rec), len(fl)
    e = _ext_default(n) if ext else None
    f = None
    if form:
        f = np.zeros(n, capi.FORMATION_IN)
        f["target_orientation"][:, 3] = 1.0
    J = PopJob(3, cost, rec, fl, ms, hz, world, nlayers=nlayers, ext=e, ndests=nf + extra_flocks + 2, blocking=blocking, form=f)
    return J, rec, fl, ms


def _spawn(J, who, flock=None, shift=0.6):
    s, m = J.one.agents_read_state(J.n)
    a = s[who].copy()
    a["pos"] += np.float32(shift); a["prev_pos"] += np.float32(shift)
    if flock is not None:
        a["flock"] = flock
    mm = m[who].copy()
    mm["next_pos"][:, 0] += np.float32(shift); mm["next_pos"][:, 2] += np.float32(shift)
    return a, mm


def _blk(k):
    b = np.zeros(k, capi.BLOCKING)
    b["faction_id"] = capi.FACTION_ID_NONE
    return b


def _none():
    return np.zeros(0, capi.AGENT), np.zeros(0, capi.MOVESTATE)


@pytest.mark.gpu
def test_symbols(pf):
    assert "pfnav_mgpu_change_population" in capi.SYMBOLS and "pfnav_group_change_population" in capi.SYMBOLS


@pytest.mark.gpu
@WORLDS
def test_removals_in_rank0_then_appends_then_both(pf, world):
    """removals only in rank 0's range (every boundary shifts down), appends only (rows move up, into an old flock and a
    flock appended in the same call), then one call that removes and appends"""
    J, rec, fl, ms = _case(world, seed=4242)
    try:
        J.ticks(2)
        lo, hi = J.ranges[0]
        rng = np.random.default_rng(1)
        J.change(rng.choice(np.arange(lo, hi), 90, replace=True), *_none())
        J.ticks(3)
        s = J.compare()
        nf = len(J.fl)
        who = np.nonzero(s["state"] == ST_MOVING)[0][:60]
        a1, m1 = _spawn(J, who[:30])
        a2, m2 = _spawn(J, who[30:], flock=nf)
        grown = np.zeros(nf + 1, capi.FLOCK); grown[:-1] = J.fl
        grown["target"][-1], grown["dest"][-1] = s["pos"][who].mean(axis=0) + 20.0, nf
        J.change([], np.concatenate([a1, a2]), np.concatenate([m1, m2]), flocks=grown)
        J.ticks(3)
        a3, m3 = _spawn(J, rng.choice(J.n, 40, replace=False), shift=-0.4)
        J.change(rng.choice(J.n, 70, replace=False), a3, m3)
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_whole_member_range_removed(pf, world):
    J, rec, fl, ms = _case(world, seed=13)
    try:
        J.ticks(2)
        lo, hi = J.ranges[world - 1]
        a, m = _spawn(J, np.arange(0, 40, 2))
        J.change(np.arange(lo, hi), a, m)
        lo, hi = J.ranges[0]
        J.change(np.arange(lo, hi), *_none())
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_blocking_units_removed_on_every_member(pf, world):
    """the C2 population with shared device blockers: units that hold device-decided blocks die on every member, and
    appended units bring blocking records"""
    J = _c2_job(pf, world)
    rng = np.random.default_rng(3)
    try:
        s = J.tick()
        stop = rng.choice(np.nonzero(s["state"] == ST_MOVING)[0], 300, replace=False).astype(np.uint32)
        J.commands(cr.deltas(stop, state=ST_ARRIVED, velocity=(0.0, 0.0)), block=(np.zeros(0, np.uint32), stop))
        bl = J.one.agents_read_blocking(J.n)
        held = np.nonzero(bl["blocking"] == 1)[0]
        assert all(len(J.own(r, held)) for r in range(world))
        before = J.one.blockers(0).copy()
        a, m = _spawn(J, np.arange(12))
        J.change(held[::2], a, m, blk=_blk(12))
        assert not (J.one.blockers(0) == before).all()
        J.ticks(3)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_foreign_surround_target_removed_and_default_records(pf, world):
    """a surround target owned by another member dies: every member's units that named it get PFNAV_NULL_UID; other
    targets are renumbered. Appended records with ext / formation tables present take the defaults (NULL records), then
    explicit ones."""
    J, rec, fl, ms = _case(world, seed=5, ext=True, form=True, nlayers=2)
    try:
        n = J.n
        lo_l, hi_l = J.ranges[-1]
        tgt, far = lo_l + 2, n - 1
        e = _ext_default(n)
        sur = np.concatenate([np.arange(10, 20), np.arange(J.ranges[1][0] + 5, J.ranges[1][0] + 15)])
        e["surround_target_uid"][sur] = tgt
        e["surround_target_uid"][30:35] = far
        s, m = J.one.agents_read_state(n)
        s["state"][sur] = ST_SURROUND
        J.one.agents_upload(s, J.fl, J.hz); J.one.agents_upload_movestate(m); J.one.agents_upload_movestate_ext(e)
        f = np.zeros(n, capi.FORMATION_IN); f["target_orientation"][:, 3] = 1.0
        J.one.agents_upload_formation(f)
        for nv, (lo, hi) in zip(J.navs, J.ranges):
            nv.agents_upload_shard(s[lo:hi], lo, hi, n, J.fl, J.hz)
        J.grp.gather()
        for nv, (lo, hi) in zip(J.navs, J.ranges):
            nv.agents_upload_movestate(m[lo:hi]); nv.agents_upload_movestate_ext(e[lo:hi]); nv.agents_upload_formation(f[lo:hi])
        J.work_lists()
        J.ticks(2)
        a, mm = _spawn(J, np.arange(0, 60, 3))
        a["radius"][::2] = 6.0                                     # layer 1
        J.change([tgt, 3], a, mm)
        x = np.concatenate([nv.agents_read_movestate_ext(hi - lo) for nv, (lo, hi) in zip(J.navs, J.ranges)])
        assert (x["surround_target_uid"][sur - (sur > 3) - (sur > tgt)] == capi.NULL_UID).all()
        assert (x["surround_target_uid"][30 - 1:35 - 1] == far - 2).all()
        J.ticks(2)
        a, mm = _spawn(J, np.arange(5, 45, 4), shift=0.3)
        ee = _ext_default(len(a)); ee["wait_ticks_left"] = 2
        ff = np.zeros(len(a), capi.FORMATION_IN); ff["target_orientation"][:, 3] = 1.0
        J.change([0], a, mm, ext=ee, form=ff)
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_last_flock_dropped(pf, world):
    J, rec, fl, ms = _case(world, seed=31)
    try:
        s = J.tick()
        last = len(J.fl) - 1
        J.change(np.nonzero(s["flock"] == last)[0], *_none(), flocks=J.fl[:last].copy())
        s = J.ticks(6)
        assert s["flock"].max() == last - 1
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_shrunk_below_world_then_zero_then_refilled(pf, world):
    J, rec, fl, ms = _case(world, seed=12, blocking=True)
    try:
        s = J.tick()
        keep_a, keep_m = J.one.agents_read_state(J.n)
        J.change(np.arange(1, J.n), *_none(), blk=np.zeros(0, capi.BLOCKING))
        assert J.n == 1 and J.ranges[-1][1] == J.ranges[-1][0]       # a member owns nothing
        J.tick()
        J.change([0], *_none(), blk=np.zeros(0, capi.BLOCKING))
        assert J.n == 0
        J.change([], keep_a, keep_m, blk=_blk(len(keep_a)))
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_growth_past_buffer_capacity(pf, world):
    """1 000 -> 6 000 entities: every member's tables and the columns regrow"""
    rng = np.random.default_rng(6)
    cw = 4
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, 0x5EED0000), cw, cw)
    a = synth.make_agents(cost, cw, cw, 6000, 3, 0x5EED0000, radius=1.0, spacing=2.2)
    rec, fl = capi.pack_agents(a)
    ms = np.zeros(len(rec), capi.MOVESTATE)
    ms["next_pos"][:, 0], ms["next_pos"][:, 2] = rec["pos"][:, 0], rec["pos"][:, 1]
    ms["step"] = 1.0; ms["next_rot"][:, 3] = 1.0; ms["combat_facing"][:, 3] = 1.0
    e = _ext_default(len(rec)); e["wait_prev"] = rng.integers(0, 3, len(rec))
    fl["dest"] = -1
    J = PopJob(cw, cost, rec[:1000], fl, ms[:1000], 20, world, ext=e[:1000], blocking=True)
    try:
        J.tick(passes=0)
        b = _blk(5000); b["faction_id"] = rng.integers(0, 16, 5000)
        J.change([], rec[1000:], ms[1000:], ext=e[1000:], blk=b)
        assert J.n == 6000
        J.ticks(3)
    finally:
        J.close()


def _c2_job(pf, world):
    """the benchmark's C2 population (100 000 entities) with device blockers shared by the group, goals requested"""
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
    J = PopJob(bench.CHUNKS, W["cost"], rec, fl, ms, 20, world, blocking=True)
    for X in J.all():
        X.pool_request_goals(np.arange(len(fl), dtype=np.int32), goals, 0)
    J.tick = lambda passes=0, _t=J.tick: _t(passes=0)
    return J


@pytest.mark.gpu
@WORLDS
def test_c2_churn_with_device_blockers(pf, world):
    """the benchmark's C2 population: 1 % removed and 1 % added every tick over several ticks, with device blockers
    shared by the group"""
    J = _c2_job(pf, world)
    rng = np.random.default_rng(8)
    try:
        for t in range(3):
            J.tick()
            k = J.n // 100
            a, m = _spawn(J, rng.choice(J.n, k, replace=False), shift=0.25)
            a["state"] = ST_MOVING
            J.change(rng.choice(J.n, k, replace=False), a, m, blk=_blk(k))
        J.tick()
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_refusals_change_nothing_anywhere(pf, world):
    """refusals every member sees, and a stranded flock index only the last member sees, fail on every member and change
    nothing; a following valid change and ticks still equal the single context that never saw them. Then the state
    errors."""
    J, rec, fl, ms = _case(world, seed=21, blocking=True)
    try:
        J.tick()
        a, m = _spawn(J, np.arange(4))
        b = _blk(4)
        bad_flock = a.copy(); bad_flock["flock"][0] = len(J.fl)
        bad_float = a.copy(); bad_float["velocity"][2, 0] = np.nan
        bad_blk = b.copy(); bad_blk["faction_id"][3] = 16
        s = J.compare()
        last = len(J.fl) - 1
        lo, hi = J.ranges[-1]
        keep = np.nonzero(s["flock"] == last)[0]
        assert len(J.own(world - 1, keep)) and len(keep) > len(J.own(world - 1, keep))
        stranded = keep[(keep < lo) | (keep >= hi)]              # the last member keeps members of the dropped flock
        before = [(nv.agents_read_state(hi - lo)[0].tobytes(), nv.agents_read_blocking(hi - lo).tobytes(), nv.blockers(0).copy())
                  for nv, (lo, hi) in zip(J.navs, J.ranges)]
        for kw in (dict(remove=[J.n]), dict(add=bad_flock), dict(add=bad_float), dict(blocking=bad_blk), dict(ms=None),
                   dict(blocking=None), dict(ext=_ext_default(4)), dict(flocks=J.fl[:1].copy())):
            args = dict(remove=[0, 1], add=a, ms=m, blocking=b)
            args.update(kw)
            with pytest.raises(capi.PfnavError, match="error -1.*member 0"):
                J.grp.change_population(args.pop("remove"), args.pop("add"), **args)
        with pytest.raises(capi.PfnavError, match="error -1.*member %d" % (world - 1)):
            J.grp.change_population(stranded, np.zeros(0, capi.AGENT), ms=np.zeros(0, capi.MOVESTATE),
                                    blocking=np.zeros(0, capi.BLOCKING), flocks=J.fl[:last].copy())
        for nv, (lo, hi), bf in zip(J.navs, J.ranges, before):
            assert nv.agents_read_state(hi - lo)[0].tobytes() == bf[0] and nv.agents_read_blocking(hi - lo).tobytes() == bf[1]
            nv.map_commit()                                        # no op was queued by a refusal
            assert (nv.blockers(0) == bf[2]).all()
        J.one.map_commit()
        J.grp.gather()
        J.work_lists()
        J.compare()
        J.change([0, 1], a, m, blk=b)
        J.ticks(4)
        # state errors
        with pytest.raises(capi.PfnavError, match="error -4"):
            J.navs[0].mgpu_change_population([0], np.zeros(0, capi.AGENT))
        lone = capi.Nav(0)
        host = capi.Nav(0, hostonly=True)
        try:
            with pytest.raises(capi.PfnavError, match="error -4"):
                lone.mgpu_change_population([0], np.zeros(0, capi.AGENT))
            with pytest.raises(capi.PfnavError, match="error -3"):
                host.mgpu_change_population([0], np.zeros(0, capi.AGENT))
        finally:
            lone.close(); host.close()
        with pytest.raises(capi.PfnavError, match="error -4"):             # the solo call still refuses on a member
            J.navs[1].agents_change_population([0], np.zeros(0, capi.AGENT))
        lo0, hi0 = J.ranges[0]
        J.navs[0].agents_upload_shard(J.navs[0].agents_read_state(hi0 - lo0, movestate=False)[0], lo0, hi0, J.n, J.fl, 20)
        with pytest.raises(capi.PfnavError, match="error -4"):
            J.grp.change_population([lo0], np.zeros(0, capi.AGENT), ms=np.zeros(0, capi.MOVESTATE), blocking=np.zeros(0, capi.BLOCKING))
        J.grp.gather()
    finally:
        J.close()
