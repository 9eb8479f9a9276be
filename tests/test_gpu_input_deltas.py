"""pfnav_agents_input_deltas and its job forms against the path they replace.

Twin contexts on the same map and population: A takes the batch through the new call; B takes the three steps --
agents_read_movestate_ext / agents_read_formation, the same records applied in numpy (inputs_ref.apply_np), and whole
uploads of both tables. After the batch both tables are compared byte for byte; then 8 resident ticks (tick,
compute_updates, apply_updates, rebuild_index, work list) compare velocities, preferred / desired velocities, LOS bits,
patches, entity state, movestate and both tables bit for bit. Orders that change a state go through
pfnav_agents_commands on both twins: only the inputs beyond point seeking take different paths.

Groups of 2 and 3 members (3: unequal ranges) against one context given the same calls: each member's tables for its
range and, through 8 ticks with the gather, every output bit for bit. The NCCL form is checked by
tests/tools/mgpu_nccl_input_deltas_check.py under torchrun."""
import numpy as np
import pytest

import cases
import commands_ref as cr
import inputs_ref as ir

capi, synth = cases.capi, cases.synth
ST_MOVING, ST_FORMATION, ST_ARRIVED, ST_SEEK, ST_WAITING, ST_SURROUND, ST_ENTER, ST_TURNING, ST_CELL = range(9)
FORM_IN = capi.FORM_HAS_FORMATION | capi.FORM_ASSIGNMENT_READY | capi.FORM_ASSIGNED_TO_CELL


def _population(seed=4242, hz=20, shuffle=False):
    """cases.update_case with desired velocities and the tables beyond point seeking: ext defaults with rot = the
    facing, some units already using a surround field; formation records all outside any formation"""
    p, cost, a, ms = cases.update_case(seed, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(seed + 3)
    a["vdes"] = rng.normal(size=(n, 2)).astype(np.float32)
    a["vdes"] /= np.linalg.norm(a["vdes"], axis=1, keepdims=True)
    rec, fl = capi.pack_agents(a)
    if shuffle:                                        # every flock on every rank
        perm = rng.permutation(n)
        rec, ms = rec[perm].copy(), ms[perm].copy()
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID
    ext["rot"] = ms["next_rot"]; ext["target_dir"] = ms["next_rot"]
    ext["target_range"] = 8.0
    ext["using_surround_field"] = rng.random(n) < 0.3
    form = np.zeros(n, capi.FORMATION_IN)
    return cost, rec, fl, ms, ext, form


def _form_records(rng, pos, flags=FORM_IN):
    k = len(pos)
    f = np.zeros(k, capi.FORMATION_IN)
    f["cell_pos"] = pos + rng.normal(scale=6.0, size=(k, 2)).astype(np.float32)
    v = rng.normal(size=(k, 2)); v /= np.linalg.norm(v, axis=1, keepdims=True)
    f["cell_arrival_vdes"] = v
    f["cohesion"] = rng.normal(scale=0.4, size=(k, 2)); f["align"] = rng.normal(scale=0.3, size=(k, 2))
    f["drag"] = rng.normal(scale=0.2, size=(k, 2))
    f["target_orientation"] = cases.dir_quat(rng.normal(size=(k, 2)))
    f["flags"] = flags
    f["flags"][::3] |= capi.FORM_IN_RANGE_OF_CELL
    return f


def _setup(X, cw, cost, hz):
    X.map_create(cw, cw, 1); X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)


class Twin:
    def __init__(self, cost, rec, fl, ms, ext, form, hz=20, cw=3):
        self.n = len(rec)
        self.has_ext, self.has_form = ext is not None, form is not None
        self.A, self.B = capi.Nav(0), capi.Nav(0)
        for X in (self.A, self.B):
            _setup(X, cw, cost, hz)
            X.agents_upload(rec, fl, hz)
            X.agents_upload_movestate(ms)
            if ext is not None:
                X.agents_upload_movestate_ext(ext)
            if form is not None:
                X.agents_upload_formation(form)
        self.work_lists()

    def close(self):
        self.A.close(); self.B.close()

    def tables(self, X):
        return (X.agents_read_movestate_ext(self.n) if self.has_ext else None,
                X.agents_read_formation(self.n) if self.has_form else None)

    def three_step(self, d):
        """B: read both tables back, apply the records in numpy, upload both whole"""
        ext, form = self.tables(self.B)
        any_form = bool((d["mask"] & capi.INPUT_FORMATION).any())
        if form is None and any_form:
            form = np.zeros(self.n, capi.FORMATION_IN)         # what the call creates
        ext, form = ir.apply_np(ext, form, d)
        if ext is not None:
            self.B.agents_upload_movestate_ext(ext)
        if form is not None:
            self.B.agents_upload_formation(form)

    def inputs(self, d, X=None):
        """the batch on one twin (X) or both, then the tables compared"""
        if X is None or X is self.A:
            self.A.agents_input_deltas(d)
        if X is None or X is self.B:
            self.three_step(d)
        self.has_form |= bool((d["mask"] & capi.INPUT_FORMATION).any())
        if X is None:
            self.compare_tables()

    def commands(self, d):
        for X in (self.A, self.B):
            X.agents_commands(d)
            X.agents_rebuild_index()

    def compare_tables(self):
        ta, tb = self.tables(self.A), self.tables(self.B)
        for name, x, y in zip(("movestate_ext", "formation"), ta, tb):
            assert (x is None) == (y is None), name
            if x is not None:
                assert x.tobytes() == y.tobytes(), (name, np.nonzero(x != y)[0][:10])
        return ta

    def work_lists(self):
        na = self.A.agents_set_work_dev()
        nb = self.B.agents_set_work_dev()
        wa, wb = self.A.agents_read_work(), self.B.agents_read_work()
        assert na == nb and np.array_equal(wa, wb)
        return wa

    def compare(self):
        sa, ma = self.A.agents_read_state(self.n)
        sb, mb = self.B.agents_read_state(self.n)
        assert sa.tobytes() == sb.tobytes(), np.nonzero(sa != sb)[0][:10]
        assert ma.tobytes() == mb.tobytes(), np.nonzero(ma != mb)[0][:10]
        self.compare_tables()
        return sa

    def tick(self, before_apply=None):
        """one resident tick on both twins, compared at every output; before_apply(X) runs between the update pass (and
        the event collection) and the apply"""
        nw = len(self.A.agents_read_work())
        out = []
        for X in (self.A, self.B):
            if nw:
                X.agents_tick(0)
                X.agents_compute_updates()
                out.append((X.agents_read_velocities(nw),) + X.agents_read_debug(nw) + (X.agents_read_patches(nw),))
                X.agents_collect_events()
            if before_apply is not None:
                before_apply(X)
            if nw:
                X.agents_apply_updates()
            X.agents_rebuild_index()
        for name, x, y in zip(("velocities", "vpref", "vdes", "los", "patches"), *out):
            assert x.tobytes() == y.tobytes(), (name, np.nonzero(x != y)[0][:10])
        self.work_lists()
        return self.compare()

    def ticks(self, k=8):
        for _ in range(k):
            s = self.tick()
        return s


def _twin(seed=4242, ext=True, form=True, **kw):
    cost, rec, fl, ms, e, f = _population(seed)
    return Twin(cost, rec, fl, ms, e if ext else None, f if form else None, **kw)


def _movers(s, k, rng, flock=None):
    m = (s["state"] == ST_MOVING) & ((s["flags"] & capi.FLAG_GARRISONED) == 0)
    if flock is not None:
        m &= s["flock"] == flock
    who = np.nonzero(m)[0]
    return np.sort(rng.choice(who, min(k, len(who)), replace=False))


@pytest.mark.gpu
def test_symbols_and_record(pf):
    assert capi.INPUT_DELTA.itemsize == 128
    for s in ("pfnav_agents_input_deltas", "pfnav_mgpu_input_deltas", "pfnav_group_input_deltas", "pfnav_agents_read_formation"):
        assert s in capi.SYMBOLS


@pytest.mark.gpu
def test_turning_order_at_and_off_its_direction(pf):
    """a turn-to-face order: STATE = TURNING through the commands, TARGET_DIR through the new call -- for half of the
    units the direction they already face (they arrive), for the others a new one"""
    T = _twin(seed=4242)
    rng = np.random.default_rng(1)
    try:
        s = T.tick()
        who = _movers(s, 120, rng)
        at, off = who[::2], who[1::2]
        ext = T.A.agents_read_movestate_ext(T.n)
        T.commands(cr.deltas(who, state=ST_TURNING, velocity=(0.0, 0.0)))
        T.inputs(np.concatenate([ir.inputs(at, target_dir=ext["rot"][at]),
                                 ir.inputs(off, target_dir=cases.dir_quat(rng.normal(size=(len(off), 2))))]))
        s = T.tick()
        assert (s["state"][at] == ST_ARRIVED).mean() >= (s["state"][off] == ST_ARRIVED).mean()
        T.ticks(7)
    finally:
        T.close()


@pytest.mark.gpu
def test_rot_write_moves_the_heading_gate(pf):
    """Entity_SetRot: MOVING units made to face along their velocity or against it (the heading gate of the MOVING
    update reads rot)"""
    T = _twin(seed=77)
    rng = np.random.default_rng(2)
    try:
        s = T.tick()
        who = _movers(s, 200, rng)
        v = s["velocity"][who]
        face = np.where((np.arange(len(who)) % 2 == 0)[:, None], v, -v)
        T.inputs(ir.inputs(who, rot=cases.dir_quat(face)))
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_surround_order_resets_prev_pos_and_field(pf):
    """a new surround order: the target through PFNAV_DELTA_TARGET, target_prev_pos = where the target stands and
    using_surround_field = 0 through the new call (some of the units were using a field for an earlier target)"""
    T = _twin(seed=5)
    rng = np.random.default_rng(3)
    try:
        s = T.tick()
        who = _movers(s, 60, rng)
        tgt = int(np.setdiff1d(_movers(s, 200, rng), who)[0])
        assert T.compare_tables()[0]["using_surround_field"][who].any()
        T.commands(cr.deltas(who, state=ST_SURROUND, target=(tgt, 0.0)))
        T.inputs(ir.inputs(who, target_prev=s["pos"][tgt], surround_field=0))
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_formation_join_and_leave(pf):
    """a flock enters a formation (ARRIVING_TO_CELL and MOVING_IN_FORMATION with their formation records), moves in
    it with new records every tick, then leaves it (records zeroed, MOVING again)"""
    T = _twin(seed=99)
    rng = np.random.default_rng(4)
    try:
        s = T.tick()
        who = _movers(s, 150, rng, flock=0)
        cell, inform = who[::2], who[1::2]
        T.commands(np.concatenate([cr.deltas(cell, state=ST_CELL), cr.deltas(inform, state=ST_FORMATION)]))
        T.inputs(ir.inputs(who, formation=_form_records(rng, s["pos"][who])))
        for _ in range(4):
            s = T.tick()
            moving = who[np.isin(s["state"][who], (ST_CELL, ST_FORMATION))]
            T.inputs(ir.inputs(moving, formation=_form_records(rng, s["pos"][moving])))
        T.ticks(4)
        T.commands(cr.deltas(who, state=ST_MOVING, clear_hist=True))
        T.inputs(ir.inputs(who, formation=np.zeros(1, capi.FORMATION_IN)))
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_formation_table_created_by_the_call(pf):
    """no formation table: a FORMATION batch creates one as an upload of zeroed records would (B uploads the zeroed
    table with the records applied), for units in ARRIVING_TO_CELL and for units whose state reads no record"""
    T = _twin(seed=31, form=False)
    rng = np.random.default_rng(5)
    try:
        s = T.tick()
        who = _movers(s, 100, rng)
        T.commands(cr.deltas(who[:50], state=ST_CELL))
        T.inputs(ir.inputs(who, formation=_form_records(rng, s["pos"][who])))
        f = T.A.agents_read_formation(T.n)
        rest = np.setdiff1d(np.arange(T.n), who)
        assert not f[rest].tobytes().strip(b"\0") and (f["flags"][who] & capi.FORM_HAS_FORMATION).all()
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_several_records_per_uid_compose(pf):
    """random batches of every mask over few uids: the folded write equals the records in order"""
    T = _twin(seed=11)
    rng = np.random.default_rng(6)
    try:
        s = T.tick()
        for _ in range(3):
            T.inputs(ir.random_inputs(rng, 900, _movers(s, 150, rng)))
            s = T.ticks(3)
    finally:
        T.close()


@pytest.mark.gpu
def test_batches_between_collect_and_apply_and_after_commands(pf):
    """a batch issued after the update pass and the event collection, before the apply, on both twins; and a batch
    issued right after a command batch of the same tick"""
    T = _twin(seed=21)
    rng = np.random.default_rng(7)
    try:
        s = T.tick()
        who = _movers(s, 100, rng)
        d = ir.random_inputs(rng, 300, who)
        T.tick(before_apply=lambda X: T.inputs(d, X))
        T.compare()
        s = T.tick()
        turn = _movers(s, 80, rng)
        T.commands(cr.deltas(turn, state=ST_TURNING))
        T.inputs(np.concatenate([ir.inputs(turn, target_dir=cases.dir_quat(rng.normal(size=(len(turn), 2)))),
                                 ir.random_inputs(rng, 200, turn)]))
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_refusals_change_nothing(pf):
    T = _twin(seed=8)
    rng = np.random.default_rng(8)
    n = T.n
    try:
        T.tick()
        good = ir.random_inputs(rng, 50, np.arange(n))
        one = lambda **kw: ir.inputs([3], **kw)
        unknown = one(rot=(0, 0, 0, 1)); unknown["mask"] |= 1 << 5
        badflags = one(formation=np.zeros(1, capi.FORMATION_IN)); badflags["formation"]["flags"] = 1 << 5
        nanform = one(formation=np.zeros(1, capi.FORMATION_IN)); nanform["formation"]["drag"] = (0.0, np.nan)
        bad = [ir.inputs([n], rot=(0, 0, 0, 1)), unknown, badflags, nanform, one(surround_field=2),
               one(target_prev=(np.inf, 0)), one(target_dir=(0, np.nan, 0, 1)), one(rot=(0, 0, -np.inf, 1))]
        before = T.compare()
        tables = T.tables(T.A)
        for b in bad:
            with pytest.raises(capi.PfnavError, match="error -1"):
                T.A.agents_input_deltas(np.concatenate([good, b]))
        T.A.agents_input_deltas(np.zeros(0, capi.INPUT_DELTA))
        for x, y in zip(tables, T.tables(T.A)):
            assert x.tobytes() == y.tobytes()
        assert T.compare().tobytes() == before.tobytes()
        T.ticks(2)
        grp = capi.Group([T.A])                              # a member of a multi-GPU job refuses
        try:
            with pytest.raises(capi.PfnavError, match="error -4"):
                T.A.agents_input_deltas(good)
        finally:
            grp.close()
        T.compare()
    finally:
        T.close()
    # the movestate_ext bits without an ext table; FORMATION creates its table on a context without one
    cost, rec, fl, ms, ext, form = _population(8)
    X = capi.Nav(0)
    host = capi.Nav(0, hostonly=True)
    try:
        _setup(X, 3, cost, 20)
        X.agents_upload(rec, fl, 20)
        for bit in ("target_prev", "target_dir", "rot", "surround_field"):
            v = {"target_prev": (1.0, 1.0), "target_dir": (0, 0, 0, 1), "rot": (0, 0, 0, 1), "surround_field": 1}[bit]
            with pytest.raises(capi.PfnavError, match="error -1"):
                X.agents_input_deltas(ir.inputs([0], **{bit: v}))
        with pytest.raises(capi.PfnavError, match="error -1"):
            X.agents_read_formation(1)
        X.agents_input_deltas(ir.inputs([4], formation=_form_records(rng, rec["pos"][4:5])))
        f = X.agents_read_formation(len(rec))
        assert f[4]["flags"] & capi.FORM_HAS_FORMATION and not np.delete(f, 4).tobytes().strip(b"\0")
        with pytest.raises(capi.PfnavError, match="error -3"):
            host.agents_input_deltas(ir.inputs([0], rot=(0, 0, 0, 1)))
    finally:
        X.close(); host.close()


@pytest.mark.gpu
def test_c2_scale(pf):
    """the benchmark's C2 population (100 000 agents): 10 000 records of every mask, then 8 ticks"""
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
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID; ext["rot"] = ms["next_rot"]; ext["target_dir"] = ms["next_rot"]
    T = Twin(W["cost"], rec, fl, ms, ext, np.zeros(n, capi.FORMATION_IN), cw=bench.CHUNKS)
    rng = np.random.default_rng(9)
    try:
        T.inputs(ir.random_inputs(rng, 10_000, rng.choice(n, 7_000, replace=False)))
        T.ticks(8)
    finally:
        T.close()


# ---- job forms: an in-process group against one context ----
def _devices(world):
    import torch
    k = torch.cuda.device_count()
    return [i % k for i in range(world)]


class Job:
    """one: a single context taking agents_input_deltas; navs: `world` sharded members of a group taking
    Group.input_deltas. ext_on / form_on: which members (and the single context, last entry) hold each table."""

    def __init__(self, world, seed=4242, hz=20, ext_on=None, form_on=None, cw=3):
        cost, rec, fl, ms, ext, form = _population(seed, hz, shuffle=True)
        self.n, self.world = len(rec), world
        self.ranges = [capi.mgpu_shard_range(self.n, r, world) for r in range(world)]
        self.one = capi.Nav(0)
        self.navs = [capi.Nav(d) for d in _devices(world)]
        self.grp = None
        for X in self.all():
            _setup(X, cw, cost, hz)
        self.grp = capi.Group(self.navs)
        self.one.agents_upload(rec, fl, hz)
        for nv, (lo, hi) in zip(self.navs, self.ranges):
            nv.agents_upload_shard(rec[lo:hi], lo, hi, self.n, fl, hz)
        self.grp.gather()
        ext_on = ext_on or [True] * (world + 1)
        form_on = form_on or [True] * (world + 1)
        for X, (lo, hi), e, f in zip(self.navs + [self.one], self.ranges + [(0, self.n)], ext_on, form_on):
            X.agents_upload_movestate(ms[lo:hi])
            if e:
                X.agents_upload_movestate_ext(ext[lo:hi])
            if f:
                X.agents_upload_formation(form[lo:hi])
        self.has_ext, self.has_form = ext_on[-1], form_on[-1]
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
        uids = np.asarray(uids)
        return uids[(uids >= lo) & (uids < hi)]

    def inputs(self, d):
        self.one.agents_input_deltas(d)
        self.grp.input_deltas(d)
        self.has_form |= bool((d["mask"] & capi.INPUT_FORMATION).any())
        return self.compare()

    def commands(self, d):
        self.one.agents_commands(d)
        self.one.agents_rebuild_index()
        self.grp.commands(d)
        self.grp.gather()
        self.work_lists()

    def member_tables(self):
        parts = []
        for nv, (lo, hi) in zip(self.navs, self.ranges):
            parts.append((nv.agents_read_movestate_ext(hi - lo) if self.has_ext else None,
                          nv.agents_read_formation(hi - lo) if self.has_form else None))
        return parts

    def compare(self):
        a1, m1 = self.one.agents_read_state(self.n)
        parts = [nv.agents_read_state(hi - lo) for nv, (lo, hi) in zip(self.navs, self.ranges)]
        assert np.concatenate([p[0] for p in parts]).tobytes() == a1.tobytes()
        assert np.concatenate([p[1] for p in parts]).tobytes() == m1.tobytes()
        tabs = self.member_tables()
        if self.has_ext:
            assert np.concatenate([t[0] for t in tabs]).tobytes() == self.one.agents_read_movestate_ext(self.n).tobytes()
        if self.has_form:
            assert np.concatenate([t[1] for t in tabs]).tobytes() == self.one.agents_read_formation(self.n).tobytes()
        return a1

    def work_lists(self):
        self.one.agents_set_work_dev()
        w1 = self.one.agents_read_work()
        for r, nv in enumerate(self.navs):
            nv.agents_set_work_dev()
            assert np.array_equal(nv.agents_read_work(), self.own(r, w1)), ("work list", r)
        return w1

    @staticmethod
    def _tick_one(X, nw):
        X.agents_tick(0)
        X.agents_compute_updates()
        out = (X.agents_read_velocities(nw),) + X.agents_read_debug(nw) + (X.agents_read_patches(nw),)
        X.agents_apply_updates()
        return out

    def tick(self):
        nw1 = len(self.one.agents_read_work())
        ref = self._tick_one(self.one, nw1) if nw1 else None
        self.one.agents_rebuild_index()
        outs = []
        for nv in self.navs:
            nw = len(nv.agents_read_work())
            if nw:
                outs.append(self._tick_one(nv, nw))
        self.grp.gather()
        if ref is not None:
            for k, name in enumerate(("velocities", "vpref", "vdes", "los", "patches")):
                assert np.concatenate([o[k] for o in outs]).tobytes() == ref[k].tobytes(), name
        self.work_lists()
        return self.compare()

    def ticks(self, k=8):
        for _ in range(k):
            s = self.tick()
        return s


WORLDS = pytest.mark.parametrize("world", [2, 3])


@pytest.mark.gpu
@WORLDS
def test_job_orders_beyond_point_seeking(pf, world):
    """turn orders, rot writes, a surround order and a formation joined, from every rank, several records per uid"""
    J = Job(world)
    rng = np.random.default_rng(10)
    try:
        s = J.tick()
        who = _movers(s, 240, rng)
        turn, rot, sur, form = who[0::4], who[1::4], who[2::4], who[3::4]
        assert all(len(J.own(r, turn)) and len(J.own(r, form)) for r in range(world))
        tgt = int(rot[0])
        J.commands(np.concatenate([cr.deltas(turn, state=ST_TURNING), cr.deltas(sur, state=ST_SURROUND, target=(tgt, 0.0)),
                                   cr.deltas(form[::2], state=ST_CELL), cr.deltas(form[1::2], state=ST_FORMATION)]))
        d = np.concatenate([ir.inputs(turn, target_dir=cases.dir_quat(rng.normal(size=(len(turn), 2)))),
                            ir.inputs(rot, rot=cases.dir_quat(-s["velocity"][rot])),
                            ir.inputs(sur, target_prev=s["pos"][tgt], surround_field=0),
                            ir.inputs(form, formation=_form_records(rng, s["pos"][form])),
                            ir.random_inputs(rng, 300, who)])
        J.inputs(d)
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_job_creates_the_formation_table_on_every_member(pf, world):
    """no member holds a formation table; a batch whose FORMATION records all name uids of the first rank creates the
    table on every member"""
    J = Job(world, seed=77, form_on=[False] * (world + 1))
    rng = np.random.default_rng(11)
    try:
        s = J.tick()
        lo, hi = J.ranges[0]
        who = _movers(s, 200, rng)
        who = who[(who >= lo) & (who < hi)][:60]
        J.commands(cr.deltas(who, state=ST_CELL))
        J.inputs(ir.inputs(who, formation=_form_records(rng, s["pos"][who])))
        for r, nv in enumerate(J.navs):
            f = nv.agents_read_formation(J.ranges[r][1] - J.ranges[r][0])
            assert r == 0 or not f.tobytes().strip(b"\0")
        J.ticks(8)
    finally:
        J.close()


@pytest.mark.gpu
@WORLDS
def test_job_refusals_change_nothing_anywhere(pf, world):
    """the last member has no movestate_ext table: an ext batch is refused by that member and fails on every member;
    a FORMATION-only batch meets members whose sets of tables differ (PFNAV_ERR_ARG); a bad record for any uid fails
    everywhere. Nothing changes on any member, and after the last member uploads its table the job goes on equal to
    the single context"""
    cost, rec, fl, ms, ext, form = _population(21, shuffle=True)
    J = Job(world, seed=21, ext_on=[True] * (world - 1) + [False, True])
    rng = np.random.default_rng(12)
    try:
        J.has_ext = False                                   # compared per member below
        s = J.compare()
        before = [(nv.agents_read_movestate_ext(hi - lo) if r < world - 1 else None, nv.agents_read_formation(hi - lo))
                  for r, (nv, (lo, hi)) in enumerate(zip(J.navs, J.ranges))]
        lo, hi = J.ranges[-1]
        with pytest.raises(capi.PfnavError, match="error -1.*member %d" % (world - 1)):
            J.grp.input_deltas(ir.inputs(np.arange(0, J.n, 97), rot=(0, 0, 0, 1)))
        with pytest.raises(capi.PfnavError, match="error -1"):
            J.grp.input_deltas(ir.inputs([lo, hi - 1], formation=np.zeros(1, capi.FORMATION_IN)))
        bad = ir.inputs([J.n - 1], formation=np.zeros(1, capi.FORMATION_IN)); bad["formation"]["flags"] = 64
        with pytest.raises(capi.PfnavError, match="error -1"):
            J.grp.input_deltas(np.concatenate([ir.inputs([0], formation=np.zeros(1, capi.FORMATION_IN)), bad]))
        for r, (nv, (lo_, hi_)) in enumerate(zip(J.navs, J.ranges)):
            e, f = before[r]
            if e is not None:
                assert nv.agents_read_movestate_ext(hi_ - lo_).tobytes() == e.tobytes()
            assert nv.agents_read_formation(hi_ - lo_).tobytes() == f.tobytes()
        J.compare()
        J.navs[-1].agents_upload_movestate_ext(ext[lo:hi])
        J.has_ext = True
        J.compare()
        who = _movers(s, 120, rng)
        J.inputs(ir.random_inputs(rng, 400, who))
        J.ticks(8)
        # state errors: the NCCL form on a group member, a context in no job
        with pytest.raises(capi.PfnavError, match="error -4"):
            J.navs[0].mgpu_input_deltas(ir.inputs([0], rot=(0, 0, 0, 1)))
        lone = capi.Nav(0)
        try:
            with pytest.raises(capi.PfnavError, match="error -4"):
                lone.mgpu_input_deltas(ir.inputs([0], rot=(0, 0, 0, 1)))
        finally:
            lone.close()
    finally:
        J.close()
