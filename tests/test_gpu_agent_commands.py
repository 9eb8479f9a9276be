"""pfnav_agents_commands + pfnav_agents_set_work_dev against the path they replace.

Twin contexts on the same map, pool and population: A takes the command batch as deltas and builds its work list on the
device; B takes the long way round: agents_read_state, the same edits in numpy (commands_ref.apply_deltas_np),
agents_upload + agents_upload_movestate (+ _ext), agents_set_work(None). After the batch: entity state byte for byte and
the work lists; after each following resident tick (tick, compute_updates, apply_updates, rebuild_index, work list):
velocities, preferred / desired velocities, LOS bits, patches and state, bit for bit -- cohesion included, which is what
pins the device-built member lists to the host's.

The movestate_ext table cannot be read back, so B re-uploads its own copy of it: the initial table plus the batch's
TARGET writes. That copy is only right while no tick has run, so populations with an ext table take their command
batches before the first tick (Twin.commands refuses otherwise)."""
import numpy as np
import pytest

import cases
import commands_ref as cr

capi, synth = cases.capi, cases.synth
ST_MOVING, ST_ARRIVED, ST_SEEK, ST_WAITING, ST_SURROUND = 0, 2, 3, 4, 5
GARR, HELD = capi.FLAG_GARRISONED, capi.FLAG_COMBAT_HELD


class Twin:
    def __init__(self, cw, cost, rec, fl, ms, hz, nlayers=1, ext=None, ndests=None, blocking=False):
        self.cw, self.hz, self.n, self.nlayers = cw, hz, len(rec), nlayers
        self.fl = np.ascontiguousarray(fl, capi.FLOCK).copy()
        self.ndests = ndests or len(fl)
        self.ext = None if ext is None else ext.copy()
        self.blocking, self.ticked = blocking, False
        self.A, self.B = capi.Nav(0), capi.Nav(0)
        for X in (self.A, self.B):
            X.map_create(cw, cw, nlayers)
            for l in range(nlayers):
                X.map_upload_layer(l, cost); X.map_build_nav(l); X.route_build(l)
            X.pool_create(self.ndests, self.ndests * cw * cw)
            X.agents_upload(rec, self.fl, hz)
            X.agents_upload_movestate(ms)
            if ext is not None:
                X.agents_upload_movestate_ext(ext)
            if blocking:
                tbl = np.zeros(self.n, capi.BLOCKING); tbl["faction_id"] = capi.FACTION_ID_NONE
                X.agents_upload_blocking(tbl)
        self.A.agents_set_work_dev()
        self.B.agents_set_work(None)

    def close(self):
        self.A.close(); self.B.close()

    def commands(self, d, flocks=None, block=None):
        """block: (uids to unblock, uids to block) through agents_set_blocking + map_commit on both twins"""
        assert self.ext is None or not self.ticked
        self.A.agents_commands(d, flocks)
        sa, ms = self.B.agents_read_state(self.n)
        cr.apply_deltas_np(d, sa, ms, self.ext)
        if flocks is not None:
            self.fl = np.ascontiguousarray(flocks, capi.FLOCK).copy()
        self.B.agents_upload(sa, self.fl, self.hz)
        self.B.agents_upload_movestate(ms)
        if self.ext is not None:
            self.B.agents_upload_movestate_ext(self.ext)
        for X in (self.A, self.B):
            if block is not None:
                X.agents_set_blocking(block[0], False); X.agents_set_blocking(block[1], True)
                X.map_commit()
        self.A.agents_rebuild_index()
        self.work_lists()
        self.compare()

    def work_lists(self):
        na = self.A.agents_set_work_dev()
        self.B.agents_set_work(None)
        wa, wb = self.A.agents_read_work(), self.B.agents_read_work()
        assert na == len(wa) and np.array_equal(wa, wb), (na, len(wb))
        return wa

    def compare(self):
        sa, ma = self.A.agents_read_state(self.n)
        sb, mb = self.B.agents_read_state(self.n)
        assert sa.tobytes() == sb.tobytes(), np.nonzero(sa != sb)[0][:10]
        assert ma.tobytes() == mb.tobytes(), np.nonzero(ma != mb)[0][:10]
        if self.blocking:
            assert self.A.agents_read_blocking(self.n).tobytes() == self.B.agents_read_blocking(self.n).tobytes()
            assert (self.A.blockers(0) == self.B.blockers(0)).all()
        return sa

    def tick(self, passes=2):
        """one resident tick on both twins, compared at every output"""
        self.ticked = True
        nw = len(self.A.agents_read_work())
        out = []
        for X in (self.A, self.B):
            for _ in range(passes):          # serve the pool misses of the new orders; the same calls on both twins
                X.agents_tick(capi.TICK_VDES_FROM_POOL)
                X.pool_repair()
            X.agents_tick(capi.TICK_VDES_FROM_POOL)
            X.agents_compute_updates()
            out.append((X.agents_read_velocities(nw),) + X.agents_read_debug(nw) + (X.agents_read_patches(nw),)
                       if nw else ())
            if self.blocking:
                X.agents_apply_updates_ex(capi.APPLY_BLOCKERS); X.map_commit()
            elif nw:
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


def _case(seed=4242, hz=20, extra_flocks=1, ext=False, **kw):
    p, cost, a, ms = cases.update_case(seed, hz)
    nf = len(a["flock_target"])
    aa = dict(a); aa["flock_dest_index"] = np.arange(nf, dtype=np.int32)
    rec, fl = capi.pack_agents(aa)
    e = None
    if ext:
        e = np.zeros(len(rec), capi.MOVESTATE_EXT); e["surround_target_uid"] = capi.NULL_UID
    return Twin(3, cost, rec, fl, ms, hz, ext=e, ndests=nf + extra_flocks + 2, **kw), rec, fl


def _grown(fl, target, dest):
    out = np.zeros(len(fl) + 1, capi.FLOCK)
    out[:-1] = fl
    out["target"][-1], out["dest"][-1], out["layer"][-1] = target, dest, 0
    return out


@pytest.mark.gpu
def test_delta_record_size(pf):
    assert capi.AGENT_DELTA.itemsize == 64
    assert "pfnav_agents_commands" in capi.SYMBOLS and "pfnav_agents_set_work_dev" in capi.SYMBOLS


@pytest.mark.gpu
@pytest.mark.parametrize("hz", [20, 5])
def test_arrived_units_ordered_to_a_new_flock(pf, hz):
    """ARRIVED units and part of a moving flock get a move order to a flock appended to the table; the order of one unit
    arrives as several deltas (a superseded flock, state and flock apart)"""
    T, rec, fl = _case(hz=hz)
    try:
        T.ticks(2)
        s = T.compare()
        who = np.concatenate([np.nonzero(s["state"] == ST_ARRIVED)[0][:60], np.nonzero((s["state"] == ST_MOVING) & (s["flock"] == 1))[0][:90]])
        new = _grown(T.fl, s["pos"][who].mean(axis=0) + 30.0, len(fl))
        d = np.concatenate([cr.deltas(who[:10], flock=0), cr.deltas(who, state=ST_MOVING, clear_hist=True), cr.deltas(who, flock=len(fl))])
        T.commands(d, new)
        assert len(T.A.agents_read_work()) >= len(who)
        s = T.ticks(8)
        assert (s["flock"][who] == len(fl)).all()
    finally:
        T.close()


@pytest.mark.gpu
def test_flock_emptied_stop_and_teleport(pf):
    """every member of flock 2 moves to flock 1 (flock 2 stays in the table, empty); a stop order (ARRIVED + zero
    velocity) and a teleport of other units in later batches"""
    T, rec, fl = _case(seed=77)
    try:
        T.tick()
        s = T.compare()
        T.commands(cr.deltas(np.nonzero(s["flock"] == 2)[0], flock=1))
        s = T.ticks(3)
        assert not (s["flock"] == 2).any()
        moving = np.nonzero(s["state"] == ST_MOVING)[0]
        T.commands(cr.deltas(moving[::7], state=ST_ARRIVED, velocity=(0.0, 0.0)))
        s = T.ticks(2)
        moving = np.nonzero(s["state"] == ST_MOVING)[0][::11]
        donors = np.nonzero(s["state"] == ST_ARRIVED)[0][:len(moving)]
        moving = moving[:len(donors)]
        T.commands(cr.deltas(moving, position=s["pos"][donors] + np.float32(0.75)))
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_flock_emptied_and_dropped_in_one_batch(pf):
    """one batch moves every member of the last flock to flock 0 and passes the table without it; a later batch appends
    a flock again"""
    T, rec, fl = _case(seed=31)
    try:
        T.tick()
        s = T.compare()
        last = len(fl) - 1
        T.commands(cr.deltas(np.nonzero(s["flock"] == last)[0], flock=0), T.fl[:last].copy())
        s = T.ticks(4)
        assert s["flock"].max() == last - 1
        who = np.nonzero(s["state"] == ST_MOVING)[0][::6]
        T.commands(cr.deltas(who, flock=last), _grown(T.fl, s["pos"][who].mean(axis=0), last))
        T.ticks(4)
    finally:
        T.close()


@pytest.mark.gpu
def test_radius_across_a_layer_boundary_and_garrison_flips(pf):
    """units grow from radius < 5 to 6 (navigation layer 0 -> 1: arrival constants of a new (flock, layer) pair, a larger
    adjacency query radius); then every GARRISONED unit leaves its garrison (the population has none left: the
    neighbour query stops filtering) and others enter one"""
    T, rec, fl = _case(seed=99, nlayers=2)
    try:
        T.tick()
        s = T.compare()
        grow = np.nonzero(s["state"] == ST_MOVING)[0][::9]
        T.commands(cr.deltas(grow, radius=6.0))
        s = T.ticks(2)
        g = np.nonzero(s["flags"] & GARR)[0]
        assert len(g)
        T.commands(cr.deltas(g, flags=s["flags"][g] & ~np.uint32(GARR)))
        s = T.ticks(3)
        g = np.nonzero(s["state"] == ST_MOVING)[0][5::13]
        T.commands(cr.deltas(g, flags=s["flags"][g] | np.uint32(GARR)))
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_seek_and_surround_targets(pf):
    """seek-enemies and surround orders: aux_dest1 names TARGET_ENEMIES / TARGET_ENTITY pool destinations, the surround
    target goes into the movestate_ext table; batches precede the first tick (see the module text)"""
    T, rec, fl = _case(seed=5, ext=True)
    try:
        nf = len(fl)
        allchunks = [(c // 3, c % 3) for c in range(9)]
        foes = np.arange(0, 40, 8)
        for X in (T.A, T.B):
            fp = X.footprints(rec["pos"], rec["radius"])
            X.pool_request_entity_fields(nf + 1, capi.TARGET_ENEMIES, fp[foes], allchunks)
            X.pool_request_entity_fields(nf + 2, capi.TARGET_ENTITY, fp[3:4], allchunks)
        mv = np.nonzero(rec["state"] == ST_MOVING)[0]
        seek, sur = mv[100:160], mv[200:240]
        d = np.concatenate([cr.deltas(seek, state=ST_SEEK, flock=-1, aux_dest1=nf + 2),
                            cr.deltas(sur, state=ST_SURROUND, aux_dest1=nf + 3, target=(3, 0.0)),
                            cr.deltas(sur[:5], target=(capi.NULL_UID, 2.5))])
        T.commands(d)
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_table_only_and_empty_batches(pf):
    """no delta and a flock table whose targets moved: the arrival constants follow; no delta and no table: nothing"""
    T, rec, fl = _case(seed=11)
    try:
        T.tick()
        before = T.compare()
        T.A.agents_commands(np.zeros(0, capi.AGENT_DELTA), None)
        assert T.compare().tobytes() == before.tobytes()
        moved = T.fl.copy()
        moved["target"][0] += np.float32(40.0)
        T.commands(np.zeros(0, capi.AGENT_DELTA), moved)
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_refused_batches_change_nothing(pf):
    T, rec, fl = _case(seed=21, nlayers=1)
    n, nf = len(rec), len(fl)
    good = cr.deltas(np.arange(20), state=ST_ARRIVED, flock=1, radius=2.0)
    bad = [cr.deltas([n], state=0), cr.deltas([0], state=9), cr.deltas([0], flock=nf), cr.deltas([0], flock=-2),
           cr.deltas([0], radius=6.0),                      # layer 1 does not exist
           cr.deltas([0], flags=capi.FLAG_AIR),             # nor the air layers
           cr.deltas([0], radius=np.nan), cr.deltas([0], velocity=(np.inf, 0)), cr.deltas([0], position=(0, np.nan)),
           cr.deltas([0], speeds=(np.nan, 1.0)), cr.deltas([0], target=(1, 1.0))]     # no ext table
    unknown = cr.deltas([0], state=0); unknown["mask"] |= 1 << 10
    bad.append(unknown)
    try:
        T.tick()
        before = T.compare()
        for b in bad:
            with pytest.raises(capi.PfnavError, match="error -1"):
                T.A.agents_commands(np.concatenate([good, b]))
        with pytest.raises(capi.PfnavError, match="error -1"):      # flock 2 keeps members: the table cannot drop it
            T.A.agents_commands(good, T.fl[:2])
        assert T.compare().tobytes() == before.tobytes()
        T.work_lists()
        before2 = T.ticks(2)
        # a member of a multi-GPU job refuses, changing nothing
        grp = capi.Group([T.A])
        try:
            with pytest.raises(capi.PfnavError, match="error -4"):
                T.A.agents_commands(good)
        finally:
            grp.close()
        assert T.compare().tobytes() == before2.tobytes()
    finally:
        T.close()


@pytest.mark.gpu
def test_host_only_context_has_no_command_path(pf):
    nav = capi.Nav(0, hostonly=True)
    try:
        with pytest.raises(capi.PfnavError, match="error -3"):
            nav.agents_commands(cr.deltas([0], state=0))
        with pytest.raises(capi.PfnavError, match="error -3"):
            nav.agents_set_work_dev()
    finally:
        nav.close()


@pytest.mark.gpu
@pytest.mark.parametrize("still,n", [("none", 70_001), ("some", 70_001), ("all", 70_001), ("some", 1_300_003)])
def test_set_work_dev_equals_set_work(pf, still, n):
    """70 001: several blocks of the compaction, a ragged tail; 1 300 003: more than 1024 x 1024 entities, so every block
    of the compaction takes more than one pass over its range"""
    rng = np.random.default_rng(1)
    cw = 4 if n < 100_000 else 16                # room for a 3.5-unit grid: the position index sorts every cell's entries
    side = int(np.ceil(np.sqrt(n)))
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, 0x5EED0000), cw, cw)
    rec = np.zeros(n, capi.AGENT)
    k = np.arange(n)
    rec["pos"] = np.stack([-(k % side) * 3.5 - 2.0, (k // side) * 3.5 + 2.0], axis=1)
    rec["prev_pos"] = rec["pos"]
    rec["radius"], rec["max_speed"], rec["speed"], rec["flags"] = 1.0, 20.0, 20.0, capi.FLAG_MOVABLE
    rec["flock"] = k % 2
    rec["vdes"] = (1.0, 0.0)
    fl = np.zeros(2, capi.FLOCK); fl["target"] = [(-100.0, 100.0), (-300.0, 300.0)]; fl["dest"] = -1
    rec["state"] = {"none": rng.choice([0, 1, 3, 5, 6, 7, 8], n), "all": rng.choice([2, 4], n), "some": rng.integers(0, 9, n)}[still]
    A, B = capi.Nav(0), capi.Nav(0)
    try:
        for X in (A, B):
            X.map_create(cw, cw, 1); X.map_upload_layer(0, cost)
            X.agents_upload(rec, fl, 20)
        nw = A.agents_set_work_dev()
        B.agents_set_work(None)
        want = np.nonzero((rec["state"] != 2) & (rec["state"] != 4))[0].astype(np.uint32)
        assert nw == len(want) and np.array_equal(A.agents_read_work(), want) and np.array_equal(B.agents_read_work(), want)
        if nw and n < 100_000:
            for X in (A, B):
                X.agents_tick(0)
            assert A.agents_read_velocities(nw).tobytes() == B.agents_read_velocities(nw).tobytes()
    finally:
        A.close(); B.close()


@pytest.mark.gpu
def test_c2_order_waves(pf):
    """the benchmark's C2 population (100 000 agents, 16 goals): every tick a wave of a few hundred orders -- stops, and
    move orders that regroup units under another goal -- with the blockers of the stopped and started units taken on the
    device (PFNAV_APPLY_BLOCKERS, agents_set_blocking, map_commit) on both twins"""
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
    T = Twin(bench.CHUNKS, W["cost"], rec, fl, ms, 20, blocking=True)
    rng = np.random.default_rng(8)
    try:
        for X in (T.A, T.B):
            X.pool_request_goals(np.arange(len(fl), dtype=np.int32), goals, 0)
        for t in range(8):
            s = T.tick(passes=0)
            moving = np.nonzero(s["state"] == ST_MOVING)[0]
            stop = rng.choice(moving, min(200, len(moving)), replace=False)     # most of this population arrives at once
            rest = np.setdiff1d(np.arange(n), stop)
            go = rng.choice(rest, 300, replace=False)
            d = np.concatenate([cr.deltas(stop, state=ST_ARRIVED, velocity=(0.0, 0.0)),
                                cr.deltas(go, state=ST_MOVING, flock=rng.integers(0, len(fl), len(go)), clear_hist=True)])
            T.commands(d, block=(go.astype(np.uint32), stop.astype(np.uint32)))
            assert len(T.A.agents_read_work()) >= len(go)
        T.tick(passes=0)
    finally:
        T.close()


@pytest.mark.gpu
def test_more_flocks_than_one_scan_pass(pf):
    """2 500 flocks (the scan over the flocks takes three passes of its block), some empty, entities without a flock:
    after a batch that reshuffles a third of the population the member lists give the same cohesion -- preferred
    velocities bit for bit -- as a fresh upload of the same population"""
    rng = np.random.default_rng(4)
    n, nf = 20_000, 2_500
    cost = synth.cost_from_pathable(synth.make_map(4, 4, 0x5EED0000), 4, 4)
    a = synth.make_agents(cost, 4, 4, n, 2, 0x5EED0000, radius=1.0, spacing=2.2)
    rec, _ = capi.pack_agents(a)
    rec["flock"] = rng.integers(-1, nf - 100, n)           # the last 100 flocks start empty
    fl = np.zeros(nf, capi.FLOCK)
    fl["target"] = rng.uniform(-900, -100, (nf, 2)) * [1, -1]; fl["dest"] = -1
    who = rng.choice(n, n // 3, replace=False)
    d = cr.deltas(who, flock=rng.integers(-1, nf, len(who)))
    A, B = capi.Nav(0), capi.Nav(0)
    try:
        for X in (A, B):
            X.map_create(4, 4, 1); X.map_upload_layer(0, cost)
            X.agents_upload(rec, fl, 20)
            X.set_cohesion_mode(2)                            # the member lists, not the windowed pass
        A.agents_commands(d)
        A.agents_rebuild_index()
        edited = rec.copy()
        cr.apply_deltas_np(d, edited, None)
        B.agents_upload(edited, fl, 20)
        assert A.agents_read_state(n, movestate=False)[0].tobytes() == edited.tobytes()
        nw = A.agents_set_work_dev()
        B.agents_set_work(None)
        assert nw == n
        for X in (A, B):
            X.agents_tick(0)
        assert A.agents_read_debug(nw)[0].tobytes() == B.agents_read_debug(nw)[0].tobytes()
        assert A.agents_read_velocities(nw).tobytes() == B.agents_read_velocities(nw).tobytes()
    finally:
        A.close(); B.close()


@pytest.mark.gpu
def test_work_list_and_flock_table_sized_by_both_writers(pf):
    """A's work list is sized in turn by agents_set_work and agents_set_work_dev, its flock table by agents_commands and
    agents_upload, each growing and shrinking; after every step the twins agree through resident ticks"""
    T, rec, fl = _case(seed=606)
    try:
        s = T.tick()
        # 1. a short explicit list
        short = np.nonzero(s["state"] == ST_MOVING)[0][:40].astype(np.uint32)
        for X in (T.A, T.B):
            X.agents_set_work(short)
        T.ticks(2)
        # 2. most units awake: Twin.commands builds A's list with agents_set_work_dev
        s = T.compare()
        still = np.nonzero((s["state"] == ST_ARRIVED) | (s["state"] == ST_WAITING))[0]
        T.commands(cr.deltas(still[: len(still) * 3 // 4], state=ST_MOVING, clear_hist=True))
        assert len(T.A.agents_read_work()) > T.n // 2
        T.ticks(3)
        # 3. a longer explicit list: every entity
        for X in (T.A, T.B):
            X.agents_set_work(np.arange(T.n, dtype=np.uint32))
        T.ticks(2)
        # 4. a flock table more than twice as long, rows copied from the current ones, and units moved into the new rows
        s = T.compare()
        nf = len(T.fl)
        big = T.fl[np.arange(2 * nf + 3) % nf].copy()
        who = np.nonzero(s["state"] == ST_MOVING)[0][::5]
        T.commands(cr.deltas(who, flock=nf + np.arange(len(who)) % (nf + 3)), big)
        T.ticks(3)
        # 5. a re-upload of the population with fewer flocks on both twins
        s, ms = T.A.agents_read_state(T.n)
        s["flock"] = np.where(s["flock"] >= nf, s["flock"] % nf, s["flock"])
        T.fl = T.fl[:nf].copy()
        for X in (T.A, T.B):
            X.agents_upload(s, T.fl, T.hz)
            X.agents_upload_movestate(ms)
        T.work_lists()
        T.compare()
        T.ticks(2)
        # 6. commands again: a table one row longer, some units moved into the new row
        s = T.compare()
        who = np.nonzero(s["state"] == ST_MOVING)[0][::7]
        T.commands(cr.deltas(who, flock=nf), _grown(T.fl, s["pos"][who].mean(axis=0), nf))
        T.ticks(3)
    finally:
        T.close()
