"""pfnav_agents_change_population against the path it replaces.

Twin contexts on the same map, pool and population: A removes and appends entities with agents_change_population and
builds its work list on the device; B takes the long way round: it reads back agents, movestate, movestate_ext and
blocking, releases the removed units' blocks with agents_set_blocking(removed, 0), deletes and appends the rows in numpy
(renumbering the surround targets by the same rule), re-uploads every table and runs agents_set_work(None). After the
change: every table byte for byte, equal blockers after map_commit and equal work lists; after each following resident
tick (tick, compute_updates, apply_updates, rebuild_index, work list): velocities, preferred / desired velocities, LOS
bits, patches and state, bit for bit -- cohesion included, which pins the device-built member lists."""
import numpy as np
import pytest

import cases

capi, synth = cases.capi, cases.synth
ST_MOVING, ST_ARRIVED, ST_SURROUND, ST_ENTER = 0, 2, 5, 6


def _ext_default(n):
    e = np.zeros(n, capi.MOVESTATE_EXT)
    e["surround_target_uid"] = capi.NULL_UID
    e["rot"][:, 3] = 1.0
    return e


def _renumber(uids, removed, n_old):
    """the numbering rule on old uids: survivors shift down past the removed ones, removed / NULL give NULL"""
    r = np.unique(np.asarray(removed, np.int64))
    u = uids.astype(np.int64)
    out = u - np.searchsorted(r, u)
    gone = (u >= n_old) | np.isin(u, r)
    return np.where(gone, capi.NULL_UID, out).astype(np.uint32)


class Twin:
    def __init__(self, cw, cost, rec, fl, ms, hz, nlayers=1, ext=None, form=None, blocking=None, ndests=None):
        self.cw, self.hz, self.n, self.nlayers = cw, hz, len(rec), nlayers
        self.fl = np.ascontiguousarray(fl, capi.FLOCK).copy()
        self.ndests = ndests or len(fl)
        self.has_ext, self.blocking = ext is not None, blocking is not None
        self.form = None if form is None else form.copy()       # formation inputs: no tick changes them, B keeps its copy
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
            if form is not None:
                X.agents_upload_formation(form)
            if blocking is not None:
                X.agents_upload_blocking(blocking)
        self.A.agents_set_work_dev()
        self.B.agents_set_work(None)

    def close(self):
        self.A.close(); self.B.close()

    def change(self, rm, add, ms, ext=None, form=None, blk=None, flocks=None):
        rm = np.asarray(rm, np.int64).reshape(-1)
        add = np.ascontiguousarray(add, capi.AGENT)
        n_new = self.n - len(np.unique(rm)) + len(add)
        self.A.agents_change_population(rm, add, ms=ms, ext=ext, formation=form, blocking=blk, flocks=flocks)
        # B: the long way round
        B = self.B
        sa, mb = B.agents_read_state(self.n)
        eb = B.agents_read_movestate_ext(self.n) if self.has_ext else None
        if self.blocking:
            B.agents_set_blocking(np.unique(rm).astype(np.uint32), False)
            bb = B.agents_read_blocking(self.n)
        if flocks is not None:
            self.fl = np.ascontiguousarray(flocks, capi.FLOCK).copy()
        keep = np.delete(np.arange(self.n), rm)
        sa = np.concatenate([sa[keep], add])
        B.agents_upload(sa, self.fl, self.hz)
        B.agents_upload_movestate(np.concatenate([mb[keep], ms]))
        if self.has_ext:
            e = eb[keep].copy()
            e["surround_target_uid"] = np.where(e["surround_target_uid"] == capi.NULL_UID, capi.NULL_UID,
                                                _renumber(e["surround_target_uid"], rm, self.n))
            B.agents_upload_movestate_ext(np.concatenate([e, _ext_default(len(add)) if ext is None else ext]))
        if self.form is not None:
            self.form = np.concatenate([self.form[keep], np.zeros(len(add), capi.FORMATION_IN) if form is None else form])
            B.agents_upload_formation(self.form)
        if self.blocking:
            B.agents_upload_blocking(np.concatenate([bb[keep], blk]))
        self.n = n_new
        for X in (self.A, self.B):
            if self.blocking:
                X.map_commit()
        assert len(self.A.agents_read_work()) == 0
        self.work_lists()
        return self.compare()

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
        if self.has_ext:
            assert self.A.agents_read_movestate_ext(self.n).tobytes() == self.B.agents_read_movestate_ext(self.n).tobytes()
        if self.blocking:
            assert self.A.agents_read_blocking(self.n).tobytes() == self.B.agents_read_blocking(self.n).tobytes()
            for l in range(self.nlayers):
                assert (self.A.blockers(l) == self.B.blockers(l)).all()
        for X in (self.A, self.B):
            assert X.agents_device_ptrs()[2] == self.n
        return sa

    def tick(self, passes=2):
        nw = len(self.A.agents_read_work())
        out = []
        for X in (self.A, self.B):
            for _ in range(passes):          # serve the pool misses of new flocks; the same calls on both twins
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
        s = None
        for _ in range(k):
            s = self.tick()
        return s


def _case(seed=4242, hz=20, extra_flocks=1, ext=False, form=False, blocking=False, nlayers=1):
    p, cost, a, ms = cases.update_case(seed, hz)
    nf = len(a["flock_target"])
    aa = dict(a); aa["flock_dest_index"] = np.arange(nf, dtype=np.int32)
    rec, fl = capi.pack_agents(aa)
    n = len(rec)
    e = _ext_default(n) if ext else None
    f = None
    if form:
        f = np.zeros(n, capi.FORMATION_IN)
        f["target_orientation"][:, 3] = 1.0
    b = None
    if blocking:
        b = np.zeros(n, capi.BLOCKING); b["faction_id"] = capi.FACTION_ID_NONE
    T = Twin(3, cost, rec, fl, ms, hz, nlayers=nlayers, ext=e, form=f, blocking=b, ndests=nf + extra_flocks + 2)
    return T, rec, fl, ms


def _spawn(s, ms_all, who, flock=None, shift=0.6):
    """new entities copied from existing ones (agents, movestate), moved a little, optionally into another flock"""
    a = s[who].copy()
    a["pos"] += np.float32(shift); a["prev_pos"] += np.float32(shift)
    if flock is not None:
        a["flock"] = flock
    m = ms_all[who].copy()
    m["next_pos"][:, 0] += np.float32(shift); m["next_pos"][:, 2] += np.float32(shift)
    return a, m


def _grown(fl, target, dest):
    out = np.zeros(len(fl) + 1, capi.FLOCK)
    out[:-1] = fl
    out["target"][-1], out["dest"][-1], out["layer"][-1] = target, dest, 0
    return out


@pytest.mark.gpu
def test_symbols(pf):
    assert "pfnav_agents_change_population" in capi.SYMBOLS and "pfnav_agents_read_movestate_ext" in capi.SYMBOLS


@pytest.mark.gpu
def test_removals_spread_over_flocks(pf):
    T, rec, fl, ms = _case(seed=71)
    try:
        T.ticks(2)
        rng = np.random.default_rng(1)
        rm = rng.choice(T.n, 120, replace=True)                  # repeats included
        T.change(rm, np.zeros(0, capi.AGENT), np.zeros(0, capi.MOVESTATE))
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_appends_into_old_and_new_flocks_then_remove_and_add(pf):
    """appends into existing flocks and into a flock appended in the same call, then after ticks one call that removes
    and adds"""
    T, rec, fl, ms = _case(seed=5)
    try:
        s = T.ticks(2)
        _, m = T.A.agents_read_state(T.n)
        nf = len(T.fl)
        who = np.nonzero(s["state"] == ST_MOVING)[0][:40]
        a1, m1 = _spawn(s, m, who[:20])
        a2, m2 = _spawn(s, m, who[20:], flock=nf)
        T.change([], np.concatenate([a1, a2]), np.concatenate([m1, m2]), flocks=_grown(T.fl, s["pos"][who].mean(axis=0) + 20.0, nf))
        s = T.ticks(4)
        _, m = T.A.agents_read_state(T.n)
        rng = np.random.default_rng(2)
        a3, m3 = _spawn(s, m, rng.choice(T.n, 30, replace=False), shift=-0.4)
        T.change(rng.choice(T.n, 50, replace=False), a3, m3)
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_removed_blocking_units_release_their_blocks(pf):
    """ARRIVED units that took their blocks on the device die: the blocker grid equals B's, where agents_set_blocking
    released them before the re-upload; new units arrive with blocking records and take no block"""
    T, rec, fl, ms = _case(seed=19, blocking=True)
    try:
        T.ticks(4)
        bl = T.A.agents_read_blocking(T.n)
        held = np.nonzero(bl["blocking"] == 1)[0]
        assert len(held) > 5
        before = T.A.blockers(0).copy()
        s, m = T.A.agents_read_state(T.n)
        a, mm = _spawn(s, m, np.arange(10))
        b = np.zeros(10, capi.BLOCKING); b["faction_id"] = capi.FACTION_ID_NONE
        T.change(held[::2], a, mm, blk=b)
        assert not (T.A.blockers(0) == before).all()
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_removed_targets_become_null_and_units_arrive(pf):
    """a surround target and an enter-range target die: the survivors' targets become PFNAV_NULL_UID on both twins and
    the units reach ARRIVED; other targets are renumbered"""
    T, rec, fl, ms = _case(seed=8, ext=True)
    try:
        n = T.n
        e = _ext_default(n)
        sur, ent, far = np.arange(100, 110), np.arange(200, 210), np.arange(300, 305)
        e["surround_target_uid"][sur] = 3
        e["surround_target_uid"][ent] = 7
        e["target_range"][ent] = 0.5
        e["surround_target_uid"][far] = n - 1                    # survives, renumbered
        s, m = T.A.agents_read_state(n)
        s["state"][sur], s["state"][ent] = ST_SURROUND, ST_ENTER
        s["state"][far] = ST_ENTER; e["target_range"][far] = 0.5
        for X in (T.A, T.B):
            X.agents_upload(s, T.fl, T.hz); X.agents_upload_movestate(m); X.agents_upload_movestate_ext(e)
        T.work_lists()
        T.ticks(2)
        T.change([3, 7, 50], np.zeros(0, capi.AGENT), np.zeros(0, capi.MOVESTATE))
        x = T.A.agents_read_movestate_ext(T.n)
        assert (x["surround_target_uid"][np.concatenate([sur, ent]) - 3] == capi.NULL_UID).all()
        assert (x["surround_target_uid"][far - 3] == n - 4).all()
        s = T.ticks(3)
        assert (s["state"][np.concatenate([sur, ent]) - 3] == ST_ARRIVED).all()
        T.ticks(5)
    finally:
        T.close()


@pytest.mark.gpu
def test_appends_across_a_layer_boundary_with_default_and_explicit_records(pf):
    """nlayers = 2: appended units of radius 6 (layer 1); ext and formation tables present, appended with NULL records
    (defaults) in one call and explicit ones in the next"""
    T, rec, fl, ms = _case(seed=99, nlayers=2, ext=True, form=True)
    try:
        s = T.ticks(2)
        _, m = T.A.agents_read_state(T.n)
        a, mm = _spawn(s, m, np.arange(0, 60, 3))
        a["radius"][::2] = 6.0
        T.change([1, 2], a, mm)
        s = T.ticks(2)
        _, m = T.A.agents_read_state(T.n)
        a, mm = _spawn(s, m, np.arange(5, 45, 4), shift=0.3)
        a["radius"][1::2] = 6.0
        e = _ext_default(len(a)); e["wait_ticks_left"] = 2; e["surround_target_uid"][0] = T.n + 1   # an appended uid
        f = np.zeros(len(a), capi.FORMATION_IN); f["target_orientation"][:, 3] = 1.0
        T.change([0], a, mm, ext=e, form=f)
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_last_flock_emptied_and_dropped(pf):
    T, rec, fl, ms = _case(seed=31)
    try:
        s = T.ticks(2)
        last = len(T.fl) - 1
        T.change(np.nonzero(s["flock"] == last)[0], np.zeros(0, capi.AGENT), np.zeros(0, capi.MOVESTATE), flocks=T.fl[:last].copy())
        s = T.ticks(6)
        assert s["flock"].max() == last - 1
    finally:
        T.close()


@pytest.mark.gpu
def test_population_to_zero_and_refilled(pf):
    T, rec, fl, ms = _case(seed=12, blocking=True)
    try:
        s = T.ticks(2)
        _, m = T.A.agents_read_state(T.n)
        keep_a, keep_m = s.copy(), m.copy()
        T.change(np.arange(T.n), np.zeros(0, capi.AGENT), np.zeros(0, capi.MOVESTATE), blk=np.zeros(0, capi.BLOCKING))
        assert T.n == 0
        b = np.zeros(len(keep_a), capi.BLOCKING); b["faction_id"] = capi.FACTION_ID_NONE
        T.change([], keep_a, keep_m, blk=b)
        T.ticks(8)
    finally:
        T.close()


@pytest.mark.gpu
def test_growth_past_buffer_capacity(pf):
    """1 000 -> 6 000 entities: every table regrows and keeps its contents"""
    rng = np.random.default_rng(6)
    cw = 4
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, 0x5EED0000), cw, cw)
    a = synth.make_agents(cost, cw, cw, 6000, 3, 0x5EED0000, radius=1.0, spacing=2.2)
    rec, fl = capi.pack_agents(a)
    ms = np.zeros(len(rec), capi.MOVESTATE)
    ms["next_pos"][:, 0], ms["next_pos"][:, 2] = rec["pos"][:, 0], rec["pos"][:, 1]
    ms["step"] = 1.0; ms["next_rot"][:, 3] = 1.0; ms["combat_facing"][:, 3] = 1.0
    b = np.zeros(len(rec), capi.BLOCKING); b["faction_id"] = rng.integers(0, 16, len(rec))
    e = _ext_default(len(rec)); e["wait_prev"] = rng.integers(0, 3, len(rec))
    fl["dest"] = -1
    T = Twin(cw, cost, rec[:1000], fl, ms[:1000], 20, ext=e[:1000], blocking=b[:1000])
    try:
        T.tick(passes=0)
        T.change([], rec[1000:], ms[1000:], ext=e[1000:], blk=b[1000:])
        assert T.n == 6000
        T.ticks(3)
    finally:
        T.close()


@pytest.mark.gpu
def test_refusals_change_nothing(pf):
    T, rec, fl, ms = _case(seed=21, blocking=True)
    try:
        s = T.ticks(2)
        _, m = T.A.agents_read_state(T.n)
        a, mm = _spawn(s, m, np.arange(4))
        b = np.zeros(4, capi.BLOCKING); b["faction_id"] = capi.FACTION_ID_NONE
        bad_flock = a.copy(); bad_flock["flock"][0] = len(T.fl)
        bad_layer = a.copy(); bad_layer["radius"][1] = 6.0
        bad_float = a.copy(); bad_float["velocity"][2, 0] = np.nan
        bad_blk = b.copy(); bad_blk["faction_id"][3] = 16
        before = (T.A.agents_read_state(T.n), T.A.agents_read_blocking(T.n).tobytes(), T.A.agents_read_work().tobytes(),
                  T.A.blockers(0).copy())
        for kw in (dict(remove=[T.n]), dict(add=bad_flock), dict(add=bad_layer), dict(add=bad_float), dict(blocking=bad_blk),
                   dict(ms=None), dict(blocking=None), dict(ext=_ext_default(4)), dict(formation=np.zeros(4, capi.FORMATION_IN)),
                   dict(flocks=T.fl[:1].copy())):
            args = dict(remove=[0, 1], add=a, ms=mm, blocking=b)
            args.update(kw)
            with pytest.raises(capi.PfnavError, match="error -1"):
                T.A.agents_change_population(args.pop("remove"), args.pop("add"), **args)
        after = (T.A.agents_read_state(T.n), T.A.agents_read_blocking(T.n).tobytes(), T.A.agents_read_work().tobytes(),
                 T.A.blockers(0))
        assert after[0][0].tobytes() == before[0][0].tobytes() and after[0][1].tobytes() == before[0][1].tobytes()
        assert after[1:3] == before[1:3] and (after[3] == before[3]).all()
        T.A.map_commit()                                          # no op was queued by a refusal
        assert (T.A.blockers(0) == before[3]).all()
        T.tick()
        grp = capi.Group([T.A])
        try:
            with pytest.raises(capi.PfnavError, match="error -4"):
                T.A.agents_change_population([0], np.zeros(0, capi.AGENT))
        finally:
            grp.close()
        T.compare()
    finally:
        T.close()


@pytest.mark.gpu
def test_host_only_context_has_no_population_path(pf):
    nav = capi.Nav(0, hostonly=True)
    try:
        with pytest.raises(capi.PfnavError, match="error -3"):
            nav.agents_change_population([0], np.zeros(0, capi.AGENT))
    finally:
        nav.close()


@pytest.mark.gpu
def test_c2_churn_with_device_blockers(pf):
    """the benchmark's C2 population (100 000 entities): 1 % removed and 1 % added every tick over several ticks, with
    the blockers of stopped units taken on the device and released when they die"""
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
    b = np.zeros(n, capi.BLOCKING); b["faction_id"] = capi.FACTION_ID_NONE
    T = Twin(bench.CHUNKS, W["cost"], rec, fl, ms, 20, blocking=b)
    rng = np.random.default_rng(8)
    try:
        for X in (T.A, T.B):
            X.pool_request_goals(np.arange(len(fl), dtype=np.int32), goals, 0)
        for t in range(4):
            s = T.tick(passes=0)
            _, m = T.A.agents_read_state(T.n)
            k = T.n // 100
            who = rng.choice(T.n, k, replace=False)
            a, mm = _spawn(s, m, who, shift=0.25)
            a["state"] = ST_MOVING
            bb = np.zeros(k, capi.BLOCKING); bb["faction_id"] = capi.FACTION_ID_NONE
            T.change(rng.choice(T.n, k, replace=False), a, mm, blk=bb)
        T.tick(passes=0)
    finally:
        T.close()
