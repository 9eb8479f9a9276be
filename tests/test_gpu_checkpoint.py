"""pfnav_agents_save / pfnav_agents_restore / pfnav_group_restore.

Run A: one context with movestate, movestate_ext, formation and device blocking tables (units stopped and holding
blocks, units in ENTER_ENTITY_RANGE, TURNING and WAITING, buildings on the map) runs k ticks of the headless loop (tick,
pool misses served, compute_updates, collect_events, apply_updates_ex(APPLY_BLOCKERS), map_commit, index, work list),
saves, clears its pool and runs m more ticks, the fields requested again through the miss path.
Run B: a fresh context with the same map and building blocks restores the save, commits and runs the same m ticks.
Every tick's velocities, patches, events, agent / movestate / movestate_ext / formation / blocking tables, blocker and
faction counts and local islands equal run A's bit for bit.
Jobs: segments saved by 1, 2 or 3 members restore onto 1, 2 and 3 members with every table, the blocker and faction
counts and the local islands of the saving job, save the same rows again, and tick bit for bit like a job of as many
members that loaded the same records through the uploads and took the blocks again on the host, and, with as many
members as saved, like the saving job's own continuation. Refusals (unapplied updates, uncommitted or unexchanged ops, a
map without pfnav_route_build, a damaged segment) return their error and change nothing."""
import numpy as np
import pytest

import cases
from test_gpu_mgpu_commands import _devices, _population

capi = cases.capi
ST_ARRIVED, ST_WAITING, ST_ENTER, ST_TURNING = 2, 4, 6, 7
K, M = 6, 6
BUILDINGS = [(-30.0, 40.0, 6.0, 2), (-150.0, 200.0, 9.0, 15)]


def population(seed=4242):
    cost, rec, fl, ms = _population(seed, 20)
    n = len(rec)
    rng = np.random.default_rng(seed)
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID
    ext["rot"][:, 3] = 1.0
    moving = np.nonzero(rec["state"] == 0)[0]
    pick = rng.choice(moving, 60, replace=False)
    enter, turn, wait = pick[:20], pick[20:40], pick[40:]
    rec["state"][enter] = ST_ENTER
    ext["surround_target_uid"][enter] = rng.choice(n, 20)
    ext["target_range"][enter] = 0.5
    rec["state"][turn] = ST_TURNING
    ang = rng.uniform(-3.0, 3.0, 20).astype(np.float32)
    ext["target_dir"][turn, 1] = np.sin(ang / 2)
    ext["target_dir"][turn, 3] = np.cos(ang / 2)
    rec["state"][wait] = ST_WAITING
    ext["wait_prev"][wait] = 0
    ext["wait_ticks_left"][wait] = rng.integers(1, 5, 20)
    form = np.zeros(n, capi.FORMATION_IN)
    form["target_orientation"][:, 3] = 1.0
    blk = np.zeros(n, capi.BLOCKING)
    blk["faction_id"] = np.where(np.arange(n) % 4 == 0, 3, capi.FACTION_ID_NONE)
    arrived = np.nonzero((rec["state"] == ST_ARRIVED) & ((rec["flags"] & capi.FLAG_GARRISONED) == 0))[0].astype(np.uint32)
    return dict(cost=cost, rec=rec, fl=fl, ms=ms, ext=ext, form=form, blk=blk, arrived=arrived)


def map_ready(X, P, route=True, buildings=True):
    X.map_create(3, 3, 1)
    X.map_upload_layer(0, P["cost"]); X.map_build_nav(0)
    if route:
        X.route_build(0)
    nd = len(P["fl"]) + 2
    X.pool_create(nd, nd * 9)
    if buildings:
        for x, z, r, f in BUILDINGS:
            X.blockers_incref(x, z, r, f)


class Run:
    """one context (grp None) or the members of a group, driven through the same headless loop"""

    def __init__(self, navs, grp=None):
        self.navs, self.grp = navs, grp

    def close(self):
        if self.grp is not None:
            self.grp.close()
        for nv in self.navs:
            nv.close()

    def n(self):
        return self.navs[0].agents_device_ptrs()[2]

    def ranges(self):
        return [capi.mgpu_shard_range(self.n(), r, len(self.navs)) for r in range(len(self.navs))]

    def commit(self):
        if self.grp is not None:
            self.grp.exchange_blocker_ops()
        nd = [nv.map_commit() for nv in self.navs]
        assert nd == [nd[0]] * len(nd)

    def settle(self):
        """after a commit: the index (gather in a group) and the work lists"""
        if self.grp is not None:
            self.grp.gather()
        else:
            self.navs[0].agents_rebuild_index()
        for nv in self.navs:
            nv.agents_set_work_dev()

    def tick(self, passes=2):
        outs = []
        for nv in self.navs:
            nw = len(nv.agents_read_work())
            if not nw:
                continue
            for _ in range(passes):
                nv.agents_tick(capi.TICK_VDES_FROM_POOL)
                nv.pool_repair()
            nv.agents_tick(capi.TICK_VDES_FROM_POOL)
            nv.agents_compute_updates()
            nv.agents_collect_events()
            outs.append((nv.agents_read_velocities(nw), nv.agents_read_patches(nw), nv.agents_read_events(nw)))
            nv.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        self.commit()
        self.settle()
        joined = tuple(np.concatenate([o[k] for o in outs]).tobytes() if outs else b"" for k in range(3))
        return joined + self.snapshot()

    def snapshot(self):
        parts = []
        for nv, (lo, hi) in zip(self.navs, self.ranges()):
            a, m = nv.agents_read_state(hi - lo)
            parts.append((a, m, nv.agents_read_movestate_ext(hi - lo), nv.agents_read_formation(hi - lo),
                          nv.agents_read_blocking(hi - lo)))
        tables = tuple(np.concatenate([p[k] for p in parts]).tobytes() for k in range(5))
        maps = [(nv.blockers(0).tobytes(), nv.faction_counts(0).tobytes(), nv.local_islands(0).tobytes()) for nv in self.navs]
        assert all(mp == maps[0] for mp in maps), "members' maps differ"
        return tables + maps[0]

    def ticks(self, k):
        return [self.tick() for _ in range(k)]

    def save(self):
        return [nv.agents_save() for nv in self.navs]


NAMES = ("velocities", "patches", "events", "agents", "movestate", "movestate_ext", "formation", "blocking", "blockers",
         "faction counts", "local islands")


def same(ref, got):
    assert len(ref) == len(got)
    for t, (r, g) in enumerate(zip(ref, got)):
        for name, x, y in zip(NAMES, r, g):
            assert x == y, ("tick", t, name)


def start_solo(P):
    X = capi.Nav(0)
    map_ready(X, P)
    X.agents_upload(P["rec"], P["fl"], 20)
    X.agents_upload_movestate(P["ms"]); X.agents_upload_movestate_ext(P["ext"])
    X.agents_upload_formation(P["form"]); X.agents_upload_blocking(P["blk"])
    X.agents_set_blocking(P["arrived"], True)
    R = Run([X])
    R.commit(); R.settle()
    return R


def start_group(P, world):
    navs = [capi.Nav(d) for d in _devices(world)]
    for nv in navs:
        map_ready(nv, P)
    grp = capi.Group(navs)
    grp.share_blockers()
    n = len(P["rec"])
    rg = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
    for nv, (lo, hi) in zip(navs, rg):
        nv.agents_upload_shard(P["rec"][lo:hi], lo, hi, n, P["fl"], 20)
    grp.gather()
    for nv, (lo, hi) in zip(navs, rg):
        nv.agents_upload_movestate(P["ms"][lo:hi]); nv.agents_upload_movestate_ext(P["ext"][lo:hi])
        nv.agents_upload_formation(P["form"][lo:hi]); nv.agents_upload_blocking(P["blk"][lo:hi])
        a = P["arrived"]
        nv.agents_set_blocking(a[(a >= lo) & (a < hi)], True)
    R = Run(navs, grp)
    R.commit(); R.settle()
    return R


def restored(P, segs, world):
    """fresh contexts, map and buildings queued, the restore, commit, gather / index, work lists"""
    navs = [capi.Nav(d) for d in _devices(world)]
    for nv in navs:
        map_ready(nv, P)
    if world == 1:
        navs[0].agents_restore(segs)
        R = Run(navs)
    else:
        grp = capi.Group(navs)
        grp.share_blockers()
        grp.restore(segs)
        R = Run(navs, grp)
    R.commit(); R.settle()
    return R


def saved_and_continued(R):
    """k ticks, the save, the snapshot at the save point, then the pool cleared and m more ticks"""
    try:
        R.ticks(K)
        segs = R.save()
        before = R.snapshot()
        for nv in R.navs:
            nv.pool_clear()
        return segs, before, R.ticks(M)
    finally:
        R.close()


@pytest.fixture(scope="module")
def run_a(pf):
    P = population()
    seg, before, ref = saved_and_continued(start_solo(P))
    return P, seg, before, ref


ROW = np.dtype([("agent", capi.AGENT), ("ms", capi.MOVESTATE), ("ext", capi.MOVESTATE_EXT), ("form", capi.FORMATION_IN),
                ("blk", capi.BLOCKING)])


def loaded_long_way(P, segs, world):
    """the state of the segments loaded the way an engine had to before the restore: the records read out of the rows,
    pfnav_agents_upload(_shard) and the four table uploads, a gather, and every recorded block taken again on the host
    (pfnav_blockers_incref on every member), committed"""
    nf = len(P["fl"])
    segs = sorted(segs, key=lambda s: int(np.frombuffer(s[40:48], np.uint64)[0]))
    rows = np.frombuffer(b"".join(s[64 + 16 * nf:] for s in segs), ROW)
    fl = np.frombuffer(segs[0][64:64 + 16 * nf], capi.FLOCK)
    n = len(rows)
    navs = [capi.Nav(d) for d in _devices(world)]
    for nv in navs:
        map_ready(nv, P)
    grp = None
    rg = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
    if world == 1:
        navs[0].agents_upload(rows["agent"].copy(), fl, 20)
    else:
        grp = capi.Group(navs)
        grp.share_blockers()
        for nv, (lo, hi) in zip(navs, rg):
            nv.agents_upload_shard(rows["agent"][lo:hi].copy(), lo, hi, n, fl, 20)
        grp.gather()
    for nv, (lo, hi) in zip(navs, rg):
        r = rows[lo:hi]
        nv.agents_upload_movestate(r["ms"].copy()); nv.agents_upload_movestate_ext(r["ext"].copy())
        nv.agents_upload_formation(r["form"].copy()); nv.agents_upload_blocking(r["blk"].copy())
    held = rows[rows["blk"]["blocking"] == 1]
    for nv in navs:
        for b, a in zip(held["blk"], held["agent"]):
            nv.blockers_incref(float(b["stop_x"]), float(b["stop_z"]), float(b["stop_radius"]), int(b["faction_id"]), int(a["flags"]))
    R = Run(navs, grp)
    R.commit(); R.settle()
    return R


@pytest.mark.gpu
def test_symbols(pf):
    assert {"pfnav_agents_save", "pfnav_agents_restore", "pfnav_group_restore"} <= set(capi.SYMBOLS)


@pytest.mark.gpu
def test_solo_restore_ticks_like_the_saved_context(run_a):
    P, seg, before, ref = run_a
    B = restored(P, seg, 1)
    try:
        assert B.snapshot() == before
        same(ref, B.ticks(M))
    finally:
        B.close()


def resaved_rows(R, nf):
    return b"".join(s[64 + 16 * nf:] for s in R.save())


@pytest.fixture(scope="module")
def saves(run_a):
    """the segments, save-point snapshot and continuation (pool cleared, m ticks) of run A and of groups of 2 and 3
    members that ran the same k ticks"""
    P, seg, before, ref = run_a
    out = {1: (seg, before, ref)}
    for w in (2, 3):
        out[w] = saved_and_continued(start_group(P, w))
    return P, out


@pytest.mark.gpu
@pytest.mark.parametrize("w_save", [1, 2, 3])
@pytest.mark.parametrize("w_new", [1, 2, 3])
def test_saves_of_1_2_3_members_restore_onto_1_2_3(saves, w_save, w_new):
    """segments of w_save members restored onto w_new members (a group when w_new > 1):
    - every table, the blocker and faction counts and the local islands equal the saving job's at its save point, and the
      restored job saves the same rows again;
    - its m ticks of the headless loop equal, bit for bit, those of a job of w_new members that loaded the same records
      through the uploads, a gather and the blocks taken again on the host -- this covers what only the tick reads: the
      gathered foreign records and flock ids, the member lists, the index and the host facts;
    - with as many members as saved, its m ticks equal the saving job's own m ticks after the save (its pool cleared):
      each member serves the field misses and in-place repairs of its own work items, so the pools, and with them the
      velocities, follow the member split, and the same split makes the same ticks."""
    P, S = saves
    segs, before, ref = S[w_save]
    nf = len(P["fl"])
    B = restored(P, segs, w_new)
    try:
        assert B.snapshot() == before
        assert resaved_rows(B, nf) == b"".join(s[64 + 16 * nf:] for s in segs)
        got = B.ticks(M)
    finally:
        B.close()
    L = loaded_long_way(P, segs, w_new)
    try:
        assert L.snapshot() == before
        same(L.ticks(M), got)
    finally:
        L.close()
    if w_new == w_save:
        same(ref, got)


@pytest.mark.gpu
def test_save_refusals(pf):
    P = population(7)
    A = start_solo(P)
    X = A.navs[0]
    try:
        A.ticks(2)
        ok = A.save()
        X.agents_tick(capi.TICK_VDES_FROM_POOL)
        X.agents_compute_updates()
        with pytest.raises(capi.PfnavError, match="error -4"):
            X.agents_save()
        X.agents_apply_updates_ex(capi.APPLY_BLOCKERS)                # ops decided, not committed
        with pytest.raises(capi.PfnavError, match="error -4"):
            X.agents_save()
        A.commit(); A.settle()
        X.agents_set_blocking(P["arrived"][:3], False)
        with pytest.raises(capi.PfnavError, match="error -4"):
            X.agents_save()
        A.commit(); A.settle()
        assert len(X.agents_save()) == len(ok[0])
    finally:
        A.close()
    G = start_group(P, 2)
    try:
        G.navs[1].agents_set_blocking(P["arrived"][-2:], False)       # decided on member 1, not exchanged
        with pytest.raises(capi.PfnavError, match="error -4"):
            G.navs[1].agents_save()
        G.commit(); G.settle()
        assert all(len(s) > 64 for s in G.save())
    finally:
        G.close()


@pytest.mark.gpu
def test_restore_refusals_change_nothing(run_a):
    P, seg = run_a[0], run_a[1]
    Q = population(11)
    for world in (1, 2):
        navs = [capi.Nav(d) for d in _devices(world)]
        try:
            for r, nv in enumerate(navs):
                map_ready(nv, Q, route=(r != world - 1), buildings=False)      # the last member lacks route_build
            grp = capi.Group(navs) if world > 1 else None
            if grp is not None:
                grp.share_blockers()
            n = len(Q["rec"])
            rg = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
            for nv, (lo, hi) in zip(navs, rg):
                if grp is None:
                    nv.agents_upload(Q["rec"], Q["fl"], 20)
                else:
                    nv.agents_upload_shard(Q["rec"][lo:hi], lo, hi, n, Q["fl"], 20)
            if grp is not None:
                grp.gather()
            for nv, (lo, hi) in zip(navs, rg):
                nv.agents_upload_movestate(Q["ms"][lo:hi]); nv.agents_upload_blocking(Q["blk"][lo:hi])
            R = Run(navs, grp)
            R.settle()
            state = [(nv.agents_read_state(hi - lo)[0].tobytes(), nv.agents_read_blocking(hi - lo).tobytes(),
                      nv.agents_read_work().tobytes(), nv.blockers(0).tobytes()) for nv, (lo, hi) in zip(navs, rg)]
            bad = bytearray(seg[0]); bad[0] ^= 1
            attempts = [(seg, "error -4"), ([bytes(bad)], "error -1"), ([seg[0][:-16]], "error -1"), (seg + seg, "error -1")]
            for segs, err in attempts:
                with pytest.raises(capi.PfnavError, match=err):
                    if grp is None:
                        navs[0].agents_restore(segs)
                    else:
                        grp.restore(segs)
            R.commit()                                                 # a refusal queued no op
            got = [(nv.agents_read_state(hi - lo)[0].tobytes(), nv.agents_read_blocking(hi - lo).tobytes(),
                    nv.agents_read_work().tobytes(), nv.blockers(0).tobytes()) for nv, (lo, hi) in zip(navs, rg)]
            assert got == state
            if grp is not None:
                grp.close()
        finally:
            for nv in navs:
                nv.close()


@pytest.mark.gpu
def test_host_only_context(pf):
    nav = capi.Nav(0, hostonly=True)
    try:
        with pytest.raises(capi.PfnavError, match="error -3"):
            nav.agents_save()
    finally:
        nav.close()
