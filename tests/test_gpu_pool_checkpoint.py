"""pfnav_pool_save / pfnav_pool_restore: the field pool saved with the population, so that a resumed game ticks exactly
like the game that was saved.

Run A: the headless loop of test_gpu_checkpoint.py (tick, misses served, compute_updates, collect_events,
apply_updates_ex(APPLY_BLOCKERS), map_commit, index, work list) runs k ticks, saves the agents and the pool, and runs m more
ticks with its pool kept. Run B: a fresh context restores the agents, commits, restores the pool, settles and runs the same
m ticks. Every tick's velocities, patches, events, tables, blocker and faction counts, local islands and every pool entry
(pfnav_pool_get over all destinations and chunks, and the whole pool segment) equal run A's bit for bit: with the serial and
the batched miss service, with a pool small enough that the continuation evicts, with zone and entity fields in the pool
and units reading the entity fields, and for jobs of 2 and 3 members. Round trips, the map digest and the refusals (each
changing nothing) are checked on their own."""
import numpy as np
import pytest

import cases
from test_gpu_checkpoint import K, M, Run, map_ready, population, same, start_group, start_solo
from test_gpu_mgpu_commands import _devices
from test_pool_checkpoint_emu import fmask_of, map_digest_np, parse

capi = cases.capi
ST_MOVING, ST_SEEK = 0, 3
CHUNKS = [(c // 3, c % 3) for c in range(9)]


def ndests(P):
    return len(P["fl"]) + 2


def pool_entries(nv, nd):
    """every (dest, chunk) entry as pfnav_pool_get reports it: has bits (through None), ff_id, flow and LOS bytes"""
    out = []
    for d in range(nd):
        for c in CHUNKS:
            f, l, ffid = nv.pool_get(d, c)
            out.append((ffid, None if f is None else f.tobytes(), None if l is None else l.tobytes()))
    return out


class PoolRun(Run):
    """Run's headless loop with the miss service chosen (pool_repair or pool_repair_batch), and after every tick each
    member's pool entries and pool segment"""

    def __init__(self, navs, grp=None, repair="pool_repair", nd=0):
        super().__init__(navs, grp)
        self.repair, self.nd = repair, nd

    @classmethod
    def of(cls, R, repair, nd):
        return cls(R.navs, R.grp, repair, nd)

    def tick(self, passes=2):
        outs = []
        for nv in self.navs:
            nw = len(nv.agents_read_work())
            if not nw:
                continue
            for _ in range(passes):
                nv.agents_tick(capi.TICK_VDES_FROM_POOL)
                getattr(nv, self.repair)()
            nv.agents_tick(capi.TICK_VDES_FROM_POOL)
            nv.agents_compute_updates()
            nv.agents_collect_events()
            outs.append((nv.agents_read_velocities(nw), nv.agents_read_patches(nw), nv.agents_read_events(nw)))
            nv.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        self.commit()
        self.settle()
        joined = tuple(np.concatenate([o[k] for o in outs]).tobytes() if outs else b"" for k in range(3))
        return joined + self.snapshot() + (self.pools(),)

    def pools(self):
        return [(pool_entries(nv, self.nd), nv.pool_save()) for nv in self.navs]


def same_pools(ref, got):
    assert len(ref) == len(got)
    for t, (r, g) in enumerate(zip(ref, got)):
        for rank, ((er, sr), (eg, sg)) in enumerate(zip(r[-1], g[-1])):
            assert er == eg, ("tick", t, "member", rank, "pool entries")
            assert sr == sg, ("tick", t, "member", rank, "pool segment")


def saved_and_kept(R, k=K, m=M):
    """k ticks, the agents' and the pools' save, then m more ticks with the pools kept"""
    try:
        R.ticks(k)
        asegs = R.save()
        psegs = [nv.pool_save() for nv in R.navs]
        return asegs, psegs, R.ticks(m)
    finally:
        R.close()


def resumed(P, asegs, psegs, world, repair="pool_repair", max_fields=None, setup=None):
    """fresh contexts in the resume order: map built, buildings queued, agents_restore, (job: exchange), map_commit,
    pool_restore, gather / index, work lists"""
    nd = ndests(P)
    navs = [capi.Nav(d) for d in _devices(world)]
    for nv in navs:
        map_ready(nv, P)
        if max_fields:
            nv.pool_create(nd, max_fields)
        if setup:
            setup(nv)
    grp = None
    if world == 1:
        navs[0].agents_restore(asegs)
    else:
        grp = capi.Group(navs)
        grp.share_blockers()
        grp.restore(asegs)
    R = PoolRun(navs, grp, repair, nd)
    R.commit()
    for nv, s in zip(navs, psegs):
        nv.pool_restore(s)
    R.settle()
    return R


def check_continuation(P, asegs, psegs, ref, world=1, **kw):
    B = resumed(P, asegs, psegs, world, **kw)
    try:
        assert [nv.pool_save() for nv in B.navs] == psegs, "the restored pools save other bytes"
        got = B.ticks(M)
    finally:
        B.close()
    same(ref, got)
    same_pools(ref, got)
    return got


@pytest.fixture(scope="module")
def run_a(pf):
    P = population()
    asegs, psegs, ref = saved_and_kept(PoolRun.of(start_solo(P), "pool_repair", ndests(P)))
    return P, asegs, psegs, ref


@pytest.mark.gpu
def test_symbols(pf):
    assert {"pfnav_pool_save", "pfnav_pool_restore"} <= set(capi.SYMBOLS)


@pytest.mark.gpu
def test_solo_continuation_without_a_clear(run_a):
    P, asegs, psegs, ref = run_a
    assert parse(psegs[0])["h"]["nstored"] > 0
    check_continuation(P, asegs, psegs, ref)


@pytest.mark.gpu
def test_solo_continuation_batched_repair(pf):
    P = population()
    asegs, psegs, ref = saved_and_kept(PoolRun.of(start_solo(P), "pool_repair_batch", ndests(P)))
    check_continuation(P, asegs, psegs, ref, repair="pool_repair_batch")


def evictions(ref, psegs):
    """keys mapped after one tick and unmapped after the next: only an eviction unmaps a key without a clear"""
    n, prev = 0, parse(psegs[0])["slot"]
    for t in ref:
        cur = parse(t[-1][0][1])["slot"]
        n += int(((prev >= 0) & (cur < 0)).sum())
        prev = cur
    return n


@pytest.mark.gpu
@pytest.mark.parametrize("repair", ["pool_repair", "pool_repair_batch"])
def test_lru_pressure(run_a, repair):
    P = population()
    nd = ndests(P)
    used = int(parse(run_a[2][0])["h"]["used"])
    small = max(6, used * 2 // 3)                       # fewer slots than run A keeps in use: the continuation evicts
    R = start_solo(P)
    R.navs[0].pool_create(nd, small)
    asegs, psegs, ref = saved_and_kept(PoolRun.of(R, repair, nd))
    assert evictions(ref, psegs) > 0, ("the continuation did not evict: the test would pass vacuously", used, small)
    check_continuation(P, asegs, psegs, ref, repair=repair, max_fields=small)


def with_seekers(seed=4242, nseek=24):
    """the checkpoint population with moving units turned into SEEK_ENEMIES units that read the TARGET_ENEMIES field of
    the last destination"""
    P = population(seed)
    rec = P["rec"]
    rng = np.random.default_rng(seed + 1)
    moving = np.nonzero(rec["state"] == ST_MOVING)[0]
    pick = rng.choice(moving, nseek, replace=False)
    rec["state"][pick] = ST_SEEK
    rec["aux_dest1"][pick] = ndests(P)                  # dest nd - 1, stored + 1
    return P


def aux_fields(nv, P):
    """a group-arrival zone field on dest nd - 2 and a TARGET_ENEMIES field on dest nd - 1 for half of the chunks (the
    seekers in the others miss, and the entity-field repair builds their fields from the remembered footprints)"""
    nd = ndests(P)
    rec = P["rec"]
    foes = np.nonzero(rec["state"] == 2)[0][:12]
    nv.pool_request_zone(nd - 2, rec["pos"][foes[0]], 6)
    fp = capi.Nav.footprints(rec["pos"][foes], rec["radius"][foes])
    nv.pool_request_entity_fields(nd - 1, capi.TARGET_ENEMIES, fp, CHUNKS[::2])


@pytest.mark.gpu
def test_zone_and_entity_fields(pf):
    P = with_seekers()
    nd = ndests(P)
    R = start_solo(P)
    aux_fields(R.navs[0], P)
    before = pool_entries(R.navs[0], nd)
    assert any(e[1] is not None for e in before[(nd - 2) * 9:(nd - 1) * 9]), "no zone field"
    asegs, psegs, ref = saved_and_kept(PoolRun.of(R, "pool_repair", nd))
    d = parse(psegs[0])
    assert d["aux"]["kind"][nd - 1] == capi.TARGET_ENEMIES and d["h"]["nfp"] > 0
    built = [sum(e[1] is not None for e in t[-1][0][0][(nd - 1) * 9:nd * 9]) for t in ref]
    assert all(built), ("the entity fields are not in the pool during the continuation", built)
    check_continuation(P, asegs, psegs, ref)


@pytest.mark.gpu
def test_round_trip_rewind_and_clear(run_a):
    P, asegs, psegs, _ = run_a
    nd = ndests(P)
    B = resumed(P, asegs, psegs, 1)
    X = B.navs[0]
    try:
        saved = pool_entries(X, nd)
        assert X.pool_save() == psegs[0]
        # further pool work without a map change (a tick's misses served, a zone field), then the restore rewinds it
        X.agents_tick(capi.TICK_VDES_FROM_POOL); X.pool_repair()
        X.agents_tick(capi.TICK_VDES_FROM_POOL)
        X.pool_request_zone(nd - 2, P["rec"]["pos"][0], 5)
        assert X.pool_save() != psegs[0]
        X.pool_restore(psegs[0])
        assert pool_entries(X, nd) == saved and X.pool_save() == psegs[0]
        # a cleared pool saves as empty and restores as empty
        X.pool_clear()
        empty = X.pool_save()
        d = parse(empty)
        assert d["h"]["used"] == 0 and d["h"]["nstored"] == 0 and (d["slot"] == -1).all()
        X.pool_restore(psegs[0])
        X.pool_restore(empty)
        assert all(e == (0, None, None) for e in pool_entries(X, nd)) and X.pool_save() == empty
    finally:
        B.close()


@pytest.fixture(scope="module")
def jobs(pf):
    P = population()
    nd = ndests(P)
    return P, {w: saved_and_kept(PoolRun.of(start_group(P, w), "pool_repair", nd)) for w in (2, 3)}


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_jobs_continue_like_the_saving_job(jobs, world):
    P, S = jobs
    asegs, psegs, ref = S[world]
    check_continuation(P, asegs, psegs, ref, world=world)


@pytest.mark.gpu
def test_refusals_change_nothing(run_a):
    P, asegs, psegs, ref = run_a
    nd = ndests(P)
    seg = psegs[0]
    B = resumed(P, asegs, psegs, 1)
    X = B.navs[0]
    try:
        state = (pool_entries(X, nd), X.pool_save(), X.agents_read_state(B.n())[0].tobytes(), X.blockers(0).tobytes(),
                 X.local_islands(0).tobytes())
        flipped = bytearray(seg); flipped[64 + 3] ^= 0x40           # the first slot-table entry
        magic = bytearray(seg); magic[0] ^= 1
        for bad in (bytes(flipped), seg[:-16], seg[:40], bytes(magic)):
            with pytest.raises(capi.PfnavError, match="error -1"):
                X.pool_restore(bad)
        got = (pool_entries(X, nd), X.pool_save(), X.agents_read_state(B.n())[0].tobytes(), X.blockers(0).tobytes(),
               X.local_islands(0).tobytes())
        assert got == state
        ticks = B.ticks(M)
    finally:
        B.close()
    same(ref, ticks)
    same_pools(ref, ticks)
    # uncommitted ops, at save and at restore
    U = resumed(P, asegs, psegs, 1)
    Y = U.navs[0]
    try:
        entries = pool_entries(Y, nd)
        Y.blockers_incref(-60.0, 60.0, 3.0)
        with pytest.raises(capi.PfnavError, match="error -4"):
            Y.pool_save()
        with pytest.raises(capi.PfnavError, match="error -4"):
            Y.pool_restore(seg)
        assert pool_entries(Y, nd) == entries
    finally:
        U.close()
    # a map with one more building, another pool geometry, no pool: refused, the target's pool as it was
    def one_more(nv):
        nv.blockers_incref(-300.0, 300.0, 5.0, 2)
    for setup, err in ((one_more, "error -1"), (lambda nv: nv.pool_create(nd, nd * 9 - 1), "error -1")):
        C = resumed(P, asegs, [], 1, setup=setup)
        Y = C.navs[0]
        try:
            empty = Y.pool_save()
            with pytest.raises(capi.PfnavError, match=err):
                Y.pool_restore(seg)
            assert Y.pool_save() == empty and all(e == (0, None, None) for e in pool_entries(Y, nd))
        finally:
            C.close()
    Z = capi.Nav(0)
    try:
        Z.map_create(3, 3, 1)
        Z.map_upload_layer(0, P["cost"]); Z.map_build_nav(0)
        for call in (lambda: Z.pool_save(), lambda: Z.pool_restore(seg)):
            with pytest.raises(capi.PfnavError, match="error -1"):
                call()
    finally:
        Z.close()
    H = capi.Nav(0, hostonly=True)
    try:
        for call in (lambda: H.pool_save(), lambda: H.pool_restore(seg)):
            with pytest.raises(capi.PfnavError, match="error -3"):
                call()
    finally:
        H.close()


@pytest.mark.gpu
def test_digest_is_the_host_function_of_the_map(run_a):
    """the segment's digest equals the CPU restatement over the map read back: cost, blocker counts, local islands and
    the faction masks of the faction counts"""
    P, asegs, psegs, _ = run_a
    B = resumed(P, asegs, psegs, 1)
    X = B.navs[0]
    try:
        cost, _, _ = X.map_get_layer(0)
        fc = X.faction_counts(0)
        assert fc.any(), "no faction-tagged blocks: the masks would not be covered"
        want = map_digest_np(cost, X.blockers(0), X.local_islands(0), fmask_of(fc), 3, 3)
        assert int(np.frombuffer(X.pool_save()[56:64], np.uint64)[0]) == want
        assert int(parse(psegs[0])["h"]["digest"]) == want
        X.set_enemy_factions(3, 1 << 2)                      # the enemy table is part of the digest
        assert int(np.frombuffer(X.pool_save()[56:64], np.uint64)[0]) != want
    finally:
        B.close()
