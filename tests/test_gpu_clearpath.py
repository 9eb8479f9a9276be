"""ClearPath on the device, case family by case family (tests/clearpath_cases.py), as populations on an open 8 x 8-chunk
map: one case per 64 x 64 wu cell, so no two cases' neighbours meet; the centre entities are the work list, each in a
flock of its own; static neighbours are ARRIVED, dynamic ones move at |vel| >= 0.3. Plus a cell with garrisoned entities
(the filter path of find_neighbours) and one with more than 512 raw hits, at 20 Hz and 1 Hz.

- The two-phase split (k_agent_velocity<1> + <2>) equals the single pass bit for bit.
- ClearPath in isolation: with the device's own preferred velocity and the neighbour lists built in the reference's
  order (ents_in_circle, find_neighbours' classification, 32 per list, the entity at prev_pos), the device velocity equals
  the port's clearpath() + vec2_truncate bit for bit, and pfnav_agents_clearpath_stats equals the sums of the per-case
  counters of the device source run on CPU threads (tests/emu/clearpath_emu.cpp) on the same inputs: the device took the
  literal replay for exactly the entities the emulation did.
- The windowed cohesion pass keeps the tick's ClearPath counters (it used to free them along with the velocity kernel's
  work-queue counter on its first tick)."""
import numpy as np
import pytest

import cases
import clearpath_cases as cc
import test_clearpath_emu as cpe

pytestmark = pytest.mark.gpu
capi = cases.capi
F = np.float32
CW = 8                      # chunks per side: 2048 wu, 32 x 32 cells of 64 wu
CELL = 64
STATE_MOVING, STATE_ARRIVED = 0, 2
MAX_SPEED = 20.0
VEL_RTOL = 1e-4


def _centres(n):
    k = np.arange(n)
    return np.stack([-(CELL // 2 + CELL * (k % 32)), CELL // 2 + CELL * (k // 32)], axis=1).astype(F)


def _families(seed, per_family):
    """every family of clearpath_cases on consecutive cells (integer cell centres)"""
    rng = np.random.default_rng(seed)
    parts, names = [], []
    for name, gen in cc.GENERATORS.items():
        n = per_family if name != "overflow" else per_family // 3
        parts.append(gen(rng, _centres(len(names) + n)[len(names):]))
        names += [name] * n
    return cc.Cases.concat(parts), names


def population(cs, garrison_cells=(), crowd_cell=None):
    """agent records: the centres first (uid = case index, the work list), then their neighbours; every entity its own
    flock. garrison_cells: cases that also get garrisoned entities among their neighbours; crowd_cell: a case whose
    cell is filled with > 512 static entities within 10 wu"""
    n = len(cs)
    pos, vel, rad, state, flags = [], [], [], [], []
    for i in range(n):
        pos.append(cs.self5[i, :2]); vel.append(cs.self5[i, 2:4]); rad.append(cs.self5[i, 4]); state.append(STATE_MOVING)
        flags.append(capi.FLAG_MOVABLE)
    for i in range(n):
        for k in range(cs.ndyn[i]):
            d = cs.dyn[i, k]
            pos.append(d[:2]); vel.append(d[2:4]); rad.append(d[4]); state.append(STATE_MOVING); flags.append(capi.FLAG_MOVABLE)
        for k in range(cs.nstat[i]):
            s = cs.stat[i, k]
            pos.append(s[:2]); vel.append((0.0, 0.0)); rad.append(s[4]); state.append(STATE_ARRIVED); flags.append(capi.FLAG_MOVABLE)
        if i in garrison_cells:
            for dx, dz in ((1.0, 1.5), (-2.0, 0.5), (0.5, -3.0), (6.0, 2.0)):
                pos.append(cs.self5[i, :2] + F((dx, dz))); vel.append((0.0, 0.0)); rad.append(1.0); state.append(STATE_ARRIVED)
                flags.append(capi.FLAG_MOVABLE | capi.FLAG_GARRISONED)
        if crowd_cell == i:
            g = np.arange(-9.0, 9.01, 0.75)
            for dx in g:
                for dz in g:
                    if 0.5 < np.hypot(dx, dz) < 9.4:
                        pos.append(cs.self5[i, :2] + F((dx, dz))); vel.append((0.0, 0.0)); rad.append(0.25)
                        state.append(STATE_ARRIVED); flags.append(capi.FLAG_MOVABLE)
    m = len(pos)
    rec = np.zeros(m, capi.AGENT)
    rec["pos"] = np.asarray(pos, F); rec["prev_pos"] = rec["pos"]; rec["velocity"] = np.asarray(vel, F)
    rec["radius"] = np.asarray(rad, F); rec["max_speed"] = MAX_SPEED; rec["speed"] = MAX_SPEED
    rec["state"] = state; rec["flags"] = flags; rec["flock"] = np.arange(m)
    vp = cs.vpref.astype(np.float64)
    ln = np.linalg.norm(vp, axis=1, keepdims=True)
    rec["vdes"][:n] = np.where(ln > 0, vp / np.maximum(ln, 1e-9), 0.0).astype(F)
    fl = np.zeros(m, capi.FLOCK)
    fl["target"] = rec["pos"]
    fl["target"][:n] = (rec["pos"][:n] + F(500.0) * rec["vdes"][:n]).astype(F)
    fl["dest"] = np.arange(m)
    return rec, fl


def reference_lists(world, rec, uid):
    """find_neighbours (movement.c:2768) as pfo_velocity_work builds it: ents_in_circle order, 32 per list"""
    p = rec["pos"][uid]
    dyn, stat = [], []
    for cu in world.ents_in_circle(float(p[0]), float(p[1]), 10.0, 512):
        o = rec[cu]
        if cu == uid or not (o["flags"] & capi.FLAG_MOVABLE) or o["radius"] == 0:
            continue
        if (rec["flags"][uid] & capi.FLAG_AIR) != (o["flags"] & capi.FLAG_AIR):
            continue
        v = o["velocity"].astype(F)
        still = o["state"] in (STATE_ARRIVED, 4) or np.sqrt(F(v[0] * v[0] + v[1] * v[1])) < F(0.3)
        row = (o["pos"][0], o["pos"][1], 0.0 if still else v[0], 0.0 if still else v[1], o["radius"])
        (stat if still else dyn).append(row)
    z = np.zeros((0, 5), F)
    return (np.asarray(dyn[:32], F) if dyn else z), (np.asarray(stat[:32], F) if stat else z)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return cpe.build_emu(tmp_path_factory.mktemp("clearpath_emu_gpu"))


@pytest.fixture(scope="module")
def fresh_nav(pf):
    n = pf.capi.Nav(0)
    cost = np.ones((CW * CW, 64, 64), np.uint8)
    n.map_create(CW, CW, 1); n.map_upload_layer(0, cost); n.map_build_nav(0)
    yield n, cost
    n.set_two_phase(1); n.set_cohesion_mode(0); n.set_los_variant(2)
    n.close()


@pytest.mark.parametrize("hz", [20, 1])
def test_clearpath_families_on_device(fresh_nav, pforacle, emu, hz):
    nav, cost = fresh_nav
    cs, names = _families(0xC1EA0 + hz, 120)
    n = len(cs)
    assert n <= 1024 - 2
    rec, fl = population(cs, garrison_cells=set(range(0, n, 97)), crowd_cell=n - 1)
    work = np.arange(n, dtype=np.uint32)
    out = {}
    try:
        nav.agents_upload(rec, fl, hz)
        nav.agents_set_work(work)
        for mode in (0, 2):
            nav.set_two_phase(mode)
            nav.clearpath_stats()                                       # reset
            nav.agents_tick(0)
            out[mode] = (nav.agents_read_velocities(n), nav.agents_read_debug(n)[0], nav.clearpath_stats())
    finally:
        nav.set_two_phase(1)
    vel, vpref, stats = out[0]
    # the two-phase split is the single pass, bit for bit (including its counters)
    assert (out[2][0] == vel).all() and (out[2][1] == vpref).all() and out[2][2] == stats

    world = pforacle.OracleWorld(pforacle.OracleMap(CW, CW, cost), rec, fl, hz)
    try:
        evel, evpref = world.velocity_work(work)
        assert cases.relerr(vpref, evpref).max() <= VEL_RTOL
        # ClearPath in isolation, on the device's own preferred velocity
        iso = cc.Cases(n)
        raw_hits = 0
        for i in range(n):
            dyn, stat = reference_lists(world, rec, i)
            iso.self5[i] = (rec["prev_pos"][i, 0], rec["prev_pos"][i, 1], rec["velocity"][i, 0], rec["velocity"][i, 1], rec["radius"][i])
            iso.vpref[i] = vpref[i]
            iso.dyn[i, :len(dyn)] = dyn; iso.ndyn[i] = len(dyn)
            iso.stat[i, :len(stat)] = stat; iso.nstat[i] = len(stat)
            iso.max_len[i] = F(MAX_SPEED) / F(hz)
            if i == n - 1:
                raw_hits = len(world.ents_in_circle(float(rec["pos"][i, 0]), float(rec["pos"][i, 1]), 10.0, 1024))
        assert raw_hits > 512
        want = cpe.run_port(pforacle, iso)
        bad = [i for i in range(n) if not cpe.bits_equal(vel[i], want[i])]
        assert not bad, [(i, names[i] if i < len(names) else "crowd", vel[i], want[i]) for i in bad[:5]]
        ev, es, _ = cpe.run_emu(emu, iso, 0)
        assert cpe.bits_equal(ev, vel)
        tot = es.sum(axis=0)
        assert stats == dict(zip(("no_admissible", "loop_possible", "literal_replays", "replay_solves"), (int(v) for v in tot)))
        print("\n[clearpath on device, %d Hz] %d entities: %s" % (hz, n, stats))
        assert stats["no_admissible"] > 0 and stats["loop_possible"] > 0
    finally:
        world.close()


def _crowd(n=20000):
    """a dense population of ~20 k entities, every one its own flock (cohesion is zero whichever pass computes it)"""
    cw = CW
    cost = np.ones((cw * cw, 64, 64), np.uint8)
    a = cases.synth.make_agents(cost, cw, cw, n, 40, 0xC0E5, radius=1.0, spacing=2.2)
    rng = np.random.default_rng(0xC0E5)
    st = a["state"].copy(); st[rng.random(n) < 0.2] = STATE_ARRIVED
    a["state"] = st
    a["prev_pos"] = a["pos"].copy()
    a["flock_target"] = a["flock_target"][a["flock_of"]]
    a["flock_of"] = np.arange(n)
    d = a["flock_target"] - a["pos"]
    a["vdes"] = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(F)
    rec, fl = capi.pack_agents(a)
    return cost, rec, fl


def test_windowed_cohesion_keeps_clearpath_counters(pf):
    """the first tick of a context with cohesion mode 1 (windowed, its rows split over blockIdx.y below ~135 k entities)
    must count the same ClearPath events as the member-list pass on the same population, and not zero"""
    cost, rec, fl = _crowd()
    work = np.nonzero(rec["state"] != STATE_ARRIVED)[0].astype(np.uint32)
    got = {}
    for mode in (1, 2):
        nav = pf.capi.Nav(0)
        try:
            nav.map_create(CW, CW, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0)
            nav.set_cohesion_mode(mode)
            nav.agents_upload(rec, fl, 20)
            nav.agents_set_work(work)
            nav.agents_tick(0)
            got[mode] = (nav.clearpath_stats(), nav.agents_read_velocities(len(work)))
        finally:
            nav.set_cohesion_mode(0)
            nav.close()
    assert got[1][0]["no_admissible"] > 0, got
    assert got[1][0] == got[2][0]
    assert (got[1][1] == got[2][1]).all()
