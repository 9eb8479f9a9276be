"""Config C4 (bench.py WORKLOADS["C4"]: the 2048 x 2048-tile map of 32 x 32 chunks, 500 k agents in 8 flocks of 62 500,
8 goals) on one device against the plain-C port and the host / numpy restatements: the map's cost grid and local
islands, the cold goal batch's every field, a 20 000-agent sample of the velocity pass with the whole population as
neighbours (both set_two_phase modes) and its position-index queries, and arrived()'s constants of every flock,
including one whose target lies in a 200 x 200-tile impassable blob (the whole-layer search tier)."""
import hashlib
import importlib
import os
import sys

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
C4_COST_SHA256 = "2ff69223c847e2a2003dc19382b29191e776eb20f500903017aad23567bcbbd3"   # the C4 map's cost grid
CW = 32
FD_STEP = {1: (-1, -1), 2: (-1, 0), 3: (-1, 1), 4: (0, -1), 5: (0, 1), 6: (1, -1), 7: (1, 0), 8: (1, 1)}
COHESION_FLOOR = 1e-6               # DESIGN.md §4 deviation 1: the cohesion floor of cases.vel_ok


@pytest.fixture(scope="module")
def c4(pf):
    bench = importlib.import_module("bench")
    bench.set_workload("C4")
    try:
        W = bench.build_workload(pf, 1, 0)
    finally:
        bench.set_workload("C2")
    assert bench.WORKLOADS["C4"]["chunks"] == CW and W["n_total"] == 500_000 and W["nflocks"] == 8
    return W


def _map(nav, cost):
    nav.map_create(CW, CW, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)


def test_c4_map_pinned(nav, c4):
    assert hashlib.sha256(c4["cost"].tobytes()).hexdigest() == C4_COST_SHA256
    _map(nav, c4["cost"])
    assert np.array_equal(nav.local_islands(0), cases.local_islands_np(c4["cost"]))


def test_c4_cold_goal_batch_vs_port(nav, c4, pforacle):
    """the 8 goals of C4 in one cold pfnav_pool_request_goals: every flow and LOS field equals plan_goal's waves run by
    the port; following the flow from sampled tiles reaches each goal over passable ground"""
    cost = c4["cost"]
    _map(nav, cost)
    targets = np.ascontiguousarray(c4["agents"]["flock_target_tile"], np.int32)
    ng = len(targets)
    nav.pool_create(ng, ng * CW * CW)
    om = pforacle.OracleMap(CW, CW, cost, None, nav.local_islands(0))
    exp = [cases.port_goal_fields(nav, om, t) for t in targets]
    nf, nl = nav.pool_request_goals(np.arange(ng, dtype=np.int32), targets)
    assert nf == sum(e[3] for e in exp) and nl == sum(len(e[1]) for e in exp)
    ncmp = cases.check_goal_pool(nav, exp, CW, CW * CW)
    depth = max(int(cases.los_depths(e[2]).max()) for e in exp)
    print(f"C4 cold goal batch: {ncmp} fields equal the port, longest LOS chain {depth}")
    assert ncmp >= ng * 1000
    img = synth.blocked_to_image(cost, CW, CW)
    passable = np.argwhere(img != 255)
    rng = np.random.default_rng(4)
    arrived = 0
    for d, (flows, _, _, _) in enumerate(exp):
        field = np.zeros(img.shape, np.uint8)
        for c, f in flows.items():
            field[(c // CW) * 64:(c // CW) * 64 + 64, (c % CW) * 64:(c % CW) * 64 + 64] = f
        gr, gc = int(targets[d, 0]) * 64 + int(targets[d, 2]), int(targets[d, 1]) * 64 + int(targets[d, 3])
        for r, c in passable[rng.integers(0, len(passable), 40)]:
            r, c = int(r), int(c)
            if field[r, c] == 0 and (r, c) != (gr, gc):
                continue                               # not connected to the goal
            for _ in range(64 * 2048):
                if (r, c) == (gr, gc):
                    arrived += 1
                    break
                step = FD_STEP[int(field[r, c])]
                r += step[0]; c += step[1]
                assert 0 <= r < img.shape[0] and 0 <= c < img.shape[1] and img[r, c] != 255, (d, r, c)
            else:
                raise AssertionError(("flow did not reach the goal", d))
    assert arrived >= 100, arrived


def _inputs(a, n, seed):
    rng = np.random.default_rng(seed)
    d = a["flock_target"][a["flock_of"]] - a["pos"]
    vdes = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(np.float32)
    aa = dict(a); aa["vdes"] = vdes; aa["has_los"] = (rng.random(n) < 0.2).astype(np.uint32)
    return aa


def _floors(vel, evel, pos):
    """cases.vel_ok, with the uses of each floor counted: -> (ok, # position-ulp floor, # cohesion floor, max rel err)"""
    ok, _ = cases.vel_ok(vel, evel, pos, COHESION_FLOOR)
    d = np.abs(vel - evel).max(axis=1)
    rel = d <= cases.VEL_RTOL * np.maximum(np.abs(evel).max(axis=1), 1e-3)
    apos = np.abs(pos).max(axis=1).astype(np.float32)
    ulp = ~rel & (d <= np.spacing(apos))
    coh = ~rel & ~ulp & (d <= COHESION_FLOOR * apos)
    return ok, int(ulp.sum()), int(coh.sum()), float(cases.relerr(vel, evel).max())


def test_c4_population_sample_vs_port(nav, c4, pforacle):
    """20 000 agents of the 500 k population (flocks of 62 500, positions up to 8 192 wu) through the velocity pass,
    every other agent present as a neighbour, against the port's move_velocity_work: preferred and new velocities within
    cases.vel_ok (1e-4 relative, else the position-ulp floor or the cohesion floor), each floor's uses counted and
    bounded; G_Pos_EntsInCircleFrom's order for 300 of them"""
    a, n = c4["agents"], c4["n_total"]
    rec, fl = capi.pack_agents(_inputs(a, n, 7))
    work = np.sort(np.random.default_rng(7).choice(n, 20_000, replace=False)).astype(np.uint32)
    world = pforacle.OracleWorld(pforacle.OracleMap(CW, CW, c4["cost"]), rec, fl, 20)
    try:
        evel, evpref = world.velocity_work(work)
        nav.map_create(CW, CW, 1); nav.map_upload_layer(0, c4["cost"])
        nav.agents_upload(rec, fl, 20)
        nav.agents_set_work(work)
        pos = a["pos"][work]
        try:
            for mode in (0, 2):
                nav.set_two_phase(mode)
                nav.agents_tick(0)
                vel = nav.agents_read_velocities(len(work))
                vpref, _, _ = nav.agents_read_debug(len(work))
                okp, up, cp, ep = _floors(vpref, evpref, pos)
                okv, uv, cv, ev = _floors(vel, evel, pos)
                print(f"C4 sample, two-phase mode {mode}: vpref max rel {ep:.2e} (ulp floor {up}, cohesion floor {cp}), "
                      f"vel max rel {ev:.2e} (ulp floor {uv}, cohesion floor {cv}) of {len(work)}")
                assert okp and okv, (mode, ep, ev)
                # the floors are rare rounding events, not a blanket over the sample
                assert up + uv <= 10 and cp + cv <= 10, (mode, up, uv, cp, cv)
        finally:
            nav.set_two_phase(1)
        assert (np.linalg.norm(evel, axis=1) == 0).mean() < 0.5 and (np.linalg.norm(evel, axis=1) > 0).mean() > 0.5
        for i in work[:300]:
            x, z = float(a["pos"][i, 0]), float(a["pos"][i, 1])
            for r, cap in ((10.0, 512), (30.0, 128)):
                got, exp = nav.ents_in_circle(x, z, r, cap), world.ents_in_circle(x, z, r, cap)
                assert len(got) == len(exp) and (got == exp).all(), (int(i), r)
    finally:
        world.close()


def _arrival_table_vs_host(nav, fl, flocks):
    """arrived()'s (flock, layer) table of the last compute_updates against route_arrival_consts; every flock of
    `flocks` has a row -> the table"""
    table = nav.agents_read_arrival_consts()
    assert sorted(int(f) for f in np.unique(table["flock"])) == list(flocks)
    for r in table:
        ok, nearest, mc = nav.route_arrival_consts(fl["target"][r["flock"]], int(r["layer"]))
        assert r["nearest_ok"] == ok, (r["flock"], r["layer"])
        if ok:
            assert tuple(r["nearest"]) == tuple(nearest), (r["flock"], r["nearest"], nearest)
        assert r["mc_n"] == len(mc) and (r["mc"][:len(mc)] == mc).all(), (r["flock"], r["mc_n"], len(mc))
    return table


def test_c4_arrival_consts(nav, c4):
    """arrived()'s constants of the 8 flocks on C4's own map after upload and one compute_updates
    (pfnav_agents_read_arrival_consts) against the host routine route_arrival_consts. Then the same on the C4 map with a
    200 x 200-tile impassable blob cut into it and a ninth flock aiming at the blob's centre, 100 tiles from the nearest
    pathable tile: its nearest tile comes from the whole-layer tier."""
    a, n = c4["agents"], c4["n_total"]
    ms = np.zeros(n, capi.MOVESTATE)
    ms["next_pos"][:, 0] = a["pos"][:, 0]; ms["next_pos"][:, 2] = a["pos"][:, 1]
    ms["step"] = 1.0
    ms["next_rot"] = cases.dir_quat(a["vel"] + 1e-6)
    ms["combat_facing"] = ms["next_rot"]
    rng = np.random.default_rng(8)
    movers = rng.choice(n, 16, replace=False)
    work = np.unique(np.concatenate([rng.choice(n, 4000, replace=False), movers])).astype(np.uint32)

    def tick(cost, aa, flocks):
        rec, fl = capi.pack_agents(aa)
        _map(nav, cost)
        nav.agents_upload(rec, fl, 20)
        nav.agents_upload_movestate(ms)
        nav.agents_set_work(work)
        nav.agents_tick(0)
        nav.agents_compute_updates()
        return _arrival_table_vs_host(nav, fl, flocks)

    table = tick(c4["cost"], _inputs(a, n, 8), range(8))
    print(f"C4 arrival constants on the C4 map: {len(table)} (flock, layer) rows equal the host routine")
    img = synth.blocked_to_image(c4["cost"], CW, CW).copy()
    img[1700:1900, 100:300] = 0xFF
    aa = _inputs(a, n, 8)
    aa["flock_of"] = a["flock_of"].copy(); aa["flock_of"][movers] = 8
    aa["flock_target"] = np.concatenate([a["flock_target"], [synth.tile_center_xz(1800 // 64, 200 // 64, 1800 % 64, 200 % 64)]]).astype(np.float32)
    aa["flock_dest_index"] = np.concatenate([a["flock_dest_index"], [0]]).astype(np.int32)
    table = tick(synth.image_to_blocked(img, CW, CW), aa, range(9))
    blob = table[table["flock"] == 8][0]
    assert blob["nearest_ok"]
    print(f"C4 map with the blob: {len(table)} (flock, layer) rows equal the host routine; blob flock's nearest "
          f"{tuple(float(v) for v in blob['nearest'])}")


def test_c4_group_of_two_equals_one_context(c4):
    """a group of 2 members on one device at C4 against single contexts: the 8-goal group batch
    (pfnav_group_request_goals_ex) leaves every member's pool entries (has bits, ff_id, flow and LOS bytes) equal to a
    single context's that ran the same batch alone, each goal's fields built on one member (test_gpu_mgpu_fields.Twins).
    Then one tick of the whole population with desired velocities read from the pool, the population split between the
    members and gathered: every member's velocities, desired velocities and LOS bits equal the single context's bit for
    bit."""
    import test_gpu_mgpu_fields as mf
    W = c4
    n, world = W["n_total"], 2
    targets = np.ascontiguousarray(W["agents"]["flock_target_tile"], np.int32)
    ng = len(targets)
    T = mf.Twins(W["cost"], CW, ng, ng * CW * CW, world)
    try:
        owner, per = T.job(np.arange(ng, dtype=np.int32), targets)
        one = T.solo[0]
        one.agents_upload(W["rec"], W["flocks"], 20)
        ranges = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
        for nv, (lo, hi) in zip(T.navs, ranges):
            nv.agents_upload_shard(W["rec"][lo:hi], lo, hi, n, W["flocks"], 20)
        T.grp.gather()
        work = np.arange(n, dtype=np.uint32)
        one.agents_set_work(work)
        one.agents_tick(capi.TICK_VDES_FROM_POOL)
        v1 = one.agents_read_velocities(n)
        _, vdes1, los1 = one.agents_read_debug(n)
        for nv, (lo, hi) in zip(T.navs, ranges):
            nv.agents_set_work(work[lo:hi])
            nv.agents_tick(capi.TICK_VDES_FROM_POOL)
        for r, (nv, (lo, hi)) in enumerate(zip(T.navs, ranges)):
            v = nv.agents_read_velocities(hi - lo)
            _, vdes, los = nv.agents_read_debug(hi - lo)
            assert np.array_equal(vdes.view(np.uint32), vdes1[lo:hi].view(np.uint32)), r
            assert np.array_equal(los, los1[lo:hi]), r
            assert np.array_equal(v.view(np.uint32), v1[lo:hi].view(np.uint32)), (r, np.nonzero((v != v1[lo:hi]).any(axis=1))[0][:10])
        assert (np.abs(vdes1).sum(axis=1) > 0).mean() > 0.9
        print(f"C4 group of {world}: {world * ng * CW * CW} pool entries and {n} velocities equal one context's "
              f"(goal owners {owner.tolist()})")
    finally:
        T.close()
