"""GPU suite at BASELINE.json sizes against the COMPILED REFERENCE (oracle/_ref/libpfref.so) where it is built; without
it each test says what it compares with instead (the plain-C port and the host / numpy restatements):
seeded >= 10k-agent samples of the bench's own C2 / C3 populations with the whole population present as neighbours,
route fields and desired velocities out of the field pool incl. the on-miss chain on the 1024 x 1024 map, 1 k dynamic
obstacles (config C5's churn) and multi-tick device-resident trajectories at 20, 10, 5 and 1 Hz. Every comparison is
an asserted maximum: integers
bit-exact, velocities within north_star's 1e-4 relative for EVERY agent."""
import hashlib
import importlib
import os
import sys

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
VEL_RTOL = 1e-4
C2_COST_SHA256 = "4d0c09dd826a03b55a8899fcd09fcd23bd075ff14573d645aa5c4654758ed304"   # the C2 / C3 map's cost grid
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


@pytest.fixture(scope="module")
def bench():
    return importlib.import_module("bench")


@pytest.fixture(scope="module")
def c2map(pf, pfref_or_golden, bench):
    """the bench's 16 x 16-chunk map in the reference (N_NewCtxForMapData: ~30 s, 2 GB) -- shared by the tests below;
    None in place of the reference when it is not built (the tests then compare with the plain-C port)"""
    bench.set_workload("C2")
    p = synth.make_map(bench.CHUNKS, bench.CHUNKS, bench.MAP_SEED)
    ref = pfref_or_golden.RefMap(bench.CHUNKS, bench.CHUNKS, p) if pfref_or_golden else None
    yield p, ref
    if ref is not None:
        ref.close()


def _population(pf, bench, workload):
    bench.set_workload(workload)
    W = bench.build_workload(pf, 1, 0)
    bench.set_workload("C2")
    return W


@pytest.mark.parametrize("workload", ["C2", "C3"])
def test_bench_population_sample_vs_reference(pf, nav, pforacle, c2map, bench, workload):
    """10 000 seeded agents of the bench population (100 k agents k10 ~ 21 / 1 M agents k10 ~ 39; every other agent is
    present as a neighbour): position-index query order (G_Pos_EntsInCircleFrom), preferred velocity and new velocity
    of move_velocity_work (movement.c:3395-3466) -- single-pass and two-phase kernels. Without the compiled reference the
    expectations come from the plain-C port (oracle/pf_oracle.c, pinned to the reference by tests/test_oracle.py)."""
    p, ref = c2map
    W = _population(pf, bench, workload)
    a, n = W["agents"], W["n_total"]
    if ref is not None:
        assert (ref.cost_base() == W["cost"]).all()
    else:       # the bench map's cost grid (compared with the reference's N_NewCtxForMapData cost where that is built)
        assert hashlib.sha256(W["cost"].tobytes()).hexdigest() == C2_COST_SHA256
    rng = np.random.default_rng(7)
    nsample = 10_000
    work = np.sort(rng.choice(n, nsample, replace=False)).astype(np.uint32)
    d = a["flock_target"][a["flock_of"]] - a["pos"]
    vdes_all = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(np.float32)
    los_all = (rng.random(n) < 0.2).astype(np.uint8)
    aa = dict(a); aa["vdes"] = vdes_all; aa["has_los"] = los_all.astype(np.uint32)
    rec, fl = capi.pack_agents(aa)
    if ref is not None:
        ref.agents_set(a["pos"], a["prev_pos"], a["vel"], a["radius"], a["max_speed"], a["state"], a["flags"],
                       a["flock_of"], a["flock_target"], np.arange(W["nflocks"], dtype=np.uint32), hz=20)
        ref.work_set(work, vdes_all[work], los_all[work], a["speed"][work])
        evel, _ = ref.velocity_work(os.cpu_count())
        evpref = ref.vpref()
        ents_in_circle = ref.ents_in_circle
    else:
        world = pforacle.OracleWorld(pforacle.OracleMap(bench.CHUNKS, bench.CHUNKS, W["cost"]), rec, fl, 20)
        evel, evpref = world.velocity_work(work)
        ents_in_circle = world.ents_in_circle
    nav.map_create(bench.CHUNKS, bench.CHUNKS, 1); nav.map_upload_layer(0, W["cost"])
    nav.agents_upload(rec, fl, 20)
    nav.agents_set_work(work)
    try:
        for mode in (0, 2):
            nav.set_two_phase(mode)
            nav.agents_tick(0)
            vel = nav.agents_read_velocities(nsample)
            vpref, _, _ = nav.agents_read_debug(nsample)
            e_vp, e_v = cases.relerr(vpref, evpref), cases.relerr(vel, evel)
            assert e_vp.max() <= VEL_RTOL, (workload, mode, e_vp.max(), work[np.nonzero(e_vp > VEL_RTOL)[0][:8]])
            assert e_v.max() <= VEL_RTOL, (workload, mode, e_v.max(), work[np.nonzero(e_v > VEL_RTOL)[0][:8]])
    finally:
        nav.set_two_phase(1)
    # the sample is representative of the hard cases: capped neighbour lists and agents without an admissible velocity
    assert (np.linalg.norm(evel, axis=1) == 0).mean() > 0.02
    for i in work[:300]:
        x, z = float(a["pos"][i, 0]), float(a["pos"][i, 1])
        for r, cap in ((10.0, 512), (30.0, 128)):
            got, exp = nav.ents_in_circle(x, z, r, cap), ents_in_circle(x, z, r, cap)
            assert len(got) == len(exp) and (got == exp).all(), (workload, int(i), r)
    if ref is None:
        world.close()


def test_windowed_cohesion_equals_member_list(pf, nav, bench):
    """cohesion_force through the position index with the exp(-0.12 d) cut-off (+ per-entity fall-back) against the plain
    sum over the flock's member list, on the bench's C2 population and on a C4-style flock of 60 000: preferred velocities
    agree to float rounding, far inside the 1e-4 budget"""
    for workload, nsel in (("C2", 20_000), ("C4", 20_000)):
        bench.set_workload(workload)
        try:
            W = bench.build_workload(pf, 1, 0) if workload == "C2" else None
            if W is None:
                # one C4 cell: 60 000 agents of radius 1.0 in one flock on an 8 x 8-chunk map
                p = synth.make_map(8, 8, 0x5EED0004)
                cost = synth.cost_from_pathable(p, 8, 8)
                a = synth.make_agents(cost, 8, 8, 60_000, 1, 0x5EED0004, radius=1.0, spacing=3.9)
                W = dict(cost=cost, agents=a, n_total=60_000, chunks=8)
            else:
                W["chunks"] = bench.CHUNKS
        finally:
            bench.set_workload("C2")
        a, n, cw = W["agents"], W["n_total"], W["chunks"]
        d = a["flock_target"][a["flock_of"]] - a["pos"]
        aa = dict(a); aa["vdes"] = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(np.float32)
        rec, fl = capi.pack_agents(aa)
        nav.map_create(cw, cw, 1); nav.map_upload_layer(0, W["cost"])
        nav.agents_upload(rec, fl, 20)
        work = np.sort(np.random.default_rng(3).choice(n, nsel, replace=False)).astype(np.uint32)
        nav.agents_set_work(work)
        out = {}
        try:
            for mode in (2, 1):
                nav.set_cohesion_mode(mode)
                nav.agents_tick(0)
                out[mode] = (nav.agents_read_debug(nsel)[0], nav.agents_read_velocities(nsel))
        finally:
            nav.set_cohesion_mode(0)
        e_vp = cases.relerr(out[1][0], out[2][0]); e_v = cases.relerr(out[1][1], out[2][1])
        assert e_vp.max() <= 2e-5, (workload, e_vp.max())
        assert e_v.max() <= VEL_RTOL, (workload, e_v.max())


def _pack_route_fields(entries):
    """(flow or None, ffid, los or None) per chunk -> has bits, ffids, the present flow and LOS fields"""
    has = np.array([(fl is not None) | ((lo is not None) << 1) for fl, _, lo in entries], np.uint8)
    ffid = np.array([ffid if fl is not None else 0 for fl, ffid, _ in entries], np.uint64)
    flows = np.array([fl for fl, _, _ in entries if fl is not None], np.uint8).reshape(-1, 64, 64)
    loss = np.array([lo for _, _, lo in entries if lo is not None], np.uint8).reshape(-1, 64, 64)
    return has, ffid, flows, loss


def test_c2_desired_velocity_from_pool_vs_reference(pf, nav, pforacle, c2map, bench):
    """A2 at full size: N_RequestPath for four flocks of the C2 population on the 1024 x 1024 map (routes of up to ~20
    hops): every route's flow and LOS fields in the pool byte for byte. Then, once the on-miss chain has settled,
    N_HasDestLOS + N_DesiredPointSeekVelocity for 2 000 of their agents (compute_los_state / compute_desired_velocity,
    movement.c:4129-4180) bit-exact and the velocity pass on top within 1e-4. Without the compiled reference the
    expectations come from the plain-C port (oracle/pf_oracle.c, pinned to the reference by tests/test_oracle.py): the
    route's requests from the host planner (route_request_path) executed by the port, desired velocities and LOS by the
    port over the pool's fields read back, velocities by the port's velocity pass with the whole population as
    neighbours. Fields that the on-miss chain adds are then consumed identically by both sides; their contents are
    covered by test_pool_repair_chain_golden."""
    p, ref = c2map
    W = _population(pf, bench, "C2")
    a, n = W["agents"], W["n_total"]
    flocks = [0, 5, 9, 14]
    rng = np.random.default_rng(11)
    work = np.sort(np.concatenate([rng.choice(np.nonzero(a["flock_of"] == f)[0], 500, replace=False) for f in flocks])).astype(np.uint32)
    dest_ids = np.zeros(W["nflocks"], np.uint32)
    nav.map_create(bench.CHUNKS, bench.CHUNKS, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0); nav.route_build(0)
    nav.pool_create(len(flocks), 2048)
    dest_index = np.full(W["nflocks"], -1, np.int32)
    nchunks = bench.CHUNKS ** 2
    om = None
    if ref is None:
        liid = cases.local_islands_np(W["cost"])
        assert (nav.local_islands(0) == liid).all()
        om = pforacle.OracleMap(bench.CHUNKS, bench.CHUNKS, W["cost"], None, liid)
    for k, f in enumerate(flocks):
        src = a["pos"][a["flock_of"] == f].mean(axis=0)
        src = a["pos"][a["flock_of"] == f][np.argmin(np.linalg.norm(a["pos"][a["flock_of"] == f] - src, axis=1))]
        src, dst = (float(src[0]), float(src[1])), (float(a["flock_target"][f][0]), float(a["flock_target"][f][1]))
        if ref is not None:
            ok_r, did_r = ref.request_path(src, dst)
            ok_r, did_r = bool(ok_r), int(did_r)
            expected = [tuple(ref.fc_flow(did_r, divmod(c, bench.CHUNKS))) + (ref.fc_los(did_r, divmod(c, bench.CHUNKS)),)
                        for c in range(nchunks)]
        else:
            # the same route's requests (the pool's dest k is still empty: nothing is skipped) run by the port in order
            ok_r, did_r, fr, fid, fc, lr, lc = nav.route_request_path(src, dst)
            fields, los = cases.execute_route(lambda r, io: om.flow_fields_update(r, inout=io), om.los_fields_create, fr, fc, lr, lc)
            last_id = {int(fc[i]): int(fid[i]) for i in range(len(fr))}
            expected = [(fields.get(c), last_id.get(c, 0), los.get(c)) for c in range(nchunks)]
        ok, did, nf, nl = nav.pool_request_path(k, src, dst)
        assert ok == ok_r and (not ok or did == did_r), f
        dest_ids[f] = did_r
        dest_index[f] = k
        # the route's field set equals the expected one, byte for byte
        g_has, g_ffid, g_flows, g_los = _pack_route_fields([(fl, ffid, lo) for fl, lo, ffid in
                                                            (nav.pool_get(k, divmod(c, bench.CHUNKS)) for c in range(nchunks))])
        e_has, e_ffid, e_flows, e_los = _pack_route_fields(expected)
        bad = np.nonzero(g_has != e_has)[0]
        assert len(bad) == 0, (f, bad[:10])
        assert (g_ffid == e_ffid).all(), (f, np.nonzero(g_ffid != e_ffid)[0][:10])
        assert (g_flows == e_flows).all() and (g_los == e_los).all(), f
    if ref is not None:
        ref.agents_set(a["pos"], a["prev_pos"], a["vel"], a["radius"], a["max_speed"], a["state"], a["flags"],
                       a["flock_of"], a["flock_target"], dest_ids, hz=20)
        ref.work_set(work, np.zeros((len(work), 2), np.float32), np.zeros(len(work), np.uint8), a["speed"][work])
        # The reference serves misses inline, entity by entity, so within the tick that fills the cache an entity can read a
        # field before a later entity's request merges another portal into it; from the next tick on every entity reads the
        # settled fields. The comparison is against that steady state (second pass), which is what the device pool converges to.
        ref.desired_from_cache()
        evdes, elos = ref.desired_from_cache()
        evel, _ = ref.velocity_work(os.cpu_count())
    aa = dict(a); aa["flock_dest_index"] = dest_index
    rec, fl = capi.pack_agents(aa)
    nav.agents_upload(rec, fl, 20)
    nav.agents_set_work(work)
    cases.settle_pool(nav)
    vel = nav.agents_read_velocities(len(work))
    _, vdes, los = nav.agents_read_debug(len(work))
    if ref is None:
        evdes, elos = om.desired_velocity(rec, fl, work, *cases.pool_fields(nav, len(flocks), nchunks))
        seeded = rec.copy(); seeded["vdes"][work] = evdes; seeded["has_dest_los"][work] = elos
        world = pforacle.OracleWorld(om, seeded, fl, 20)
        evel, _ = world.velocity_work(work)
        world.close()
    assert (los == elos).all(), np.nonzero(los != elos)[0][:10]
    bad = np.nonzero((vdes != evdes).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), work[bad[:10]], vdes[bad[:3]], evdes[bad[:3]])
    assert (np.abs(evdes).sum(axis=1) > 0).mean() > 0.95
    assert cases.relerr(vel, evel).max() <= VEL_RTOL


def test_c5_churn_vs_reference(pf, nav, pforacle, c2map, bench):
    """config C5's dynamic-obstacle churn on the 1024 x 1024 map: 1 000 circular blockers placed, then every one moved
    by one tile (N_BlockersDecref + N_BlockersIncref) over three ticks with N_Update in between: blocker refcounts and
    local islands of all 256 chunks bit-exact after every commit; then flow (tile + portal) and chained LOS fields of
    dirtied chunks, and the velocity pass of 3 000 agents standing among the blockers. Without the compiled reference:
    refcounts from the host restatement (a host-only context, pinned to the reference by tests/test_oracle.py), islands
    from the numpy restatement, fields and velocities from the plain-C port (oracle/pf_oracle.c)."""
    p, ref = c2map
    W = _population(pf, bench, "C2")
    a, n = W["agents"], W["n_total"]
    cw = bench.CHUNKS
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0); nav.route_build(0)
    host = None
    if ref is None:
        host = capi.Nav(hostonly=True)
        host.map_create(cw, cw, 1); host.map_upload_layer(0, W["cost"]); host.map_build_nav(0); host.route_build(0)
    rng = np.random.default_rng(55)
    # blockers of radius 6 near the agents of four flocks (so that the tile probes of the steering see them) + anywhere
    near = a["pos"][rng.choice(np.nonzero(np.isin(a["flock_of"], [1, 4, 7, 12]))[0], 600, replace=False)] + rng.normal(scale=25.0, size=(600, 2))
    far = np.stack([-rng.uniform(20, cw * 256 - 20, 400), rng.uniform(20, cw * 256 - 20, 400)], 1)
    bpos = np.concatenate([near, far]).astype(np.float32)
    bpos[:, 0] = np.clip(bpos[:, 0], -(cw * 256 - 20), -20); bpos[:, 1] = np.clip(bpos[:, 1], 20, cw * 256 - 20)
    placed = []

    def blockers(delta, x, z):
        if ref is not None:
            (ref.blockers_incref if delta > 0 else ref.blockers_decref)(x, z, 6.0)
        for nv in (nav, host) if host is not None else (nav,):
            (nv.blockers_incref if delta > 0 else nv.blockers_decref)(x, z, 6.0, 0, capi.FLAG_MOVABLE)

    def commit():
        if ref is not None:
            ref.update()
        else:
            host.map_commit()
        return nav.map_commit()

    def expected_grids():
        if ref is not None:
            return ref.blockers(), ref.local_islands()
        blk = host.blockers(0)
        return blk, cases.local_islands_np(W["cost"], blk)
    try:
        for x, z in bpos:
            blockers(+1, float(x), float(z))
            placed.append((float(x), float(z)))
        for tick in range(3):
            nd = commit()
            eblk, eliid = expected_grids()
            assert (nav.blockers(0) == eblk).all(), tick
            assert (nav.local_islands(0) == eliid).all(), tick
            assert nd > 0
            step = rng.integers(-1, 2, size=(len(placed), 2)).astype(np.float32) * 4.0
            for k, (x, z) in enumerate(placed):
                nx = float(np.clip(x + step[k, 0], -(cw * 256 - 20), -20)); nz = float(np.clip(z + step[k, 1], 20, cw * 256 - 20))
                blockers(-1, x, z); blockers(+1, nx, nz)
                placed[k] = (nx, nz)
        commit()
        blk, liid = expected_grids()
        assert (nav.blockers(0) == blk).all() and (nav.local_islands(0) == liid).all()
        # fields of chunks that hold blockers: tile targets, portal targets, chained LOS
        dirty = np.nonzero(blk.reshape(cw * cw, -1).any(axis=1))[0]
        assert len(dirty) >= 100
        ports = ref.portals() if ref is not None else nav.portals(0)
        om = pforacle.OracleMap(cw, cw, W["cost"], blk, liid)
        reqs, exp = [], []
        for c in dirty[:48]:
            free = np.argwhere((W["cost"][c] != 255) & (blk[c] == 0))
            t = free[rng.integers(len(free))]
            reqs.append(capi.tile_req((c // cw, c % cw), (int(t[0]), int(t[1]))))
            if ref is not None:
                exp.append(ref.flow_tile((c // cw, c % cw), (int(t[0]), int(t[1]))))
        specs = [s_ for s_ in cases.portal_specs(ports, liid, cw) if (s_[0][0] * cw + s_[0][1]) in set(dirty[:24].tolist())][:64]
        for s_ in specs:
            reqs.append(cases.portal_reqs([s_]))
            if ref is not None:
                exp.append(ref.flow_portal(s_[0], s_[1], s_[5], s_[6]))
        reqs = np.concatenate(reqs)
        exp = np.stack(exp) if ref is not None else om.flow_fields_update(reqs)
        got = nav.flow_fields_update(reqs)
        assert (got == exp).all(), np.nonzero((got != exp).reshape(len(exp), -1).any(axis=1))[0][:10]
        eff = np.where(blk > 0, 255, W["cost"]).astype(np.uint8)
        lr = cases.los_case(eff, cw, cw, 77, ntargets=6)
        assert (nav.los_fields_create(lr) == (cases.ref_los_batch(ref, lr) if ref is not None else om.los_fields_create(lr))).all()
        # velocity pass among the blockers (nullify_impass_components reads the blocked tiles, movement.c:1831)
        work = np.sort(rng.choice(np.nonzero(np.isin(a["flock_of"], [1, 4, 7, 12]))[0], 3000, replace=False)).astype(np.uint32)
        d = a["flock_target"][a["flock_of"]] - a["pos"]
        vdes_all = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(np.float32)
        aa = dict(a); aa["vdes"] = vdes_all
        rec, fl = capi.pack_agents(aa)
        if ref is not None:
            ref.agents_set(a["pos"], a["prev_pos"], a["vel"], a["radius"], a["max_speed"], a["state"], a["flags"],
                           a["flock_of"], a["flock_target"], np.arange(W["nflocks"], dtype=np.uint32), hz=20)
            ref.work_set(work, vdes_all[work], np.zeros(len(work), np.uint8), a["speed"][work])
            evel, _ = ref.velocity_work(os.cpu_count())
            evpref = ref.vpref()
        else:
            world = pforacle.OracleWorld(om, rec, fl, 20)
            evel, evpref = world.velocity_work(work)
            world.close()
        nav.agents_upload(rec, fl, 20); nav.agents_set_work(work); nav.agents_tick(0)
        vel = nav.agents_read_velocities(len(work)); vpref, _, _ = nav.agents_read_debug(len(work))
        assert cases.relerr(vpref, evpref).max() <= VEL_RTOL and cases.relerr(vel, evel).max() <= VEL_RTOL
        # the steering did see blocked tiles
        assert (np.abs(vpref - (a["vel"][work] + 0)).sum() > 0)
    finally:
        if ref is not None:
            for x, z in placed:                           # leave the shared reference map as it was
                ref.blockers_decref(x, z, 6.0)
            ref.update()
        if host is not None:
            host.close()


@pytest.mark.parametrize("hz", [20, 10, 5, 1])
def test_device_resident_trajectory_vs_reference(pf, nav, pforacle, pfref_or_golden, hz):
    """SURVEY 8f-3: positions never leave the device between ticks. Eight ticks of a marching crowd (1 500 agents, three
    flocks, 3 x 3 chunks, goals far away: pure motion, heading gate, interpolation below 20 Hz) and one tick of an
    arriving crowd (arrivals, adjacent-arrived cascade, WAITING, interpolations left unfinished, blockers taken by the
    stopped entities and the N_Update that follows), at each of the four tick rates (movement.c:2210): against the
    reference's own entity_compute_update / entity_apply_update (movement.c:2303-2766) where it is built, else against
    the plain-C port (oracle/pf_oracle.c) re-seeded with the device's state every tick (cases.run_trajectory). At 1 Hz an
    agent moves up to 20 wu per tick: across index cells, tiles and chunk borders."""
    cw = 3
    # marching crowd
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
        out = cases.run_trajectory(nav, ref, pforacle, a, ms, cw, cost, hz, 8, with_blockers=True, follow=True)
        assert len(out) == 8 and out[-1][0] > 1000, out
    finally:
        if ref is not None:
            ref.close()
    # arriving crowd: one tick on a settled cache -- arrivals, adjacent-arrived cascade, WAITING, then the engine's share of the
    # apply on our side (entity_block -> N_BlockersIncref for every stopped entity) and the N_Update that follows:
    # identical states, positions, blocker refcounts and local islands. (Later ticks of this scenario re-request half the
    # fields through the on-miss chain while the reference is still walking its entities; those transients depend on the
    # reference's serial order, see test_c2_desired_velocity_from_pool_vs_reference.)
    p, cost, a, ms = cases.update_case(4242, hz)
    ref = pfref_or_golden.RefMap(cw, cw, p) if pfref_or_golden else None
    try:
        out = cases.run_trajectory(nav, ref, pforacle, a, ms, cw, cost, hz, 1, with_blockers=True)
        assert len(out) == 1 and out[0][0] > 1000, out
    finally:
        if ref is not None:
            ref.close()
