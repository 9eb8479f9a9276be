"""CPU suite (-m "not gpu"): the oracle port against the committed golden vectors (generated from the
compiled reference by tests/golden/make_golden.py), against the compiled reference itself when it is
available, plus host-side logic and the C-ABI surface (no compute calls: there is no GPU here)."""
import ctypes
import os
import re

import numpy as np
import pytest

import cases

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
capi, synth = cases.capi, cases.synth


def gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


# ---------------------------------------------------------------- oracle port vs golden vectors
def test_port_flow_tile_golden(pforacle):
    g = gold("flow_tile")
    for k in range(3):
        om = pforacle.OracleMap(1, 1, g[f"cost{k}"])
        reqs = g[f"reqs{k}"].view(capi.FIELD_REQ)
        got = om.flow_fields_update(reqs)
        assert (got == g[f"exp{k}"]).all()
        # empty frontier (impassable target) leaves the initialised field untouched: all FD_NONE
        if (g[f"cost{k}"][0][reqs[-1]["tile_r"], reqs[-1]["tile_c"]] == 255):
            assert (got[-1] == 0).all()


def test_port_flow_portal_and_merge_golden(pforacle):
    g = gold("portal_los")
    om = pforacle.OracleMap(3, 3, g["cost"], None, g["liid"])
    reqs = g["reqs"].view(capi.FIELD_REQ)
    assert (om.flow_fields_update(reqs) == g["exp"]).all()
    q = reqs[:1].copy(); q["init"] = 0
    assert (om.flow_fields_update(q, inout=g["merge_base"][None])[0] == g["merge_exp"]).all()


def test_port_los_golden(pforacle):
    g = gold("portal_los")
    om = pforacle.OracleMap(3, 3, g["cost"])
    got = om.los_fields_create(g["los_reqs"].view(capi.LOS_REQ))
    assert (got == g["los_exp"]).all()


def _port_repair(pforacle, om, gisl, T, K, A, B):
    out = []
    for i in range(len(K)):
        q = T[i:i + 1]
        if K[i] == 0:
            out.append(om.flow_nearest_pathable((int(q["chunk_r"][0]), int(q["chunk_c"][0])), (int(A[i]) >> 8, int(A[i]) & 255), B[i]))
        else:
            out.append(om.flow_island_to_nearest(gisl, q, int(A[i]), B[i]))
    return np.stack(out)


def test_port_repair_chain_golden(pforacle):
    """N_FlowFieldUpdateToNearestPathable / N_FlowFieldUpdateIslandToNearest (field.c:2247, 2307)"""
    g = gold("repair")
    om = pforacle.OracleMap(2, 2, g["cost"], g["blk"], g["liid"])
    T = g["targets"].view(capi.FIELD_REQ)
    got = _port_repair(pforacle, om, g["islands"], T, g["kinds"], g["args"], g["base"])
    assert (got == g["exp"]).all()
    assert (g["base"] != g["exp"]).any()


def test_port_repair_chain_vs_ref(pfref, pforacle):
    p = cases.noise_map(3, 2, 91, 0.25)
    ref = pfref.RefMap(3, 2, p)
    rng = np.random.default_rng(17)
    for _ in range(70):
        ref.blockers_incref(float(-rng.uniform(10, 3 * 256 - 10)), float(rng.uniform(10, 2 * 256 - 10)),
                            float(rng.uniform(2, 16)), 0, 0)
    ref.update()
    T, K, A, B, E = cases.repair_case(ref, 3, 2, 23, per_chunk=3)
    om = pforacle.OracleMap(3, 2, ref.cost_base(), ref.blockers(), ref.local_islands())
    got = _port_repair(pforacle, om, ref.islands(), T, K, A, B)
    assert (got == E).all()
    ref.close()


def test_repair_chain_sequence_golden(pforacle):
    """the SEQUENCE of the on-miss chain (nav.c:3484-3554) as pfnav_pool_repair runs it -- misses in work order, one
    representative per (chunk, local island | blocked tile), path request from its position, repair only when that
    request succeeded and the tile is still FD_NONE -- executed here with the host planner + the oracle port in
    place of the kernels, against the reference's steady-state desired velocities."""
    g = gold("repair_pool")
    cw = ch = 2
    pos, target, liid = g["pos"], g["target"], g["liid"]
    n = len(pos)
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, g["cost"], g["blk"], liid); nav.map_build_nav(0); nav.route_build(0)
    gisl = nav.route_islands(0)
    om = pforacle.OracleMap(cw, ch, g["cost"], g["blk"], liid)
    flow, last, ffid = {}, {}, np.zeros(cw * ch, np.uint64)

    def tile_of(p):
        ar, ac = min(int(abs(p[1]) / 4), ch * 64 - 1), min(int(abs(p[0]) / 4), cw * 64 - 1)
        return (ar >> 6) * cw + (ac >> 6), ar & 63, ac & 63

    def request(src):
        ok, did, fr, fid, fc, lr, lc = nav.route_request_path((float(src[0]), float(src[1])), (float(target[0]), float(target[1])),
                                                              0, ffid.copy(), np.ones(cw * ch, np.uint8))
        for k in range(len(fr)):
            c = int(fc[k])
            flow[c] = om.flow_fields_update(fr[k:k + 1], None if fr[k]["init"] else flow[c][None])[0]
            ffid[c] = fid[k]; last[c] = fr[k:k + 1].copy()
        return ok, len(fr)

    assert request(pos[0])[0]
    for _ in range(4):
        reps, seen = [], set()
        for i in range(n):
            c, r, cc = tile_of(pos[i])
            if c in flow and flow[c][r, cc] != 0:
                continue
            li = int(liid[c][r, cc])
            key = (c, ("t", r, cc) if li == 0xFFFF else li)
            if key not in seen:
                seen.add(key); reps.append((i, c, r, cc, li))
        done = 0
        oks = {}
        for i, c, r, cc, li in reps:
            oks[i], nf = request(pos[i]); done += nf > 0
        for i, c, r, cc, li in reps:
            if not oks[i] or c not in flow or flow[c][r, cc] != 0:
                continue
            flow[c] = om.flow_nearest_pathable((c // cw, c % cw), (r, cc), flow[c]) if li == 0xFFFF \
                else om.flow_island_to_nearest(gisl, last[c], li, flow[c])
            done += 1
        if not done:
            break
    rec = np.zeros(n, capi.AGENT); rec["pos"] = pos; rec["prev_pos"] = pos; rec["flock"] = 0
    fl = np.zeros(1, capi.FLOCK); fl["target"] = target; fl["dest"] = 0
    slot = np.full((1, cw * ch), -1, np.int32); F = np.zeros((cw * ch, 64, 64), np.uint8)
    for k, c in enumerate(sorted(flow)):
        slot[0, c] = k; F[k] = flow[c]
    vd, _ = om.desired_velocity(rec, fl, np.arange(n, dtype=np.uint32), slot, F, np.zeros_like(F))
    assert (vd == g["vdes"]).all()
    nav.close()


def test_port_faction_fields_golden(pforacle):
    """attacking requests: field_tile_passable_no_enemies (field.c:179) in flow (tile, portal) and LOS fields"""
    g = gold("faction")
    om = pforacle.OracleMap(2, 2, g["cost"], g["blk"], g["liid"], factions=g["factions"], enemies=g["enemies"])
    assert (om.flow_fields_update(g["treq"].view(capi.FIELD_REQ)) == g["texp"]).all()
    assert (om.flow_fields_update(g["preq"].view(capi.FIELD_REQ)) == g["pexp"]).all()
    assert (om.los_fields_create(g["lreq"].view(capi.LOS_REQ)) == g["lexp"]).all()


@pytest.mark.parametrize("dim", [96, 32])
def test_port_region_fields_golden(pforacle, dim):
    """cell arrival fields (+ fix-up) and group arrival fields vs the compiled reference's output (region.npz):
    regions over every map edge, the aliasing flood (rows < columns), the base shift, overlays, enemy masks"""
    g = gold("region")
    om = pforacle.OracleMap(3, 3, g["cost"], g["blk"], None, factions=g["factions"])
    reqs = cases.region_reqs_from_golden(g["req%d" % dim], g["ov%d" % dim])
    for i, q in enumerate(reqs):
        f = om.region_field_create(dim, q["enemies"], 1, [q["target"]], q["center"], q["overlay"])
        assert (f == g["create%d" % dim][i]).all(), i
        if q["start"] is not None:
            f = om.region_field_fixup(dim, q["start"], q["center"], f, q["overlay"])
        assert (f == g["exp%d" % dim][i]).all(), i
    for k in range(len(g["gx%d" % dim])):
        f = om.group_arrival_field(dim, int(g["ge%d" % dim][k]), g["gt%d" % dim][k], g["gc%d" % dim][k])
        assert (f == g["gx%d" % dim][k]).all(), k


def test_port_region_fields_vs_ref(pfref, pforacle):
    cw = ch = 2
    p, blockers, wars, reqs = cases.region_case(77, cw, ch, 32, 96)
    ref = pfref.RefMap(cw, ch, p)
    for a, b in wars:
        ref.set_war(a, b)
    for b in blockers:
        ref.blockers_incref(b[0], b[1], b[2], b[3], 0)
    ref.update()
    cost, blk, fac = ref.cost_base(), ref.blockers(), ref.factions()
    cases.region_pick_starts(reqs, cost, blk, cw, ch, 77, 96)
    om = pforacle.OracleMap(cw, ch, cost, blk, None, factions=fac)
    for q in reqs:
        e = ref.cell_arrival_field(96, q["target"], q["center"], q["enemies"], q["overlay"], q["start"])
        f = om.region_field_create(96, q["enemies"], 1, [q["target"]], q["center"], q["overlay"])
        if q["start"] is not None:
            f = om.region_field_fixup(96, q["start"], q["center"], f, q["overlay"])
        assert (e == f).all(), q
    ref.close()


def _zone_chunks(centre_xz, radius, cw, ch):
    """N_RequestAsyncGroupArrivalField's chunk selection (nav.c:3945-3951) for a map at the origin"""
    ct_r = min(int(abs(centre_xz[1]) / 4), ch * 64 - 1); ct_c = min(int(abs(centre_xz[0]) / 4), cw * 64 - 1)
    clamp = lambda a, lo, hi: max(lo, min(hi, a))
    tdiv = lambda a: int(a / 64)                       # C division truncates toward zero
    reach = 2 * radius
    return (ct_r, ct_c), [(cr, cc) for cr in range(clamp(tdiv(ct_r - reach), 0, ch - 1), clamp(tdiv(ct_r + reach), 0, ch - 1) + 1)
                          for cc in range(clamp(tdiv(ct_c - reach), 0, cw - 1), clamp(tdiv(ct_c + reach), 0, cw - 1) + 1)]


def test_port_zone_fields_golden(pforacle):
    """TARGET_ZONE chunk fields (field_update_zone, field.c:1810) and N_DesiredGroupArrivalVelocity (nav.c:3561)"""
    g = gold("region")
    cw = ch = 3
    om = pforacle.OracleMap(cw, ch, g["cost"], g["blk"], None)
    for k in range(len(g["zc"])):
        for c in range(cw * ch):
            assert (om.flow_field_zone((c // cw, c % cw), g["zc"][k], int(g["zrad"][k])) == g["zexp"][k, c]).all(), (k, c)
    for k in range(len(g["gv_radius"])):
        cxz, rad = g["gv_centre"][k], int(g["gv_radius"][k])
        fields = np.zeros((cw * ch, 64, 64), np.uint8); has = np.zeros(cw * ch, np.uint8)
        inside = (0 <= -cxz[0] <= cw * 256) and (0 <= cxz[1] <= ch * 256)
        if inside:
            ct, chunks = _zone_chunks(cxz, rad, cw, ch)
            for cr, cc in chunks:
                fields[cr * cw + cc] = om.flow_field_zone((cr, cc), ct, rad); has[cr * cw + cc] = 1
        assert int(has.sum()) == int(g["gv_nfields"][k])
        v, f = om.group_arrival_velocity(fields, has, cxz, rad, g["gv_pos"][k])
        assert (f == g["gv_flags"][k]).all() and (v == g["gv_vel"][k]).all(), k


def test_zone_seeds_host_vs_port(pforacle):
    """the host-side seed flood of the CUDA path (pfnav_zone_seeds, no device needed) == the port's, order included"""
    g = gold("region")
    cw = ch = 3
    om = pforacle.OracleMap(cw, ch, g["cost"], g["blk"], None)
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, g["cost"], g["blk"])
    rng = np.random.default_rng(2)
    for k in range(40):
        centre = (int(rng.integers(0, ch * 64)), int(rng.integers(0, cw * 64))); radius = int(rng.integers(0, 60))
        for cr in range(ch):
            for cc in range(cw):
                a, b = nav.zone_seeds((cr, cc), centre, radius), om.zone_seeds((cr, cc), centre, radius)
                assert a.shape == b.shape and (a == b).all(), (centre, radius, cr, cc)
    nav.map_create(1, 3, 1)
    with pytest.raises(Exception):
        nav.zone_seeds((0, 0), (10, 10), 3)            # one chunk column: the reference's stride overruns its buffer
    nav.close()


def test_entity_and_enemies_fields_golden(pforacle):
    """TARGET_ENTITY / TARGET_ENEMIES: the host seed code of the CUDA path (pfnav_entity_seeds: footprint tiles,
    contour rings per reference layer, the enemies' search rectangle) + the port's padded-chunk integration
    == the compiled reference's N_FlowFieldUpdate through a nav_unit_query_ctx"""
    g = gold("targets")
    cw = ch = 3
    wars = [tuple(w) for w in g["wars"]]
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, g["cost_0"], g["blk_0"])
    fp = nav.footprints(g["pos"], g["radius"])
    for L in (0, 2):
        om = pforacle.OracleMap(cw, ch, g["cost_%d" % L], g["blk_%d" % L], None)
        for k, u in enumerate(g["uids"]):
            for c in range(cw * ch):
                sd = nav.entity_seeds(capi.TARGET_ENTITY, fp[u:u + 1], (c // cw, c % cw), ref_layer=L)
                assert (om.chunk_field_seeded((c // cw, c % cw), sd) == g["ent_%d" % L][k, c]).all(), (L, u, c)
        for f in range(4):
            sel = cases.enemies_of(f, wars, g["factions"], g["flags"])
            for c in range(cw * ch):
                sd = nav.entity_seeds(capi.TARGET_ENEMIES, fp[sel], (c // cw, c % cw), ref_layer=L)
                assert (om.chunk_field_seeded((c // cw, c % cw), sd) == g["foe_%d" % L][f, c]).all(), (L, f, c)
    with pytest.raises(capi.PfnavError):
        nav.entity_seeds(capi.TARGET_ENTITY, fp[:2], (0, 0))              # one target entity only
    nav.close()


TILE_CASES = ((2, 2), (3, 2))


def test_port_cost_from_tiles_golden(pforacle):
    g = gold("tiles")
    for k, (cw, ch) in enumerate(TILE_CASES):
        t = g[f"tiles{k}"].astype(np.int32)
        for layer in (0, 3, 4, 8):
            assert (pforacle.cost_from_tiles(cw, ch, t, layer) == g[f"cost{k}_{layer}"]).all(), (k, layer)


def test_port_cost_from_tiles_vs_ref(pfref, pforacle):
    for seed, terrain in ((51, False), (52, True), (53, False)):
        t = cases.tile_attr_case(2, 3, seed, terrain)
        ref = pfref.RefMap(2, 3, tiles=t)
        for layer in range(12):
            assert (pforacle.cost_from_tiles(2, 3, t, layer) == ref.cost_base(layer)).all(), (seed, layer)
        ref.close()


def test_local_islands_restatement_golden():
    g = gold("portal_los")
    assert (cases.local_islands_np(g["cost"]) == g["liid"]).all()


def _agents_from_gold(g):
    a = {k[2:]: g[k] for k in g.files if k.startswith("a_")}
    a["vdes"] = np.zeros((len(a["radius"]), 2), np.float32); a["vdes"][g["work"]] = g["vdes"]
    a["has_los"] = np.zeros(len(a["radius"]), np.uint32); a["has_los"][g["work"]] = g["los"]
    return a


@pytest.mark.parametrize("name,cw", [("agents_1x1", 1), ("agents_dense", 1), ("agents_3x3", 3)])
def test_port_agents_golden(pforacle, name, cw):
    g = gold(name)
    a = _agents_from_gold(g)
    rec, fl = capi.pack_agents(a)
    om = pforacle.OracleMap(cw, cw, g["cost"])
    w = pforacle.OracleWorld(om, rec, fl, 20)
    # spatial index: same hits in the same order as bg_ent_inrange_circle
    o10 = np.cumsum(np.concatenate([[0], g["q10_len"]])); o30 = np.cumsum(np.concatenate([[0], g["q30_len"]]))
    for k, i in enumerate(g["qi"]):
        x, z = float(a["pos"][i, 0]), float(a["pos"][i, 1])
        assert (w.ents_in_circle(x, z, 10.0, 512) == g["q10"][o10[k]:o10[k + 1]]).all()
        assert (w.ents_in_circle(x, z, 30.0, 128) == g["q30"][o30[k]:o30[k + 1]]).all()
    vel, vpref = w.velocity_work(g["work"])
    # tolerance: north_star's 1e-4 relative. (Cohesion sums flock members in khash bucket order in the
    # reference and in ascending uid here; with one flock of dense uids the two coincide bit for bit.)
    assert cases.relerr(vpref, g["vpref"]).max() <= 1e-4
    assert cases.relerr(vel, g["vel"]).max() <= 1e-4
    if name != "agents_3x3":
        assert (vel == g["vel"]).all() and (vpref == g["vpref"]).all()
    w.close()


@pytest.mark.parametrize("name", ["update_hz20", "update_hz10"])
def test_port_velocity_with_garrisoned_and_los_golden(pforacle, name):
    """the state-update fixtures also pin the velocity pass where the older ones are blind: agents with
    line of sight next to their goal, zero-velocity movers, COMBAT_HELD units, and GARRISONED entities,
    which G_Pos_EntsInCircleFrom swap-removes from every radius query (position.c:100-119, 379)"""
    g = gold(name)
    a = _agents_from_gold(g)
    assert (a["flags"] & capi.FLAG_GARRISONED).any() and g["los"].any()
    rec, fl = capi.pack_agents(a)
    om = pforacle.OracleMap(3, 3, g["cost"])
    w = pforacle.OracleWorld(om, rec, fl, int(g["hz"]))
    vel, _ = w.velocity_work(g["work"])
    assert (cases.relerr(vel, g["vel"]) <= 1e-6).all()
    w.close()


@pytest.mark.parametrize("name", ["update_hz20", "update_hz10"])
def test_port_entity_update_golden(pforacle, name):
    """a-8 in the restatement: entity_compute_update (movement.c:2303) patches from the reference's velocities; flags,
    states and all 25 floats identical. The two map searches of arrived() come from the host code of the CUDA path
    (pfnav_route_arrival_consts), which this pins as well."""
    g = gold(name)
    a = _agents_from_gold(g)
    rec, fl = capi.pack_agents(a)
    nav = capi.Nav(hostonly=True)
    nav.map_create(3, 3, 1); nav.map_upload_layer(0, g["cost"]); nav.map_build_nav(0); nav.route_build(0)
    arrival = [nav.route_arrival_consts(t) for t in a["flock_target"]]
    nav.close()
    w = pforacle.OracleWorld(pforacle.OracleMap(3, 3, g["cost"]), rec, fl, int(g["hz"]))
    p = w.entity_updates(g["ms"].view(capi.MOVESTATE), arrival, g["work"], g["vel"], g["vdes"], capi.PATCH)
    oi, of = g["patch_i"], g["patch_f"]
    assert (p["flags"] == oi[:, 0].astype(np.uint32)).all() and (p["next_state"] == oi[:, 1]).all() and (p["next_block"] == oi[:, 2]).all()
    got = np.concatenate([p["next_velocity"], p["next_pos"], p["next_rot"], p["next_ppos"], p["next_npos"],
                          p["next_step"][:, None], p["next_left"][:, None], p["next_nrot"], p["next_prot"]], axis=1)
    assert (got == of[:, :25]).all()
    w.close()
    # entity_apply_update's movestate part: velocity history after the patches
    a2, ms2 = pforacle.entity_apply(rec, g["ms"].view(capi.MOVESTATE), g["work"], p)
    assert (ms2["vel_hist"][g["work"]] == g["hist"]).all() and (ms2["vel_hist_idx"][g["work"]] == g["hidx"]).all()


@pytest.mark.parametrize("name", ["update_hz20", "update_hz10"])
def test_port_tick_golden(pforacle, name):
    """cases.port_tick, the per-tick expectation of the device-resident trajectory test, composed end to end on the
    reference's state-update fixtures: from the reference's desired velocities it must reproduce the reference's
    velocities, patches and velocity history. Velocities within 1e-6 relative (the port's own bound,
    test_port_velocity_with_garrisoned_and_los_golden); flags, states, blocking and the history index identical for
    every work item; the 25 patch floats and the history bit-exact wherever the port's velocity is the reference's,
    within 1e-4 of max(|x|, 1) elsewhere."""
    g = gold(name)
    a = _agents_from_gold(g)
    rec, fl = capi.pack_agents(a)
    nav = capi.Nav(hostonly=True)
    nav.map_create(3, 3, 1); nav.map_upload_layer(0, g["cost"]); nav.map_build_nav(0); nav.route_build(0)
    arrival = [nav.route_arrival_consts(t) for t in a["flock_target"]]
    nav.close()
    work = g["work"]
    t = cases.port_tick(pforacle.OracleMap(3, 3, g["cost"]), rec, fl, g["ms"].view(capi.MOVESTATE), work, int(g["hz"]),
                        arrival, vdes=g["vdes"], los=g["los"])
    assert (cases.relerr(t["vel"], g["vel"]) <= 1e-6).all()
    p, oi, of = t["patches"], g["patch_i"], g["patch_f"][:, :25]
    assert (p["flags"] == oi[:, 0].astype(np.uint32)).all() and (p["next_state"] == oi[:, 1]).all() and (p["next_block"] == oi[:, 2]).all()
    assert {-1, 2, 4} <= set(p["next_state"].tolist())
    exact = (t["vel"] == g["vel"]).all(axis=1)
    assert exact.mean() > 0.95
    got = cases.patch_floats(p)
    assert (got[exact] == of[exact]).all()
    assert (np.abs(got - of) <= 1e-4 * np.maximum(np.abs(of), 1.0)).all()
    ms2 = t["movestate"]
    assert (ms2["vel_hist_idx"][work] == g["hidx"]).all()
    assert (ms2["vel_hist"][work][exact] == g["hist"][exact]).all()
    assert (np.abs(ms2["vel_hist"][work] - g["hist"]) <= 1e-4 * np.maximum(np.abs(g["hist"]), 1.0)).all()
    # the agent records after the apply: garrisoned entities untouched, everyone else moved to the patch's position
    garr = (a["flags"][work] & capi.FLAG_GARRISONED) != 0
    setpos = ((oi[:, 0] & 4) != 0) & ~garr
    assert (t["agents"]["pos"][work][setpos] == got[setpos][:, [2, 4]]).all()
    assert (t["agents"]["state"][work][garr] == a["state"][work][garr]).all()


# ---- every movement state: the steering variants and the state machine beyond point seeking -------------------------
UNPINNED = ("the port's states beyond point seeking (formation, cell arrival, enemy seek, entity range, turning, the "
            "waiting countdown, surround) follow the CUDA kernels' structure and stay UNPINNED to the reference: ")


def _states_case(hz):
    """test_gpu_states' all-states scenario and its work inputs, and the port's tick on them"""
    import test_gpu_states as S
    p, cost, a, ms, form, ext = S._scenario(5151, hz)
    work, vdes, los = S._work_inputs(a, form)
    aa = dict(a)
    n = len(a["radius"])
    aa["vdes"] = np.zeros((n, 2), np.float32); aa["vdes"][work] = vdes
    aa["has_los"] = np.zeros(n, np.uint32); aa["has_los"][work] = los
    rec, fl = capi.pack_agents(aa)
    host = capi.Nav(hostonly=True)
    host.map_create(3, 3, 1); host.map_upload_layer(0, cost); host.map_build_nav(0); host.route_build(0)
    try:
        t = cases.states_port_tick(host, {0: cases.pforacle_map(3, 3, cost)}, rec, fl, ms, form, ext, work, hz)
    finally:
        host.close()
    return dict(cost=cost, a=a, ms=ms, form=form, ext=ext, work=work, vdes=vdes, los=los, rec=rec, fl=fl, port=t)


def _port_patches_from(c, vel, hz):
    """the port's entity_compute_update on given velocities (the reference's), with the scenario's arrival constants"""
    import pforacle
    host = capi.Nav(hostonly=True)
    host.map_create(3, 3, 1); host.map_upload_layer(0, c["cost"]); host.map_build_nav(0); host.route_build(0)
    try:
        arrival = [host.route_arrival_consts(t) for t in c["fl"]["target"]]
        tarr = cases.target_arrivals(host, c["rec"], c["ext"], c["work"])
    finally:
        host.close()
    rec = c["rec"].copy(); rec["vdes"][c["work"]] = c["vdes"]; rec["has_dest_los"][c["work"]] = c["los"]
    w = pforacle.OracleWorld(cases.pforacle_map(3, 3, c["cost"]), rec, c["fl"], hz, c["form"], c["ext"])
    try:
        return w.entity_updates(c["ms"], arrival, c["work"], vel, c["vdes"], capi.PATCH, tarr)
    finally:
        w.close()


def _check_port_states(c, hz, evel, oi, of, ox):
    """the port against reference values of the all-states scenario: velocities within 1e-4; from the reference's
    velocities, flags / states / blocking / wait ticks identical and the patch floats within 1e-4 of max(|x|, 1)"""
    assert cases.vel_ok(c["port"]["vel"], evel, c["a"]["pos"][c["work"]])[0]
    p = _port_patches_from(c, evel, hz)
    assert (p["flags"] == oi[:, 0].astype(np.uint32)).all() and (p["next_state"] == oi[:, 1]).all()
    assert (p["next_block"] == oi[:, 2]).all() and (p["wait_ticks_left"] == oi[:, 3]).all()
    got = cases.patch_floats(p)
    assert (np.abs(got - of[:, :25]) <= 1e-4 * np.maximum(np.abs(of[:, :25]), 1.0)).all()
    gx = np.concatenate([p["next_dest"], p["next_target_prev"], p["next_target_dir"], p["next_attack"][:, None].astype(np.float32)], axis=1)
    assert np.abs(gx - ox).max() <= 1e-5


@pytest.mark.parametrize("hz", [20, 10])
def test_port_all_states_vs_ref(pforacle, hz):
    """the port's every-state tick on test_gpu_states' scenario against the compiled reference"""
    import pfref
    if not pfref.available():
        pytest.skip(UNPINNED + "oracle/_ref/libpfref.so is not built")
    import test_gpu_states as S
    c = _states_case(hz)
    p, cost, a, ms, form, ext = S._scenario(5151, hz)
    ref = pfref.RefMap(3, 3, p)
    try:
        S._ref_setup(ref, a, ms, form, ext, hz, c["work"], c["vdes"], c["los"])
        evel, _ = ref.velocity_work(os.cpu_count())
        oi, of, ox = ref.compute_updates_ext(evel)
    finally:
        ref.close()
    _check_port_states(c, hz, evel, oi, of, ox)


@pytest.mark.parametrize("hz", [20, 10])
def test_port_all_states_golden(pforacle, hz):
    """the port's every-state tick against movement_states_hz*.npz where those hold reference values (recorded with the
    compiled reference, PFNAV_RECORD_GOLDEN without _SELF); a file recorded from the CUDA path pins nothing"""
    g = gold("movement_states_hz%d" % hz)
    if str(g["source"]) != "reference":
        pytest.skip(UNPINNED + "movement_states_hz%d.npz was recorded from the CUDA path, not from the reference" % hz)
    c = _states_case(hz)
    _check_port_states(c, hz, g["vel"], g["patch_i"], g["patch_f"], g["patch_x"])


@pytest.mark.parametrize("hz", [20, 10, 5, 1])
def test_port_all_states_cover_the_state_machine(pforacle, hz):
    """the port's every-state tick on test_gpu_states' scenario reaches every state and every kind of transition that
    tests/test_gpu_states_port.py compares the device with, at every tick rate"""
    c = _states_case(hz)
    stw = c["a"]["state"][c["work"]]
    for s_ in (0, 1, 3, 4, 5, 6, 7, 8):
        assert (stw == s_).sum() > 10, s_
    p = c["port"]["patches"]
    assert {-1, 0, 1, 2, 4, 7, 8} <= set(p["next_state"].tolist())
    for bit in (10, 11, 12, 13, 14):
        assert (p["flags"] & (1 << bit)).any(), bit
    # WAITING counts down by one (not garrisoned or stuck units, which return before the state switch); on 0 the unit
    # returns to wait_prev (SET_MOVING) and the apply leaves it there
    wt = stw == 4
    before = c["ext"]["wait_ticks_left"][c["work"]]
    assert np.isin(p["wait_ticks_left"][wt] - before[wt], (-1, 0)).all() and (p["wait_ticks_left"][wt] == before[wt] - 1).mean() > 0.9
    back = wt & (p["wait_ticks_left"] == 0)
    assert back.any() and ((p["flags"][back] & (1 << 12)) != 0).all()
    assert (c["port"]["agents"]["state"][c["work"]][back] == c["ext"]["wait_prev"][c["work"]][back]).all()


def test_port_desired_velocity_golden(pforacle):
    g = gold("agents_3x3")
    a = _agents_from_gold(g)
    rec, fl = capi.pack_agents(a)
    om = pforacle.OracleMap(3, 3, g["cost"])
    slot = np.full(3 * 9, -1, np.int32)
    for s, (f, cr, cc, hf, hl) in enumerate(g["pool_chunks"]):
        slot[f * 9 + cr * 3 + cc] = s
    vdes, los = om.desired_velocity(rec, fl, g["work"], slot, g["pool_flow"], g["pool_los"])
    assert (los == g["los"]).all()
    assert (vdes == g["vdes"]).all()       # bit-exact: pure float ops, no transcendental


# ---------------------------------------------------------------- oracle port vs compiled reference
@pytest.mark.parametrize("seed,dens", [(3, 0.05), (5, 0.3)])
def test_port_vs_ref_fields(pfref, pforacle, seed, dens):
    cw = ch = 2
    p = cases.noise_map(cw, ch, seed, dens)
    ref = pfref.RefMap(cw, ch, p)
    cost, liid = ref.cost_base(), ref.local_islands()
    assert (cost == synth.cost_from_pathable(p, cw, ch)).all()
    assert (liid == cases.local_islands_np(cost)).all()
    om = pforacle.OracleMap(cw, ch, cost, None, liid)
    specs = cases.portal_specs(ref.portals(), liid, cw, limit=24)
    got = om.flow_fields_update(cases.portal_reqs(specs))
    for k, s in enumerate(specs):
        assert (ref.flow_portal(s[0], s[1], s[5], s[6]) == got[k]).all()
    lr = cases.los_case(cost, cw, ch, seed, ntargets=2)
    assert (om.los_fields_create(lr) == cases.ref_los_batch(ref, lr)).all()
    ref.close()


def test_port_vs_ref_blockers(pfref, pforacle):
    """dynamic obstacles: N_BlockersIncref + N_Update on the reference, then fields with blockers > 0"""
    p = cases.noise_map(1, 1, 9, 0.05)
    ref = pfref.RefMap(1, 1, p)
    rng = np.random.default_rng(9)
    for _ in range(25):
        x, z = -rng.uniform(10, 246), rng.uniform(10, 246)
        ref.blockers_incref(float(x), float(z), 3.0, 0, 1 << 3)
    ref.update()
    cost, blk, liid = ref.cost_base(), ref.blockers(), ref.local_islands()
    assert (blk > 0).any()
    assert (liid == cases.local_islands_np(cost, blk)).all()
    om = pforacle.OracleMap(1, 1, cost, blk, liid)
    free = np.argwhere((cost[0] != 255) & (blk[0] == 0))
    for r, c in free[::501]:
        q = capi.tile_req((0, 0), (int(r), int(c)))
        assert (om.flow_fields_update(q)[0] == ref.flow_tile((0, 0), (int(r), int(c)))).all()
        lq = capi.los_req((0, 0), (0, 0, int(r), int(c)))
        assert (om.los_fields_create(lq)[0] == ref.los((0, 0), (0, 0, int(r), int(c)))).all()
    ref.close()


# ---------------------------------------------------------------- host-side planner (host-only context: no compute)
def test_route_request_path_attacking_vs_ref(pfref, pforacle):
    """N_RequestPathAttacking (nav.c:3393): same route, faction packed into the dest_id and applied to every field"""
    cw = ch = 3
    p = cases.noise_map(cw, ch, 57, 0.1)
    ref = pfref.RefMap(cw, ch, p)
    rng = np.random.default_rng(8)
    ref.set_war(0, 1); ref.set_war(0, 2)
    for _ in range(50):
        ref.blockers_incref(float(-rng.uniform(10, cw * 256 - 10)), float(rng.uniform(10, ch * 256 - 10)),
                            float(rng.uniform(2, 9)), int(rng.integers(0, 4)), 0)
    ref.update()
    cost, blk, liid, fac = ref.cost_base(), ref.blockers(), ref.local_islands(), ref.factions()
    enemies = np.zeros(16, np.uint16); enemies[0] = 0b110; enemies[1] = 0b001; enemies[2] = 0b001
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, cost, blk, liid); nav.map_build_nav(0); nav.route_build(0)
    om = pforacle.OracleMap(cw, ch, cost, blk, liid, factions=fac, enemies=enemies)
    free = synth.blocked_to_image(cost, cw, ch) != 255
    pairs = [pr for pr in cases.route_pairs(cost, cw, ch, 57, 40)][:12]
    oks, dids, ffids, flows, loss, has = [], [], [], [], [], []
    for src, dst in pairs:
        ref.fc_clear()
        ok, did = ref.request_path(src, dst, faction=0)
        oks.append(ok); dids.append(did)
        fid = np.zeros(cw * ch, np.uint64); hs = np.zeros(cw * ch, np.uint8)
        fl = np.zeros((cw * ch, 64, 64), np.uint8); ls = np.zeros((cw * ch, 64, 64), np.uint8)
        for c in range(cw * ch):
            f, i = ref.fc_flow(did, (c // cw, c % cw)) if ok else (None, None)
            l = ref.fc_los(did, (c // cw, c % cw)) if ok else None
            if f is not None:
                fl[c] = f; fid[c] = i; hs[c] |= 1
            if l is not None:
                ls[c] = l; hs[c] |= 2
        ffids.append(fid); flows.append(fl); loss.append(ls); has.append(hs)
    assert any(oks) and all((d & 0xF) == 0 for d, o in zip(dids, oks) if o)
    nav.request_faction(0)
    _check_route_against(nav, om, cw, ch, pairs, oks, dids, ffids, flows, loss, has)
    nav.request_faction()
    ref.close(); nav.close()


def _check_route_against(nav, om, cw, ch, pairs, ok_e, did_e, ffid_e, flow_e, los_e, has_e):
    for k, (src, dst) in enumerate(pairs):
        ok, did, fr, fid, fc, lr, lc = nav.route_request_path(tuple(src), tuple(dst))
        assert ok == bool(ok_e[k])
        if not ok:
            continue
        assert did == int(did_e[k])
        fields, los = cases.execute_route(lambda r, io: om.flow_fields_update(r, inout=io), om.los_fields_create, fr, fc, lr, lc)
        last_id = {int(fc[i]): int(fid[i]) for i in range(len(fr))}
        for c in range(cw * ch):
            assert bool(has_e[k][c] & 1) == (c in fields) and bool(has_e[k][c] & 2) == (c in los)
            if c in fields:
                assert last_id[c] == int(ffid_e[k][c])                 # N_FlowFieldID of the mapped field
                assert (fields[c] == flow_e[k][c]).all()
            if c in los:
                assert (los[c] == los_e[k][c]).all()


def test_route_request_path_golden(pforacle):
    """n_request_path restated on the host (pfnav_route.cu), fields executed by the oracle port: identical
    (chunk -> ff_id) mapping, flow fields and chained LOS fields as the reference's field cache holds"""
    g = gold("route_3x3")
    for k in range(2):
        nav = capi.Nav(hostonly=True)
        nav.map_create(3, 3, 1); nav.map_upload_layer(0, g[f"cost{k}"]); nav.map_build_nav(0); nav.route_build(0)
        assert (nav.local_islands(0) == g[f"liid{k}"]).all()
        assert (nav.route_islands(0) == g[f"islands{k}"]).all()          # global island ids
        ports = nav.portals(0)
        assert (ports[:, :9] == g[f"portals{k}"][:, :9]).all()
        e, off = g[f"edges{k}"], 0
        for row in ports:                                                   # portal-graph edges: ref, state, cost bits
            n = int(e[off]); exp = e[off + 1:off + 1 + 3 * n].reshape(n, 3); off += 1 + 3 * n
            assert (nav.route_edges(int(row[0]) * 3 + int(row[1]), int(row[2])) == exp).all()
        om = pforacle.OracleMap(3, 3, g[f"cost{k}"], None, g[f"liid{k}"])
        _check_route_against(nav, om, 3, 3, g[f"pairs{k}"], g[f"ok{k}"], g[f"did{k}"], g[f"ffid{k}"], g[f"flow{k}"], g[f"los{k}"], g[f"has{k}"])
        with pytest.raises(capi.PfnavError):                                # host-only context: no compute path
            nav.flow_fields_update(capi.tile_req((0, 0), (1, 1)))
        nav.close()


def test_pfmap_parse_roundtrip_and_errors():
    """pfnav_pfmap_parse (docs/pfmap.txt; al_parse_pfmap_header asset_load.c:168, m_al_parse_tile map_asset_load.c:103):
    host code, no device"""
    t = cases.tile_attr_case(3, 2, 5)
    want = np.concatenate([(t[..., :1] != 0).astype(np.int32), t[..., 1:]], -1)
    txt = capi.pfmap_write(t)
    assert (capi.pfmap_parse(txt) == want).all()
    assert (capi.pfmap_parse(capi.pfmap_write(t, version="1.2", per_line=8)) == want).all()       # num_splats line, 8 tiles per line
    assert (capi.pfmap_parse(txt.replace(b"\n", b"\r\n")) == want).all()
    for bad in (b"", b"version 1.0\nnum_materials 0\nnum_rows 1\nnum_cols 1\n0+00", txt[:-30], txt.replace(b"0+", b"0+0", 1),
                txt.replace(b"num_rows", b"rows", 1)):
        with pytest.raises(capi.PfnavError):
            capi.pfmap_parse(bad)
    demo = os.path.join(os.environ.get("PFNAV_REFERENCE", ""), "assets", "maps", "demo.pfmap")
    if os.path.exists(demo):                       # the engine's own demo map: the tiles the golden was built from
        assert (capi.pfmap_parse(open(demo, "rb").read()) == gold("demo_map")["tiles"]).all()


def test_demo_map_nav_build_golden(pforacle):
    """the engine's demo map (4 x 4 chunks, every tile type, heights -3..9) through the reference's nav build: per-layer
    cost grids (port), local / global islands, portals and 16 path requests (host planner + port fields)"""
    g = gold("demo_map")
    tiles = g["tiles"].astype(np.int32)
    for layer in (0, 1, 3, 4, 8):
        assert (pforacle.cost_from_tiles(4, 4, tiles, layer) == g["cost_%d" % layer]).all(), layer
    nav = capi.Nav(hostonly=True)
    nav.map_create(4, 4, 1); nav.map_upload_layer(0, g["cost_0"]); nav.map_build_nav(0); nav.route_build(0)
    assert (nav.local_islands(0) == g["liid_0"]).all()
    assert (nav.route_islands(0) == g["islands_0"]).all()
    assert (nav.portals(0)[:, :9] == g["portals_0"][:, :9]).all()
    om = pforacle.OracleMap(4, 4, g["cost_0"], None, g["liid_0"])
    _check_route_against(nav, om, 4, 4, g["pairs"], g["ok"], g["did"], g["ffid"], g["flow"], g["los"], g["has"])
    nav.close()


def test_stress_scenario_golden(pforacle):
    """the reference's own stress test (scripts/test_stress.py) on its plain map CENTRED AT THE ORIGIN (map position
    (+512, -512), M_CenterAtOrigin map.c:420): both path requests (planner + port fields), vdes / LOS per unit out of the
    settled field cache, and the velocity pass of 512 units"""
    g = gold("stress")
    mx, mz = [float(v) for v in g["map_origin"]]
    assert (pforacle.cost_from_tiles(4, 4, g["tiles"].astype(np.int32), 0) == g["cost"]).all()
    nav = capi.Nav(hostonly=True)
    nav.map_create(4, 4, 1, mx, mz); nav.map_upload_layer(0, g["cost"]); nav.map_build_nav(0); nav.route_build(0)
    assert (nav.local_islands(0) == g["liid"]).all() and (nav.route_islands(0) == g["islands"]).all()
    om = pforacle.OracleMap(4, 4, g["cost"], None, g["liid"], map_x=mx, map_z=mz)
    _check_route_against(nav, om, 4, 4, g["pairs"], g["ok"], g["did"], g["ffid"], g["flow"], g["los_f"], g["has"])
    nav.close()
    a = _agents_from_gold(g)
    rec, fl = capi.pack_agents(a)
    slot = np.full(2 * 16, -1, np.int32)
    for k, (f, cr, cc, hf, hl) in enumerate(g["pool_chunks"]):
        slot[f * 16 + cr * 4 + cc] = k
    vdes, los = om.desired_velocity(rec, fl, g["work"], slot, g["pool_flow"], g["pool_los"])
    assert (los == g["los"]).all() and (vdes == g["vdes"]).all()
    w = pforacle.OracleWorld(om, rec, fl, 20)
    vel, vpref = w.velocity_work(g["work"])
    assert cases.relerr(vpref, g["vpref"]).max() <= 1e-4 and cases.relerr(vel, g["vel"]).max() <= 1e-4
    w.close()


def test_route_request_path_vs_ref(pfref, pforacle):
    cw = ch = 4
    p = cases.noise_map(cw, ch, 91, 0.1)
    ref = pfref.RefMap(cw, ch, p)
    cost = ref.cost_base()
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    om = pforacle.OracleMap(cw, ch, cost, None, ref.local_islands())
    pairs = cases.route_pairs(cost, cw, ch, 91, 16)
    oks, dids, ffids, flows, loss, has = [], [], [], [], [], []
    for src, dst in pairs:
        ref.fc_clear()
        ok, did = ref.request_path(src, dst)
        oks.append(ok); dids.append(did)
        fid = np.zeros(cw * ch, np.uint64); hs = np.zeros(cw * ch, np.uint8)
        fl = np.zeros((cw * ch, 64, 64), np.uint8); ls = np.zeros((cw * ch, 64, 64), np.uint8)
        for c in range(cw * ch):
            f, i = ref.fc_flow(did, (c // cw, c % cw)) if ok else (None, None)
            l = ref.fc_los(did, (c // cw, c % cw)) if ok else None
            if f is not None:
                fl[c] = f; fid[c] = i; hs[c] |= 1
            if l is not None:
                ls[c] = l; hs[c] |= 2
        ffids.append(fid); flows.append(fl); loss.append(ls); has.append(hs)
    _check_route_against(nav, om, cw, ch, pairs, oks, dids, ffids, flows, loss, has)
    ref.close(); nav.close()


def test_blockers_commit_and_route_vs_ref(pfref, pforacle):
    """N_BlockersIncref/Decref (circle + contour rings on the 4 ground layers), N_Update (islands, edge
    states) and path requests on the churned map: identical counts, island ids, edges, routes, fields"""
    cw = ch = 2
    p = cases.noise_map(cw, ch, 9, 0.05)
    ref = pfref.RefMap(cw, ch, p)
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 4)
    for l in range(4):
        nav.map_upload_layer(l, ref.cost_base(l)); nav.map_build_nav(l)
    nav.route_build(0)
    rng = np.random.default_rng(9)
    placed = []
    for it in range(60):
        x, z, r = -float(rng.uniform(2, 510)), float(rng.uniform(2, 510)), float(rng.choice([1.5, 3.0, 6.0, 11.0]))
        ref.blockers_incref(x, z, r, 0, capi.FLAG_MOVABLE); nav.blockers_incref(x, z, r, 0, capi.FLAG_MOVABLE)
        placed.append((x, z, r))
        if it % 3 == 2:
            x, z, r = placed.pop(int(rng.integers(0, len(placed))))
            ref.blockers_decref(x, z, r, 0, capi.FLAG_MOVABLE); nav.blockers_decref(x, z, r, 0, capi.FLAG_MOVABLE)
    ref.update()
    assert nav.map_commit() > 0
    for l in range(4):
        assert (ref.blockers(l) == nav.blockers(l)).all()
        assert (ref.local_islands(l) == nav.local_islands(l)).all()
    for row in ref.portals():
        ci = int(row[0]) * cw + int(row[1])
        assert (ref.portal_edges(0, ci, int(row[2])) == nav.route_edges(ci, int(row[2]))).all()
    cost, blk = ref.cost_base(), ref.blockers()
    om = pforacle.OracleMap(cw, ch, cost, blk, ref.local_islands())
    pairs = cases.route_pairs(np.where(blk > 0, 255, cost).astype(np.uint8), cw, ch, 9, 12)
    oks, dids, ffids, flows, loss, has = [], [], [], [], [], []
    for src, dst in pairs:
        ref.fc_clear()
        ok, did = ref.request_path(src, dst)
        oks.append(ok); dids.append(did)
        fid = np.zeros(cw * ch, np.uint64); hs = np.zeros(cw * ch, np.uint8)
        fl = np.zeros((cw * ch, 64, 64), np.uint8); ls = np.zeros((cw * ch, 64, 64), np.uint8)
        for c in range(cw * ch):
            f, i = ref.fc_flow(did, (c // cw, c % cw)) if ok else (None, None)
            l = ref.fc_los(did, (c // cw, c % cw)) if ok else None
            if f is not None:
                fl[c] = f; fid[c] = i; hs[c] |= 1
            if l is not None:
                ls[c] = l; hs[c] |= 2
        ffids.append(fid); flows.append(fl); loss.append(ls); has.append(hs)
    _check_route_against(nav, om, cw, ch, pairs, oks, dids, ffids, flows, loss, has)
    ref.close(); nav.close()


# ---------------------------------------------------------------- host logic + ABI surface
def test_blockers_obb_vs_ref(pfref):
    """N_BlockersIncrefOBB / DecrefOBB (nav.c:4685): rotated building footprints -> M_Tile_AllUnderObj supercover +
    interior + contour rings on the four ground layers, duplicates and all; identical refcounts"""
    cw = ch = 2
    p = cases.noise_map(cw, ch, 13, 0.05)
    ref = pfref.RefMap(cw, ch, p)
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 4)
    for l in range(4):
        nav.map_upload_layer(l, ref.cost_base(0))
    rng = np.random.default_rng(4)
    boxes = []
    for _ in range(40):
        c = np.array([-rng.uniform(60, cw * 256 - 60), rng.uniform(60, ch * 256 - 60)])
        hw, hh, ang = rng.uniform(3, 30), rng.uniform(3, 30), rng.uniform(0, np.pi)
        ax, ay = np.array([np.cos(ang), np.sin(ang)]), np.array([-np.sin(ang), np.cos(ang)])
        b = np.array([c - ax * hw - ay * hh, c + ax * hw - ay * hh, c + ax * hw + ay * hh, c - ax * hw + ay * hh], np.float32)
        boxes.append(b)
        ref.blockers_obb(b, True, 0, 0); nav.blockers_obb(b, True, 0, 0)
    for l in range(4):
        assert (ref.blockers(l) == nav.blockers(l)).all(), l
    assert ref.blockers(0).max() >= 2          # overlaps and the corner duplicates are counted
    for b in boxes[:25]:
        ref.blockers_obb(b, False, 0, 0); nav.blockers_obb(b, False, 0, 0)
    for l in range(4):
        assert (ref.blockers(l) == nav.blockers(l)).all(), l
    with pytest.raises(capi.PfnavError):
        nav.blockers_obb(np.array([[10.0, 5.0], [-5.0, 5.0], [-5.0, 20.0], [10.0, 20.0]], np.float32))   # corner outside
    ref.close(); nav.close()


def test_map_origin_blockers_and_fields_vs_ref(pfref, pforacle):
    """a map that is not at the origin (the engine centres its maps, map.c:420) and is not square: circle + OBB
    blockers on the four ground layers, islands, faction counts, world-space group arrival fields"""
    cw, ch, mx, mz = 4, 3, 512.0, -384.0
    p = cases.noise_map(cw, cw, 17, 0.1)[:ch * 32]
    ref = pfref.RefMap(cw, ch, p, map_x=mx, map_z=mz)
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 4, mx, mz)
    for L in range(4):
        nav.map_upload_layer(L, ref.cost_base(L)); nav.map_build_nav(L)
    rng = np.random.default_rng(5)
    for _ in range(80):
        x, z, r, f = mx - rng.uniform(6, cw * 256 - 6), mz + rng.uniform(6, ch * 256 - 6), rng.uniform(1, 14), int(rng.integers(0, 4))
        ref.blockers_incref(float(x), float(z), float(r), f, 0); nav.blockers_incref(float(x), float(z), float(r), f, 0)
    for _ in range(12):
        c = np.array([mx - rng.uniform(40, cw * 256 - 40), mz + rng.uniform(40, ch * 256 - 40)])
        ang, hx, hz = rng.uniform(0, np.pi), rng.uniform(4, 30), rng.uniform(4, 30)
        ax, az = np.array([np.cos(ang), np.sin(ang)]), np.array([-np.sin(ang), np.cos(ang)])
        corners = np.array([c - ax * hx - az * hz, c + ax * hx - az * hz, c + ax * hx + az * hz, c - ax * hx + az * hz], np.float32)
        ref.blockers_obb(corners, True, 1, 0); nav.blockers_obb(corners, True, 1, 0)
    ref.update(); nav.map_commit()
    for L in range(4):
        assert (nav.blockers(L) == ref.blockers(L)).all(), L
        assert (nav.local_islands(L) == ref.local_islands(L)).all(), L
        assert (nav.faction_counts(L) == ref.factions(L)).all(), L
    om = pforacle.OracleMap(cw, ch, ref.cost_base(0), ref.blockers(0), None, map_x=mx, map_z=mz)
    for _ in range(12):
        c = (mx - rng.uniform(-5, cw * 256 + 5), mz + rng.uniform(-5, ch * 256 + 5))
        t = np.stack([c[0] + rng.uniform(-200, 200, 10), c[1] + rng.uniform(-200, 200, 10)], 1)
        assert (ref.group_arrival_field(96, t, c) == om.group_arrival_field(96, 0, t, c)).all()
    ref.close(); nav.close()


def test_map_create_drops_state_of_previous_map():
    """dirty sets / routes / per-faction counts of an earlier, larger map must not leak into the next one"""
    nav = capi.Nav(hostonly=True)
    p = cases.noise_map(3, 3, 5, 0.05)
    nav.map_create(3, 3, 1); nav.map_upload_layer(0, synth.cost_from_pathable(p, 3, 3)); nav.map_build_nav(0)
    nav.blockers_incref(-700.0, 700.0, 9.0, 2, 0)           # lands in chunk (2, 2): out of range for the next map
    p2 = cases.noise_map(1, 1, 6, 0.05)
    nav.map_create(1, 1, 1); nav.map_upload_layer(0, synth.cost_from_pathable(p2, 1, 1)); nav.map_build_nav(0)
    assert nav.map_commit() == 0
    assert not nav.blockers(0).any()
    nav.close()


def test_synth_is_deterministic():
    p1 = synth.make_map(2, 2, 0x5EED0002); p2 = synth.make_map(2, 2, 0x5EED0002)
    assert (p1 == p2).all() and 0.05 < (p1 == 0).mean() < 0.5
    c = synth.cost_from_pathable(p1, 2, 2)
    a1 = synth.make_agents(c, 2, 2, 500, 2, 7); a2 = synth.make_agents(c, 2, 2, 500, 2, 7)
    for k in ("pos", "vel", "flock_target"):
        assert (a1[k] == a2[k]).all()
    img = synth.blocked_to_image(c, 2, 2)
    assert (synth.image_to_blocked(img, 2, 2) == c).all()
    tr, tc = synth.tile_for_xz(a1["pos"][:, 0], a1["pos"][:, 1], 2, 2)
    assert (img[tr, tc] != 0xFF).all()          # agents stand on passable ground


def test_record_layouts_match_header():
    hdr = open(os.path.join(os.path.dirname(GOLD), "..", "include", "pfnav.h")).read()
    assert capi.FIELD_REQ.itemsize == 64 and capi.LOS_REQ.itemsize == 48
    assert capi.AGENT.itemsize == 64 and capi.FLOCK.itemsize == 16
    for name in capi.SYMBOLS:
        assert re.search(r"\b%s\s*\(" % name, hdr), name + " is bound but not declared in include/pfnav.h"
    declared = set(re.findall(r"\b(pfnav_[a-z0-9_]+)\s*\(", hdr))
    assert declared <= set(capi.SYMBOLS), declared - set(capi.SYMBOLS)


def test_abi_library_loads_and_exports_every_symbol():
    L = capi.load()
    for name in capi.SYMBOLS:
        assert hasattr(L, name), name
    assert L.pfnav_version() >= 100


def test_no_cpu_fallback_without_gpu():
    """On a box without a usable GPU the product path must fail loudly, not fall back."""
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(capi.PfnavError):
        capi.Nav(0)


def test_product_does_not_touch_oracle():
    """the package and tools/ (benchmark / trace helpers that ship with it) never reference the checker; whatever needs
    it lives under tests/ (tests/tools: GPU checks, offline fuzzers)"""
    top = os.path.join(os.path.dirname(GOLD), "..")
    for root in (os.path.join(top, "permafrost-engine_b200"), os.path.join(top, "tools"), os.path.join(top, "include")):
        for dp, _, files in os.walk(root):
            for f in files:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                    src = open(os.path.join(dp, f)).read()
                    assert "pforacle" not in src and "pfref" not in src and "oracle/" not in src, f


def test_port_los_blocked_destination_tile_vs_ref(pforacle, pfref):
    """pins the port on the reference's behaviour for a blocked destination tile (the NaN-slope line, field.c:463-517)"""
    cw = ch = 3
    p = cases.noise_map(cw, ch, 8181, 0.08)
    ref = pfref.RefMap(cw, ch, p)
    try:
        rng = np.random.default_rng(8181)
        for _ in range(40):
            x, z, r = float(-rng.uniform(10, cw * 256 - 10)), float(rng.uniform(10, ch * 256 - 10)), float(rng.uniform(2, 9))
            ref.blockers_incref(x, z, r)
        ref.update()
        cost, blk, liid = ref.cost_base(), ref.blockers(), ref.local_islands()
        om = pforacle.OracleMap(cw, ch, cost, blk, liid)
        n = 0
        for chunk in range(cw * ch):
            for r_, c_ in np.argwhere((cost[chunk] != 255) & (blk[chunk] > 0))[::23][:6]:
                td = (chunk // cw, chunk % cw, int(r_), int(c_))
                exp = ref.los((td[0], td[1]), td)
                got = om.los_fields_create(capi.los_req((td[0], td[1]), td))[0]
                assert (got == exp).all(), td
                n += 1
        assert n >= 12
    finally:
        ref.close()


@pytest.mark.parametrize("family", ["random", "forced_retries", "equal_distances", "point_ties", "degenerate_neighbours",
                                    "early_end", "degenerate_geometry", "overflow"])
def test_port_clearpath_vs_ref(pfref, pforacle, family):
    """pfo_clearpath (the port's clearpath() + vec2_truncate) against the reference's G_ClearPath_NewVelocity on the case
    families the device source is checked with (tests/test_clearpath_emu.py), bit for bit"""
    import clearpath_cases as cc
    cs = cc.FAMILIES[family](np.random.default_rng(0xC1EA9), 200)
    for i in range(len(cs)):
        s5, vp, dyn, stat, _ = cs.case(i)
        got = pforacle.clearpath(s5, vp, dyn, stat)
        want = pfref.clearpath(s5, vp, dyn, stat)
        assert not np.isnan(got).any() and (got == want).all(), (family, i, got, want)
