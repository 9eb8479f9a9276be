"""GPU suite (-m gpu): the CUDA path, called through the C ABI, against (1) the committed golden
vectors from the compiled reference, (2) the oracle port on further seeds, (3) the compiled reference
itself when oracle/_ref travelled with the snapshot, and (4) size-independent properties at the
full BASELINE.json sizes.  Integer outputs (flow dirs, LOS bits, islands, portal indices, neighbour
order) must be bit-exact; velocities within north_star's 1e-4 relative."""
import os

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
capi, synth = cases.capi, cases.synth
VEL_RTOL = 1e-4


def gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


def _upload(nav, cw, ch, cost, blockers=None, liid=None):
    nav.map_create(cw, ch, 1)
    nav.map_upload_layer(0, cost, blockers, liid)


# ------------------------------------------------------------------ fields vs golden
@pytest.mark.parametrize("tma", [0, 1])
def test_flow_tile_golden(nav, tma):
    g = gold("flow_tile")
    nav.set_tma(tma)
    for k in range(3):
        _upload(nav, 1, 1, g[f"cost{k}"])
        got = nav.flow_fields_update(g[f"reqs{k}"].view(capi.FIELD_REQ))
        assert (got == g[f"exp{k}"]).all()
    nav.set_tma(1)


@pytest.mark.parametrize("tma", [0, 1])
def test_flow_portal_and_merge_golden(nav, tma):
    g = gold("portal_los")
    nav.set_tma(tma)
    _upload(nav, 3, 3, g["cost"], None, g["liid"])
    reqs = g["reqs"].view(capi.FIELD_REQ)
    assert (nav.flow_fields_update(reqs) == g["exp"]).all()
    q = reqs[:1].copy(); q["init"] = 0
    assert (nav.flow_fields_update(q, inout=g["merge_base"][None])[0] == g["merge_exp"]).all()
    nav.set_tma(1)


@pytest.mark.parametrize("variant", [0, 1])
def test_los_golden(nav, variant):
    nav.set_los_variant(variant)
    try:
        _los_golden(nav)
    finally:
        nav.set_los_variant(2)          # the shipped default (k_los_level)


def _los_golden(nav):
    g = gold("portal_los")
    _upload(nav, 3, 3, g["cost"])
    assert (nav.los_fields_create(g["los_reqs"].view(capi.LOS_REQ)) == g["los_exp"]).all()
    # chained LOS along real routes (order-sensitive cases) from the route fixture
    r = gold("route_3x3")
    for k in range(2):
        _upload(nav, 3, 3, r[f"cost{k}"])
        nav.map_build_nav(0); nav.route_build(0)
        for i, (src, dst) in enumerate(r[f"pairs{k}"]):
            if not r[f"ok{k}"][i]:
                continue
            nav.pool_create(1, 9)
            nav.pool_request_path(0, tuple(src), tuple(dst))
            for c in range(9):
                if r[f"has{k}"][i][c] & 2:
                    assert (nav.pool_get(0, (c // 3, c % 3))[1] == r[f"los{k}"][i][c]).all()


def test_islands_and_portals_golden(nav):
    """bit-exact local-island ids and portal indices/endpoints (north_star: 'bit-exact ... portal indices')"""
    g = gold("portal_los")
    _upload(nav, 3, 3, g["cost"])
    nav.map_build_nav(0)
    assert (nav.local_islands(0) == g["liid"]).all()
    assert (nav.portals(0)[:, :9] == g["portals"][:, :9]).all()


def test_empty_and_error_paths(nav):
    g = gold("flow_tile")
    _upload(nav, 1, 1, g["cost0"])
    assert nav.flow_fields_update(np.zeros(0, capi.FIELD_REQ)).shape[0] == 0
    assert nav.los_fields_create(np.zeros(0, capi.LOS_REQ)).shape[0] == 0
    bad = capi.tile_req((0, 0), (64, 0))
    with pytest.raises(capi.PfnavError):
        nav.flow_fields_update(bad)
    bad = capi.tile_req((1, 0), (3, 3))          # chunk outside the map
    with pytest.raises(capi.PfnavError):
        nav.flow_fields_update(bad)
    att = capi.tile_req((0, 0), (3, 3)); att["faction_id"] = 2
    with pytest.raises(capi.PfnavError):           # attacking (faction-aware) request before pfnav_set_enemy_factions: refused
        nav.flow_fields_update(att)


# ------------------------------------------------------------------ fields vs the oracle port (more seeds)
@pytest.mark.parametrize("seed,dens", [(41, 0.0), (42, 0.1), (43, 0.35)])
def test_fields_vs_port(nav, pforacle, seed, dens):
    cw = ch = 2
    p = cases.noise_map(cw, ch, seed, dens)
    cost = synth.cost_from_pathable(p, cw, ch)
    _upload(nav, cw, ch, cost)
    nav.map_build_nav(0)
    liid, ports = nav.local_islands(0), nav.portals(0)
    assert (liid == cases.local_islands_np(cost)).all()
    om = pforacle.OracleMap(cw, ch, cost, None, liid)
    specs = cases.portal_specs(ports, liid, cw, limit=64)
    reqs = cases.portal_reqs(specs)
    rng = np.random.default_rng(seed)
    for c in range(cw * ch):
        tiles = np.argwhere(cost[c] != 255)
        for r_, c_ in tiles[rng.integers(0, len(tiles), 6)]:
            reqs = np.concatenate([reqs, capi.tile_req((c // cw, c % cw), (int(r_), int(c_)))])
    assert (nav.flow_fields_update(reqs) == om.flow_fields_update(reqs)).all()
    lr = cases.los_case(cost, cw, ch, seed, ntargets=6)
    assert (nav.los_fields_create(lr) == om.los_fields_create(lr)).all()


def test_general_cost_kernel_vs_port(nav, pforacle):
    """costs other than 1/0xFF (transient 0 of n_clear_cost_for_tile, nav.c:359, and arbitrary weights)"""
    p = cases.noise_map(1, 1, 51, 0.1)
    cost = synth.cost_from_pathable(p, 1, 1)
    rng = np.random.default_rng(51)
    w = rng.integers(0, 6, cost.shape).astype(np.uint8)
    cost = np.where(cost == 255, 255, np.where(rng.random(cost.shape) < 0.3, w, 1)).astype(np.uint8)
    _upload(nav, 1, 1, cost)
    om = pforacle.OracleMap(1, 1, cost)
    tiles = np.argwhere(cost[0] != 255)
    reqs = np.concatenate([capi.tile_req((0, 0), (int(r), int(c))) for r, c in tiles[::397]])
    assert (nav.flow_fields_update(reqs) == om.flow_fields_update(reqs)).all()


def test_blockers_and_chunk_update(nav, pforacle):
    """pfnav_map_update_chunk + pfnav_map_refresh_chunk (N_BlockersIncref / n_update_dirty_local_islands)"""
    cw = ch = 2
    p = cases.noise_map(cw, ch, 61, 0.05)
    cost = synth.cost_from_pathable(p, cw, ch)
    _upload(nav, cw, ch, cost)
    nav.map_build_nav(0)
    rng = np.random.default_rng(61)
    blk = np.zeros(cost.shape, np.uint16)
    for c in range(cw * ch):
        for _ in range(30):
            r0, c0 = rng.integers(0, 60, 2)
            blk[c, r0:r0 + 3, c0:c0 + 3] += 1
        nav.map_update_chunk(0, (c // cw, c % cw), None, blk[c], None)
        nav.map_refresh_chunk(0, (c // cw, c % cw))
    liid = nav.local_islands(0)
    assert (liid == cases.local_islands_np(cost, blk)).all()
    om = pforacle.OracleMap(cw, ch, cost, blk, liid)
    specs = cases.portal_specs(nav.portals(0), liid, cw, limit=40)
    reqs = cases.portal_reqs(specs)
    assert (nav.flow_fields_update(reqs) == om.flow_fields_update(reqs)).all()
    lr = cases.los_case(np.where(blk > 0, 255, cost).astype(np.uint8), cw, ch, 61, ntargets=4)
    assert (nav.los_fields_create(lr) == om.los_fields_create(lr)).all()


# ------------------------------------------------------------------ agents vs golden
def _agents_from_gold(g):
    a = {k[2:]: g[k] for k in g.files if k.startswith("a_")}
    a["vdes"] = np.zeros((len(a["radius"]), 2), np.float32); a["vdes"][g["work"]] = g["vdes"]
    a["has_los"] = np.zeros(len(a["radius"]), np.uint32); a["has_los"][g["work"]] = g["los"]
    return a


@pytest.mark.parametrize("name,cw", [("agents_1x1", 1), ("agents_dense", 1), ("agents_3x3", 3)])
def test_agents_golden(nav, name, cw):
    g = gold(name)
    a = _agents_from_gold(g)
    rec, fl = capi.pack_agents(a)
    _upload(nav, cw, cw, g["cost"])
    nav.agents_upload(rec, fl, 20)
    o10 = np.cumsum(np.concatenate([[0], g["q10_len"]])); o30 = np.cumsum(np.concatenate([[0], g["q30_len"]]))
    for k, i in enumerate(g["qi"]):
        x, z = float(a["pos"][i, 0]), float(a["pos"][i, 1])
        assert (nav.ents_in_circle(x, z, 10.0, 512) == g["q10"][o10[k]:o10[k + 1]]).all()
        assert (nav.ents_in_circle(x, z, 30.0, 128) == g["q30"][o30[k]:o30[k + 1]]).all()
    nav.agents_set_work(g["work"])
    nav.agents_tick(0)
    vel = nav.agents_read_velocities(len(g["work"]))
    vpref, vdes, los = nav.agents_read_debug(len(g["work"]))
    assert (vdes == g["vdes"]).all() and (los == g["los"]).all()
    e_vp, e_v = cases.relerr(vpref, g["vpref"]), cases.relerr(vel, g["vel"])
    # EVERY agent within north_star's 1e-4 relative (no agent of any committed population lands on the other side of an
    # epsilon-threshold branch of ClearPath)
    assert e_vp.max() <= VEL_RTOL, (e_vp.max(), np.nonzero(e_vp > VEL_RTOL)[0][:10])
    assert e_v.max() <= VEL_RTOL, (e_v.max(), np.nonzero(e_v > VEL_RTOL)[0][:10])


def test_agents_vdes_from_pool_golden(nav):
    g = gold("agents_3x3")
    a = _agents_from_gold(g)
    a["vdes"][:] = 0; a["has_los"][:] = 0           # must come from the pool
    rec, fl = capi.pack_agents(a)
    _upload(nav, 3, 3, g["cost"])
    nav.pool_create(3, 27)
    for s, (f, cr, cc, hf, hl) in enumerate(g["pool_chunks"]):
        nav.pool_put(int(f), (int(cr), int(cc)), g["pool_flow"][s] if hf else None, g["pool_los"][s] if hl else None)
    nav.agents_upload(rec, fl, 20)
    nav.agents_set_work(g["work"])
    nav.agents_tick(capi.TICK_VDES_FROM_POOL)
    vel = nav.agents_read_velocities(len(g["work"]))
    vpref, vdes, los = nav.agents_read_debug(len(g["work"]))
    assert (los == g["los"]).all()
    assert (vdes == g["vdes"]).all()
    assert cases.relerr(vel, g["vel"]).max() <= VEL_RTOL


def test_agents_vs_port_dense_crowd(nav, pforacle):
    """32+32 neighbour caps, drop-furthest retries, static neighbours: a tightly packed crowd"""
    p, cost, a = cases.agent_case(1, 900, 2, 71, 0.02, 2.2)
    rng = np.random.default_rng(71)
    a["vdes"] = rng.normal(size=(900, 2)).astype(np.float32)
    a["vdes"] /= np.linalg.norm(a["vdes"], axis=1, keepdims=True)
    a["has_los"] = (rng.random(900) < 0.3).astype(np.uint32)
    rec, fl = capi.pack_agents(a)
    work = np.nonzero((a["state"] != 2) & (a["state"] != 4))[0].astype(np.uint32)
    om = pforacle.OracleMap(1, 1, cost)
    w = pforacle.OracleWorld(om, rec, fl, 20)
    evel, evpref = w.velocity_work(work)
    _upload(nav, 1, 1, cost)
    nav.agents_upload(rec, fl, 20)
    nav.agents_set_work(work)
    nav.agents_tick(0)
    vel = nav.agents_read_velocities(len(work))
    vpref, _, _ = nav.agents_read_debug(len(work))
    assert cases.relerr(vpref, evpref).max() <= VEL_RTOL
    assert cases.relerr(vel, evel).max() <= VEL_RTOL
    w.close()
    # the other tick rates (SCALED_MAX_FORCE and max_speed / hz, movement.c:93) and a COMBAT_HELD agent
    rec2 = rec.copy(); rec2["flags"][work[0]] |= capi.FLAG_COMBAT_HELD
    for hz in (10, 5, 1):
        w2 = pforacle.OracleWorld(om, rec2, fl, hz)
        evel2, evpref2 = w2.velocity_work(work[:200])
        w2.close()
        nav.agents_upload(rec2, fl, hz)
        nav.agents_set_work(work[:200])
        nav.agents_tick(0)
        vel2 = nav.agents_read_velocities(200)
        vpref2, _, _ = nav.agents_read_debug(200)
        assert (vel2[0] == 0).all(), hz
        assert cases.relerr(vpref2, evpref2).max() <= VEL_RTOL, hz
        assert cases.relerr(vel2, evel2).max() <= VEL_RTOL, hz


# ------------------------------------------------------------------ against the compiled reference, if it travelled
def test_request_goal_fields_vs_ref(nav, pfref_or_golden, pforacle):
    """every field pfnav_pool_request_goal builds on the device equals what the reference's own
    N_FlowFieldUpdate / N_LOSFieldCreate returns for the same request. Without the compiled reference the fields come from
    the plain-C port (oracle/pf_oracle.c, pinned to the reference by tests/test_oracle.py) and the islands from the numpy
    restatement; the portal table is then compared only by test_islands_and_portals_golden (reference vectors)."""
    cw = ch = 3
    p = cases.noise_map(cw, ch, 81, 0.08)
    ref = pfref_or_golden.RefMap(cw, ch, p) if pfref_or_golden else None
    cost = ref.cost_base() if ref is not None else synth.cost_from_pathable(p, cw, ch)
    _upload(nav, cw, ch, cost)
    nav.map_build_nav(0)
    liid = nav.local_islands(0)
    assert (liid == (ref.local_islands() if ref is not None else cases.local_islands_np(cost))).all()
    if ref is not None:
        ports = ref.portals()
        assert (nav.portals(0)[:, :9] == ports[:, :9]).all()
    tiles = np.argwhere(cost[4] != 255)
    tr, tc = [int(v) for v in tiles[len(tiles) // 2]]
    td = (1, 1, tr, tc)
    fr, fc, fw, lr, lc = nav.plan_goal(td)
    assert len(fr) >= 9 and len(lr) == len(np.unique(fc))
    om = pforacle.OracleMap(cw, ch, cost, None, liid)
    # wave 0 requests, one per chunk
    got = nav.flow_fields_update(fr[fw == 0])
    if ref is None:
        exp = om.flow_fields_update(fr[fw == 0])
    else:
        exp = []
        for q in fr[fw == 0]:
            chunk = (int(q["chunk_r"]), int(q["chunk_c"]))
            if q["target_type"] == capi.TARGET_TILE:
                exp.append(ref.flow_tile(chunk, (int(q["tile_r"]), int(q["tile_c"]))))
            else:
                sel = ports[(ports[:, 0] == chunk[0]) & (ports[:, 1] == chunk[1]) & (ports[:, 3] == q["port_r0"]) &
                            (ports[:, 4] == q["port_c0"]) & (ports[:, 5] == q["port_r1"]) & (ports[:, 6] == q["port_c1"])]
                exp.append(ref.flow_portal(chunk, int(sel[0][2]), int(q["port_iid"]), int(q["next_iid"])))
        exp = np.stack(exp)
    assert (got == exp).all()
    exp_los = cases.ref_los_batch(ref, lr) if ref is not None else om.los_fields_create(lr)
    assert (nav.los_fields_create(lr) == exp_los).all()
    if ref is not None:
        ref.close()


def test_pool_request_path_golden(nav):
    """N_RequestPath end to end on the device: route on the host (cost-faithful), fields built into the
    pool by the kernels; (chunk -> ff_id) mapping, flow and chained LOS fields equal the reference's cache"""
    g = gold("route_3x3")
    for k in range(2):
        _upload(nav, 3, 3, g[f"cost{k}"])
        nav.map_build_nav(0); nav.route_build(0)
        for i, (src, dst) in enumerate(g[f"pairs{k}"]):
            nav.pool_create(1, 9)                      # cold cache per request, like the fixture
            ok, did, nf, nl = nav.pool_request_path(0, tuple(src), tuple(dst))
            assert ok == bool(g[f"ok{k}"][i])
            if not ok:
                continue
            assert did == int(g[f"did{k}"][i])
            for c in range(9):
                f, l, ffid = nav.pool_get(0, (c // 3, c % 3))
                assert (f is not None) == bool(g[f"has{k}"][i][c] & 1) and (l is not None) == bool(g[f"has{k}"][i][c] & 2)
                if f is not None:
                    assert ffid == int(g[f"ffid{k}"][i][c]) and (f == g[f"flow{k}"][i][c]).all()
                if l is not None:
                    assert (l == g[f"los{k}"][i][c]).all()
        # warm cache: a second request from another source reuses / merges into the cached fields
        nav.pool_create(1, 9)
        (s0, d0), (s1, _) = g[f"pairs{k}"][0], g[f"pairs{k}"][1]
        ok0, _, nf0, nl0 = nav.pool_request_path(0, tuple(s0), tuple(d0))
        ok1, _, nf1, nl1 = nav.pool_request_path(0, tuple(s0), tuple(d0))
        assert ok0 == ok1 and nf1 == 0 and nl1 == 0          # everything cached the second time


def test_pool_request_goals_vs_port(nav, pforacle):
    """batched goal requests (flow waves + dependency-scheduled LOS chains straight into the pool), the
    resident-plan fast path on a repeated batch, and invalidation of that plan when the map changes"""
    cw = ch = 4
    p = cases.noise_map(cw, ch, 95, 0.1)
    cost = synth.cost_from_pathable(p, cw, ch)
    _upload(nav, cw, ch, cost)
    nav.map_build_nav(0)
    liid = nav.local_islands(0)
    om = pforacle.OracleMap(cw, ch, cost, None, liid)
    rng = np.random.default_rng(95)
    tiles = synth.random_passable_tiles(cost, 5, rng)
    targets = np.array([[int(t[0]) // cw, int(t[0]) % cw, int(t[1]), int(t[2])] for t in tiles], np.int32)
    nav.pool_create(5, 5 * cw * ch)

    def expected(om_):
        exp = []
        for d in range(5):
            fr, fc, fw, lr, lc = nav.plan_goal(tuple(int(v) for v in targets[d]))
            fields = {}
            for w in range(int(fw.max()) + 1):
                sel = np.nonzero(fw == w)[0]
                base = np.stack([fields.get(int(fc[i]), np.zeros((64, 64), np.uint8)) for i in sel])
                out = om_.flow_fields_update(fr[sel], inout=base)
                for k, i in enumerate(sel):
                    fields[int(fc[i])] = out[k]
            los = om_.los_fields_create(lr)
            exp.append((fields, {int(lc[k]): los[k] for k in range(len(lr))}))
        return exp

    def check(exp):
        for d in range(5):
            for c in range(cw * ch):
                f, l, _ = nav.pool_get(d, (c // cw, c % cw))
                assert (f is not None) == (c in exp[d][0]) and (l is not None) == (c in exp[d][1])
                if f is not None:
                    assert (f == exp[d][0][c]).all()
                if l is not None:
                    assert (l == exp[d][1][c]).all()

    exp = expected(om)
    for _ in range(3):                                   # 2nd and 3rd call take the resident-plan path
        nf, nl = nav.pool_request_goals(np.arange(5, dtype=np.int32), targets)
        assert nf >= 5 and nl >= 5
        check(exp)
    # block a band of tiles in one chunk: islands change, the resident plan must be dropped
    blk = np.zeros((64, 64), np.uint16); blk[20:23, 5:60] = 1
    nav.map_update_chunk(0, (1, 1), None, blk, None)
    nav.map_refresh_chunk(0, (1, 1))
    blk_all = np.zeros(cost.shape, np.uint16); blk_all[1 * cw + 1] = blk
    om2 = pforacle.OracleMap(cw, ch, cost, blk_all, nav.local_islands(0))
    nav.pool_create(5, 5 * cw * ch)
    nav.pool_request_goals(np.arange(5, dtype=np.int32), targets)
    check(expected(om2))


# ------------------------------------------------------------------ full-size properties (BASELINE configs[1])
FD_STEP = {1: (-1, -1), 2: (-1, 0), 3: (-1, 1), 4: (0, -1), 5: (0, 1), 6: (1, -1), 7: (1, 0), 8: (1, 1)}


def test_full_size_goal_properties(nav):
    """1024x1024 tiles (16x16 chunks): following the flow from any reached tile arrives at the goal
    without ever stepping on an impassable tile; rebuilding is idempotent; LOS visibility only on
    passable tiles and never within 1 tile of a wavefront-blocked tile."""
    import torch
    cw = ch = 16
    p = synth.make_map(cw, ch, 0x5EED0001)
    cost = synth.cost_from_pathable(p, cw, ch)
    _upload(nav, cw, ch, cost)
    nav.map_build_nav(0)
    img = synth.blocked_to_image(cost, cw, ch)
    passable = np.argwhere(img != 255)
    gr, gc = [int(v) for v in passable[len(passable) // 3]]
    td = (gr // 64, gc // 64, gr % 64, gc % 64)
    nav.pool_create(1, 256)
    nf, nl = nav.pool_request_goal(0, td)
    torch.cuda.synchronize()
    fr, fc, fw, lr, lc = nav.plan_goal(td)
    assert nf == len(fr) and nl == len(lr) and nl == len(np.unique(fc))
    # read the pool back through the host API by recomputing with the host-buffer entry points
    flows = {}
    for w in range(int(fw.max()) + 1):
        sel = np.nonzero(fw == w)[0]
        base = np.stack([flows.get(int(fc[i]), np.zeros((64, 64), np.uint8)) for i in sel])
        out = nav.flow_fields_update(fr[sel], inout=base)
        for k, i in enumerate(sel):
            flows[int(fc[i])] = out[k]
    # idempotence
    sel = np.nonzero(fw == 0)[0]
    again = nav.flow_fields_update(fr[sel])
    if int(fw.max()) == 0:
        for k, i in enumerate(sel):
            assert (again[k] == flows[int(fc[i])]).all()
    field = np.zeros((ch * 64, cw * 64), np.uint8)
    for c, f in flows.items():
        field[(c // cw) * 64:(c // cw) * 64 + 64, (c % cw) * 64:(c % cw) * 64 + 64] = f
    rng = np.random.default_rng(1)
    starts = passable[rng.integers(0, len(passable), 300)]
    arrived = 0
    for r, c in starts:
        r, c = int(r), int(c)
        if field[r, c] == 0 and (r, c) != (gr, gc):
            continue                                   # not connected to the goal
        for _ in range(8 * 1024):
            if (r, c) == (gr, gc):
                arrived += 1
                break
            d = int(field[r, c])
            assert d != 0, "flow led to a tile without direction"
            r += FD_STEP[d][0]; c += FD_STEP[d][1]
            assert 0 <= r < ch * 64 and 0 <= c < cw * 64 and img[r, c] != 255, "flow left passable ground"
        else:
            raise AssertionError("flow did not reach the goal")
    assert arrived > 100
    los = nav.los_fields_create(lr)
    for k in range(len(lr)):
        c = int(lc[k])
        cimg = cost[c]
        vis, blk = los[k] & 1, (los[k] >> 1) & 1
        assert not (vis & (cimg == 255)).any()
        dil = np.zeros((66, 66), np.uint8)
        for dr in range(3):
            for dc in range(3):
                dil[dr:dr + 64, dc:dc + 64] |= blk
        assert not (vis & dil[1:65, 1:65]).any()
    assert (los[0] & 1).sum() > 0


def test_full_size_agents_properties(nav):
    """100k agents on the 1024^2 map: speed clamp, finite outputs, work-list order, determinism"""
    cw = ch = 16
    p = synth.make_map(cw, ch, 0x5EED0001)
    cost = synth.cost_from_pathable(p, cw, ch)
    _upload(nav, cw, ch, cost)
    a = synth.make_agents(cost, cw, ch, 100_000, 16, 0x5EED0001, radius=1.0, spacing=2.6)
    rng = np.random.default_rng(2)
    a["vdes"] = rng.normal(size=(100_000, 2)).astype(np.float32)
    a["vdes"] /= np.linalg.norm(a["vdes"], axis=1, keepdims=True)
    rec, fl = capi.pack_agents(a)
    nav.agents_upload(rec, fl, 20)
    work = np.arange(0, 100_000, 7, dtype=np.uint32)
    nav.agents_set_work(work)
    nav.agents_tick(0)
    v1 = nav.agents_read_velocities(len(work))
    nav.agents_tick(0)
    v2 = nav.agents_read_velocities(len(work))
    assert np.isfinite(v1).all()
    assert (v1 == v2).all(), "tick is not deterministic"
    assert (np.linalg.norm(v1, axis=1) <= 20.0 / 20 * (1 + 1e-5)).all()      # truncate(max_speed / hz)
    # neighbour query: inclusive int64 distance test, ids unique, all within range
    i = 12345
    ids = nav.ents_in_circle(float(a["pos"][i, 0]), float(a["pos"][i, 1]), 30.0, 512)
    assert len(np.unique(ids)) == len(ids) and i in ids
    d = np.linalg.norm(a["pos"][ids] - a["pos"][i], axis=1)
    assert (d <= 30.0 + 1e-2).all()


def test_cost_from_tiles_golden(nav, pforacle):
    """a-11: n_set_cost_for_tile + n_make_cliff_edges on the device, every tile type; then the
    structural build (local islands, portals) on top of the device-made costs."""
    g = gold("tiles")
    for k, (cw, ch) in enumerate(((2, 2), (3, 2))):
        t = g[f"tiles{k}"].astype(np.int32)
        nav.map_create(cw, ch, 4)
        for slot, layer in enumerate((0, 3, 4, 8)):
            nav.map_cost_from_tiles(slot, layer, t)
            cost, blk, _ = nav.map_get_layer(slot)
            assert (cost == g[f"cost{k}_{layer}"]).all(), (k, layer)
            assert (cost == pforacle.cost_from_tiles(cw, ch, t, layer)).all()
            assert not blk.any()
        nav.map_build_nav(0)
        assert (nav.local_islands(0) == g[f"liid{k}"]).all()
        ports = nav.portals(0)
        assert len(ports) == len(g[f"portals{k}"])
        assert (ports[:, :9] == g[f"portals{k}"][:, :9]).all()


@pytest.mark.parametrize("name", ["update_hz20", "update_hz10"])
def test_entity_update_golden(nav, name):
    """a-8: entity_compute_update patches (movement.c:2303) and the movestate part of entity_apply_update
    (movement.c:2693) against the compiled reference: flags / states identical, floats within 1e-4."""
    g = gold(name)
    hz = int(g["hz"])
    a = _agents_from_gold(g)
    rec, fl = capi.pack_agents(a)
    ms = g["ms"].view(capi.MOVESTATE)
    work = g["work"]
    nav.map_create(3, 3, 1); nav.map_upload_layer(0, g["cost"]); nav.map_build_nav(0); nav.route_build(0)
    nav.agents_upload(rec, fl, hz)
    nav.agents_upload_movestate(ms)
    nav.agents_set_work(work)
    nav.agents_tick(0)
    vel = nav.agents_read_velocities(len(work))
    assert cases.relerr(vel, g["vel"]).max() <= VEL_RTOL
    nav.agents_compute_updates()
    p = nav.agents_read_patches(len(work))
    oi, of = g["patch_i"], g["patch_f"]
    # discrete outcome (flags, next state, blocking): identical for EVERY work item
    same = (p["flags"] == oi[:, 0].astype(np.uint32)) & (p["next_state"] == oi[:, 1]) & (p["next_block"] == oi[:, 2])
    assert same.all(), np.nonzero(~same)[0][:10]
    sel = same
    got = np.concatenate([p["next_velocity"], p["next_pos"], p["next_rot"], p["next_ppos"], p["next_npos"],
                          p["next_step"][:, None], p["next_left"][:, None], p["next_nrot"], p["next_prot"]], axis=1)
    exp = of[:, :25]
    err = np.abs(got[sel] - exp[sel]) / np.maximum(np.abs(exp[sel]), 1.0)
    assert err.max() <= 1e-4, (err.max(), np.unravel_index(err.argmax(), err.shape))
    # every transition kind is present in the fixture
    assert {-1, 2, 4} <= set(np.unique(oi[:, 1]).tolist())
    # device-side apply: velocity history + interpolation fields
    nav.agents_apply_updates()
    a2, ms2 = nav.agents_read_state(len(rec))
    herr = np.abs(ms2["vel_hist"][work][sel] - g["hist"][sel]).max()
    assert herr <= 1e-4, herr
    assert (ms2["vel_hist_idx"][work][sel] == g["hidx"][sel]).all()
    setpos = sel & ((oi[:, 0] & 4) != 0) & ((a["flags"][work] & capi.FLAG_GARRISONED) == 0)
    assert np.abs(a2["pos"][work][setpos] - of[setpos][:, [2, 4]]).max() <= 1e-3
    # entity_apply_update skips garrisoned entities altogether (movement.c:2697)
    garr = (a["flags"][work] & capi.FLAG_GARRISONED) != 0
    setst = sel & ((oi[:, 0] & 1) != 0) & ~garr
    assert (a2["state"][work][setst] == oi[setst, 1]).all()
    assert (a2["state"][work][garr] == a["state"][work][garr]).all()


def test_repair_chain_golden(nav, pforacle):
    """a-4: the on-miss repair chain of N_DesiredPointSeekVelocity (nav.c:3508-3554): both field updates, tile and
    portal targets, on a map whose local islands were cut by blockers -- bit-exact vs the compiled reference."""
    g = gold("repair")
    nav.map_create(2, 2, 1)
    nav.map_upload_layer(0, g["cost"], g["blk"], g["liid"])
    nav.map_build_nav(0); nav.route_build(0)
    assert (nav.local_islands(0) == g["liid"]).all()
    T = g["targets"].view(capi.FIELD_REQ)
    got = nav.flow_fields_repair(T, g["kinds"], g["args"], g["base"])
    bad = np.nonzero((got != g["exp"]).reshape(len(T), -1).any(axis=1))[0]
    assert len(bad) == 0, (bad[:10], g["kinds"][bad[:10]])


@pytest.mark.parametrize("seed", [41, 42])
def test_repair_chain_vs_port(nav, pforacle, seed):
    """pfnav_flow_fields_repair against the plain-C port (field.c:2247, 2307) on maps whose blockers were committed
    through the device: both kinds, tile targets (passable and blocked) and portal targets, every chunk, many start
    tiles and islands. Blocker operations queued after the commit do not reach the repair: kind-0 seeds are flooded
    on the device images, the start check and kind-1 seeds come from the host mirrors, and both are the committed map."""
    cw, ch = 3, 2
    rng = np.random.default_rng(seed)
    cost = synth.cost_from_pathable(cases.noise_map(cw, ch, seed, 0.2), cw, ch)
    nav.map_create(cw, ch, 1)
    nav.map_upload_layer(0, cost)
    nav.map_build_nav(0)

    def place_blockers(n):
        for _ in range(n):
            nav.blockers_incref(float(-rng.uniform(10, cw * 256 - 10)), float(rng.uniform(10, ch * 256 - 10)),
                                float(rng.uniform(2, 16)), 0, 0)

    place_blockers(70)
    assert nav.map_commit() > 0
    nav.route_build(0)
    blk, liid, gisl = nav.blockers(0), nav.local_islands(0), nav.route_islands(0)
    om = pforacle.OracleMap(cw, ch, cost, blk, liid)
    specs = cases.portal_specs(nav.portals(0), liid, cw)
    T, K, A, B, E = [], [], [], [], []
    for chunk in range(cw * ch):
        cr, cc = divmod(chunk, cw)
        free = np.argwhere((cost[chunk] != 255) & (blk[chunk] == 0))
        blocked = np.argwhere((cost[chunk] != 255) & (blk[chunk] > 0))
        nonp = np.argwhere((cost[chunk] == 255) | (blk[chunk] > 0))
        reqs = [capi.tile_req((cr, cc), tuple(int(v) for v in t[rng.integers(len(t))])) for t in (free, blocked) if len(t)]
        reqs += [cases.portal_reqs([s]) for s in specs if s[0] == (cr, cc)][:3]
        iids = [int(i) for i in np.unique(liid[chunk]) if i != 0xFFFF]
        for q in reqs:
            base = om.flow_fields_update(q)[0]
            for s in nonp[rng.integers(0, len(nonp), 8)] if len(nonp) else []:
                T.append(q); K.append(0); A.append((int(s[0]) << 8) | int(s[1])); B.append(base)
                E.append(om.flow_nearest_pathable((cr, cc), (int(s[0]), int(s[1])), base))
            for iid in iids[:8]:
                T.append(q); K.append(1); A.append(iid); B.append(base)
                E.append(om.flow_island_to_nearest(gisl, q, iid, base))
    T, K, A, B, E = np.concatenate(T), np.array(K, np.int32), np.array(A, np.int32), np.stack(B), np.stack(E)
    assert (T["target_type"] == capi.TARGET_PORTAL).any() and (K == 0).any() and (K == 1).any()
    assert (B != E).any()
    place_blockers(30)                                   # queued, not committed
    got = nav.flow_fields_repair(T, K, A, B)
    bad = np.nonzero((got != E).reshape(len(T), -1).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), len(T), bad[:10], K[bad[:10]])


def test_pool_repair_chain_golden(nav):
    """a-4 end to end: N_DesiredPointSeekVelocity's on-miss chain (nav.c:3484-3554) against the device pool.
    Entities on blocked tiles, inside walls, on islands cut off by blockers and in chunks the first request never
    touched; steady-state answers equal the reference's bit for bit."""
    g = gold("repair_pool")
    pos, target = g["pos"], g["target"]
    n = len(pos)
    nav.map_create(2, 2, 1)
    nav.map_upload_layer(0, g["cost"], g["blk"], g["liid"])
    nav.map_build_nav(0); nav.route_build(0)
    nav.pool_create(1, 8)
    ok, did, nf, nl = nav.pool_request_path(0, (float(pos[0, 0]), float(pos[0, 1])), (float(target[0]), float(target[1])))
    assert ok and did == int(g["did"])
    rec = np.zeros(n, capi.AGENT)
    rec["pos"] = pos; rec["prev_pos"] = pos; rec["radius"] = 1.0; rec["max_speed"] = 20.0; rec["speed"] = 20.0
    rec["flags"] = capi.FLAG_MOVABLE; rec["flock"] = 0
    fl = np.zeros(1, capi.FLOCK); fl["target"] = target; fl["dest"] = 0; fl["layer"] = 0
    nav.agents_upload(rec, fl, 20)
    nav.agents_set_work(np.arange(n, dtype=np.uint32))
    total = 0
    for _ in range(4):
        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        nreq, nrep = nav.pool_repair()
        total += nreq + nrep
        if nreq + nrep == 0:
            break
    assert total > 0
    nav.agents_tick(capi.TICK_VDES_FROM_POOL)
    _, vdes, los = nav.agents_read_debug(n)
    bad = np.nonzero((vdes != g["vdes"]).any(axis=1))[0]
    assert len(bad) == 0, (len(bad), bad[:10], vdes[bad[:5]], g["vdes"][bad[:5]])
    assert (los == g["los"]).all()


def test_faction_fields_golden(nav):
    """"attacking" requests (N_RequestPathAttacking): flow + LOS fields over per-faction blocker refcounts, first with
    the reference's counts uploaded, then with the counts rebuilt by pfnav_blockers_incref(faction) + pfnav_map_commit"""
    g = gold("faction")
    treq, preq, lreq = g["treq"].view(capi.FIELD_REQ), g["preq"].view(capi.FIELD_REQ), g["lreq"].view(capi.LOS_REQ)
    for mode in ("upload", "incref"):
        nav.map_create(2, 2, 1)
        for f in range(15):
            nav.set_enemy_factions(f, int(g["enemies"][f]))
        if mode == "upload":
            nav.map_upload_layer(0, g["cost"], g["blk"], g["liid"])
            nav.map_upload_factions(0, g["factions"])
        else:
            nav.map_upload_layer(0, g["cost"]); nav.map_build_nav(0)
            for x, z, r, f in g["blockers"]:
                nav.blockers_incref(float(x), float(z), float(r), int(f), 0)
            nav.map_commit()
            assert (nav.blockers(0) == g["blk"]).all() and (nav.local_islands(0) == g["liid"]).all()
        assert (nav.flow_fields_update(treq) == g["texp"]).all(), mode
        assert (nav.flow_fields_update(preq) == g["pexp"]).all(), mode
        assert (nav.los_fields_create(lreq) == g["lexp"]).all(), mode
    # a faction id without an enemy table is refused, not guessed
    nav2_req = treq[:1].copy(); nav2_req["faction_id"] = 20
    with pytest.raises(Exception):
        nav.flow_fields_update(nav2_req)


@pytest.mark.parametrize("name,cw", [("agents_dense", 1), ("agents_3x3", 3), ("update_hz20", 3)])
def test_two_phase_velocity_update_is_bit_identical(nav, name, cw):
    """the split velocity update (phase A before the field join, phase B after) returns exactly what the single
    pass returns -- and both match the reference -- including agents with no admissible velocity, COMBAT_HELD
    and GARRISONED entities"""
    g = gold(name)
    a = _agents_from_gold(g)
    rec, fl = capi.pack_agents(a)
    _upload(nav, cw, cw, g["cost"])
    out = {}
    try:
        for mode in (0, 2):
            nav.set_two_phase(mode)
            nav.agents_upload(rec, fl, 20)
            nav.agents_set_work(g["work"])
            nav.agents_tick(0)
            out[mode] = (nav.agents_read_velocities(len(g["work"])), nav.agents_read_debug(len(g["work"]))[0])
    finally:
        nav.set_two_phase(1)
    assert (out[0][0] == out[2][0]).all() and (out[0][1] == out[2][1]).all()
    assert cases.relerr(out[2][0], g["vel"]).max() <= VEL_RTOL


def test_los_with_caller_held_prev_field(nav):
    """N_LOSFieldCreate(..., prev) one field at a time, the previous chunk's field held by the caller
    (PFNAV_LOS_PREV_INPLACE), equals the chained batch -- and the golden fields"""
    g = gold("portal_los")
    _upload(nav, 3, 3, g["cost"])
    reqs = g["los_reqs"].view(capi.LOS_REQ)
    exp = g["los_exp"]
    done = 0
    for i in range(len(reqs)):
        q = reqs[i:i + 1].copy()
        if q["prev_index"][0] < 0:
            got = nav.los_fields_create(q)[0]
        else:
            p = int(q["prev_index"][0])
            q["prev_index"] = capi.LOS_PREV_INPLACE
            got = nav.los_fields_create(q, prev_fields={0: exp[p]})[0]
            done += 1
        assert (got == exp[i]).all(), i
    assert done > 0


# ------------------------------------------------------------------ region ("cell arrival") fields
def _region_map(nav, g):
    nav.map_create(3, 3, 1)
    nav.map_upload_layer(0, g["cost"], g["blk"])
    nav.map_upload_factions(0, g["factions"])


@pytest.mark.parametrize("dim", [96, 32])
def test_region_fields_golden(nav, dim):
    """N_CellArrivalFieldCreate [+ N_CellArrivalFieldUpdateToNearestPathable] and N_GroupArrivalFieldCreate
    (field.c:2445, 2603, 2525) vs the compiled reference: one batched launch, bit-exact packed directions"""
    g = gold("region")
    _region_map(nav, g)
    reqs = cases.region_reqs_from_golden(g["req%d" % dim], g["ov%d" % dim])
    got = nav.region_fields(dim, reqs)
    bad = [i for i in range(len(reqs)) if (got[i] != g["exp%d" % dim][i]).any()]
    assert not bad, bad
    # create alone, then the fix-up in place on the caller's field (the reference's two separate calls)
    create = nav.region_fields(dim, [dict(q, start=None) for q in reqs])
    assert (create == g["create%d" % dim]).all()
    fix = [i for i, q in enumerate(reqs) if q["start"] is not None]
    upd = nav.region_fields(dim, [dict(reqs[i], no_create=True) for i in fix], inout=create[fix])
    assert (upd == g["exp%d" % dim][fix]).all()
    for k in range(len(g["gx%d" % dim])):
        f = nav.group_arrival_field(dim, g["gt%d" % dim][k], g["gc%d" % dim][k], int(g["ge%d" % dim][k]))
        assert (f == g["gx%d" % dim][k]).all(), k


def test_region_fields_vs_port(nav, pforacle):
    """a formation-sized batch (one 96 x 96 field per cell, formation.c:3152) on a 4 x 4-chunk map vs the port;
    dims 96, 64 and 128 (PFNAV_REGION_DIM_MAX)"""
    cw = ch = 4
    for seed, dim, n in ((91, 96, 300), (92, 64, 64), (93, 128, 24)):
        p, blockers, wars, reqs = cases.region_case(seed, cw, ch, n, dim)
        cost = synth.cost_from_pathable(p, cw, ch)
        nav.map_create(cw, ch, 1)
        nav.map_upload_layer(0, cost); nav.map_build_nav(0)
        enemies = np.zeros(16, np.uint16)
        for a, b in wars:
            enemies[a] |= 1 << b; enemies[b] |= 1 << a
        for f in range(15):
            nav.set_enemy_factions(f, int(enemies[f]))
        for x, z, r, f in blockers:
            nav.blockers_incref(float(x), float(z), float(r), int(f), 0)
        nav.map_commit()
        blk = nav.blockers(0)
        fac = nav.faction_counts(0)         # nav_chunk::factions as counted by pfnav_blockers_incref (pinned by faction.npz)
        cases.region_pick_starts(reqs, cost, blk, cw, ch, seed, dim)
        om = pforacle.OracleMap(cw, ch, cost, blk, None, factions=fac)
        got = nav.region_fields(dim, reqs)
        for i, q in enumerate(reqs):
            e = om.region_field_create(dim, q["enemies"], 1, [q["target"]], q["center"], q["overlay"])
            if q["start"] is not None:
                e = om.region_field_fixup(dim, q["start"], q["center"], e, q["overlay"])
            assert (got[i] == e).all(), (seed, dim, i, q)
        # many seeds per field (tile-space group arrival), no base shift
        rng = np.random.default_rng(seed)
        greqs = []
        for q in reqs[:16]:
            sd = np.stack([rng.integers(0, ch * 64, 20), rng.integers(0, cw * 64, 20)], 1)
            greqs.append(dict(center=q["center"], seeds=sd, enemies=q["enemies"], overlay=q["overlay"], start=None, cell=False))
        gg = nav.region_fields(dim, greqs)
        for i, q in enumerate(greqs):
            assert (gg[i] == om.region_field_create(dim, q["enemies"], 0, q["seeds"], q["center"], q["overlay"])).all(), (seed, i)


def test_region_fields_argument_errors(nav):
    g = gold("region")
    _region_map(nav, g)
    ok = dict(center=(96, 96), target=(100, 100), enemies=0, overlay=None, start=None)
    assert nav.region_fields(96, [ok]).shape == (1, 96, 48)
    with pytest.raises(Exception):
        nav.region_fields(95, [ok])                                        # odd dim
    with pytest.raises(Exception):
        nav.region_fields(130, [ok])                                       # > PFNAV_REGION_DIM_MAX
    with pytest.raises(Exception):
        nav.region_fields(96, [dict(ok, center=(400, 10))])                # centre outside the map
    with pytest.raises(Exception):
        nav.region_fields(96, [dict(ok, target=(10, 100))])                # cell tile before the region base
    with pytest.raises(Exception):
        nav.region_fields(96, [dict(ok, start=(190, 190))])                # fix-up start outside the clamped region
    with pytest.raises(Exception):
        nav.region_fields(96, [dict(ok, seeds=[(100, 100), (101, 101)], cell=True)])
    assert nav.region_fields(96, []).shape == (0, 96, 48)


def test_zone_fields_and_group_arrival_golden(nav):
    """TARGET_ZONE chunk fields (seeds on the host in the reference's heap order, integration on the device) and
    N_DesiredGroupArrivalVelocity out of the pool, vs the compiled reference"""
    g = gold("region")
    cw = ch = 3
    _region_map(nav, g)
    allchunks = [(c // cw, c % cw) for c in range(cw * ch)]
    for k in range(len(g["zc"])):
        got = nav.zone_fields(g["zc"][k], int(g["zrad"][k]), allchunks)
        bad = [c for c in range(cw * ch) if (got[c] != g["zexp"][k, c]).any()]
        assert not bad, (k, bad)
    nav.pool_create(8, 64)
    for k in range(len(g["gv_radius"])):
        n = nav.pool_request_zone(k, g["gv_centre"][k], int(g["gv_radius"][k]))
        assert n == int(g["gv_nfields"][k]), k
        v, f = nav.group_arrival_velocity(k, g["gv_centre"][k], int(g["gv_radius"][k]), g["gv_pos"][k])
        assert (f == g["gv_flags"][k]).all(), k
        assert (v == g["gv_vel"][k]).all(), k
    # a destination without zone fields: every call "returns false"
    v, f = nav.group_arrival_velocity(7, g["gv_centre"][1], int(g["gv_radius"][1]), g["gv_pos"][1])
    assert not f.any() and not v.any()


def test_demo_map_pfmap_ingestion_golden(nav):
    """SURVEY 8f-4: the engine's demo map as PFMAP text -> pfnav_map_load_pfmap (parse, device cost pass for five
    reference layers, islands, portals) -> N_RequestPath into the pool; everything equals the reference's build"""
    g = gold("demo_map")
    text = capi.pfmap_write(g["tiles"].astype(np.int32), version="1.2")
    layers = (0, 1, 3, 4, 8)
    nav.map_load_pfmap(text, layers)
    for slot, layer in enumerate(layers):
        cost, blk, _ = nav.map_get_layer(slot)
        assert (cost == g["cost_%d" % layer]).all(), layer
        assert not blk.any()
    assert (nav.local_islands(0) == g["liid_0"]).all()
    assert (nav.portals(0)[:, :9] == g["portals_0"][:, :9]).all()
    nav.route_build(0)
    for i, (src, dst) in enumerate(g["pairs"]):
        nav.pool_create(1, 16)
        ok, did, nf, nl = nav.pool_request_path(0, tuple(src), tuple(dst))
        assert ok == bool(g["ok"][i]) and (not ok or did == int(g["did"][i]))
        for c in range(16):
            f, l, ffid = nav.pool_get(0, (c // 4, c % 4))
            assert (f is not None) == bool(g["has"][i][c] & 1) and (l is not None) == bool(g["has"][i][c] & 2), (i, c)
            if f is not None:
                assert ffid == int(g["ffid"][i][c]) and (f == g["flow"][i][c]).all(), (i, c)
            if l is not None:
                assert (l == g["los"][i][c]).all(), (i, c)


def test_entity_and_enemies_fields_golden(nav):
    """N_FlowFieldUpdate with TARGET_ENTITY / TARGET_ENEMIES (field.c:2040-2048) on reference layers 0 and 2: every
    chunk of the map in one launch per target, vs the compiled reference"""
    g = gold("targets")
    cw = ch = 3
    wars = [tuple(w) for w in g["wars"]]
    allchunks = [(c // cw, c % cw) for c in range(cw * ch)]
    nav.map_create(cw, ch, 2)
    for slot, L in enumerate((0, 2)):
        nav.map_upload_layer(slot, g["cost_%d" % L], g["blk_%d" % L])
    fp = nav.footprints(g["pos"], g["radius"])
    for slot, L in enumerate((0, 2)):
        for k, u in enumerate(g["uids"]):
            got = nav.entity_fields(capi.TARGET_ENTITY, fp[u:u + 1], allchunks, layer=slot, ref_layer=L)
            assert (got == g["ent_%d" % L][k]).all(), (L, u)
        for f in range(4):
            sel = cases.enemies_of(f, wars, g["factions"], g["flags"])
            got = nav.entity_fields(capi.TARGET_ENEMIES, fp[sel], allchunks, layer=slot, ref_layer=L)
            assert (got == g["foe_%d" % L][f]).all(), (L, f)


def test_stress_scenario_golden(nav):
    """the reference's stress test layout on its plain map centred at the origin (map position (+512, -512)): PFMAP
    ingestion, both path requests into the pool, one tick with vdes / LOS from the pool, vs the compiled reference"""
    g = gold("stress")
    mx, mz = [float(v) for v in g["map_origin"]]
    nav.map_load_pfmap(capi.pfmap_write(g["tiles"].astype(np.int32)), (0,), mx, mz)
    cost, _, liid = nav.map_get_layer(0)
    assert (cost == g["cost"]).all() and (liid == g["liid"]).all()
    nav.route_build(0)
    nav.pool_create(2, 32)
    for f, (src, dst) in enumerate(g["pairs"]):
        ok, did, nf, nl = nav.pool_request_path(f, tuple(src), tuple(dst))
        assert ok and did == int(g["did"][f])
        for c in range(16):
            fl_, lo_, ffid = nav.pool_get(f, (c // 4, c % 4))
            assert (fl_ is not None) == bool(g["has"][f][c] & 1) and (lo_ is not None) == bool(g["has"][f][c] & 2), (f, c)
            if fl_ is not None:
                assert ffid == int(g["ffid"][f][c]) and (fl_ == g["flow"][f][c]).all(), (f, c)
            if lo_ is not None:
                assert (lo_ == g["los_f"][f][c]).all(), (f, c)
    # the tick reads the SETTLED field cache of the reference (its per-unit on-miss requests have added the chunks the
    # two requests above never touched): first put exactly those fields, then let the on-miss chain rebuild them
    a = {k[2:]: g[k] for k in g.files if k.startswith("a_")}
    rec, fl = capi.pack_agents(a)
    n = len(g["work"])

    def tick_and_check(tag):
        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        vel = nav.agents_read_velocities(n)
        vpref, vdes, los = nav.agents_read_debug(n)
        assert (los == g["los"]).all(), tag
        assert (vdes == g["vdes"]).all(), tag
        assert (cases.relerr(vpref, g["vpref"]) <= VEL_RTOL).all(), tag
        assert cases.relerr(vel, g["vel"]).max() <= VEL_RTOL, tag

    nav.pool_create(2, 32)
    for k, (f, cr, cc, hf, hl) in enumerate(g["pool_chunks"]):
        nav.pool_put(int(f), (int(cr), int(cc)), g["pool_flow"][k] if hf else None, g["pool_los"][k] if hl else None)
    nav.agents_upload(rec, fl, 20)
    nav.agents_set_work(g["work"])
    tick_and_check("settled cache put")
    nav.pool_create(2, 32)
    for f, (src, dst) in enumerate(g["pairs"]):
        assert nav.pool_request_path(f, tuple(src), tuple(dst))[0]
    for _ in range(6):
        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        nreq, nrep = nav.pool_repair()
        if nreq + nrep == 0:
            break
    for k, (f, cr, cc, hf, hl) in enumerate(g["pool_chunks"]):
        fl_, lo_, _ = nav.pool_get(int(f), (int(cr), int(cc)))
        assert (fl_ is not None) == bool(hf) and (lo_ is not None) == bool(hl), (f, cr, cc)
        assert (not hf or (fl_ == g["pool_flow"][k]).all()) and (not hl or (lo_ == g["pool_los"][k]).all()), (f, cr, cc)
    tick_and_check("on-miss chain")


def test_los_blocked_destination_tile(nav, pforacle):
    """the destination tile itself is blocked: its neighbour sees it as a corner and casts the `wavefront blocked` line
    from the tile to ITSELF -- a 0/0 slope whose x86 float->int conversions (INT_MIN) and wrapped error term make the
    reference mark the whole row towards column 0 (field.c:463-517). Found by the link-swap test; the port reproduces it."""
    cw = ch = 3
    p = cases.noise_map(cw, ch, 8181, 0.08)
    cost = synth.cost_from_pathable(p, cw, ch)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0)
    rng = np.random.default_rng(8181)
    for _ in range(40):
        x, z, r = float(-rng.uniform(10, cw * 256 - 10)), float(rng.uniform(10, ch * 256 - 10)), float(rng.uniform(2, 9))
        nav.blockers_incref(x, z, r, 0, 0)
    nav.map_commit()
    blk, liid = nav.blockers(0), nav.local_islands(0)
    om = pforacle.OracleMap(cw, ch, cost, blk, liid)
    reqs = []
    for chunk in range(cw * ch):
        for r_, c_ in np.argwhere((cost[chunk] != 255) & (blk[chunk] > 0))[::23][:6]:       # blocked, passable by cost
            td = (chunk // cw, chunk % cw, int(r_), int(c_))
            reqs.append(capi.los_req((td[0], td[1]), td))
    assert len(reqs) >= 12
    reqs = np.concatenate(reqs)
    for variant in (2, 1, 0):
        nav.set_los_variant(variant)
        try:
            got = nav.los_fields_create(reqs)
        finally:
            nav.set_los_variant(2)
        exp = om.los_fields_create(reqs)
        bad = np.nonzero((got != exp).reshape(len(reqs), -1).any(axis=1))[0]
        assert len(bad) == 0, (variant, bad[:10])
    assert ((exp >> 1) & 1).sum() > 100
