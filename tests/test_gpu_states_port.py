"""Every movement state of the device tick against the plain-C port (oracle/pf_oracle.c), never against a recording:
the steering variants of move_velocity_work (point_seek_vpref, enemy_seek_vpref, cell_arrival_seek_vpref,
formation_seek_vpref, movement.c:3414-3448) and entity_compute_update / the movestate part of entity_apply_update for all
nine states (movement.c:2303-2757). The population is test_gpu_states._scenario's: MOVING, MOVING_IN_FORMATION,
ARRIVING_TO_CELL, SEEK_ENEMIES, ENTER_ENTITY_RANGE, TURNING, SURROUND_ENTITY and WAITING units among ARRIVED ones, with
formation inputs and movestate beyond point seeking; here some SURROUND_ENTITY units also have live targets, near and far,
so that the surround-field hysteresis bits are exercised.

For the states beyond point seeking the port follows the structure of the CUDA kernels (no reference source was at hand
when it was written; tests/golden/README.md): this file checks the device against a serial, scalar C statement of the same
rules -- index pre-selection, layer choice, float contraction, races, state carried between ticks -- not reference parity.
tests/test_oracle.py pins the port to the reference where oracle/_ref is built.

Tolerances: integer outputs (flags, next_state, next_block, wait ticks, engine_todo) equal; preferred velocities and
velocities within 1e-4 relative or one float spacing of the entity's position (cases.vel_ok, DESIGN.md deviation 7), the
uses of that floor bounded as in the trajectory test; patch floats and the state after the apply within 1e-4 of
max(|x|, 1)."""
import numpy as np
import pytest

import cases
from test_gpu_states import (ST_ARRIVED, ST_CELL, ST_ENTER, ST_FORMATION, ST_MOVING, ST_SEEK, ST_SURROUND, ST_TURNING,
                             ST_WAITING, _scenario, _spread_states, _work_inputs)

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
SEED = 5151
ALL_STATES = (ST_MOVING, ST_FORMATION, ST_SEEK, ST_WAITING, ST_SURROUND, ST_ENTER, ST_TURNING, ST_CELL)
EXTRA = ("next_dest", "next_target_prev", "next_target_dir")
INTS = ("flags", "next_state", "next_block", "next_attack", "wait_ticks_left", "engine_todo")


def _live_surround(a, ext, seed):
    """give two thirds of the SURROUND_ENTITY units a live target: alternately the nearest other unit, not yet using the
    surround field (inside a third of a chunk: start using it), and a random unit, already using it (mostly beyond half
    a chunk: stop); every fourth near one already uses it too"""
    rng = np.random.default_rng(seed)
    su = np.nonzero(a["state"] == ST_SURROUND)[0]
    live = su[: 2 * len(su) // 3]
    for i, u in enumerate(live):
        if i % 2 == 0:
            d = np.linalg.norm(a["pos"] - a["pos"][u], axis=1); d[u] = np.inf
            ext["surround_target_uid"][u] = np.argmin(d)
            ext["using_surround_field"][u] = 1 if i % 8 == 0 else 0
        else:
            ext["surround_target_uid"][u] = rng.integers(0, len(a["radius"]))
            ext["using_surround_field"][u] = 1


def _records(a, work, vdes, los):
    aa = dict(a)
    n = len(a["radius"])
    aa["vdes"] = np.zeros((n, 2), np.float32); aa["vdes"][work] = vdes
    aa["has_los"] = np.zeros(n, np.uint32); aa["has_los"][work] = los
    rec, fl = capi.pack_agents(aa)
    if "flock_layer" in a:
        fl["layer"] = a["flock_layer"]
    return rec, fl


def _host(cw, ch, costs, map_xz=(0.0, 0.0)):
    host = capi.Nav(hostonly=True)
    host.map_create(cw, ch, len(costs), *map_xz)
    for L, c in enumerate(costs):
        host.map_upload_layer(L, c); host.map_build_nav(L); host.route_build(L)
    return host


def _device_setup(nav, cw, ch, costs, rec, fl, ms, form, ext, hz, map_xz=(0.0, 0.0)):
    nav.map_create(cw, ch, len(costs), *map_xz)
    for L, c in enumerate(costs):
        nav.map_upload_layer(L, c); nav.map_build_nav(L); nav.route_build(L)
    nav.agents_upload(rec, fl, hz)
    nav.agents_upload_movestate(ms)
    nav.agents_upload_formation(form)
    nav.agents_upload_movestate_ext(ext)


def _device_tick(nav, work, n):
    """velocity pass (desired velocities of the records), entity_compute_update, apply -> dict like the port's"""
    nav.agents_set_work(work)
    nav.agents_tick(0)
    vel = nav.agents_read_velocities(len(work))
    vpref, vdes, los = nav.agents_read_debug(len(work))
    nav.agents_compute_updates()
    patches = nav.agents_read_patches(len(work))
    nav.agents_apply_updates()
    agents, ms = nav.agents_read_state(n)
    return dict(vel=vel, vpref=vpref, vdes=vdes, los=los, patches=patches, agents=agents, movestate=ms,
                ext=nav.agents_read_movestate_ext(n))


def _compare(tag, dev, exp, work, pos, pos_tol):
    """device tick vs port tick on identical inputs -> number of uses of the position-ulp floor"""
    assert (dev["vdes"] == exp["vdes"]).all() and (dev["los"] == exp["los"]).all(), tag
    nfloor = 0
    for k in ("vpref", "vel"):
        ok, nf = cases.vel_ok(dev[k], exp[k], pos[work])
        bad = cases.relerr(dev[k], exp[k])
        assert ok, (tag, k, bad.max(), work[np.argmax(bad)])
        nfloor += nf
    pg, pe = dev["patches"], exp["patches"]
    for k in INTS:
        same = pg[k] == pe[k]
        assert same.all(), (tag, k, work[np.nonzero(~same)[0][:10]], pg[k][~same][:5], pe[k][~same][:5])
    fg = np.concatenate([cases.patch_floats(pg)] + [pg[k] for k in EXTRA], axis=1)
    fe = np.concatenate([cases.patch_floats(pe)] + [pe[k] for k in EXTRA], axis=1)
    err = np.abs(fg - fe) / np.maximum(np.abs(fe), 1.0)
    assert err.max() <= 1e-4, (tag, err.max(), np.unravel_index(err.argmax(), err.shape))
    # the state after the apply, whole population
    ga, ea = dev["agents"], exp["agents"]
    assert (ga["state"] == ea["state"]).all(), (tag, np.nonzero(ga["state"] != ea["state"])[0][:10])
    for k in ("pos", "prev_pos"):
        e = np.abs(ga[k] - ea[k]).max(axis=1)
        assert (e <= pos_tol).all(), (tag, k, e.max())
    assert cases.vel_ok(ga["velocity"], ea["velocity"], pos)[0], tag
    gm, em = dev["movestate"], exp["movestate"]
    for k in ("vel_hist_idx", "left", "step"):
        assert (gm[k] == em[k]).all(), (tag, k, np.nonzero(gm[k] != em[k])[0][:10])
    for k in ("vel_hist", "next_rot"):
        e = np.abs(gm[k] - em[k]) / np.maximum(np.abs(em[k]), 1.0)
        assert e.max() <= 1e-4, (tag, k, e.max())
    assert (np.abs(gm["next_pos"] - em["next_pos"]).max(axis=1) <= pos_tol).all(), tag
    gx, ex = dev["ext"], exp["ext"]
    for k in ("wait_prev", "wait_ticks_left", "surround_target_uid", "using_surround_field"):
        assert (gx[k] == ex[k]).all(), (tag, k, np.nonzero(gx[k] != ex[k])[0][:10])
    for k in ("target_range", "target_prev_pos", "target_dir", "rot"):
        e = np.abs(gx[k] - ex[k]) / np.maximum(np.abs(ex[k]), 1.0)
        assert e.max() <= 1e-4, (tag, k, e.max())
    return nfloor


def _coverage(a, work, patches):
    stw = a["state"][work]
    for s_ in ALL_STATES:
        assert (stw == s_).sum() > 10, s_
    nxt = set(np.unique(patches["next_state"]).tolist())
    assert {-1, ST_MOVING, ST_FORMATION, ST_ARRIVED, ST_WAITING, ST_TURNING, ST_CELL} <= nxt, nxt
    for bit in (10, 11, 12, 13, 14):          # SET_DEST, SET_TARGET_PREV, SET_MOVING, SET_TARGET_DIR, TURNING_IN_PLACE
        assert (patches["flags"] & (1 << bit)).any(), bit
    for todo in (capi.TODO_SURROUND_QUERY, capi.TODO_USE_SURROUND_FIELD, capi.TODO_DROP_SURROUND_FIELD):
        assert (patches["engine_todo"] & todo).any(), todo


def _one_tick(nav, hz, tweak=None):
    p, cost, a, ms, form, ext = _scenario(SEED, hz)
    _live_surround(a, ext, SEED)
    work, vdes, los = _work_inputs(a, form)
    if tweak is not None:
        work, vdes, los = tweak(cost, a, ms, form, ext, work, vdes, los)
    rec, fl = _records(a, work, vdes, los)
    host = _host(3, 3, [cost])
    try:
        exp = cases.states_port_tick(host, {0: cases.pforacle_map(3, 3, cost)}, rec, fl, ms, form, ext, work, hz)
    finally:
        host.close()
    _device_setup(nav, 3, 3, [cost], rec, fl, ms, form, ext, hz)
    dev = _device_tick(nav, work, len(rec))
    pos_tol = np.maximum(1e-4 * np.maximum(1.0, a["max_speed"] / hz), np.spacing(np.float32(768.0)))
    nfloor = _compare("hz%d" % hz, dev, exp, work, a["pos"], pos_tol)
    assert nfloor <= 4, nfloor
    return a, work, dev, exp


@pytest.mark.parametrize("hz", [20, 10, 5, 1])
def test_all_states_one_tick_vs_port(nav, hz):
    """one tick of every state at every tick rate: velocities, patches and the state after the device apply"""
    a, work, dev, _ = _one_tick(nav, hz)
    _coverage(a, work, dev["patches"])


def test_all_states_resident_trajectory_vs_port(nav):
    """8 device-resident ticks through the mixed-state population at 10 Hz (interpolation in flight): the device state is
    uploaded once; before every tick the port is re-seeded with the device's state read back (agents, movestates,
    movestate_ext) and the tick is compared on identical inputs. The work list is every unit not ARRIVED."""
    hz, nticks = 10, 8
    p, cost, a, ms, form, ext = _scenario(SEED, hz)
    _live_surround(a, ext, SEED)
    work, vdes, los = _work_inputs(a, form)
    rec, fl = _records(a, work, vdes, los)
    n = len(rec)
    host = _host(3, 3, [cost])
    omap = {0: cases.pforacle_map(3, 3, cost)}
    _device_setup(nav, 3, 3, [cost], rec, fl, ms, form, ext, hz)
    pos_tol = np.maximum(1e-4 * np.maximum(1.0, a["max_speed"] / hz), np.spacing(np.float32(768.0)))
    nfloor, seen = 0, set()
    try:
        for tick in range(nticks):
            seed_a, seed_ms = nav.agents_read_state(n)
            seed_ext = nav.agents_read_movestate_ext(n)
            work = np.nonzero(seed_a["state"] != ST_ARRIVED)[0].astype(np.uint32)
            exp = cases.states_port_tick(host, omap, seed_a, fl, seed_ms, form, seed_ext, work, hz)
            dev = _device_tick(nav, work, n)
            nav.agents_rebuild_index()
            nfloor += _compare("tick %d" % tick, dev, exp, work, seed_a["pos"], pos_tol)
            seen |= set(seed_a["state"][work].tolist())
            seen |= set(dev["patches"]["next_state"].tolist())
    finally:
        host.close()
    assert set(ALL_STATES) | {ST_ARRIVED} <= seen, seen
    assert nfloor <= max(2, nticks // 2), nfloor


# ------------------------------------------------------------------------------------ non-zero layer, offset map
@pytest.mark.parametrize("shape", ["2x5_offset", "5x2_centred"])
def test_all_states_layers_and_offset_vs_port(nav, shape):
    """the same tick on test_gpu_tick_layers' maps: units on every navigation layer (flocks whose fields are on a non-zero
    layer) on a 2 x 5-chunk map at a non-tile-aligned offset and a 5 x 2-chunk map centred at the origin; the port runs
    once per layer in use (cases.port_tick_layers)"""
    import test_gpu_tick_layers as TL
    hz = 20
    case = TL.layer_case(shape, hz)
    cw, ch, map_xz, a, ms, layers = case["cw"], case["ch"], case["map_xz"], case["a"], case["ms"], case["layers"]
    ms["combat_facing"] = cases.dir_quat(np.random.default_rng(3).normal(size=(len(ms), 2)))
    form, ext = _spread_states(a, ms, SEED)
    _live_surround(a, ext, SEED)
    work, vdes, los = _work_inputs(a, form)
    rec, fl = _records(a, work, vdes, los)
    costs = list(case["costs"])
    host = _host(cw, ch, costs, map_xz)
    try:
        omaps = {L: cases.pforacle_map(cw, ch, costs[L], map_xz) for L in range(len(costs))}
        exp = cases.states_port_tick(host, omaps, rec, fl, ms, form, ext, work, hz, layers)
    finally:
        host.close()
    _device_setup(nav, cw, ch, costs, rec, fl, ms, form, ext, hz, map_xz)
    dev = _device_tick(nav, work, len(rec))
    extent = max(abs(map_xz[0]), abs(map_xz[0] - cw * 256.0), abs(map_xz[1]), abs(map_xz[1] + ch * 256.0))
    pos_tol = np.maximum(1e-4 * np.maximum(1.0, a["max_speed"] / hz), np.spacing(np.float32(extent)))
    ok_floor = _compare(shape, dev, exp, work, a["pos"], pos_tol)
    assert ok_floor <= 4, ok_floor
    lw = layers[work]
    assert len(np.unique(lw)) >= 4 and (lw > 0).sum() > 100
    for s_ in ALL_STATES:
        assert ((a["state"][work] == s_) & (lw > 0)).sum() > 0, s_          # every state on a non-zero layer too


# ------------------------------------------------------------------------------------ edge inputs aimed at branches
def _quat_deg(deg):
    """a heading `deg` degrees away from dir_quat((1, 0)) about the y axis"""
    ang = np.deg2rad(deg)
    return cases.dir_quat(np.array([[np.cos(ang), np.sin(ang)]]))[0]


def _free_spots(cost, a, k, seed):
    """k passable tile centres with all eight neighbour tiles passable, > 45 wu from every unit and from each other"""
    rng = np.random.default_rng(seed)
    img = synth.blocked_to_image(cost, 3, 3)
    pas = img != 255
    inner = pas.copy()
    for dr in (-1, 0, 1):
        for dc in (-1, 0, 1):
            inner &= np.roll(np.roll(pas, dr, 0), dc, 1)
    cand = np.argwhere(inner[2:-2, 2:-2]) + 2
    cand = cand[rng.permutation(len(cand))]
    xz = np.stack([-(cand[:, 1] + 0.5) * 4.0, (cand[:, 0] + 0.5) * 4.0], 1).astype(np.float32)
    out = []
    for p in xz:
        if np.min(np.linalg.norm(a["pos"] - p, axis=1)) > 45.0 and all(np.linalg.norm(p - q) > 45.0 for q in out):
            out.append(p)
            if len(out) == k:
                break
    assert len(out) == k
    return np.array(out, np.float32)


# TURNING's completion test `fabs(degrees) <= 5.0f` (movement.c:2611) at its edge: `degrees` is PFM_Quat_PitchDiff in
# degrees, in the reference's float/double arithmetic. Against TURN_TARGET these rotations give exactly 5.0f and the float
# on either side of it (found by a search over float neighbours of a 5-degree rotation; each double value lies at least
# 0.18 of a float spacing inside its float's rounding interval)
TURN_TARGET = np.array([0.0, -0.5, 0.0, 0.8660253882408142], np.float32)
TURN_AT_5 = {"turn_5_below": [0.0, -0.4617488384246826, 0.0, 0.8870097398757935],
             "turn_5_exact": [0.0, -0.46174904704093933, 0.0, 0.8870087265968323],
             "turn_5_above": [0.0, -0.4617490768432617, 0.0, 0.887008547782898]}
# the heading gate (movement.c:2323-2335): units whose facing is `deg` degrees off the desired direction, from rest
# (tolerance 10 degrees) or moving (90 degrees)
GATE = [("gate_%s_%s_%d" % (st, "moving" if mv else "rest", deg), st, mv, deg)
        for st in ("moving", "formation") for mv, deg in ((False, 11), (False, 89), (True, 11), (True, 89), (True, 91))]


def _f32_len(d):
    """v2_len of a float32 difference: the float sum of float squares, square-rooted"""
    d = np.asarray(d, np.float32)
    return np.float32(np.sqrt(np.float64(np.float32(d[0] * d[0]) + np.float32(d[1] * d[1]))))


def test_branch_edges_vs_port(nav):
    """single units at the edges of the state machine's and the steering's branches, each with an assertion that its
    branch was taken, on top of the whole 20 Hz population (compared with the port as in the other tests)"""
    E = {}

    def tweak(cost, a, ms, form, ext, work, vdes, los):
        hz = 20
        movers = [int(u) for u in np.nonzero(a["state"] == ST_MOVING)[0]]
        names = ["turn_exact", "turn_ulp", "turn_4_5", "turn_5_5", "range_exact", "range_below", "wait1", "wait0",
                 "cell_arrived_not_in_range", "cell_arrived_in_range", "cell_zero_vdes", "drag_cap", "no_drag",
                 "drag_below_cap", "enter_null", "enter_self", "surround_null"] + list(TURN_AT_5) + [g[0] for g in GATE]
        spots = _free_spots(cost, a, len(names), 7)
        for name, u, p in zip(names, movers, spots):
            E[name] = u
            a["pos"][u] = p; a["prev_pos"][u] = p; a["flock_of"][u] = -1
            ms["next_pos"][u] = (p[0], 0.0, p[1]); ms["left"][u] = 0
            a["flags"][u] &= ~np.uint32(capi.FLAG_COMBAT_HELD | capi.FLAG_GARRISONED)
            form[u] = np.zeros(1, capi.FORMATION_IN)
            ext["surround_target_uid"][u] = capi.NULL_UID
        # TURNING: exactly at the target direction, one ulp off it, 4.5 and 5.5 degrees off (the 5-degree test, :2611)
        for name, rot in (("turn_exact", _quat_deg(30.0)), ("turn_ulp", _quat_deg(30.0)), ("turn_4_5", _quat_deg(34.5)),
                          ("turn_5_5", _quat_deg(35.5))):
            u = E[name]
            a["state"][u] = ST_TURNING; a["vel"][u] = 0
            ext["target_dir"][u] = _quat_deg(30.0); ext["rot"][u] = rot
        ext["rot"][E["turn_ulp"], 1] = np.nextafter(ext["rot"][E["turn_ulp"], 1], np.float32(1))
        for name, rot in TURN_AT_5.items():
            u = E[name]
            a["state"][u] = ST_TURNING; a["vel"][u] = 0
            ext["target_dir"][u] = TURN_TARGET; ext["rot"][u] = rot
        # the heading gate: a MOVING unit turns in place when its facing is off the desired direction by more than the
        # tolerance; MOVING_IN_FORMATION is outside the gate (DESIGN.md row a-8)
        for name, st, mv, deg in GATE:
            u = E[name]
            a["state"][u] = ST_MOVING if st == "moving" else ST_FORMATION
            form["flags"][u] = capi.FORM_HAS_FORMATION | capi.FORM_ASSIGNMENT_READY if st == "formation" else 0
            a["vel"][u] = (0.05, 0.0) if mv else (0.0, 0.0); a["prev_pos"][u] = a["pos"][u] - a["vel"][u]
            ms["next_rot"][u] = _quat_deg(float(deg))
        # ENTER_ENTITY_RANGE with target_range exactly the distance to the target, and one float below it: combat-held, so
        # the new position is the current one
        tgt = E["wait0"]
        for name in ("range_exact", "range_below"):
            u = E[name]
            a["state"][u] = ST_ENTER; a["flags"][u] |= capi.FLAG_COMBAT_HELD
            ext["surround_target_uid"][u] = tgt
            d = _f32_len(a["pos"][u] - a["pos"][tgt])
            ext["target_range"][u] = d if name == "range_exact" else np.nextafter(d, np.float32(0))
            ext["target_prev_pos"][u] = a["pos"][tgt] + np.float32(10.0)      # the target moved: re-issue the order
        # WAITING with 1 and 0 ticks left (:2633)
        for name, t in (("wait1", 1), ("wait0", 0)):
            u = E[name]
            a["state"][u] = ST_WAITING; a["vel"][u] = 0
            ext["wait_ticks_left"][u] = t; ext["wait_prev"][u] = ST_SEEK
        # ARRIVING_TO_CELL: arrived at the cell but not in range of it -> back to MOVING_IN_FORMATION; in range -> TURNING
        ready = capi.FORM_HAS_FORMATION | capi.FORM_ASSIGNMENT_READY | capi.FORM_ASSIGNED_TO_CELL
        for name, extra in (("cell_arrived_not_in_range", 0), ("cell_arrived_in_range", capi.FORM_IN_RANGE_OF_CELL)):
            u = E[name]
            a["state"][u] = ST_CELL
            form["flags"][u] = ready | capi.FORM_ARRIVED_AT_CELL | extra
            form["cell_pos"][u] = a["pos"][u] + np.float32(3.0)
            form["target_orientation"][u] = _quat_deg(77.0)
        # a zero cell_arrival_vdes with the cell 20 wu away: no arrival force, no cohesion (inside 30 wu), no neighbours
        u = E["cell_zero_vdes"]
        a["state"][u] = ST_CELL
        form["flags"][u] = ready | capi.FORM_IN_RANGE_OF_CELL
        form["cell_pos"][u] = a["pos"][u] + np.float32([20.0, 0.0]); form["cell_arrival_vdes"][u] = 0
        form["cohesion"][u] = (0.3, 0.2); form["align"][u] = (0.1, -0.2)
        a["vel"][u] = (0.03, -0.04); a["prev_pos"][u] = a["pos"][u] - a["vel"][u]
        # formation drag: full speed along the desired direction; with a drag the preferred speed is capped at 75 %
        # (drag_cap: no steering force, so the cap applies to the preferred velocity, not to the force added to the
        # current velocity nor to ClearPath's output, which equals the preferred velocity for a unit without neighbours);
        # below the cap the drag changes nothing
        for name, drag, frac in (("drag_cap", (0.3, 0.1), 1.0), ("no_drag", (0.0, 0.0), 1.0), ("drag_below_cap", (0.3, 0.1), 0.5)):
            u = E[name]
            a["state"][u] = ST_FORMATION
            form["flags"][u] = capi.FORM_HAS_FORMATION | capi.FORM_ASSIGNMENT_READY
            form["drag"][u] = drag
            a["vel"][u] = (np.float32(frac) * a["speed"][u] / hz, 0.0); a["prev_pos"][u] = a["pos"][u] - a["vel"][u]
            a["max_speed"][u] = np.float32(frac) * a["speed"][u]          # the desired velocity equals the current one
            ms["next_rot"][u] = cases.dir_quat(np.array([[1.0, 0.0]]))[0]
        # ENTER_ENTITY_RANGE whose target is NULL, or itself (range 0, combat-held: distance 0 <= 0)
        u = E["enter_null"]; a["state"][u] = ST_ENTER
        u = E["enter_self"]; a["state"][u] = ST_ENTER; a["flags"][u] |= capi.FLAG_COMBAT_HELD
        ext["surround_target_uid"][u] = u; ext["target_range"][u] = 0.0; ext["target_prev_pos"][u] = a["pos"][u]
        u = E["surround_null"]; a["state"][u] = ST_SURROUND
        work, vdes, los = _work_inputs(a, form)
        wi = {k: int(np.nonzero(work == u)[0][0]) for k, u in E.items()}
        for k in ["drag_cap", "no_drag", "drag_below_cap"] + [g[0] for g in GATE]:
            vdes[wi[k]] = (1.0, 0.0); los[wi[k]] = 0
        vdes[wi["cell_zero_vdes"]] = 0
        E["_wi"] = wi
        return work, vdes, los

    a, work, dev, exp = _one_tick(nav, 20, tweak)
    wi, hz = E["_wi"], 20
    for side in (dev, exp):
        pt = side["patches"]
        st = {k: int(pt["next_state"][i]) for k, i in wi.items()}
        fl = {k: int(pt["flags"][i]) for k, i in wi.items()}
        assert st["turn_exact"] == ST_ARRIVED and st["turn_ulp"] == ST_ARRIVED and st["turn_4_5"] == ST_ARRIVED
        assert st["turn_5_5"] == -1 and fl["turn_5_5"] & (1 << 3) and fl["turn_5_5"] & (1 << 9)     # ROTATION | PREV_ROT
        assert st["range_exact"] == ST_WAITING and pt["next_block"][wi["range_exact"]] == 1
        assert st["range_below"] == -1 and fl["range_below"] & (1 << 10) and fl["range_below"] & (1 << 11)
        assert st["wait1"] == ST_SEEK and fl["wait1"] & (1 << 12) and pt["wait_ticks_left"][wi["wait1"]] == 0
        assert st["wait0"] == -1 and pt["wait_ticks_left"][wi["wait0"]] == -1
        assert st["cell_arrived_not_in_range"] == ST_FORMATION
        assert st["cell_arrived_in_range"] == ST_TURNING and fl["cell_arrived_in_range"] & (1 << 13)
        assert (pt["next_target_dir"][wi["cell_arrived_in_range"]] == _quat_deg(77.0)).all()
        assert st["enter_null"] == ST_ARRIVED and st["enter_self"] == ST_WAITING and st["surround_null"] == ST_ARRIVED
        vp = side["vpref"]
        u = E["cell_zero_vdes"]
        assert (vp[wi["cell_zero_vdes"]] == a["vel"][u]).all(), vp[wi["cell_zero_vdes"]]
        cap = np.float32((np.float64(a["speed"][E["drag_cap"]]) * 0.75) / hz)
        assert abs(np.linalg.norm(vp[wi["drag_cap"]]) - cap) <= 1e-6 * cap, (np.linalg.norm(vp[wi["drag_cap"]]), cap)
        assert np.linalg.norm(vp[wi["no_drag"]]) > 1.2 * cap
        assert (vp[wi["drag_below_cap"]] == a["vel"][E["drag_below_cap"]]).all()
        assert st["turn_5_exact"] == ST_ARRIVED and st["turn_5_below"] == ST_ARRIVED
        assert st["turn_5_above"] == -1 and fl["turn_5_above"] & (1 << 3)
        for name, stt, mv, deg in GATE:
            gated = stt == "moving" and deg > (90 if mv else 10)
            assert bool(fl[name] & (1 << 14)) == gated, name                  # TURNING_IN_PLACE
            assert (np.abs(pt["next_velocity"][wi[name]]).max() == 0) == gated, name
    # the apply: WAITING entered from ENTER_ENTITY_RANGE records the state it left and WAIT_TICKS; wait1 moves on
    gx, ga = dev["ext"], dev["agents"]
    assert gx["wait_prev"][E["range_exact"]] == ST_ENTER and gx["wait_ticks_left"][E["range_exact"]] == 60
    assert ga["state"][E["wait1"]] == ST_SEEK and gx["wait_ticks_left"][E["wait0"]] == -1
    assert (gx["target_dir"][E["cell_arrived_in_range"]] == _quat_deg(77.0)).all()
    assert (gx["target_prev_pos"][E["range_below"]] == a["pos"][E["wait0"]]).all()
