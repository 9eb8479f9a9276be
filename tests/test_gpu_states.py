"""GPU suite: every movement state of move_velocity_work / entity_compute_update (movement.c:3395-3466, 2303-2670) against
the COMPILED REFERENCE on the box: the steering variants (enemy_seek_vpref, cell_arrival_seek_vpref, formation_seek_vpref,
movement.c:1946, 1908, 1985), the formation inputs, the state machine of SEEK_ENEMIES / ENTER_ENTITY_RANGE / TURNING /
WAITING / ARRIVING_TO_CELL / MOVING_IN_FORMATION, and the TARGET_ENEMIES / TARGET_ENTITY field consumers
(N_DesiredEnemySeekVelocity / N_DesiredSurroundVelocity, nav.c:3603, 3687)."""
import os

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
VEL_RTOL = 1e-4
ST_MOVING, ST_FORMATION, ST_ARRIVED, ST_SEEK, ST_WAITING, ST_SURROUND, ST_ENTER, ST_TURNING, ST_CELL = range(9)


def _scenario(seed, hz):
    """1 500 agents of cases.update_case with the movement states spread over them and all the inputs those states read"""
    p, cost, a, ms = cases.update_case(seed, hz)
    form, ext = _spread_states(a, ms, seed)
    return p, cost, a, ms, form, ext


def _spread_states(a, ms, seed):
    """spread the movement states over the MOVING units of `a` (in place: state, flock_of) -> the formation inputs and
    the movestate beyond point seeking those states read (FORMATION_IN, MOVESTATE_EXT)"""
    n = len(a["radius"])
    rng = np.random.default_rng(seed + 7)
    st = a["state"].copy()
    movers = np.nonzero(st == 0)[0]
    pick = rng.permutation(movers)
    k = len(pick) // 8
    st[pick[0 * k:1 * k]] = ST_FORMATION
    st[pick[1 * k:2 * k]] = ST_CELL
    st[pick[2 * k:3 * k]] = ST_SEEK
    st[pick[3 * k:4 * k]] = ST_ENTER
    st[pick[4 * k:4 * k + k // 2]] = ST_TURNING
    st[pick[4 * k + k // 2:5 * k]] = ST_SURROUND
    st[pick[5 * k:6 * k]] = ST_WAITING
    a["state"] = st
    flock_of = a["flock_of"].copy()
    flock_of[st == ST_SEEK] = -1                            # seekers have no flock (movement.c:3420)
    a["flock_of"] = flock_of
    # formation inputs
    form = np.zeros(n, capi.FORMATION_IN)
    inform = (st == ST_FORMATION) | (st == ST_CELL) | ((st == ST_MOVING) & (rng.random(n) < 0.15))
    form["flags"][inform] = capi.FORM_HAS_FORMATION
    for bit, prob in ((capi.FORM_ASSIGNMENT_READY, 0.85), (capi.FORM_ASSIGNED_TO_CELL, 0.6), (capi.FORM_IN_RANGE_OF_CELL, 0.5),
                      (capi.FORM_ARRIVED_AT_CELL, 0.3)):
        form["flags"][inform & (rng.random(n) < prob)] |= bit
    form["cell_pos"] = a["pos"] + rng.normal(scale=25.0, size=(n, 2)).astype(np.float32)
    near = rng.random(n) < 0.3
    form["cell_pos"][near] = (a["pos"] + rng.normal(scale=3.0, size=(n, 2)))[near]
    v = rng.normal(size=(n, 2)); v /= np.linalg.norm(v, axis=1, keepdims=True)
    form["cell_arrival_vdes"] = v.astype(np.float32)
    form["cell_arrival_vdes"][rng.random(n) < 0.1] = 0
    form["cohesion"] = rng.normal(scale=0.4, size=(n, 2)); form["align"] = rng.normal(scale=0.3, size=(n, 2))
    form["drag"] = rng.normal(scale=0.2, size=(n, 2)) * (rng.random((n, 1)) < 0.5)
    form["target_orientation"] = cases.dir_quat(rng.normal(size=(n, 2)))
    # movestate beyond point seeking
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID
    enter = np.nonzero(st == ST_ENTER)[0]
    tgt = rng.integers(0, n, len(enter)).astype(np.uint32)
    tgt[: len(enter) // 6] = capi.NULL_UID
    ext["surround_target_uid"][enter] = tgt
    ext["target_range"] = rng.uniform(2.0, 60.0, n)
    ext["target_prev_pos"] = a["pos"] + rng.normal(scale=6.0, size=(n, 2)).astype(np.float32)
    have = enter[tgt != capi.NULL_UID]
    ext["target_prev_pos"][have] = (a["pos"][ext["surround_target_uid"][have]] + rng.normal(scale=4.0, size=(len(have), 2))).astype(np.float32)
    ext["target_dir"] = cases.dir_quat(rng.normal(size=(n, 2)))
    ext["rot"] = ms["next_rot"]
    turning = np.nonzero(st == ST_TURNING)[0]
    close = turning[: len(turning) // 3]
    ext["target_dir"][close] = ext["rot"][close]            # already facing the target direction -> ARRIVED
    ext["wait_prev"] = ST_MOVING
    ext["wait_ticks_left"] = rng.integers(1, 5, n)
    return form, ext


def _work_inputs(a, form, seed=99):
    """the work list of a one-tick all-states case (every state but ARRIVED: the WAITING countdown runs in
    entity_compute_update, movement.c:2630) and its desired velocities and LOS bits -> (work, vdes, los)"""
    rng = np.random.default_rng(seed)
    work = np.nonzero(a["state"] != ST_ARRIVED)[0].astype(np.uint32)
    vdes = rng.normal(size=(len(work), 2)).astype(np.float32)
    vdes /= np.linalg.norm(vdes, axis=1, keepdims=True)
    vdes[rng.random(len(work)) < 0.08] = 0
    cell = a["state"][work] == ST_CELL
    vdes[cell] = form["cell_arrival_vdes"][work][cell]       # ent_desired_velocity (movement.c:1507)
    vdes[a["state"][work] == ST_TURNING] = 0
    los = (rng.random(len(work)) < 0.25).astype(np.uint8)
    los[a["flock_of"][work] < 0] = 0
    return work, vdes, los


def _ref_setup(ref, a, ms, form, ext, hz, work, vdes, los):
    n = len(a["radius"])
    dest_ids = np.array([ref.dest_id((float(t[0]), float(t[1]))) for t in a["flock_target"]], np.uint32)
    ref.agents_set(a["pos"], a["prev_pos"], a["vel"], a["radius"], a["max_speed"], a["state"], a["flags"],
                   a["flock_of"], a["flock_target"], dest_ids, hz=hz)
    ref.movestate_set(ms["next_pos"][:, [0, 2]], ms["next_rot"], ms["step"], ms["left"], ms["vel_hist"], ms["vel_hist_idx"],
                      ext["wait_prev"], ext["wait_ticks_left"], ms["combat_facing"])
    ints = np.stack([ext["wait_prev"], ext["wait_ticks_left"], ext["surround_target_uid"].astype(np.int64).astype(np.int32),
                     ext["using_surround_field"].astype(np.int32)], axis=1)
    flo = np.concatenate([ext["target_range"][:, None], ext["target_prev_pos"], ext["target_dir"], ext["rot"]], axis=1)
    ref.movestate_ext_set(ints, flo)
    ref.work_set(work, vdes, los, a["speed"][work])
    f14 = np.concatenate([form["cell_pos"], form["cell_arrival_vdes"], form["cohesion"], form["align"], form["drag"],
                          form["target_orientation"]], axis=1)[work]
    ref.work_set_formation(f14, form["flags"][work])


@pytest.mark.parametrize("hz", [20, 10])
def test_all_movement_states_vs_reference(nav, pfref_or_golden, hz):
    """every movement state's velocity, entity_compute_update patch and device-side apply vs the compiled reference.
    Without the compiled reference it compares with a regression baseline recorded from the CUDA path
    (tests/golden/README.md), not with reference values."""
    p, cost, a, ms, form, ext = _scenario(5151, hz)
    n = len(a["radius"])
    cw = 3
    work, vdes, los = _work_inputs(a, form)
    ref = pfref_or_golden.RefMap(cw, cw, p) if pfref_or_golden else None
    E = cases.Expected("movement_states_hz%d" % hz, ref)
    ref_out = {}

    def reference():
        if not ref_out:
            try:
                _ref_setup(ref, a, ms, form, ext, hz, work, vdes, los)
                ref_out["vel"], _ = ref.velocity_work(os.cpu_count())
                ref_out["upd"] = ref.compute_updates_ext(ref_out["vel"])
            finally:
                ref.close()
        return ref_out
    aa = dict(a)
    aa["vdes"] = np.zeros((n, 2), np.float32); aa["vdes"][work] = vdes
    aa["has_los"] = np.zeros(n, np.uint32); aa["has_los"][work] = los
    rec, fl = capi.pack_agents(aa)
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.agents_upload(rec, fl, hz)
    nav.agents_upload_movestate(ms)
    nav.agents_upload_formation(form)
    nav.agents_upload_movestate_ext(ext)
    nav.agents_set_work(work)
    try:
        vels = {}
        for mode in (0, 2):
            nav.set_two_phase(mode)
            nav.agents_tick(0)
            vels[mode] = nav.agents_read_velocities(len(work))
        assert (vels[0] == vels[2]).all()
    finally:
        nav.set_two_phase(1)
    vel = vels[0]
    evel = E("vel", lambda: reference()["vel"], vel)
    e = cases.relerr(vel, evel)
    bad = np.nonzero(e > VEL_RTOL)[0]
    assert len(bad) == 0, (e.max(), work[bad[:8]], a["state"][work][bad[:8]])
    nav.agents_compute_updates()
    pt = nav.agents_read_patches(len(work))
    got_oi = np.stack([pt["flags"].astype(np.int64), pt["next_state"], pt["next_block"], pt["wait_ticks_left"]], axis=1)
    got = np.concatenate([pt["next_velocity"], pt["next_pos"], pt["next_rot"], pt["next_ppos"], pt["next_npos"],
                          pt["next_step"][:, None], pt["next_left"][:, None], pt["next_nrot"], pt["next_prot"]], axis=1)
    gx = np.concatenate([pt["next_dest"], pt["next_target_prev"], pt["next_target_dir"], pt["next_attack"][:, None].astype(np.float32)], axis=1)
    oi = E("patch_i", lambda: reference()["upd"][0], got_oi)
    of = E("patch_f", lambda: reference()["upd"][1], got)
    ox = E("patch_x", lambda: reference()["upd"][2], gx)
    E.save()
    stw = a["state"][work]
    surround_live = (stw == ST_SURROUND) & (ext["surround_target_uid"][work] != capi.NULL_UID)
    assert not surround_live.any()                         # the scenario keeps surround targets NULL (engine geometry otherwise)
    flags_same = (pt["flags"] == oi[:, 0].astype(np.uint32))
    assert flags_same.all(), (np.nonzero(~flags_same)[0][:10], stw[~flags_same][:10], pt["flags"][~flags_same][:5], oi[~flags_same][:5, 0])
    assert (pt["next_state"] == oi[:, 1]).all(), np.nonzero(pt["next_state"] != oi[:, 1])[0][:10]
    assert (pt["next_block"] == oi[:, 2]).all()
    assert (pt["wait_ticks_left"] == oi[:, 3]).all()
    err = np.abs(got - of[:, :25]) / np.maximum(np.abs(of[:, :25]), 1.0)
    assert err.max() <= 1e-4, (err.max(), np.unravel_index(err.argmax(), err.shape))
    assert np.abs(gx - ox).max() <= 1e-5, np.abs(gx - ox).max()
    # every state and every transition kind is present
    for s_ in (ST_MOVING, ST_FORMATION, ST_SEEK, ST_WAITING, ST_SURROUND, ST_ENTER, ST_TURNING, ST_CELL):
        assert (stw == s_).sum() > 10, s_
    assert {-1, ST_ARRIVED, ST_WAITING, ST_MOVING, ST_FORMATION, ST_TURNING, ST_CELL} <= set(np.unique(oi[:, 1]).tolist())
    assert (oi[:, 0] & (1 << 10)).any() and (oi[:, 0] & (1 << 12)).any() and (oi[:, 0] & (1 << 13)).any()
    # device-side apply of the new fields
    nav.agents_apply_updates()
    a2, _ = nav.agents_read_state(n)
    moved = (pt["flags"] & (1 | (1 << 12))) != 0
    garr = (a["flags"][work] & capi.FLAG_GARRISONED) != 0
    assert (a2["state"][work][moved & ~garr] == oi[moved & ~garr, 1]).all()


def test_enemy_seek_and_surround_field_consumers(nav):
    """N_DesiredEnemySeekVelocity / N_DesiredSurroundVelocity: SEEK_ENEMIES entities and surround-field users read the own
    tile's direction out of TARGET_ENEMIES / TARGET_ENTITY pool destinations (pfnav_pool_request_entity_fields); the field
    bytes equal the reference's N_FlowFieldUpdate for those targets and the desired velocity is N_FlowDir of the tile."""
    g = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "targets.npz"))
    cw = ch = 3
    wars = [tuple(w) for w in g["wars"]]
    nav.map_create(cw, ch, 1)
    nav.map_upload_layer(0, g["cost_0"], g["blk_0"]); nav.map_build_nav(0); nav.route_build(0)
    fp = nav.footprints(g["pos"], g["radius"])
    allchunks = [(c // cw, c % cw) for c in range(cw * ch)]
    nav.pool_create(4, 4 * cw * ch)
    foes = cases.enemies_of(1, wars, g["factions"], g["flags"])
    nav.pool_request_entity_fields(0, capi.TARGET_ENEMIES, fp[foes], allchunks)
    u = int(g["uids"][0])
    nav.pool_request_entity_fields(1, capi.TARGET_ENTITY, fp[u:u + 1], allchunks)
    for c in range(cw * ch):
        assert (nav.pool_get(0, (c // cw, c % cw))[0] == g["foe_0"][1][c]).all(), c
        assert (nav.pool_get(1, (c // cw, c % cw))[0] == g["ent_0"][0][c]).all(), c
    rng = np.random.default_rng(3)
    n = 600
    img = synth.blocked_to_image(g["cost_0"], cw, ch)
    blk_img = synth.blocked_to_image(g["blk_0"], cw, ch)
    pas = np.argwhere((img != 255) & (blk_img == 0))
    t = pas[rng.integers(0, len(pas), n)]
    pos = np.stack([-(t[:, 1] + rng.uniform(0.05, 0.95, n)) * 4.0, (t[:, 0] + rng.uniform(0.05, 0.95, n)) * 4.0], 1).astype(np.float32)
    rec = np.zeros(n, capi.AGENT)
    rec["pos"] = pos; rec["prev_pos"] = pos; rec["radius"] = 1.0; rec["max_speed"] = 20.0; rec["speed"] = 20.0
    rec["flags"] = capi.FLAG_MOVABLE
    rec["state"][: n // 2] = ST_SEEK; rec["flock"][: n // 2] = -1; rec["aux_dest1"][: n // 2] = 1
    rec["state"][n // 2:] = ST_SURROUND; rec["flock"][n // 2:] = 0; rec["aux_dest1"][n // 2:] = 2
    fl = np.zeros(1, capi.FLOCK); fl["target"] = g["pos"][u]; fl["dest"] = -1
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID
    ext["surround_target_uid"][n // 2:] = 0; ext["using_surround_field"][n // 2:] = 1
    nav.agents_upload(rec, fl, 20)
    nav.agents_upload_movestate_ext(ext)
    nav.agents_set_work(np.arange(n, dtype=np.uint32))
    nav.agents_tick(capi.TICK_VDES_FROM_POOL)
    _, vdes, los = nav.agents_read_debug(n)
    d = np.float32(1.0 / np.sqrt(2.0))
    DIR = np.array([[0, 0], [d, -d], [0, -1], [-d, -d], [1, 0], [-1, 0], [d, d], [0, 1], [-d, d]], np.float32)    # N_FlowDir (field.c:2429)
    field = [np.zeros((ch * 64, cw * 64), np.uint8) for _ in range(2)]
    for c in range(cw * ch):
        field[0][(c // cw) * 64:(c // cw) * 64 + 64, (c % cw) * 64:(c % cw) * 64 + 64] = g["foe_0"][1][c]
        field[1][(c // cw) * 64:(c // cw) * 64 + 64, (c % cw) * 64:(c % cw) * 64 + 64] = g["ent_0"][0][c]
    exp = np.concatenate([DIR[field[0][t[: n // 2, 0], t[: n // 2, 1]]], DIR[field[1][t[n // 2:, 0], t[n // 2:, 1]]]])
    assert (vdes == exp).all(), np.nonzero((vdes != exp).any(axis=1))[0][:10]
    assert not los.any()
    assert (np.abs(exp).sum(axis=1) > 0).mean() > 0.5
