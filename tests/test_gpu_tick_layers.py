"""The whole device tick against the plain-C port (oracle/pf_oracle.c) for units on every navigation layer, on non-square
maps placed where the engine places them: ground units of all four radius classes (radii on both sides of 5, 10 and
15 wu), water and air units, flocks whose fields are on a non-zero layer and flocks whose members span several
layers, on a 5 x 2-chunk map centred at the origin as M_CenterAtOrigin does (map.c:420), a 2 x 5-chunk map at an
offset that is not tile-aligned and a 1 x 6 strip at the origin. Every layer is built from one tile image
(map_cost_from_tiles) with the port's cost pass as its expectation.

The port's world holds one layer, and a unit's layer only changes its own tile probes and arrival constants, so every
tick runs the port once per layer in use and takes each unit's results from the run of its own layer
(cases.port_tick_layers); neighbours are the whole population in every run. Per tick (cases.run_trajectory, re-seeded
from the device state every tick): LOS bits and desired velocities out of the settled field pool bit-exact,
preferred velocities and velocities within 1e-4 (or one position ulp, or 1e-6 |pos| where the cohesion term nearly
cancels the position: cases.vel_ok), once with the member-list cohesion pass and once with the windowed one, patches, states and the state after the apply; then the blockers taken by the stopped
units and the local islands of all twelve layers against a host-only context and the numpy restatement. After the run:
the position index's circle queries near every map edge against the port's.

python tests/test_gpu_tick_layers.py runs the port side of every scenario without a GPU and prints its coverage."""
import os
import sys

import numpy as np
import pytest

if __name__ == "__main__":      # run from the command line: the paths tests/conftest.py sets up
    _ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [_ROOT, os.path.join(_ROOT, "oracle")]
import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
NLAYERS = 12
ST_ARRIVED = 2
# (chunk_w, chunk_h, (map_x, map_z), seed)
SHAPES = {
    "5x2_centred": (5, 2, (5 * 256 / 2.0, -(2 * 256 / 2.0)), 0x1A7E0),
    "2x5_offset": (2, 5, (601.3, -250.9), 0x1A7E1),
    "1x6_strip": (1, 6, (0.0, 0.0), 0x1A7E2),
}
# one flock each: (flags, member radii (cycled), members, spacing in radii, goal)
#   march   the generator's goal, >= 150 wu away
#   shore   a tile deep inside terrain the flock's layer cannot enter; a few members stand next to the nearest pathable
#           point, where only the (flock, layer) arrival constants can stop them
#   centre  the flock's own centre
GROUPS = [
    (0, (1.0,), 700, 2.6, "march"),
    (0, (1.0,), 500, 2.6, "march"),
    (0, (4.99, 5.0), 300, 2.2, "shore"),
    (0, (9.99, 10.0), 160, 2.2, "shore"),
    (0, (14.99, 15.0), 80, 2.2, "shore"),
    (capi.FLAG_WATER, (2.0, 5.0), 150, 2.2, "shore"),
    (capi.FLAG_AIR, (1.5, 10.0), 300, 2.6, "centre"),
]
LONE_FLOCK = 1          # one member of this flock stands far from the others: the windowed cohesion pass hands it back
# flocks of hundreds at |pos| up to ~1000 wu: the cohesion term's summation noise (cases.vel_ok)
COHESION_FLOOR = 1e-6
SHORE_UNITS = 8         # members per "shore" flock placed next to the nearest pathable point of their goal


def _tile_xz(gr, gc, map_xz):
    return np.stack([map_xz[0] - (gc + 0.5) * 4.0, map_xz[1] + (gr + 0.5) * 4.0], axis=-1).astype(np.float32)


def _passable_at(costs, layer, xz, cw, ch, map_xz):
    gr, gc = synth.tile_for_xz(xz[..., 0], xz[..., 1], cw, ch, *map_xz)
    return synth.blocked_to_image(costs[layer], cw, ch)[gr, gc] != 0xFF


def layer_case(shape, hz):
    """-> dict(cw, ch, map_xz, tiles, costs[12], a (agents + flock_layer), ms, layers (per unit), requests,
    shore (uids that only the arrival constants stop), lone (uid))"""
    import pforacle
    from scipy import ndimage
    cw, ch, map_xz, seed = SHAPES[shape]
    tiles = cases.tile_attr_case(cw, ch, seed, terrain=True)
    rng = np.random.default_rng(seed)
    for _ in range(max(2, cw * ch // 3)):            # lakes wide enough to hold goals more than 1.5 x 15 wu from the shore
        r, c = rng.integers(0, ch * 32 - 14), rng.integers(0, cw * 32 - 14)
        tiles[r:r + 14, c:c + 14] = (1, 0, -2, 0)
    costs = np.stack([pforacle.cost_from_tiles(cw, ch, tiles, L) for L in range(NLAYERS)])
    host = capi.Nav(hostonly=True)
    host.map_create(cw, ch, NLAYERS, *map_xz)
    for L in range(NLAYERS):
        host.map_upload_layer(L, costs[L]); host.map_build_nav(L); host.route_build(L)
    parts, flock_layer, shore = [], [], []
    n0 = 0
    try:
        for f, (flags, radii, n, spacing, goal) in enumerate(GROUPS):
            radius = np.array(radii, np.float32)[np.arange(n) % len(radii)]
            layers = cases.nav_layer(np.full(n, flags | capi.FLAG_MOVABLE), radius)
            L = int(layers.max())
            g = synth.make_agents(costs[L], cw, ch, n, 1, seed + 17 * f, radius=float(radius.max()), spacing=spacing,
                                  hz=hz, map_x=map_xz[0], map_z=map_xz[1], goal_min_dist=150.0)
            g["radius"] = radius
            g["flags"] = np.full(n, flags | capi.FLAG_MOVABLE, np.uint32)
            centre = g["pos"].mean(axis=0)
            if goal == "centre":
                g["flock_target"][0] = centre
            elif goal == "shore":
                img = synth.blocked_to_image(costs[L], cw, ch)
                depth = ndimage.distance_transform_edt(img == 0xFF) * 4.0          # wu to the nearest pathable tile
                thresh = 1.5 * float(radius.max())
                deep = np.argwhere(depth >= thresh + 8.0)
                assert len(deep), (shape, f)
                xz = _tile_xz(deep[:, 0], deep[:, 1], map_xz)
                tgt = xz[np.argmin(((xz - centre) ** 2).sum(axis=1))]
                g["flock_target"][0] = tgt
                ok, nearest, _ = host.route_arrival_consts(tgt, L)
                assert ok, (shape, f)
                # members on the flock's (non-zero) layer placed around the nearest pathable point: further than 1.5 r from
                # the goal, within 0.4 * 1.5 r of the point, on a passable tile; slow, so that they stay there for the tick
                picked = []
                for u in np.nonzero(layers == L)[0]:
                    for _ in range(50):
                        p = (nearest + rng.uniform(-0.4, 0.4, 2) * 1.5 * radius[u] / np.sqrt(2)).astype(np.float32)
                        if np.linalg.norm(p - tgt) > 1.5 * radius[u] + 1.0 and _passable_at(costs, int(layers[u]), p, cw, ch, map_xz):
                            g["pos"][u] = p
                            picked.append(u)
                            break
                    if len(picked) == SHORE_UNITS:
                        break
                assert len(picked) == SHORE_UNITS, (shape, f, len(picked))
                g["max_speed"][picked] = 4.0; g["speed"][picked] = 4.0
                shore += [n0 + u for u in picked]
            d = g["flock_target"][0] - g["pos"]
            dist = np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-3)
            g["vel"] = (d / dist * (0.5 * g["max_speed"][:, None] / hz)).astype(np.float32)
            g["vel"][rng.random(n) < 0.1] *= np.float32(0.05)
            g["prev_pos"] = (g["pos"] - g["vel"]).astype(np.float32)
            if f >= 2:                  # ARRIVED members start the adjacent-arrived cascade (movement.c:2457) on every layer
                st = np.where(rng.random(n) < 0.05, ST_ARRIVED, 0).astype(np.int32)
                st[[u - n0 for u in shore if u >= n0]] = 0
                g["state"] = st
            g["flock_of"][:] = f
            parts.append(g)
            flock_layer.append(L)
            n0 += n
    finally:
        host.close()
    a = {k: np.concatenate([g[k] for g in parts]) for k in ("pos", "prev_pos", "vel", "radius", "max_speed", "speed", "state",
                                                            "flags", "flock_of")}
    a["flock_target"] = np.concatenate([g["flock_target"] for g in parts])
    a["flock_layer"] = np.array(flock_layer, np.int32)
    # the lone member: the ground tile furthest from the rest of its flock
    mem = np.nonzero(a["flock_of"] == LONE_FLOCK)[0]
    lone, rest = int(mem[0]), a["pos"][mem[1:]]
    img = synth.blocked_to_image(costs[0], cw, ch)
    cand = np.argwhere(img != 0xFF)[rng.choice(int((img != 0xFF).sum()), 4000, replace=False)]
    xz = _tile_xz(cand[:, 0], cand[:, 1], map_xz)
    far = np.sqrt(((xz[:, None, :] - rest[None, :, :]) ** 2).sum(axis=2)).min(axis=1)
    a["pos"][lone] = xz[np.argmax(far)]
    a["prev_pos"][lone] = a["pos"][lone] - a["vel"][lone]
    layers = cases.nav_layer(a["flags"], a["radius"])
    n = len(layers)
    for u in range(n):
        assert _passable_at(costs, int(layers[u]), a["pos"][u], cw, ch, map_xz), (shape, u, int(layers[u]))
    ms = np.zeros(n, capi.MOVESTATE)
    ms["next_pos"][:, 0] = a["pos"][:, 0]; ms["next_pos"][:, 2] = a["pos"][:, 1]
    ms["step"] = 1.0 / (20 // hz)
    ms["next_rot"] = cases.dir_quat(a["vel"] + 1e-6)
    ms["combat_facing"] = ms["next_rot"]
    ms["vel_hist"] = np.repeat(a["vel"][:, None, :], 14, axis=1)
    # every flock's fields requested up front on its own layer, from the member nearest to the flock's centre
    requests = []
    for f in range(len(GROUPS)):
        m = np.nonzero(a["flock_of"] == f)[0]
        requests.append((f, a["pos"][m[np.argmin(np.linalg.norm(a["pos"][m] - a["pos"][m].mean(axis=0), axis=1))]]))
    return dict(cw=cw, ch=ch, map_xz=map_xz, tiles=tiles, costs=costs, a=a, ms=ms, layers=layers, requests=requests,
                shore=np.array(shore), lone=lone, lone_dist=float(far.max()))


def coverage(case):
    """per layer: units, work items (not ARRIVED), "shore" members; the lone member's distance to its flock"""
    a, layers = case["a"], case["layers"]
    out = {}
    for L in np.unique(layers):
        on = layers == L
        out[int(L)] = dict(units=int(on.sum()), work=int((on & (a["state"] != ST_ARRIVED)).sum()),
                           arrived=int((on & (a["state"] == ST_ARRIVED)).sum()), shore=int(np.isin(np.nonzero(on)[0], case["shore"]).sum()))
    return out


def _check_case(case):
    """what the scenario must hold for the comparison to mean something"""
    cov = coverage(case)
    # all four ground classes, water and air
    assert {0, 1, 2, 3, 4, 5, 8, 10} <= set(cov), cov
    for L, c in cov.items():
        assert c["work"] >= 30, (L, c)
    a = case["a"]
    # flocks whose members span several layers, and flocks whose fields are on a non-zero layer
    assert sum(len(np.unique(case["layers"][a["flock_of"] == f])) > 1 for f in range(len(GROUPS))) >= 4
    assert (a["flock_layer"] != 0).sum() >= 4
    # the arrival constants decide for members on non-zero layers
    assert len(case["shore"]) and (case["layers"][case["shore"]] != 0).all()
    # alone beyond the cohesion window (COH_R = 230 wu plus one index cell either side) in a flock of more than one
    assert case["lone_dist"] > 300.0, case["lone_dist"]
    return cov


def _nsplit(n, sm_count):
    """the row split of k_cohesion_window for a population of n (pfnav_agents_tick)"""
    nblk = (n + 127) // 128
    return max(1, min(8, (sm_count * 8 + nblk - 1) // nblk))


def _query_centres(cw, ch, map_xz):
    """points 2 wu inside every edge and corner of the map, and its centre"""
    x0, x1 = map_xz[0] - cw * 256.0 + 2.0, map_xz[0] - 2.0
    z0, z1 = map_xz[1] + 2.0, map_xz[1] + ch * 256.0 - 2.0
    xm, zm = (x0 + x1) / 2, (z0 + z1) / 2
    return [(x, z) for x in (x0, xm, x1) for z in (z0, zm, z1)]


@pytest.mark.parametrize("hz", [20, 5])
@pytest.mark.parametrize("shape", list(SHAPES))
def test_tick_on_every_layer_vs_port(pf, nav, pforacle, shape, hz):
    """three ticks of the scenario (layer_case) with both cohesion passes: see the module docstring"""
    import torch
    case = layer_case(shape, hz)
    _check_case(case)
    cw, ch, map_xz, a = case["cw"], case["ch"], case["map_xz"], case["a"]
    n = len(a["radius"])
    # the windowed cohesion pass splits its rows over blockIdx.y at this population size
    assert _nsplit(n, torch.cuda.get_device_properties(0).multi_processor_count) > 1
    log = []
    out = cases.run_trajectory(nav, None, pforacle, a, case["ms"], cw, case["costs"], hz, 3, with_blockers=True, ch=ch,
                               map_xz=map_xz, nlayers=NLAYERS, layer_of_unit=case["layers"], tiles=case["tiles"],
                               requests=case["requests"], cohesion_modes=(0, 1), log=log, cohesion_floor=COHESION_FLOOR)
    assert len(out) == 3, out
    # the "shore" members were stopped by their (flock, layer) arrival constants in the first tick (a few may have been
    # pushed away by their neighbours)
    t0 = log[0]
    arrived = ((t0["patches"]["flags"] & 1) != 0) & (t0["patches"]["next_state"] == ST_ARRIVED)
    nshore = int(np.isin(case["shore"], t0["work"][arrived]).sum())
    assert nshore * 4 >= len(case["shore"]) * 3, (nshore, len(case["shore"]))
    # arrivals on non-zero layers beyond the shore members (the adjacent-arrived cascade)
    assert (arrived & (t0["layers"] != 0)).sum() > 2 * len(case["shore"]), int((arrived & (t0["layers"] != 0)).sum())
    # the position index after the last apply: circle queries near every edge, in the port's order
    got, _ = nav.agents_read_state(n)
    rec = np.array(got, capi.AGENT)
    world = pforacle.OracleWorld(pforacle.OracleMap(cw, ch, case["costs"][0], None, None, *map_xz), rec,
                                 np.zeros(len(GROUPS), capi.FLOCK), hz)
    try:
        for x, z in _query_centres(cw, ch, map_xz):
            for r in (12.0, 60.0, 250.0, 1000.0):
                for cap in (512, n):
                    g, e = nav.ents_in_circle(x, z, r, cap), world.ents_in_circle(x, z, r, cap)
                    assert len(g) == len(e) and (g == e).all(), (x, z, r, cap, len(g), len(e))
    finally:
        world.close()


def _rehearse(shape, hz):
    """the port side of one scenario without a GPU: one port tick per layer in use on the initial state (desired
    velocities straight at the goals), the host-only context's arrival constants and the blockers of the stopped units"""
    import pforacle
    case = layer_case(shape, hz)
    cov = _check_case(case)
    cw, ch, map_xz, a, layers = case["cw"], case["ch"], case["map_xz"], case["a"], case["layers"]
    d = a["flock_target"][a["flock_of"]] - a["pos"]
    aa = dict(a); aa["vdes"] = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(np.float32)
    rec, fl = capi.pack_agents(aa)
    fl["layer"] = a["flock_layer"]
    work = np.nonzero(a["state"] != ST_ARRIVED)[0].astype(np.uint32)
    host = capi.Nav(hostonly=True)
    host.map_create(cw, ch, NLAYERS, *map_xz)
    try:
        for L in range(NLAYERS):
            host.map_upload_layer(L, case["costs"][L]); host.map_build_nav(L); host.route_build(L)
        used = np.unique(layers[work])
        omaps = {L: pforacle.OracleMap(cw, ch, case["costs"][L], None, None, *map_xz) for L in used}
        arrivals = {L: [host.route_arrival_consts(t, int(L)) for t in a["flock_target"]] for L in used}
        exp = cases.port_tick_layers(omaps, rec, fl, case["ms"], work, hz, arrivals, layers, None)
        p = exp["patches"]
        stop = ((p["flags"] & 1) != 0) & (p["next_block"] != 0)
        for w in np.nonzero(stop)[0]:
            u = work[w]
            host.blockers_incref(float(a["pos"][u, 0]), float(a["pos"][u, 1]), float(a["radius"][u]), 0, int(a["flags"][u]))
        host.map_commit()
        arrived = stop & (p["next_state"] == ST_ARRIVED)
        print("%s @ %d Hz: %d units, nsplit on 132 SMs %d, lone member %.0f wu from its flock" % (
            shape, hz, len(layers), _nsplit(len(layers), 132), case["lone_dist"]))
        for L in sorted(cov):
            on = layers[work] == L
            print("  layer %2d: %s  arrivals %d  stopped %d  blocked tiles %d" % (
                L, cov[L], int((arrived & on).sum()), int((stop & on).sum()), int((host.blockers(int(L)) > 0).sum())))
        shore_w = np.isin(work, case["shore"])
        print("  shore members stopped by the arrival constants: %d of %d" % (int((arrived & shore_w).sum()), len(case["shore"])))
    finally:
        host.close()


if __name__ == "__main__":
    for s in SHAPES:
        for hz in (20, 5):
            _rehearse(s, hz)
