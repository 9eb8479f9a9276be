"""Inputs and the host reference for pfnav_map_query tests (tests/test_map_query_emu.py, tests/test_gpu_map_query.py).

The reference answers of the two searches come from pfnav_route_arrival_consts (Nav.route_arrival_consts), the host
routine the tick's arrived() constants use; the tolerance test of N_IsMaximallyClose is restated in float32."""
import numpy as np

import cases

capi, synth = cases.capi, cases.synth


def image(a, cw, ch):
    """[chunks][64][64] -> row-major [H64][W64] (the device layout)"""
    return np.ascontiguousarray(a.reshape(ch, cw, 64, 64).transpose(0, 2, 1, 3).reshape(ch * 64, cw * 64))


def tile_xz(r, c, map_xz=(0.0, 0.0)):
    """world (x, z) of the centre of absolute nav tile (r, c)"""
    return synth.tile_center_xz(r // 64, c // 64, r % 64, c % 64, map_xz[0], map_xz[1])


def on_map(x, z, cw, ch, map_xz=(0.0, 0.0)):
    """M_Tile_DescForPoint2D's box test, in float32"""
    f = np.float32
    mx, mz = f(map_xz[0]), f(map_xz[1])
    return not (f(x) > mx or f(x) < mx - f(cw * 256) or f(z) < mz or f(z) > mz + f(ch * 256))


def blocked_rect_map(cw, ch, seed, rects):
    """a synthetic map (chunk-blocked cost) with the given absolute impassable rectangles (r0, c0, r1, c1) added"""
    img = synth.blocked_to_image(synth.cost_from_pathable(synth.make_map(cw, ch, seed, frac_blocked=0.2, rivers=cw > 1), cw, ch),
                                 cw, ch).copy()
    for r0, c0, r1, c1 in rects:
        img[r0:r1, c0:c1] = 0xFF
    return synth.image_to_blocked(img, cw, ch)


def search_tiles(cost_c, cw, ch, rng, n, extra=()):
    """random tiles, impassable tiles, the four corners, chunk borders and the given extra tiles"""
    H, W = ch * 64, cw * 64
    img = synth.blocked_to_image(cost_c, cw, ch)
    out = [(int(rng.integers(0, H)), int(rng.integers(0, W))) for _ in range(n)]
    imp = np.argwhere(img == 0xFF)
    if len(imp):
        out += [tuple(int(v) for v in imp[rng.integers(0, len(imp))]) for _ in range(n)]
    out += [(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1)]
    for _ in range(n // 2):
        out.append((64 * int(rng.integers(0, ch)) + int(rng.choice([0, 63])), int(rng.integers(0, W))))
        out.append((int(rng.integers(0, H)), 64 * int(rng.integers(0, cw)) + int(rng.choice([0, 63]))))
    return out + list(extra)


def search_queries(tiles, layer=0, tolerances=(0.0,), map_xz=(0.0, 0.0), rng=None):
    """for every tile: a CLOSEST_PATHABLE query at its centre, and MAXIMALLY_CLOSE queries towards it from the centre and
    from a point a few tiles away, one per tolerance"""
    q = []
    for k, (r, c) in enumerate(tiles):
        x, z = tile_xz(r, c, map_xz)
        q.append((capi.QUERY_CLOSEST_PATHABLE, layer, x, z, 0.0, 0.0, 0.0, 0))
        for t in tolerances:
            q.append((capi.QUERY_MAXIMALLY_CLOSE, layer, x, z, x, z, t, 0))
            dx, dz = (rng.uniform(-12.0, 12.0, 2) if rng is not None else (4.0 * (k % 3 - 1), 4.0 * ((k // 3) % 3 - 1)))
            q.append((capi.QUERY_MAXIMALLY_CLOSE, layer, x + dx, z + dz, x, z, t, 0))
    return np.array(q, capi.MAP_QUERY)


def reference(nav, q, cw, ch, map_xz=(0.0, 0.0)):
    """the expected MAP_QUERY_RESULT of the search kinds, from pfnav_route_arrival_consts, and the expected tile lists of
    the MAXIMALLY_CLOSE queries (float32 (x, z) centres, None off the map)"""
    out = np.zeros(len(q), capi.MAP_QUERY_RESULT)
    lists = [None] * len(q)
    f = np.float32
    for i, a in enumerate(q):
        if a["kind"] == capi.QUERY_CLOSEST_PATHABLE:
            if not on_map(a["x"], a["z"], cw, ch, map_xz):
                continue
            ok, nearest, _ = nav.route_arrival_consts((a["x"], a["z"]), int(a["layer"]))
            out[i]["ok"] = ok
            if ok:
                out[i]["x"], out[i]["z"] = nearest
        elif a["kind"] == capi.QUERY_MAXIMALLY_CLOSE:
            if not (on_map(a["x"], a["z"], cw, ch, map_xz) and on_map(a["dst_x"], a["dst_z"], cw, ch, map_xz)):
                continue
            _, _, mc = nav.route_arrival_consts((a["dst_x"], a["dst_z"]), int(a["layer"]))
            lists[i] = mc
            dx, dz = mc[:, 0] - f(a["x"]), mc[:, 1] - f(a["z"])
            out[i]["ok"] = bool((np.sqrt(dx * dx + dz * dz) <= f(a["tolerance"])).any())
    return out, lists
