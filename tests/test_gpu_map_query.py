"""pfnav_map_query on the device: the probe kinds against a numpy restatement over the committed layer grids, DEST_ID
against the dest_id pfnav_pool_request_path reports (and the compiled reference when it is built), the two searches
against the host routine pfnav_route_arrival_consts plus the float tolerance test, commit ordering and argument errors."""
import numpy as np
import pytest

import map_query_cases as mq

capi, synth = mq.capi, mq.synth
pytestmark = pytest.mark.gpu
C2_SEED, CW = 0x5EED0001, 16          # bench.py's C2 map
f32 = np.float32


def _desc(x, z, cw, ch, map_xz):
    """M_Tile_DescForPoint2D (tile.c:547) over arrays, in the device's arithmetic -> (inside, abs row, abs col)"""
    x, z = x.astype(f32), z.astype(f32)
    mx, mz = f32(map_xz[0]), f32(map_xz[1])
    inside = ~((x > mx) | (x < mx - f32(cw * 256)) | (z < mz) | (z > mz + f32(ch * 256)))
    cr = np.clip((np.abs((mz - z).astype(np.float64)) / 256.0).astype(np.int64), 0, ch - 1)
    cc = np.clip((np.abs((mx - x).astype(np.float64)) / 256.0).astype(np.int64), 0, cw - 1)
    bx, bz = mx - cc.astype(f32) * f32(256), mz + cr.astype(f32) * f32(256)
    tr = np.clip((np.abs((bz - z).astype(np.float64)) / 4).astype(np.int64), 0, 63)
    tc = np.clip((np.abs((bx - x).astype(np.float64)) / 4).astype(np.int64), 0, 63)
    return inside, cr * 64 + tr, cc * 64 + tc


def _probe_expected(nav, layer, x, z, cw, ch, map_xz):
    cost, blk, _ = nav.map_get_layer(layer)
    cost, blk = mq.image(cost, cw, ch), mq.image(blk, cw, ch)
    inside, r, c = _desc(x, z, cw, ch, map_xz)
    bad = (cost == 0xFF) | (blk > 0)
    H, W = bad.shape
    adj = np.zeros(len(x), bool)
    for dr, dc in ((-1, 0), (0, -1), (0, 1), (1, 0)):
        nr, nc = r + dr, c + dc
        ok = (nr >= 0) & (nr < H) & (nc >= 0) & (nc < W)
        adj |= ok & bad[np.clip(nr, 0, H - 1), np.clip(nc, 0, W - 1)]
    return inside & (cost[r, c] != 0xFF), inside & (blk[r, c] > 0), inside & adj


def _points(rng, n, cw, ch, map_xz):
    """random points over (and a little beyond) the map box, points exactly on its edges, on the last row and column"""
    mx, mz = map_xz
    W, H = cw * 256.0, ch * 256.0
    x = rng.uniform(mx - W - 8, mx + 8, n).astype(f32)
    z = rng.uniform(mz - 8, mz + H + 8, n).astype(f32)
    k = n // 8
    x[:k] = rng.choice([mx, mx - W, mx - W + 1.0, mx - W + 3.999, np.nextafter(f32(mx - W), f32(-1e9))], k)
    z[k:2 * k] = rng.choice([mz, mz + H, mz + H - 1.0, mz + H - 3.999, np.nextafter(f32(mz + H), f32(1e9))], k)
    return x, z


def _c2_nav(nlayers=2):
    nav = capi.Nav(0)
    nav.map_create(CW, CW, nlayers)
    costs = []
    for layer in range(nlayers):
        cost = synth.cost_from_pathable(synth.make_map(CW, CW, C2_SEED + 17 * layer, rivers=True), CW, CW)
        nav.map_upload_layer(layer, cost)
        nav.map_build_nav(layer)
        nav.route_build(layer)
        costs.append(cost)
    return nav, costs


def _query(kind, layer, x, z, dst=(0.0, 0.0), tol=0.0, faction=capi.FACTION_ID_NONE):
    q = np.zeros(len(x), capi.MAP_QUERY)
    q["kind"], q["layer"], q["x"], q["z"] = kind, layer, x, z
    q["dst_x"], q["dst_z"], q["tolerance"], q["faction_id"] = dst[0], dst[1], tol, faction
    return q


def test_probe_kinds_vs_numpy_c2():
    nav, costs = _c2_nav()
    try:
        rng = np.random.default_rng(1)
        x, z = _points(rng, 1 << 20, CW, CW, (0.0, 0.0))
        for phase in range(2):
            if phase:         # committed blockers on both layer groups (ground 0..3)
                for _ in range(200):
                    nav.blockers_incref(float(rng.uniform(-CW * 256, 0)), float(rng.uniform(0, CW * 256)), float(rng.uniform(1, 12)))
                nav.map_commit()
                assert nav.blockers(0).any() and nav.blockers(1).any()
            for layer in range(2):
                want = _probe_expected(nav, layer, x, z, CW, CW, (0.0, 0.0))
                for kind, w in zip((capi.QUERY_PATHABLE, capi.QUERY_BLOCKED, capi.QUERY_ADJACENT_IMPASSABLE), want):
                    got = nav.map_query(_query(kind, layer, x, z))
                    assert (got["ok"].astype(bool) == w).all(), (phase, layer, kind, int((got["ok"].astype(bool) != w).sum()))
                    assert (~w).any() and (w.any() or (kind == capi.QUERY_BLOCKED and phase == 0))
    finally:
        nav.close()


def test_probe_kinds_shifted_origin_1x1():
    nav = capi.Nav(0)
    try:
        map_xz = (300.0, -77.0)
        cost = mq.blocked_rect_map(1, 1, 0x5EED0500, [(10, 10, 30, 20)])
        nav.map_create(1, 1, 1, *map_xz)
        nav.map_upload_layer(0, cost)
        nav.map_build_nav(0)
        nav.blockers_incref(*mq.tile_xz(40, 40, map_xz), 5.0)
        nav.map_commit()
        x, z = _points(np.random.default_rng(2), 1 << 16, 1, 1, map_xz)
        want = _probe_expected(nav, 0, x, z, 1, 1, map_xz)
        for kind, w in zip((capi.QUERY_PATHABLE, capi.QUERY_BLOCKED, capi.QUERY_ADJACENT_IMPASSABLE), want):
            assert (nav.map_query(_query(kind, 0, x, z))["ok"].astype(bool) == w).all()
    finally:
        nav.close()


def test_dest_id_vs_request_path(pfref_or_golden):
    nav, costs = _c2_nav(nlayers=1)
    try:
        nav.pool_create(64, 4096)
        rng = np.random.default_rng(3)
        img = synth.blocked_to_image(costs[0], CW, CW)
        free = np.argwhere(img != 0xFF)
        src = mq.tile_xz(*[int(v) for v in free[0]])
        dst = [mq.tile_xz(*[int(v) for v in free[rng.integers(0, len(free))]]) for _ in range(24)]
        dst += [(float(rng.uniform(-CW * 256, 0)), float(rng.uniform(0, CW * 256))) for _ in range(8)]
        x, z = np.array([d[0] for d in dst], f32), np.array([d[1] for d in dst], f32)
        for faction in (capi.FACTION_ID_NONE, 3):
            nav.request_faction(faction)
            want = [nav.pool_request_path(i, src, d)[1] for i, d in enumerate(dst)]
            got = nav.map_query(_query(capi.QUERY_DEST_ID, 0, x, z, faction=faction))
            assert (got["ok"] == 1).all() and list(got["dest_id"]) == want, faction
        nav.request_faction(capi.FACTION_ID_NONE)
        off = nav.map_query(_query(capi.QUERY_DEST_ID, 0, np.array([10.0], f32), np.array([10.0], f32)))
        assert off["ok"][0] == 0
        if pfref_or_golden is not None:
            ref = pfref_or_golden.RefMap(CW, CW, synth.make_map(CW, CW, C2_SEED, rivers=True))
            got = nav.map_query(_query(capi.QUERY_DEST_ID, 0, x, z))
            assert list(got["dest_id"]) == [ref.dest_id(d) for d in dst]
    finally:
        nav.close()


def _check_searches(nav, q, cw, ch, map_xz=(0.0, 0.0)):
    got = nav.map_query(q)
    want, _ = mq.reference(nav, q, cw, ch, map_xz)
    bad = [(tuple(q[i]), tuple(got[i]), tuple(want[i])) for i in range(len(q)) if got[i] != want[i]]
    assert not bad, bad[:5]
    return got


@pytest.mark.parametrize("cw", [1, 16])
def test_searches_vs_host_synthetic(cw):
    """1 x 1 and 16 x 16 maps with impassable rectangles and committed blockers, tolerances 0 and 1.5 x radius"""
    rng = np.random.default_rng(10 + cw)
    side = min(40, 64 * cw - 8)
    r0, c0 = int(rng.integers(0, cw * 64 - side + 1)), int(rng.integers(0, cw * 64 - side + 1))
    cost = mq.blocked_rect_map(cw, cw, 0x5EED0600 + cw, [(r0, c0, r0 + side, c0 + side)])
    nav = capi.Nav(0)
    try:
        nav.map_create(cw, cw, 1)
        nav.map_upload_layer(0, cost)
        nav.map_build_nav(0)
        nav.route_build(0)
        for _ in range(10 * cw):
            nav.blockers_incref(float(rng.uniform(-cw * 256, 0)), float(rng.uniform(0, cw * 256)), float(rng.uniform(1, 8)))
        nav.map_commit()
        tiles = mq.search_tiles(cost, cw, cw, rng, 40, [(r0 + side // 2, c0 + side // 2)])
        _check_searches(nav, mq.search_queries(tiles, tolerances=(0.0, 1.5 * 3.0, 1.5 * 7.5), rng=rng), cw, cw)
    finally:
        nav.close()


def test_searches_vs_host_c2_two_layers():
    nav, costs = _c2_nav()
    try:
        rng = np.random.default_rng(4)
        for _ in range(300):
            nav.blockers_incref(float(rng.uniform(-CW * 256, 0)), float(rng.uniform(0, CW * 256)), float(rng.uniform(1, 12)))
        nav.map_commit()
        q = np.concatenate([mq.search_queries(mq.search_tiles(costs[layer], CW, CW, rng, 60), layer=layer,
                                              tolerances=(0.0, 1.5 * 5.0), rng=rng) for layer in range(2)])
        _check_searches(nav, q, CW, CW)
    finally:
        nav.close()


def test_searches_host_fallback():
    """searches that leave the kernel's 128 x 128 window are finished on the host with the same answers"""
    img = np.ones((256, 256), np.uint8)
    img[28:228, 28:228] = 0xFF
    img[60, 128] = 1
    nav = capi.Nav(0)
    try:
        nav.map_create(4, 4, 1)
        nav.map_upload_layer(0, synth.image_to_blocked(img, 4, 4))
        nav.map_build_nav(0)
        nav.route_build(0)
        cx, cz = mq.tile_xz(128, 128)
        ix, iz = mq.tile_xz(60, 128)
        q = np.array([(capi.QUERY_CLOSEST_PATHABLE, 0, cx, cz, 0, 0, 0, 0),
                      (capi.QUERY_MAXIMALLY_CLOSE, 0, ix, iz, ix, iz, 100.0, 0),
                      (capi.QUERY_MAXIMALLY_CLOSE, 0, cx, cz, cx, cz, 0.0, 0)], capi.MAP_QUERY)
        got = _check_searches(nav, q, 4, 4)
        assert got["ok"][0] == 1 and got["ok"][1] == 0
    finally:
        nav.close()


def test_commit_ordering():
    nav, costs = _c2_nav(nlayers=1)
    try:
        img = synth.blocked_to_image(costs[0], CW, CW)
        free = np.argwhere(img != 0xFF)
        r, c = [int(v) for v in free[len(free) // 2]]
        x, z = mq.tile_xz(r, c)
        q = np.concatenate([_query(k, 0, np.array([x], f32), np.array([z], f32)) for k in
                            (capi.QUERY_BLOCKED, capi.QUERY_CLOSEST_PATHABLE)])
        before = nav.map_query(q)
        assert before["ok"][0] == 0 and before["ok"][1] == 1 and before["x"][1] == f32(x)
        nav.blockers_incref(x, z, 6.0)
        assert (nav.map_query(q) == before).all(), "an increment that is not committed must not be seen"
        nav.map_commit()
        after = nav.map_query(q)
        assert after["ok"][0] == 1 and after["ok"][1] == 1 and after["x"][1] != f32(x)
        _check_searches(nav, q[1:], CW, CW)
    finally:
        nav.close()


def test_errors():
    nav = capi.Nav(0)
    try:
        nav.map_create(1, 1, 2)
        cost = mq.blocked_rect_map(1, 1, 0x5EED0700, [])
        nav.map_upload_layer(0, cost)
        nav.map_build_nav(0)
        good = _query(capi.QUERY_PATHABLE, 0, np.array([-2.0], f32), np.array([2.0], f32))
        for bad in (dict(kind=6), dict(kind=-1), dict(layer=2), dict(layer=-1),
                    dict(kind=capi.QUERY_MAXIMALLY_CLOSE, tolerance=np.nan),
                    dict(kind=capi.QUERY_MAXIMALLY_CLOSE),                      # before pfnav_route_build
                    dict(kind=capi.QUERY_DEST_ID, faction_id=16)):
            q = np.concatenate([good, good])
            for k, v in bad.items():
                q[k][1] = v
            sentinel = np.array([(7, 7, 7.0, 7.0)] * 2, capi.MAP_QUERY_RESULT)
            out = sentinel.copy()
            with pytest.raises(capi.PfnavError, match="error -1"):
                nav.map_query(q, out=out)
            assert (out == sentinel).all(), bad
        nav.route_build(0)
        q = _query(capi.QUERY_MAXIMALLY_CLOSE, 0, np.array([-2.0], f32), np.array([2.0], f32), dst=(-2.0, 2.0))
        nav.map_query(q)
        q["tolerance"] = np.inf
        with pytest.raises(capi.PfnavError, match="error -1"):
            nav.map_query(q)
        assert len(nav.map_query(np.zeros(0, capi.MAP_QUERY))) == 0
    finally:
        nav.close()
    host = capi.Nav(hostonly=True)
    try:
        host.map_create(1, 1, 1)
        with pytest.raises(capi.PfnavError, match="error -3"):
            host.map_query(np.zeros(1, capi.MAP_QUERY))
    finally:
        host.close()
