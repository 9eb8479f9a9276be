"""The device source of pfnav_map_query's search kernel (csrc/pfnav_query_kernel.cuh) run as one warp on CPU threads
(tests/emu/query_emu.cpp) against the host routine pfnav_route_arrival_consts on a host-only context: the answer of
N_ClosestPathable and the tile list of n_closest_island_tiles that N_IsMaximallyClose compares with. Both searches return
the first tiles in the reference's queue order, so the window replay must give the same tile and the same list in the same
order; a search that leaves the 128 x 128 window must say so instead. Test infrastructure, not a product path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import map_query_cases as mq

capi, synth = mq.capi, mq.synth
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libquery_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fno-strict-aliasing", "-fPIC", "-shared", "-pthread",
                    os.path.join(HERE, "emu", "query_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_map_search.argtypes = [C.c_void_p] * 3 + [C.c_int, C.c_int, C.c_float, C.c_float] + [C.c_void_p, C.c_int] + [C.c_void_p] * 4
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _host_nav(cw, ch, cost_c, blk_c=None, map_xz=(0.0, 0.0), blockers=()):
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1, *map_xz)
    nav.map_upload_layer(0, cost_c, blk_c)
    nav.map_build_nav(0)
    nav.route_build(0)
    for x, z, radius in blockers:            # committed blockers: N_BlockersIncref + N_Update
        nav.blockers_incref(x, z, radius)
    if blockers:
        nav.map_commit()
    return nav


def _check(emu, nav, cw, ch, cost_c, q, map_xz=(0.0, 0.0)):
    """run the emulated kernel on the search queries q; compare every query it finished with the host routine.
    Returns the fallback flags."""
    cost = mq.image(np.ascontiguousarray(cost_c, np.uint8), cw, ch)
    blk = mq.image(nav.blockers(0), cw, ch)
    gisl = mq.image(nav.route_islands(0), cw, ch)
    n = len(q)
    out = np.zeros(n, capi.MAP_QUERY_RESULT)
    fb = np.zeros(n, np.uint8)
    mc_rc = np.zeros((n, 256, 2), np.int32)
    mc_n = np.zeros(n, np.int32)
    assert emu.emu_map_search(_p(cost), _p(blk), _p(gisl), cw, ch, map_xz[0], map_xz[1], _p(q), n, _p(out), _p(fb),
                              _p(mc_rc), _p(mc_n)) == 0
    want, lists = mq.reference(nav, q, cw, ch, map_xz)
    f = np.float32
    bad = []
    for i in range(n):
        if fb[i]:
            continue
        if out[i] != want[i]:
            bad.append((i, tuple(q[i]), tuple(out[i]), tuple(want[i])))
        if lists[i] is not None:
            rc = mc_rc[i, :mc_n[i]]
            got = np.stack([f(map_xz[0]) - rc[:, 1].astype(f) * f(4), f(map_xz[1]) + rc[:, 0].astype(f) * f(4)], 1)
            if mc_n[i] < 0 or got.shape != lists[i].shape or (got != lists[i]).any():
                bad.append((i, tuple(q[i]), "list", int(mc_n[i]), len(lists[i])))
    assert not bad, bad[:5]
    return fb


def _golden_maps():
    g = np.load(os.path.join(HERE, "golden", "route_3x3.npz"))
    yield "route_3x3", 3, 3, g["cost0"]
    yield "route_3x3_1", 3, 3, g["cost1"]
    g = np.load(os.path.join(HERE, "golden", "demo_map.npz"))
    yield "demo_map", 4, 4, g["cost_0"]
    g = np.load(os.path.join(HERE, "golden", "stress.npz"))
    yield "stress", 4, 4, g["cost"]


@pytest.mark.parametrize("name", ["route_3x3", "route_3x3_1", "demo_map", "stress"])
def test_map_search_source_vs_host_golden(emu, name):
    _, cw, ch, cost_c = next(m for m in _golden_maps() if m[0] == name)
    rng = np.random.default_rng(len(name))
    nav = _host_nav(cw, ch, cost_c)
    try:
        q = mq.search_queries(mq.search_tiles(cost_c, cw, ch, rng, 40), tolerances=(0.0, 6.0), rng=rng)
        fb = _check(emu, nav, cw, ch, cost_c, q)
        assert not fb.any(), "no golden-map search leaves the window"
    finally:
        nav.close()


@pytest.mark.parametrize("cw,ch", [(1, 1), (3, 3), (16, 16)])
def test_map_search_source_vs_host_synthetic(emu, cw, ch):
    """impassable rectangles with targets inside them, corners, chunk borders, committed blockers, a shifted map origin"""
    rng = np.random.default_rng(cw)
    side = min(40, 64 * min(cw, ch) - 8)
    r0, c0 = int(rng.integers(0, ch * 64 - side + 1)), int(rng.integers(0, cw * 64 - side + 1))
    cost_c = mq.blocked_rect_map(cw, ch, 0x5EED0400 + cw, [(r0, c0, r0 + side, c0 + side), (0, 0, 6, 9)])
    map_xz = (512.0, -256.0)
    # blockers: one on a free tile (a search target below), others at random
    img = synth.blocked_to_image(cost_c, cw, ch)
    free = np.argwhere(img != 0xFF)
    bt = [tuple(int(v) for v in free[rng.integers(0, len(free))]) for _ in range(6)]
    blockers = [(*mq.tile_xz(r, c, map_xz), float(rng.choice([1.0, 3.0, 7.0]))) for r, c in bt]
    nav = _host_nav(cw, ch, cost_c, map_xz=map_xz, blockers=blockers)
    try:
        assert nav.blockers(0).any()
        extra = [(r0 + side // 2, c0 + side // 2), (r0, c0), (r0 + side - 1, c0 + side - 1), (2, 3)] + bt
        q = mq.search_queries(mq.search_tiles(cost_c, cw, ch, rng, 30 if cw < 16 else 20, extra), tolerances=(0.0, 6.0),
                              map_xz=map_xz, rng=rng)
        _check(emu, nav, cw, ch, cost_c, q, map_xz)
    finally:
        nav.close()


def test_map_search_window_overflow(emu):
    """a 200 x 200 impassable blob: N_ClosestPathable from its centre and n_closest_island_tiles of a one-tile island in
    it both need tiles outside the 128 x 128 window, and the kernel must flag them for the host"""
    cw = ch = 4
    img = np.zeros((256, 256), np.uint8) + 1
    img[28:228, 28:228] = 0xFF
    img[60, 128] = 1                                     # a one-tile island 68 tiles from the centre
    cost_c = synth.image_to_blocked(img, cw, ch)
    nav = _host_nav(cw, ch, cost_c)
    try:
        cx, cz = mq.tile_xz(128, 128)
        ix, iz = mq.tile_xz(60, 128)
        q = np.array([(capi.QUERY_CLOSEST_PATHABLE, 0, cx, cz, 0, 0, 0, 0),
                      (capi.QUERY_MAXIMALLY_CLOSE, 0, ix, iz, ix, iz, 100.0, 0),
                      (capi.QUERY_CLOSEST_PATHABLE, 0, *mq.tile_xz(70, 128), 0, 0, 0, 0),        # finds the island in the window
                      (capi.QUERY_MAXIMALLY_CLOSE, 0, cx, cz, cx, cz, 0.0, 0)], capi.MAP_QUERY)
        fb = _check(emu, nav, cw, ch, cost_c, q)
        assert list(fb) == [1, 1, 0, 0]
        want, lists = mq.reference(nav, q, cw, ch)
        assert want[0]["ok"] == 1 and len(lists[1]) == 0    # what the host finishes: a corner 100 tiles away, no tiles
    finally:
        nav.close()
