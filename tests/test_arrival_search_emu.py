"""The whole-layer search tier (mq_layer_search in csrc/pfnav_layer_search.cuh) run as one CTA on CPU threads
(tests/emu/arrival_emu.cpp) against the host routine pfnav_route_arrival_consts on host-only contexts. It must return the
nearest tile of N_ClosestPathable and the tile list of n_closest_island_tiles in the same order, with the same 256 cap, on
searches that reach far past any window: large impassable blobs, cuts that fall on the next Chebyshev level, map corners,
one-chunk and non-square maps, shifted map origins and blocked targets. Test infrastructure, not a product path."""
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
    so = str(tmp_path_factory.mktemp("emu") / "libarrival_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fno-strict-aliasing", "-fPIC", "-shared", "-pthread",
                    os.path.join(HERE, "emu", "arrival_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_layer_search.argtypes = [C.c_void_p] * 3 + [C.c_int, C.c_int, C.c_float, C.c_float, C.c_int] + \
        [C.c_void_p] * 3 + [C.c_int, C.c_int] + [C.c_void_p] * 3
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _host_nav(cw, ch, img, map_xz=(0.0, 0.0), blockers=()):
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1, *map_xz)
    nav.map_upload_layer(0, synth.image_to_blocked(np.ascontiguousarray(img, np.uint8), cw, ch))
    nav.map_build_nav(0)
    nav.route_build(0)
    for x, z, radius in blockers:
        nav.blockers_incref(x, z, radius)
    if blockers:
        nav.map_commit()
    return nav


def _check(emu, cw, ch, img, tiles, map_xz=(0.0, 0.0), blockers=(), nt=64):
    """both searches from every (row, col) in tiles, on the tier and on the host; returns the host's answers"""
    nav = _host_nav(cw, ch, img, map_xz, blockers)
    try:
        cost = np.ascontiguousarray(img, np.uint8)
        blk = mq.image(nav.blockers(0), cw, ch)
        gisl = mq.image(nav.route_islands(0), cw, ch)
        W = cw * 64
        want, searches = [], []
        for r, c in tiles:
            ok, nearest, mc = nav.route_arrival_consts(mq.tile_xz(r, c, map_xz))
            want.append((ok, nearest, mc))
            if cost[r, c] == 0xFF or blk[r, c] > 0:      # N_ClosestPathable searches from blocked targets only
                searches.append((1, r, c, len(want) - 1))
            searches.append((0, r, c, len(want) - 1))
        n = len(searches)
        cp, tr, tc = (np.array([s[k] for s in searches], np.int32) for k in range(3))
        out_tile, out_n = np.zeros(n, np.int32), np.zeros(n, np.int32)
        lists = np.zeros((n, 256, 2), np.float32)
        assert emu.emu_layer_search(_p(cost), _p(blk), _p(gisl), cw, ch, map_xz[0], map_xz[1], 0, _p(cp), _p(tr), _p(tc),
                                    n, nt, _p(out_tile), _p(lists), _p(out_n)) == 0
        f = np.float32
        bad = []
        for i, (is_cp, r, c, w) in enumerate(searches):
            ok, nearest, mc = want[w]
            if is_cp:
                t = int(out_tile[i])
                got = (0, None) if t < 0 else (1, (f(map_xz[0]) - f((t % W) // 64 * 256) - f(t % W % 64 * 4),
                                                   f(map_xz[1]) + f(t // W // 64 * 256) + f(t // W % 64 * 4)))
                if got[0] != ok or (ok and tuple(nearest) != got[1]):
                    bad.append(("nearest", r, c, got, ok, tuple(nearest)))
            elif out_n[i] != len(mc) or (lists[i, :out_n[i]] != mc).any():
                bad.append(("list", r, c, int(out_n[i]), len(mc)))
        assert not bad, bad[:5]
        return want
    finally:
        nav.close()


def test_layer_tier_window_overflow_blob(emu):
    """the 200 x 200 blob of test_map_search_window_overflow: both of its flagged searches, and more inside the blob"""
    img = np.zeros((256, 256), np.uint8) + 1
    img[28:228, 28:228] = 0xFF
    img[60, 128] = 1
    want = _check(emu, 4, 4, img, [(128, 128), (60, 128), (70, 128), (100, 200), (227, 28)])
    assert want[0][0] == 1 and len(want[1][2]) == 0


def test_layer_tier_far_nearest(emu):
    """a target whose nearest pathable tile is more than 300 tiles away"""
    img = np.zeros((384, 384), np.uint8) + 0xFF
    img[383, 0] = 1
    img[0, 383] = 1
    want = _check(emu, 6, 6, img, [(10, 40), (300, 300)], nt=128)
    assert all(w[0] == 1 for w in want)


def _square_blob(n, d0):
    """an impassable map with a passable square of Chebyshev radius d0 around its centre, whose centre and top-left
    corner are impassable: from the centre, n_closest_island_tiles first lists that corner (Manhattan 2 * d0, met last
    on its level), so the cut at mh > 2 * d0 falls on the next level"""
    rr, cc = np.mgrid[0:n, 0:n]
    c = n // 2
    img = np.where(np.maximum(np.abs(rr - c), np.abs(cc - c)) <= d0, 1, 0xFF).astype(np.uint8)
    img[c, c] = 0xFF
    img[c - d0, c - d0] = 0xFF
    return img


def test_layer_tier_list_cut_at_256(emu):
    """a hole of radius 130 around the target: its list is cut at 256 tiles on the next Chebyshev level"""
    want = _check(emu, 6, 6, _square_blob(384, 130), [(192, 192)], nt=128)
    assert len(want[0][2]) == 256


def test_layer_tier_cut_on_next_level(emu):
    """the same layout with a small hole: the Manhattan cut, not the cap, ends the list on the next level"""
    want = _check(emu, 2, 2, _square_blob(128, 10), [(64, 64), (54, 54), (64, 75)])
    assert 1 < len(want[0][2]) < 256


@pytest.mark.parametrize("cw,ch,map_xz", [(1, 1, (0.0, 0.0)), (5, 2, (640.0, -256.0)), (2, 5, (101.5, -37.25))])
def test_layer_tier_corners_and_shapes(emu, cw, ch, map_xz):
    """map corners, one chunk, a 5 x 2 map centred on the origin and a 2 x 5 one at a non-tile-aligned offset, with
    committed blockers (one on a search target)"""
    rng = np.random.default_rng(cw * 10 + ch)
    H, W = ch * 64, cw * 64
    img = np.where(rng.random((H, W)) < 0.35, 0xFF, 1).astype(np.uint8)
    img[H // 3:H // 3 + 20, :W - 5] = 0xFF
    tiles = [(0, 0), (0, W - 1), (H - 1, 0), (H - 1, W - 1), (H // 3 + 10, W // 2)]
    tiles += [(int(rng.integers(0, H)), int(rng.integers(0, W))) for _ in range(8)]
    free = np.argwhere(img != 0xFF)
    br, bc = (int(v) for v in free[rng.integers(0, len(free))])
    tiles.append((br, bc))
    blockers = [(*mq.tile_xz(br, bc, map_xz), 3.0)]
    _check(emu, cw, ch, img, tiles, map_xz, blockers, nt=32)


def test_layer_tier_blocked_target(emu):
    """a target tile covered by a committed blocker: N_ClosestPathable searches, and the island list skips blocked tiles"""
    img = np.zeros((128, 192), np.uint8) + 1
    img[:, 100:103] = 0xFF
    r, c = 64, 60
    _check(emu, 3, 2, img, [(r, c), (r, 99), (0, 103)], blockers=[(*mq.tile_xz(r, c), 7.0), (*mq.tile_xz(r, 99), 3.0)])
