"""The device source of the kind-0 repair seeds (csrc/pfnav_repair_kernel.cuh, the bit-row flood k_repair_chain runs for
N_FlowFieldUpdateToNearestPathable) run as one CTA on CPU threads (tests/emu/repair_emu.cpp) against the host's
breadth-first search (pfnav_repair_seeds through pfnav_repair_seed_mask on a host-only context). The repaired field
depends on the exact seed set, so the bitmaps must be equal. Test infrastructure, not a product path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

capi, synth = cases.capi, cases.synth
HERE = os.path.dirname(os.path.abspath(__file__))
NEAREST_PATHABLE = 0          # PFNAV_REPAIR_NEAREST_PATHABLE


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "librepair_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", "-pthread", os.path.join(HERE, "emu", "repair_emu.cpp"),
                    "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_repair_seeds.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _check(emu, img, blk, cw, ch, chunk, starts):
    """img / blk: row-major [ch*64][cw*64] images; starts: (r, c) inside `chunk`, every one non-passable"""
    cost_c, blk_c = synth.image_to_blocked(img, cw, ch), synth.image_to_blocked(blk, cw, ch)
    nav = capi.Nav(hostonly=True)
    try:
        nav.map_create(cw, ch, 1)
        nav.map_upload_layer(0, cost_c, blk_c)
        want = [nav.repair_seed_mask(chunk, NEAREST_PATHABLE, (r << 8) | c) for r, c in starts]
    finally:
        nav.close()
    st = np.array([(r << 6) | c for r, c in starts], np.int32)
    out = np.zeros((len(starts), 64), np.uint64)
    assert emu.emu_repair_seeds(_p(np.ascontiguousarray(img, np.uint8)), _p(np.ascontiguousarray(blk, np.uint16)), cw * 64,
                                chunk[0], chunk[1], _p(st), len(st), _p(out)) == 0
    got = np.unpackbits(out.view(np.uint8), bitorder="little").reshape(len(starts), 64, 64).astype(bool)
    bad = [starts[i] for i in range(len(starts)) if (got[i] != want[i]).any()]
    assert not bad, bad[:5]
    return want


def _nonpass_tiles(img, blk, chunk, rng, n):
    sub = (img[chunk[0] * 64:(chunk[0] + 1) * 64, chunk[1] * 64:(chunk[1] + 1) * 64] == 0xFF) | \
          (blk[chunk[0] * 64:(chunk[0] + 1) * 64, chunk[1] * 64:(chunk[1] + 1) * 64] > 0)
    t = np.argwhere(sub)
    if len(t) == 0:
        return []
    return [tuple(int(v) for v in t[k]) for k in rng.choice(len(t), min(n, len(t)), replace=False)]


@pytest.mark.parametrize("cw,ch,chunk", [(1, 1, (0, 0)), (2, 2, (1, 0)), (3, 3, (1, 1))])
def test_repair_seed_flood_synthetic(emu, cw, ch, chunk):
    """random walls and rivers, rectangular blobs touching the chunk edges, scattered blockers"""
    rng = np.random.default_rng(0x5EED0400 + cw)
    img = synth.blocked_to_image(synth.cost_from_pathable(synth.make_map(cw, ch, 11 + cw, frac_blocked=0.3, rivers=cw > 1),
                                                          cw, ch), cw, ch).copy()
    r0, c0 = chunk[0] * 64, chunk[1] * 64
    img[r0:r0 + 20, c0:c0 + 9] = 0xFF                 # touches the top and left edges
    img[r0 + 50:r0 + 64, c0 + 30:c0 + 64] = 0xFF      # touches the bottom and right edges
    blk = np.zeros_like(img, dtype=np.uint16)
    for _ in range(40):
        r, c = int(rng.integers(r0, r0 + 64)), int(rng.integers(c0, c0 + 64))
        blk[r:r + int(rng.integers(1, 5)), c:c + int(rng.integers(1, 5))] = 1
    starts = _nonpass_tiles(img, blk, chunk, rng, 120) + [(0, 0), (63, 63), (10, 0), (63, 40)]
    want = _check(emu, img, blk, cw, ch, chunk, starts)
    assert sum(int(w.sum()) for w in want) > 0


def test_repair_seed_flood_single_tiles_and_blockers(emu):
    """single-tile blobs (cost and blocker), and start tiles blocked only by a blocker, at corners and edges"""
    img = np.ones((128, 128), np.uint8)
    blk = np.zeros((128, 128), np.uint16)
    singles = [(0, 0), (0, 63), (63, 0), (63, 63), (31, 32), (5, 17)]
    for r, c in singles:
        img[64 + r, 64 + c] = 0xFF
    only_blk = [(10, 10), (0, 40), (40, 0), (62, 63)]
    for r, c in only_blk:
        blk[64 + r, 64 + c] = 3
    blk[64 + 20:64 + 23, 64 + 20:64 + 40] = 1          # a blocker bar next to a wall tile
    img[64 + 23, 64 + 30] = 0xFF
    starts = singles + only_blk + [(21, 25), (23, 30)]
    want = _check(emu, img, blk, 2, 2, (1, 1), starts)
    assert all(w.sum() >= 2 for w in want)


def test_repair_seed_flood_full_chunk(emu):
    """a blob that fills the chunk: the flood reaches every tile and there are no seeds; the same with one open tile"""
    img = np.ones((64, 64), np.uint8)
    img[:] = 0xFF
    blk = np.zeros((64, 64), np.uint16)
    want = _check(emu, img, blk, 1, 1, (0, 0), [(0, 0), (37, 12), (63, 63)])
    assert not any(w.any() for w in want)
    img[40, 40] = 1
    want = _check(emu, img, blk, 1, 1, (0, 0), [(0, 0), (39, 40)])
    assert all(w.sum() == 1 and w[40, 40] for w in want)
