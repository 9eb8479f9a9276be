"""The device source of k_zone_seed_bits (csrc/pfnav_zone_kernel.cuh), the TARGET_ZONE seed flood of
pfnav_pool_request_zones, run as one warp on CPU threads (tests/emu/zone_emu.cpp) against the host flood
(pfnav_zone_seeds on a host-only context). The field bytes depend on the exact seed set, which the budget cuts in the
reference's heap order, so the bitmaps must be equal. Test infrastructure, not a product path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

capi, synth = cases.capi, cases.synth
HERE = os.path.dirname(os.path.abspath(__file__))
ZONE_JOB = np.dtype([("layer", "<i4"), ("centre_r", "<i4"), ("centre_c", "<i4"), ("base_r", "<i4"), ("base_c", "<i4"),
                     ("budget", "<i4")])
RADII = (0, 1, 2, 5, 13, 40, 73, 90)


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libzone_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fno-strict-aliasing", "-fPIC", "-shared", "-pthread",
                    os.path.join(HERE, "emu", "zone_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_zone_seed_bits.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
    return L


def _image(a, cw, ch):
    """[chunks][64][64] -> row-major [H64][W64] (the device layout)"""
    return np.ascontiguousarray(a.reshape(ch, cw, 64, 64).transpose(0, 2, 1, 3).reshape(ch * 64, cw * 64))


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _base(dim, cr, cc):
    return (cr * 64 - 32 if cr > 0 and dim > 64 else cr * 64), (cc * 64 - 32 if cc > 0 and dim > 64 else cc * 64)


def _budget(dim, radius):
    return min(int(np.pi * radius * radius + 0.5), dim * dim)


def _synthetic(cw, ch, seed):
    """a synthetic map with a large blocked square and scattered blockers (chunk-blocked cost and blocker arrays)"""
    rng = np.random.default_rng(seed)
    img = synth.blocked_to_image(synth.cost_from_pathable(synth.make_map(cw, ch, seed, frac_blocked=0.3, rivers=cw > 1), cw, ch), cw, ch)
    img = img.copy()
    side = min(40, 64 * min(cw, ch) - 8)
    r0, c0 = int(rng.integers(0, ch * 64 - side + 1)), int(rng.integers(0, cw * 64 - side + 1))
    img[r0:r0 + side, c0:c0 + side] = 0xFF
    blk = np.zeros_like(img, dtype=np.uint16)
    for _ in range(30 * cw * ch):
        r, c = int(rng.integers(0, ch * 64)), int(rng.integers(0, cw * 64))
        blk[r:r + int(rng.integers(1, 5)), c:c + int(rng.integers(1, 5))] = 1
    return synth.image_to_blocked(img, cw, ch), synth.image_to_blocked(blk, cw, ch), (r0 + side // 2, c0 + side // 2)


def _centres(cw, ch, cost_c, rng, n, inside):
    """random tiles, blocked tiles, the middle of the blocked square, chunk borders, map edges and corners"""
    H, W = ch * 64, cw * 64
    img = synth.blocked_to_image(cost_c, cw, ch)
    blocked = np.argwhere(img == 0xFF)
    out = [(int(rng.integers(0, H)), int(rng.integers(0, W))) for _ in range(n)]
    out += [tuple(int(v) for v in blocked[rng.integers(0, len(blocked))]) for _ in range(n // 2)] if len(blocked) else []
    out += [inside, (0, 0), (H - 1, W - 1), (0, W - 1), (H - 1, 0), (H // 2, 0), (0, W // 2)]
    for _ in range(n // 2):
        out.append((64 * int(rng.integers(0, ch)) + int(rng.choice([0, 31, 32, 63])), int(rng.integers(0, W))))
        out.append((int(rng.integers(0, H)), 64 * int(rng.integers(0, cw)) + int(rng.choice([0, 31, 32, 63]))))
    return out


def _check(emu, cw, ch, cost_c, blk_c, centres, rng):
    dim = 64 if cw == ch == 1 else 128
    nav = capi.Nav(hostonly=True)
    try:
        nav.map_create(cw, ch, 1)
        nav.map_upload_layer(0, cost_c, blk_c)
        cost, blk = _image(cost_c, cw, ch), _image(blk_c, cw, ch)
        jobs, want = [], []
        for k, centre in enumerate(centres):
            radius = RADII[k % len(RADII)]
            # every chunk whose window holds the centre, and one whose window does not
            chunks = [(cr, cc) for cr in range(ch) for cc in range(cw)
                      if 0 <= centre[0] - _base(dim, cr, cc)[0] < dim and 0 <= centre[1] - _base(dim, cr, cc)[1] < dim]
            away = [(cr, cc) for cr in range(ch) for cc in range(cw) if (cr, cc) not in chunks]
            if away:
                chunks.append(away[int(rng.integers(0, len(away)))])
            for cr, cc in chunks:
                br, bc = _base(dim, cr, cc)
                jobs.append((0, centre[0], centre[1], br, bc, _budget(dim, radius)))
                s = nav.zone_seeds((cr, cc), centre, radius)
                bm = np.zeros((dim, dim), bool)
                bm[s[:, 0] - br, s[:, 1] - bc] = True
                want.append(bm)
        jobs = np.array(jobs, ZONE_JOB)
        bits = np.zeros((len(jobs), dim * dim // 32), np.uint32)
        assert emu.emu_zone_seed_bits(_p(cost), _p(blk), ch * 64, cw * 64, dim, _p(jobs), len(jobs), _p(bits)) == 0
        got = np.unpackbits(bits.view(np.uint8), bitorder="little").reshape(len(jobs), dim, dim).astype(bool)
        bad = [i for i in range(len(jobs)) if (got[i] != want[i]).any()]
        assert not bad, [tuple(jobs[i]) for i in bad[:5]]
        assert sum(int(w.sum()) for w in want) > 0
    finally:
        nav.close()


@pytest.mark.parametrize("cw,ch", [(1, 1), (3, 3), (16, 16)])
def test_zone_flood_source_vs_host_flood_synthetic(emu, cw, ch):
    cost_c, blk_c, inside = _synthetic(cw, ch, 0x5EED0300 + cw)
    rng = np.random.default_rng(cw)
    _check(emu, cw, ch, cost_c, blk_c, _centres(cw, ch, cost_c, rng, 40 if cw < 16 else 24, inside), rng)


def test_zone_flood_source_vs_host_flood_golden_map(emu):
    g = np.load(os.path.join(HERE, "golden", "region.npz"))
    cw = ch = 3
    rng = np.random.default_rng(7)
    centres = [tuple(int(v) for v in c) for c in g["zc"]] + _centres(cw, ch, g["cost"], rng, 30, (96, 96))
    _check(emu, cw, ch, g["cost"], g["blk"], centres, rng)
