"""The device source of k_region_fields (csrc/pfnav_region_kernel.cuh) run as one thread block on CPU threads
(tests/emu/region_emu.cpp: CUDA keywords as plain C++, __syncthreads = a pthread barrier) against the golden vectors
of the compiled reference. It checks the kernel's index arithmetic and fixed-point logic without a GPU; it is test
infrastructure, not a product path (libpfnav.so has no CPU fallback)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

capi, synth = cases.capi, cases.synth
HERE = os.path.dirname(os.path.abspath(__file__))
GOLD = os.path.join(HERE, "golden")


def gold(name):
    return np.load(os.path.join(GOLD, name + ".npz"))


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libregion_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O1", "-fPIC", "-shared", "-pthread", os.path.join(HERE, "emu", "region_emu.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    L.emu_region_fields.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                    C.c_void_p, C.c_void_p, C.c_int]
    return L


def _image(a, cw, ch):
    """[chunks][64][64] -> row-major [H64][W64] (the device layout)"""
    return np.ascontiguousarray(a.reshape(ch, cw, 64, 64).transpose(0, 2, 1, 3).reshape(ch * 64, cw * 64))


def _fmask(fac, cw, ch):
    m = np.zeros((cw * ch, 64, 64), np.uint16)
    for f in range(15):
        m |= (fac[:, f] > 0).astype(np.uint16) << f
    return _image(m, cw, ch)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _run(emu, cost, blk, fmask, dim, rec, sd, ov, out, chunk_out):
    sd = np.ascontiguousarray(np.concatenate([sd, np.zeros((1, 2), np.int32)]))
    ov = np.ascontiguousarray(np.concatenate([ov, np.zeros((1, 2), np.int32)]))
    emu.emu_region_fields(_p(cost), _p(blk), _p(fmask), cost.shape[1], cost.shape[0], dim, _p(rec), len(rec), _p(sd), _p(ov), _p(out),
                          chunk_out)
    return out


@pytest.mark.parametrize("dim", [96, 32])
def test_region_kernel_source_on_cpu_threads(emu, dim):
    g = gold("region")
    cw = ch = 3
    cost, blk, fmask = _image(g["cost"], cw, ch), _image(g["blk"], cw, ch), _fmask(g["factions"], cw, ch)
    reqs = cases.region_reqs_from_golden(g["req%d" % dim], g["ov%d" % dim])
    rec, sd, ov = capi.pack_region_reqs(reqs)
    got = _run(emu, cost, blk, fmask, dim, rec, sd, ov, np.zeros((len(reqs), dim, dim // 2), np.uint8), 0)
    bad = [i for i in range(len(reqs)) if (got[i] != g["exp%d" % dim][i]).any()]
    assert not bad, bad
    # the fix-up alone, in place on the create-only fields
    fix = [i for i, q in enumerate(reqs) if q["start"] is not None]
    rec, sd, ov = capi.pack_region_reqs([dict(reqs[i], no_create=True) for i in fix])
    upd = _run(emu, cost, blk, fmask, dim, rec, sd, ov, np.ascontiguousarray(g["create%d" % dim][fix]), 0)
    assert (upd == g["exp%d" % dim][fix]).all()


def test_chunk_window_kernel_source_on_cpu_threads(emu, pforacle):
    """the padded-chunk mode (zone / entity / enemies fields): seeds from the port / the host code, integration + the
    64 x 64 window from the kernel source"""
    g = gold("region")
    cw = ch = 3
    cost, blk = _image(g["cost"], cw, ch), _image(g["blk"], cw, ch)
    fmask = np.zeros_like(blk)
    om = pforacle.OracleMap(cw, ch, g["cost"], g["blk"], None)
    for k in (3, 6, 9, 11):
        rec = np.zeros(cw * ch, capi.REGION_REQ); sds = []
        for c in range(cw * ch):
            s = om.zone_seeds((c // cw, c % cw), g["zc"][k], int(g["zrad"][k]))
            rec["center_r"][c], rec["center_c"][c] = c // cw, c % cw
            rec["seed_off"][c], rec["seed_n"][c] = sum(len(x) for x in sds), len(s)
            rec["flags"][c] = capi.REGION_CREATE
            sds.append(s)
        got = _run(emu, cost, blk, fmask, 128, rec, np.concatenate(sds).astype(np.int32), np.zeros((0, 2), np.int32),
                   np.full((cw * ch, 64, 64), 0xEE, np.uint8), 1)
        assert (got == g["zexp"][k]).all(), k


@pytest.mark.parametrize("cw,ch,map_xz,seed", [(2, 5, (601.3, -250.9), 0x5EED0C10), (1, 1, (0.0, 0.0), 0x5EED0C11)],
                         ids=["2x5_offset", "1x1"])
def test_chunk_window_kernel_source_vs_port(emu, pforacle, cw, ch, map_xz, seed):
    """the padded-chunk mode on generated inputs: a non-square 2 x 5 map at an offset that is not tile-aligned (windows
    of 128, the last row's and column's running past the map) and a 1 x 1 map (a window of 64), with committed
    blockers. Zone seeds from the port, entity / enemies seeds from the host code; every chunk's field from the kernel
    source on CPU threads == OracleMap.flow_field_zone / chunk_field_seeded"""
    rng = np.random.default_rng(seed)
    H, W = ch * 64, cw * 64
    cost = synth.cost_from_pathable(synth.make_map(cw, ch, seed, rivers=cw > 1 and ch > 1), cw, ch)
    nav = capi.Nav(hostonly=True)
    try:
        nav.map_create(cw, ch, 1, *map_xz); nav.map_upload_layer(0, cost); nav.map_build_nav(0)
        for _ in range(30 * cw * ch):
            nav.blockers_incref(map_xz[0] - rng.uniform(0, W * 4), map_xz[1] + rng.uniform(0, H * 4), rng.uniform(2, 12), 0)
        nav.map_commit()
        blk = nav.blockers(0)
        om = pforacle.OracleMap(cw, ch, cost, blk, None, map_x=map_xz[0], map_z=map_xz[1])
        chunks = [divmod(c, cw) for c in range(cw * ch)]
        open_ = np.argwhere(synth.blocked_to_image(cost, cw, ch) != 0xFF)
        zones = [(tuple(int(v) for v in open_[i]), r) for i, r in zip(rng.integers(0, len(open_), 6), (0, 2, 13, 40, 73, 90))]
        zones += [((0, 0), 20), ((H - 1, W - 1), 50), ((H - 1, 0), 90)]
        fp = capi.Nav.footprints(np.stack([map_xz[0] - rng.uniform(0, W * 4, 40), map_xz[1] + rng.uniform(0, H * 4, 40)], 1),
                                 rng.choice(np.array([0.0, 6.0, 20.0, 40.0, 60.0], np.float32), 40))
        ents = [(capi.TARGET_ENEMIES, fp, L) for L in (0, 3)] + [(capi.TARGET_ENTITY, fp[i:i + 1], 1) for i in range(0, 40, 8)]
        jobs, sds = [], []
        for c in chunks:
            for centre, r in zones:
                jobs.append((c, om.flow_field_zone(c, centre, r)))
                sds.append(om.zone_seeds(c, centre, r))
            for kind, f, L in ents:
                s = nav.entity_seeds(kind, f, c, L)
                jobs.append((c, om.chunk_field_seeded(c, s)))
                sds.append(s)
    finally:
        nav.close()
    rec = np.zeros(len(jobs), capi.REGION_REQ)
    for i, ((cr, cc), _) in enumerate(jobs):
        rec["center_r"][i], rec["center_c"][i] = cr, cc
        rec["seed_off"][i], rec["seed_n"][i] = sum(len(x) for x in sds[:i]), len(sds[i])
        rec["flags"][i] = capi.REGION_CREATE
    dim = 128 if cw > 1 and ch > 1 else 64
    got = _run(emu, _image(cost, cw, ch), _image(blk, cw, ch), np.zeros((H, W), np.uint16), dim, rec,
               np.concatenate(sds).astype(np.int32).reshape(-1, 2), np.zeros((0, 2), np.int32),
               np.zeros((len(jobs), 64, 64), np.uint8), 1)
    bad = [(i, jobs[i][0]) for i in range(len(jobs)) if (got[i] != jobs[i][1]).any()]
    assert not bad, bad[:8]
    # the fields reach the last chunk row and column, and some seed sets are empty (windows without the zone centre)
    nonempty = [jobs[i][0] for i in range(len(jobs)) if jobs[i][1].any()]
    assert any(c[0] == ch - 1 for c in nonempty) and any(c[1] == cw - 1 for c in nonempty)
    assert any(len(s) == 0 for s in sds) and sum(len(s) > 0 for s in sds) > len(sds) // 4


@pytest.mark.parametrize("seed,dim,n", [(92, 64, 40), (93, 128, 16), (94, 96, 60)])
def test_region_kernel_source_vs_port(emu, pforacle, seed, dim, n):
    """further window sizes (incl. PFNAV_REGION_DIM_MAX) and a 4 x 4-chunk map: kernel source on CPU threads vs the port"""
    cw = ch = 4
    p, blockers, wars, reqs = cases.region_case(seed, cw, ch, n, dim)
    cost_c = synth.cost_from_pathable(p, cw, ch)
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, cost_c); nav.map_build_nav(0)
    for x, z, r, f in blockers:
        nav.blockers_incref(float(x), float(z), float(r), int(f), 0)
    nav.map_commit()
    blk_c, fac = nav.blockers(0), nav.faction_counts(0)
    nav.close()
    cases.region_pick_starts(reqs, cost_c, blk_c, cw, ch, seed, dim)
    om = pforacle.OracleMap(cw, ch, cost_c, blk_c, None, factions=fac)
    rec, sd, ov = capi.pack_region_reqs(reqs)
    got = _run(emu, _image(cost_c, cw, ch), _image(blk_c, cw, ch), _fmask(fac, cw, ch), dim, rec, sd, ov,
               np.zeros((len(reqs), dim, dim // 2), np.uint8), 0)
    for i, q in enumerate(reqs):
        e = om.region_field_create(dim, q["enemies"], 1, [q["target"]], q["center"], q["overlay"])
        if q["start"] is not None:
            e = om.region_field_fixup(dim, q["start"], q["center"], e, q["overlay"])
        assert (got[i] == e).all(), (seed, dim, i, q)
