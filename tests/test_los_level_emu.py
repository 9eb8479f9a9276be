"""The device source of k_los_level (csrc/pfnav_los_kernel.cuh), the level-parallel LOS pass with its certificate and
the byte-state replay as fallback, run as one warp on CPU threads (tests/emu/los_emu.cpp) against the plain-C port's
N_LOSFieldCreate. The fields must be equal byte for byte. Two more builds of the same source check the certificate
itself: with it compiled out (-DLOS_LEVEL_NO_CERTIFICATE) the level pass must get a field of the C2 batch wrong, so the
test can see an ordering error; with the replay forced for every field (-DLOS_LEVEL_ALWAYS_REPLAY) it must match the
port. Test infrastructure, not a product path."""
import collections
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

capi, synth = cases.capi, cases.synth
HERE = os.path.dirname(os.path.abspath(__file__))
REPLAYED = 1 << 31          # LOS_TRACE_REPLAYED in the trace's fourth word


def _build(tmp, name, defines=()):
    so = str(tmp / ("liblos_emu_%s.so" % name))
    subprocess.run(["g++", "-std=c++17", "-O2", "-fno-strict-aliasing", "-fPIC", "-shared", "-pthread", *defines,
                    os.path.join(HERE, "emu", "los_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_los_fields.argtypes = [C.c_void_p] * 4 + [C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p, C.c_int, C.c_void_p,
                                                    C.c_void_p, C.c_int]
    return L


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("los_emu")
    return {"level": _build(tmp, "level"), "nocert": _build(tmp, "nocert", ["-DLOS_LEVEL_NO_CERTIFICATE"]),
            "replay": _build(tmp, "replay", ["-DLOS_LEVEL_ALWAYS_REPLAY"])}


def _image(a, cw, ch):
    """[chunks][64][64] -> row-major [H64][W64] (the device layout)"""
    return np.ascontiguousarray(a.reshape(ch, cw, 64, 64).transpose(0, 2, 1, 3).reshape(ch * 64, cw * 64))


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def run_emu(L, cw, ch, cost, reqs, blk=None, factions=None, enemies=None, variant=2):
    """-> (fields [n][64][64], trace [n][4]) of one batch; cost / blk / factions chunk-blocked as the port takes them"""
    reqs = np.ascontiguousarray(reqs)
    assert all(int(q["prev_index"]) < i for i, q in enumerate(reqs))
    ci = _image(np.asarray(cost, np.uint8), cw, ch)
    bi = _image(np.zeros(cost.shape, np.uint16) if blk is None else np.asarray(blk, np.uint16), cw, ch)
    fi = None
    if factions is not None:
        fm = np.zeros(cost.shape, np.uint16)
        for f in range(factions.shape[1]):
            fm |= (factions[:, f] > 0).astype(np.uint16) << f
        fi = _image(fm, cw, ch)
    en = None if enemies is None else np.ascontiguousarray(enemies, np.uint16)
    out = np.zeros((len(reqs), 64, 64), np.uint8)
    trace = np.zeros((len(reqs), 4), np.uint64)
    assert L.emu_los_fields(_p(ci), _p(bi), _p(fi), _p(en), ch * 64, cw * 64, 0.0, 0.0, _p(reqs), len(reqs), _p(out),
                            _p(trace), variant) == 0
    return out, trace


def replayed(trace):
    return (trace[:, 3] & np.uint64(REPLAYED)) != 0


def c2_batch(ngoals=16):
    """the C2 map and `ngoals` goals on random passable tiles, every chunk of the 16 x 16 map chained to its goal through a
    breadth-first tree over chunks: 16 x 256 fields, the count of the C2 cold step"""
    cw = 16
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, 0x5EED0001, rivers=True), cw, cw)
    rng = np.random.default_rng(7)
    reqs = []
    for t in synth.random_passable_tiles(cost, ngoals, rng):
        ci, tr, tc = int(t[0]), int(t[1]), int(t[2])
        cr, cc = ci // cw, ci % cw
        td = (cr, cc, tr, tc)
        idx = {(cr, cc): len(reqs)}
        reqs.append(capi.los_req((cr, cc), td))
        dq = collections.deque([(cr, cc)])
        while dq:
            a = dq.popleft()
            for nb in ((a[0] + 1, a[1]), (a[0] - 1, a[1]), (a[0], a[1] + 1), (a[0], a[1] - 1)):
                if 0 <= nb[0] < cw and 0 <= nb[1] < cw and nb not in idx:
                    idx[nb] = len(reqs)
                    reqs.append(capi.los_req(nb, td, prev_index=idx[a], prev_chunk=a))
                    dq.append(nb)
    return cw, cost, np.concatenate(reqs)


def _bad(got, want):
    return [i for i in range(len(want)) if (got[i] != want[i]).any()]


def test_los_level_portal_los_golden(emu, pforacle):
    g = np.load(os.path.join(HERE, "golden", "portal_los.npz"))
    reqs = g["los_reqs"].view(capi.LOS_REQ)
    got, _ = run_emu(emu["level"], 3, 3, g["cost"], reqs)
    assert not _bad(got, g["los_exp"])
    assert not _bad(got, pforacle.OracleMap(3, 3, g["cost"]).los_fields_create(reqs))


@pytest.mark.parametrize("cw", [1, 4, 16])
def test_los_level_los_case_vs_port(emu, pforacle, cw):
    cost = synth.cost_from_pathable(cases.noise_map(cw, cw, 0x10500 + cw, 0.06), cw, cw)
    reqs = cases.los_case(cost, cw, cw, 0x10500 + cw, ntargets=6 if cw < 16 else 10)
    got, trace = run_emu(emu["level"], cw, cw, cost, reqs)
    assert not _bad(got, pforacle.OracleMap(cw, cw, cost).los_fields_create(reqs))
    assert (trace[:, 3] & np.uint64(0xFFFF) > 1).any()          # fields with pops, not only zero-filled ones


def test_los_level_blocked_destination_tile_vs_port(emu, pforacle):
    """targets on blocked tiles (the NaN-slope line from the target to itself) and on impassable ones"""
    cw = ch = 3
    cost = synth.cost_from_pathable(cases.noise_map(cw, ch, 8181, 0.08), cw, ch)
    rng = np.random.default_rng(8181)
    blk = np.zeros(cost.shape, np.uint16)
    for _ in range(60):
        k, r, c = int(rng.integers(0, cw * ch)), int(rng.integers(0, 62)), int(rng.integers(0, 62))
        blk[k, r:r + int(rng.integers(1, 4)), c:c + int(rng.integers(1, 4))] = 1
    reqs = []
    for chunk in range(cw * ch):
        tiles = list(np.argwhere((cost[chunk] != 255) & (blk[chunk] > 0))[::17][:4]) + list(np.argwhere(cost[chunk] == 255)[:1])
        for r_, c_ in tiles:
            td = (chunk // cw, chunk % cw, int(r_), int(c_))
            i0 = len(reqs)
            reqs.append(capi.los_req((td[0], td[1]), td))
            for nb in ((td[0] + 1, td[1]), (td[0], td[1] - 1)):
                if 0 <= nb[0] < ch and 0 <= nb[1] < cw:
                    reqs.append(capi.los_req(nb, td, prev_index=i0, prev_chunk=(td[0], td[1])))
    reqs = np.concatenate(reqs)
    assert len(reqs) >= 20
    got, _ = run_emu(emu["level"], cw, ch, cost, reqs, blk=blk)
    assert not _bad(got, pforacle.OracleMap(cw, ch, cost, blk).los_fields_create(reqs))


def test_los_level_attacking_faction_golden(emu, pforacle):
    """attacking requests walk over tiles blocked only by their enemies (field.c:179); the corner rule keeps the plain one"""
    g = np.load(os.path.join(HERE, "golden", "faction.npz"))
    reqs = g["lreq"].view(capi.LOS_REQ)
    assert (reqs["faction_id"] != capi.FACTION_ID_NONE).any()
    got, _ = run_emu(emu["level"], 2, 2, g["cost"], reqs, blk=g["blk"], factions=g["factions"], enemies=g["enemies"])
    assert not _bad(got, g["lexp"])
    om = pforacle.OracleMap(2, 2, g["cost"], g["blk"], g["liid"], factions=g["factions"], enemies=g["enemies"])
    assert not _bad(got, om.los_fields_create(reqs))


@pytest.fixture(scope="module")
def c2(pforacle):
    cw, cost, reqs = c2_batch()
    return cw, cost, reqs, pforacle.OracleMap(cw, cw, cost).los_fields_create(reqs)


def test_los_level_c2_batch_vs_port(emu, c2):
    """the whole C2-sized batch; it holds fields whose certificate fails, and those are replayed"""
    cw, cost, reqs, want = c2
    got, trace = run_emu(emu["level"], cw, cw, cost, reqs)
    assert not _bad(got, want)
    nrep = int(replayed(trace).sum())
    assert 0 < nrep < (trace[:, 3] & np.uint64(0xFFFF) > 0).sum() // 4


def test_los_level_certificate_catches_order_errors(emu, c2):
    """without the certificate the level pass gets a field of the C2 batch wrong; with the replay forced everywhere the
    same source matches the port"""
    cw, cost, reqs, want = c2
    got, trace = run_emu(emu["nocert"], cw, cw, cost, reqs)
    assert not replayed(trace).any()
    assert _bad(got, want)
    got, trace = run_emu(emu["replay"], cw, cw, cost, reqs)
    assert not _bad(got, want)
    nonzero = (trace[:, 3] & np.uint64(0xFFFF)) > 0
    assert replayed(trace)[nonzero].all()
