"""The host rule of the entity-field batches named by uid (csrc/pfnav_resident_host.h, compiled with g++ through
tests/emu/resident_emu.cpp) on synthetic record arrays, against a Python restatement of the contract in
include/pfnav.h: given and named footprints mixed, each request's seeker chunks listed once in the order of their first
seeker, and every argument error, with nothing written on an error."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

HERE = os.path.dirname(os.path.abspath(__file__))
capi = cases.capi
REQ, FP, NULL = capi.ENTITY_FIELD_REQ, capi.FOOTPRINT, capi.NULL_UID
CW, CH = 5, 3


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libresident_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", os.path.join(HERE, "emu", "resident_emu.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    p, z = C.c_void_p, C.c_size_t
    L.emu_last_error.restype = C.c_char_p
    L.emu_resolve.argtypes = [p, z, p, p, z, p, z, p, p, z, C.c_int, C.c_int, p, p, p, z, C.POINTER(z), C.POINTER(C.c_int)]
    return L


def _p(a):
    return None if a is None or len(a) == 0 else a.ctypes.data_as(C.c_void_p)


def _records(n, seed):
    """{x, z, vx, vz, radius, state_flags} per entity, and the chunk under each (-1 for a few off the map)"""
    rng = np.random.default_rng(seed)
    rec = np.zeros((n, 6), np.float32)
    rec[:, 0] = -rng.uniform(0, CW * 256, n)
    rec[:, 1] = rng.uniform(0, CH * 256, n)
    rec[:, 4] = rng.uniform(0.5, 40.0, n)
    chunk = (rec[:, 1] // 256).astype(np.int32) * CW + (-rec[:, 0] // 256).astype(np.int32)
    off = rng.choice(n, max(1, n // 50), replace=False)
    chunk[off] = -1
    return rec, chunk


def _fp(n, seed):
    rng = np.random.default_rng(seed)
    fp = np.zeros(n, FP)
    fp["x"] = -rng.uniform(0, CW * 256, n); fp["z"] = rng.uniform(0, CH * 256, n); fp["sel_radius"] = rng.uniform(0, 9, n)
    b = rng.random(n) < 0.3
    fp["is_building"][b] = 1
    fp["corners_xz"][b] = rng.uniform(1, 100, (int(b.sum()), 8))
    return fp


def _req(dest, kind, ent, sk):
    r = np.zeros(1, REQ)
    r["dest"], r["target_kind"] = dest, kind
    r["ent_off"], r["ent_n"], r["chunk_off"], r["chunk_n"] = ent[0], ent[1], sk[0], sk[1]
    return r


def run(L, reqs, fp, uids, seekers, rec, chunk, population=None):
    reqs = np.ascontiguousarray(reqs, REQ)
    nents = len(fp) if fp is not None else (0 if uids is None else len(uids))
    seekers = np.ascontiguousarray(seekers, np.uint32)
    out_r = np.zeros(len(reqs), REQ); out_r["dest"] = -77
    out_e = np.zeros(nents, FP); out_e["x"] = -77.0
    cap = 4096
    out_c = np.full((cap, 2), -77, np.int32)
    nc, kept = C.c_size_t(12345), C.c_int(-1)
    rc = L.emu_resolve(_p(reqs), len(reqs), _p(fp), _p(uids), nents, _p(seekers), len(seekers), _p(rec), _p(chunk),
                       len(rec) if population is None else population, CW, CH, _p(out_r), _p(out_e), _p(out_c), cap,
                       C.byref(nc), C.byref(kept))
    if rc:
        # nothing written: neither the outputs nor the batch the rule merges into
        assert (out_r["dest"] == -77).all() and (out_e["x"] == -77.0).all() and (out_c == -77).all() and nc.value == 12345
        assert kept.value in (-1, 1)
        return rc, L.emu_last_error().decode()
    return rc, (out_r, out_e, out_c[:nc.value].copy())


def restate(reqs, fp, uids, seekers, rec, chunk):
    """the contract of include/pfnav.h in Python"""
    nents = len(fp) if fp is not None else len(uids)
    ents = np.zeros(nents, FP) if fp is None else fp.copy()
    for k in range(nents):
        if uids is not None and uids[k] != NULL:
            e = np.zeros(1, FP)[0]
            e["x"], e["z"], e["sel_radius"] = rec[uids[k], 0], rec[uids[k], 1], rec[uids[k], 4]
            ents[k] = e
    out, chunks = reqs.copy(), []
    for i, q in enumerate(reqs):
        seen = []
        for s in seekers[int(q["chunk_off"]):int(q["chunk_off"]) + int(q["chunk_n"])]:
            c = int(chunk[s])
            if c not in seen:
                seen.append(c)
        out[i]["chunk_off"], out[i]["chunk_n"] = len(chunks), len(seen)
        chunks += [divmod(c, CW) for c in seen]
    return out, ents, np.array(chunks, np.int32).reshape(-1, 2)


def _same(got, want):
    assert got[0].tobytes() == want[0].tobytes()
    assert got[1].tobytes() == want[1].tobytes()
    assert np.array_equal(got[2], want[2])


def test_mixed_footprints_and_first_seen_chunks(emu):
    """given and named footprints in one array, overlapping ranges, TARGET_ENTITY by uid, repeated seekers; chunks
    listed once per request in the order of their first seeker"""
    rec, chunk = _records(500, 1)
    on = np.nonzero(chunk >= 0)[0]
    rng = np.random.default_rng(2)
    nents = 200
    fp = _fp(nents, 3)
    uids = np.full(nents, NULL, np.uint32)
    named = rng.random(nents) < 0.7
    uids[named] = rng.choice(on, int(named.sum()))
    seekers = rng.choice(on, 300).astype(np.uint32)
    seekers[100:110] = seekers[0]                           # one seeker repeated
    reqs = np.concatenate([_req(0, capi.TARGET_ENEMIES, (0, 200), (0, 300)), _req(1, capi.TARGET_ENEMIES, (50, 100), (40, 80)),
                           _req(2, capi.TARGET_ENTITY, (int(np.nonzero(named)[0][0]), 1), (290, 10)),
                           _req(0, capi.TARGET_ENEMIES, (0, 0), (0, 0)), _req(3, capi.TARGET_ENEMIES, (10, 20), (0, 300))])
    rc, got = run(emu, reqs, fp, uids, seekers, rec, chunk)
    assert rc == 0, got
    want = restate(reqs, fp, uids, seekers, rec, chunk)
    _same(got, want)
    assert got[0]["chunk_n"][0] == len(set(chunk[seekers].tolist()))
    assert got[0]["chunk_n"][3] == 0
    # a named entry ignores what ents holds there: building flag and corners cleared
    k = int(np.nonzero(named & (fp["is_building"] == 1))[0][0])
    assert got[1]["is_building"][k] == 0 and (got[1]["corners_xz"][k] == 0).all()


def test_all_named_without_ents_and_all_given_without_uids(emu):
    rec, chunk = _records(100, 4)
    on = np.nonzero(chunk >= 0)[0]
    uids = on[:30].astype(np.uint32)
    seekers = on[::-1][:20].astype(np.uint32)
    reqs = np.concatenate([_req(0, capi.TARGET_ENEMIES, (0, 30), (0, 20)), _req(1, capi.TARGET_ENTITY, (5, 1), (3, 4))])
    rc, got = run(emu, reqs, None, uids, seekers, rec, chunk)
    assert rc == 0
    _same(got, restate(reqs, None, uids, seekers, rec, chunk))
    fp = _fp(30, 5)
    rc, got = run(emu, reqs, fp, None, seekers, rec, chunk)
    assert rc == 0
    _same(got, restate(reqs, fp, None, seekers, rec, chunk))
    assert got[1].tobytes() == fp.tobytes()


def test_order_is_first_seen(emu):
    """chunks c2, c0, c2, c1, c0 -> c2, c0, c1 (not sorted, not last seen)"""
    rec = np.zeros((5, 6), np.float32)
    chunk = np.array([2 * CW + 1, 0, 2 * CW + 1, 4, 0], np.int32)
    rc, got = run(emu, _req(0, capi.TARGET_ENEMIES, (0, 0), (0, 5)), None, None, np.arange(5), rec, chunk)
    assert rc == 0
    assert got[2].tolist() == [[2, 1], [0, 0], [0, 4]]


def test_m_zero_resolves_nothing(emu):
    rec, chunk = _records(10, 6)
    chunk[:] = -1                                           # every seeker off the map: not looked at
    rc, _ = run(emu, np.zeros(0, REQ), None, np.arange(3, dtype=np.uint32), np.arange(4), rec, chunk)
    assert rc == 0


def test_errors_write_nothing(emu):
    rec, chunk = _records(60, 7)
    on = np.nonzero(chunk >= 0)[0]
    offmap = int(np.nonzero(chunk < 0)[0][0])
    fp = _fp(10, 8)
    uids = on[:10].astype(np.uint32)
    sk = on[:8].astype(np.uint32)
    ok = _req(0, capi.TARGET_ENEMIES, (0, 10), (0, 8))
    half = uids.copy(); half[3] = NULL
    cases_ = [
        ("uid outside", ok, fp, np.where(np.arange(10) == 4, 60, uids).astype(np.uint32), sk, None),
        ("seeker outside", ok, fp, uids, np.append(sk[:7], 60).astype(np.uint32), None),
        ("seeker NULL_UID", ok, fp, uids, np.append(sk[:7], NULL).astype(np.uint32), None),
        ("ents NULL, an entry names no uid", ok, None, half, sk, None),
        ("footprint range", _req(0, capi.TARGET_ENEMIES, (5, 6), (0, 8)), fp, uids, sk, None),
        ("seeker range", _req(0, capi.TARGET_ENEMIES, (0, 10), (4, 5)), fp, uids, sk, None),
        ("seeker off the map", ok, fp, uids, np.append(sk[:7], offmap).astype(np.uint32), None),
        ("population", ok, fp, uids, sk, int(max(uids.max(), sk.max()))),
    ]
    for name, r, f, u, s, pop in cases_:
        rc, err = run(emu, r, f, u, s, rec, chunk, pop)
        assert rc == capi.ERR_ARG, name
        assert err, name
    # a seeker off the map in no request's range still refuses: every seeker is resolved
    rc, _ = run(emu, _req(0, capi.TARGET_ENEMIES, (0, 10), (0, 7)), fp, uids, np.append(sk[:7], offmap).astype(np.uint32), rec, chunk)
    assert rc == capi.ERR_ARG
    # NULL pointers with counts, and the 2^24 bounds, through the raw ABI
    L = emu
    z = C.c_size_t(0)
    k = C.c_int(0)
    r = np.ascontiguousarray(ok, REQ)
    assert L.emu_resolve(_p(r), 1, None, None, 10, _p(sk), 8, _p(rec), _p(chunk), 60, CW, CH, None, None, None, 0,
                         C.byref(z), C.byref(k)) == capi.ERR_ARG
    assert L.emu_resolve(_p(r), 1, _p(fp), None, 10, None, 8, _p(rec), _p(chunk), 60, CW, CH, None, None, None, 0,
                         C.byref(z), C.byref(k)) == capi.ERR_ARG
    assert L.emu_resolve(None, 1, _p(fp), None, 10, _p(sk), 8, _p(rec), _p(chunk), 60, CW, CH, None, None, None, 0,
                         C.byref(z), C.byref(k)) == capi.ERR_ARG
    for m, ne, ns in [(1 << 24, 0, 0), (0, 1 << 24, 0), (0, 0, 1 << 24)]:
        assert L.emu_resolve(_p(r), m, _p(fp), None, ne, _p(sk), ns, _p(rec), _p(chunk), 60, CW, CH, None, None, None, 0,
                             C.byref(z), C.byref(k)) == capi.ERR_ARG


def test_merge_error_keeps_the_batch(emu):
    """a seeker off the map is found by the merge: it leaves the batch it merges into as it was"""
    rec, chunk = _records(40, 9)
    offmap = int(np.nonzero(chunk < 0)[0][0])
    out_r, out_e = np.zeros(1, REQ), np.zeros(1, FP)
    out_c = np.zeros((8, 2), np.int32)
    z, k = C.c_size_t(0), C.c_int(0)
    r = np.ascontiguousarray(_req(0, capi.TARGET_ENEMIES, (0, 0), (0, 1)), REQ)
    sk = np.array([offmap], np.uint32)
    assert emu.emu_resolve(_p(r), 1, None, None, 0, _p(sk), 1, _p(rec), _p(chunk), 40, CW, CH, _p(out_r), _p(out_e),
                           _p(out_c), 8, C.byref(z), C.byref(k)) == capi.ERR_ARG
    assert k.value == 1
