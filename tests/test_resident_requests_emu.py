"""The host rule of the calls whose positions may name resident entities (pf_resident_points_check in
csrc/pfnav_resident_host.h, compiled with g++ through tests/emu/resident_points_emu.cpp) on synthetic record arrays,
against a Python restatement of the contract in include/pfnav.h (pfnav_pool_request_paths_resident,
pfnav_map_query_resident, pfnav_group_arrival_velocity_resident): named and given entries mixed, every entry named with
no given positions, no uid arrays, n == 0, and every argument error, with nothing written on an error."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
NULL = 0xFFFFFFFF
ERR_ARG = -1


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libresident_points_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", os.path.join(HERE, "emu", "resident_points_emu.cpp"),
                    "-o", so], check=True)
    L = C.CDLL(so)
    p, z, i = C.c_void_p, C.c_size_t, C.c_int
    L.emu_last_error.restype = C.c_char_p
    L.emu_points.argtypes = [z, p, i, p, i, z, p, i, i, i, p, p, p, C.POINTER(z), C.POINTER(z)]
    return L


def _p(a):
    return None if a is None or len(a) == 0 else a.ctypes.data_as(C.c_void_p)


def _records(n, seed):
    rng = np.random.default_rng(seed)
    rec = rng.uniform(-1000, 1000, (n, 6)).astype(np.float32)
    return rec


# the three layouts: path requests (sources then destinations, 2 floats each), map queries (32-byte records, x, z at
# floats 2, 3 and dst_x, dst_z at 4, 5), group arrival (one float2 per entity)
LAYOUTS = {"paths": lambda n: (2, 0, 2 * n, 4 * n), "map_query": lambda n: (8, 2, 4, 8 * n), "arrival": lambda n: (2, 0, 0, 2 * n)}


def run(L, n, ua, ga, ub, gb, pop, rec, layout, buf):
    """-> rc, error text, pairs (entry, uid), n0; buf is written in place on success"""
    stride, off_a, off_b, _ = LAYOUTS[layout](n)
    ent = np.full(2 * n + 1, 0xDEAD, np.uint32)
    uid = np.full(2 * n + 1, 0xDEAD, np.uint32)
    npairs, n0 = C.c_size_t(777), C.c_size_t(777)
    rc = L.emu_points(n, _p(ua), int(ga), _p(ub), int(gb), pop, _p(rec), stride, off_a, off_b, _p(buf), _p(ent), _p(uid),
                      C.byref(npairs), C.byref(n0))
    if rc:
        assert (ent == 0xDEAD).all() and (uid == 0xDEAD).all() and npairs.value == 777 and n0.value == 777
        return rc, L.emu_last_error().decode(), None, None
    return rc, "", (ent[:npairs.value].copy(), uid[:npairs.value].copy()), n0.value


def restate(n, ua, ga, ub, gb, pop, rec, layout, buf):
    """the contract: -> None on an argument error, else the pairs, n0 and the buffer after the substitution"""
    if n >= 1 << 24:
        return None
    pairs, buf = [], buf.copy()
    stride, off_a, off_b, _ = LAYOUTS[layout](n)
    for uids, given, off in ((ua, ga, off_a), (ub, gb, off_b)):
        for k in range(n):
            u = NULL if uids is None else int(uids[k])
            if u == NULL:
                if not given:
                    return None
                continue
            if u >= pop:
                return None
            pairs.append((k, u))
            buf[k * stride + off: k * stride + off + 2] = rec[u, :2]
        if off == off_a:
            n0 = len(pairs)
    e = np.array([p[0] for p in pairs], np.uint32)
    u = np.array([p[1] for p in pairs], np.uint32)
    return (e, u), n0, buf


def check(L, n, ua, ga, ub, gb, pop, rec, layout, seed=0):
    """the emulated rule against the restatement; -> rc"""
    size = LAYOUTS[layout](n)[3]
    buf0 = np.random.default_rng(seed).uniform(-5, 5, max(size, 1)).astype(np.float32)
    buf = buf0.copy()
    rc, err, pairs, n0 = run(L, n, ua, ga, ub, gb, pop, rec, layout, buf)
    want = restate(n, ua, ga, ub, gb, pop, rec, layout, buf0)
    if want is None:
        assert rc == ERR_ARG and err
        assert buf.tobytes() == buf0.tobytes()
        return rc
    assert rc == 0, err
    assert np.array_equal(pairs[0], want[0][0]) and np.array_equal(pairs[1], want[0][1])
    assert n0 == want[1]
    assert buf.tobytes() == want[2].tobytes()
    return rc


@pytest.mark.parametrize("layout", list(LAYOUTS))
@pytest.mark.parametrize("n", [1, 7, 300, 5000])
def test_mixed_named_and_given(emu, layout, n):
    pop = 4000
    rec = _records(pop, 1)
    rng = np.random.default_rng(n)
    ua = rng.integers(0, pop, n).astype(np.uint32)
    ua[rng.random(n) < 0.4] = NULL
    ub = None if layout == "arrival" else rng.integers(0, pop, n).astype(np.uint32)
    if ub is not None:
        ub[rng.random(n) < 0.5] = NULL
        ub[:2] = ua[:2]                               # one entity as both positions of a request
    assert check(emu, n, ua, True, ub, True, pop, rec, layout, seed=n) == 0


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_all_named_without_given_positions(emu, layout):
    pop, n = 900, 600
    rec = _records(pop, 2)
    rng = np.random.default_rng(3)
    ua = rng.integers(0, pop, n).astype(np.uint32)
    ub = None if layout == "arrival" else rng.integers(0, pop, n).astype(np.uint32)
    assert check(emu, n, ua, False, ub, layout == "arrival", pop, rec, layout) == 0
    ua[0] = pop - 1                                   # the last entity of the population
    assert check(emu, n, ua, False, ub, layout == "arrival", pop, rec, layout) == 0


@pytest.mark.parametrize("layout", list(LAYOUTS))
def test_no_uid_arrays(emu, layout):
    """NULL uid arrays name nothing: the given positions stand, no pairs"""
    rec = _records(10, 4)
    for n in (0, 1, 33):
        assert check(emu, n, None, True, None, True, 10, rec, layout) == 0
    rng = np.random.default_rng(5)
    ub = rng.integers(0, 10, 20).astype(np.uint32)
    assert check(emu, 20, None, True, ub, False, 10, rec, "paths") == 0   # sources given, destinations named


def test_n_zero(emu):
    """n == 0 checks nothing and names nothing, whatever the arrays"""
    rec = _records(4, 6)
    for layout in LAYOUTS:
        assert check(emu, 0, None, False, None, False, 0, rec, layout) == 0
        assert check(emu, 0, np.zeros(1, np.uint32), False, None, False, 0, rec, layout) == 0


def test_errors_write_nothing(emu):
    pop, n = 50, 40
    rec = _records(pop, 7)
    rng = np.random.default_rng(8)
    ua = rng.integers(0, pop, n).astype(np.uint32)
    ub = rng.integers(0, pop, n).astype(np.uint32)
    cases = {
        "a: uid == population": (np.where(np.arange(n) == 17, pop, ua).astype(np.uint32), True, ub, True),
        "a: uid far outside": (np.where(np.arange(n) == 0, 0xFFFFFFFE, ua).astype(np.uint32), True, ub, True),
        "b: uid outside, after a named a": (ua, True, np.where(np.arange(n) == n - 1, pop + 3, ub).astype(np.uint32), True),
        "a: NULL given, an entry unnamed": (np.where(np.arange(n) == 5, NULL, ua).astype(np.uint32), False, ub, True),
        "b: NULL given, an entry unnamed": (ua, True, np.where(np.arange(n) == n - 1, NULL, ub).astype(np.uint32), False),
        "a: no uids and no given": (None, False, ub, True),
        "b: no uids and no given": (ua, True, None, False),
        "empty population": (ua, True, ub, True),
    }
    for name, (a, ga, b, gb) in cases.items():
        p = 0 if name == "empty population" else pop
        for layout in ("paths", "map_query"):
            assert check(emu, n, a, ga, b, gb, p, rec, layout) == ERR_ARG, (name, layout)
    # n at 2^24: refused before any array is read (NULL arrays with "given" set are never dereferenced)
    buf = np.zeros(1, np.float32)
    ent = np.zeros(1, np.uint32)
    npairs, n0 = C.c_size_t(777), C.c_size_t(777)
    assert emu.emu_points(1 << 24, None, 1, None, 1, pop, _p(rec), 2, 0, 0, _p(buf), _p(ent), _p(ent), C.byref(npairs),
                          C.byref(n0)) == ERR_ARG
    assert npairs.value == 777 and emu.emu_last_error()
