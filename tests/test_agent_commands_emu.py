"""The host side of pfnav_agents_commands (csrc/pfnav_commands_host.h, compiled with g++ through
tests/emu/commands_emu.cpp): delta validation, per-uid merging in array order, the per-entity write rule the device
kernel runs (here on the CPU), the navigation layer rule, and the (flock, layer) mirror that keeps flock_layer_used
equal to what a fresh upload of the resulting population computes."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
D = capi.AGENT_DELTA
HELD, GARR, WATER, AIR = capi.FLAG_COMBAT_HELD, capi.FLAG_GARRISONED, capi.FLAG_WATER, capi.FLAG_AIR


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libcommands_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-D_GLIBCXX_ASSERTIONS", "-fPIC", "-shared", os.path.join(HERE, "emu", "commands_emu.cpp"), "-o", so],
                   check=True)
    L = C.CDLL(so)
    p = C.c_void_p
    L.emu_cmd_merge.argtypes = [p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, p, C.c_char_p]
    L.emu_cmd_apply.argtypes = [p, p, p, p, C.c_int]
    L.emu_layer.argtypes = [C.c_uint32, C.c_float]
    L.emu_mirror_new.restype = p
    L.emu_mirror_new.argtypes = [p, C.c_int, C.c_int]
    L.emu_mirror_delete.argtypes = [p]
    L.emu_mirror_batch.argtypes = [p, p, C.c_int, C.c_int, C.c_int, C.c_char_p]
    L.emu_mirror_state.argtypes = [p, p, p, p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def merge(L, d, n_agents, nflocks, lo=0, hi=None, ms=True, ext=True):
    d = np.ascontiguousarray(d, D)
    out = np.zeros(max(len(d), 1), D)
    err = C.create_string_buffer(256)
    k = L.emu_cmd_merge(_p(d), len(d), lo, n_agents if hi is None else hi, n_agents, nflocks, int(ms), int(ext), _p(out), err)
    return (None, err.value.decode()) if k < 0 else (out[:k].copy(), None)


def population(rng, n, nflocks):
    a = np.zeros(n, capi.AGENT)
    a["pos"] = rng.random((n, 2)) * 100
    a["prev_pos"] = a["pos"]
    a["radius"] = rng.choice([1.5, 5.0, 12.0, 16.0], n)
    a["flags"] = rng.choice([0, HELD, WATER, AIR | GARR, HELD | GARR], n).astype(np.uint32) | capi.FLAG_MOVABLE
    a["flock"] = rng.integers(-1, nflocks, n)
    a["state"] = rng.integers(0, 9, n)
    ms = np.zeros(n, capi.MOVESTATE)
    ms["vel_hist"] = rng.random((n, 14, 2)) + 1
    ms["step"], ms["left"] = 0.5, 3
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID
    return a, ms, ext


def random_deltas(rng, k, n, nflocks):
    d = np.zeros(k, D)
    d["uid"] = rng.integers(0, n, k)
    d["mask"] = rng.integers(0, 1 << 10, k)
    d["state"] = rng.integers(0, 9, k)
    d["flock"] = rng.integers(-1, nflocks, k)
    d["aux_dest1"] = rng.integers(0, 5, k)
    d["flags"] = rng.choice([0, HELD, WATER, AIR, GARR, HELD | GARR], k).astype(np.uint32) | capi.FLAG_MOVABLE
    d["position"] = rng.random((k, 2)) * 100
    d["velocity"] = rng.random((k, 2))
    d["max_speed"], d["speed"] = rng.random(k) * 10, rng.random(k) * 10
    d["radius"] = rng.choice([1.5, 4.99, 5.0, 10.0, 14.9, 15.0], k)
    d["target_uid"] = np.where(rng.random(k) < 0.3, capi.NULL_UID, rng.integers(0, n, k))
    d["target_range"] = rng.random(k) * 20
    return d


def test_delta_layout():
    assert D.itemsize == 64
    assert [D.fields[f][1] for f in ("uid", "mask", "state", "flock", "aux_dest1", "flags", "position", "velocity", "max_speed",
                                     "speed", "radius", "target_uid", "target_range", "_pad")] == list(range(0, 64, 4))[:6] + [24, 32, 40, 44, 48, 52, 56, 60]


def test_layer_rule(emu):
    for flags, base in ((0, 0), (WATER, 4), (AIR, 8), (WATER | AIR, 4), (GARR | HELD, 0)):
        for r, cls in ((0.0, 0), (4.999, 0), (5.0, 1), (9.99, 1), (10.0, 2), (14.99, 2), (15.0, 3), (80.0, 3), (-1.0, 0)):
            assert emu.emu_layer(flags, r) == base + cls


@pytest.mark.parametrize("seed", range(6))
def test_merged_batch_equals_deltas_in_order(emu, seed):
    """several deltas per uid: applying the merged records (one per uid, first-occurrence order) leaves every table as
    applying the raw deltas one after the other does -- including the CLEAR_HIST rule against the flags of the moment"""
    rng = np.random.default_rng(seed)
    n, nflocks = 40, 5
    a, ms, ext = population(rng, n, nflocks)
    d = random_deltas(rng, 300, n, nflocks)
    m, err = merge(emu, d, n, nflocks)
    assert err is None
    first = list(dict.fromkeys(int(u) for u in d["uid"]))
    assert list(m["uid"]) == first and not (m["mask"] & capi.DELTA_CLEAR_HIST).any()
    a1, ms1, ext1 = a.copy(), ms.copy(), ext.copy()
    emu.emu_cmd_apply(_p(a1), _p(ms1), _p(ext1), _p(d), len(d))
    a2, ms2, ext2 = a.copy(), ms.copy(), ext.copy()
    emu.emu_cmd_apply(_p(a2), _p(ms2), _p(ext2), _p(m), len(m))
    assert a1.tobytes() == a2.tobytes() and ms1.tobytes() == ms2.tobytes() and ext1.tobytes() == ext2.tobytes()
    # and against a numpy restatement of the field writes, delta by delta
    a3, ms3, ext3 = a.copy(), ms.copy(), ext.copy()
    for x in d:
        u, k = int(x["uid"]), int(x["mask"])
        if k & capi.DELTA_STATE: a3["state"][u] = x["state"]
        if k & capi.DELTA_FLOCK: a3["flock"][u] = x["flock"]
        if k & capi.DELTA_AUX_DEST: a3["aux_dest1"][u] = x["aux_dest1"]
        if k & capi.DELTA_FLAGS: a3["flags"][u] = x["flags"] & 0xFFFFFF
        if k & capi.DELTA_SPEEDS: a3["max_speed"][u], a3["speed"][u] = x["max_speed"], x["speed"]
        if k & capi.DELTA_RADIUS: a3["radius"][u] = x["radius"]
        if k & capi.DELTA_VELOCITY: a3["velocity"][u] = x["velocity"]
        if k & capi.DELTA_POSITION:
            a3["pos"][u] = a3["prev_pos"][u] = x["position"]
            ms3["next_pos"][u, 0], ms3["next_pos"][u, 2] = x["position"]
            ms3["step"][u], ms3["left"][u] = 0, 0
        if (k & capi.DELTA_CLEAR_HIST) and not (a3["flags"][u] & HELD): ms3["vel_hist"][u] = 0
        if k & capi.DELTA_TARGET: ext3["surround_target_uid"][u], ext3["target_range"][u] = x["target_uid"], x["target_range"]
    assert a1.tobytes() == a3.tobytes() and ms1.tobytes() == ms3.tobytes() and ext1.tobytes() == ext3.tobytes()


def test_validation(emu):
    n, nflocks = 10, 3
    def one(**kw):
        d = np.zeros(1, D)
        for k, v in kw.items():
            d[k] = v
        return d
    ok = lambda d, **kw: merge(emu, d, n, nflocks, **kw)[1] is None
    assert ok(one(uid=9, mask=capi.DELTA_STATE, state=8))
    assert ok(np.zeros(0, D))
    assert not ok(one(uid=10, mask=0))
    assert not ok(one(uid=3, mask=0), lo=4)                       # outside the own range
    assert not ok(one(uid=8, mask=0), hi=8)
    assert not ok(one(uid=0, mask=1 << 10))
    assert not ok(one(uid=0, mask=capi.DELTA_STATE, state=9))
    assert ok(one(uid=0, mask=0, state=99))                       # not carried, not checked
    assert ok(one(uid=0, mask=capi.DELTA_FLOCK, flock=-1)) and ok(one(uid=0, mask=capi.DELTA_FLOCK, flock=2))
    assert not ok(one(uid=0, mask=capi.DELTA_FLOCK, flock=3)) and not ok(one(uid=0, mask=capi.DELTA_FLOCK, flock=-2))
    for bad in (np.nan, np.inf, -np.inf):
        assert not ok(one(uid=0, mask=capi.DELTA_RADIUS, radius=bad))
        assert not ok(one(uid=0, mask=capi.DELTA_SPEEDS, speed=bad)) and not ok(one(uid=0, mask=capi.DELTA_SPEEDS, max_speed=bad))
        assert not ok(one(uid=0, mask=capi.DELTA_VELOCITY, velocity=(0, bad)))
        assert not ok(one(uid=0, mask=capi.DELTA_POSITION, position=(bad, 0)))
        assert not ok(one(uid=0, mask=capi.DELTA_TARGET, target_uid=1, target_range=bad))
        assert ok(one(uid=0, mask=capi.DELTA_STATE, radius=bad))
    assert ok(one(uid=0, mask=capi.DELTA_TARGET, target_uid=capi.NULL_UID)) and ok(one(uid=0, mask=capi.DELTA_TARGET, target_uid=9))
    assert not ok(one(uid=0, mask=capi.DELTA_TARGET, target_uid=10))
    assert not ok(one(uid=0, mask=capi.DELTA_TARGET, target_uid=1), ext=False)
    assert not ok(one(uid=0, mask=capi.DELTA_POSITION), ms=False) and not ok(one(uid=0, mask=capi.DELTA_CLEAR_HIST), ms=False)
    # one bad delta anywhere refuses the batch
    d = np.concatenate([one(uid=1, mask=capi.DELTA_STATE)] * 5 + [one(uid=1, mask=capi.DELTA_STATE, state=77)])
    assert not ok(d)


@pytest.mark.parametrize("seed", range(4))
def test_mirror_tracks_a_fresh_upload(emu, seed):
    """batches of merged deltas, with the flock table growing and shrinking: the mirror's (flock, layer) per entity and the
    flock_layer_used table equal a brute-force recount over the resulting population; refused batches change nothing"""
    rng = np.random.default_rng(100 + seed)
    n, nflocks, nlayers = 60, 4, 8                 # ground and water layers exist, air does not
    a, ms, ext = population(rng, n, nflocks)
    a["flags"] &= ~np.uint32(AIR)
    h = emu.emu_mirror_new(_p(a), n, nflocks)
    err = C.create_string_buffer(256)

    def recount(a, nflocks):
        layer = np.array([emu.emu_layer(int(f), float(r)) for f, r in zip(a["flags"], a["radius"])], np.uint8)
        used = np.zeros((nflocks, 12), np.uint8)
        for f, l in zip(a["flock"], layer):
            if f >= 0:
                used[f, l] = 1
        return layer, used

    def check(a, nflocks):
        fl, ly, us = np.zeros(n, np.int32), np.zeros(n, np.uint8), np.zeros((nflocks, 12), np.uint8)
        emu.emu_mirror_state(h, _p(fl), _p(ly), _p(us))
        layer, used = recount(a, nflocks)
        assert (fl == a["flock"]).all() and (ly == layer).all() and (us == used).all()

    try:
        check(a, nflocks)
        refused = 0
        for it in range(40):
            new_nf = max(1, nflocks + int(rng.integers(-1, 3)))
            d = random_deltas(rng, int(rng.integers(0, 30)), n, new_nf)
            d["mask"] &= capi.DELTA_FLOCK | capi.DELTA_FLAGS | capi.DELTA_RADIUS | capi.DELTA_STATE
            if it % 3:
                d["flags"] &= ~np.uint32(AIR)
            m, e = merge(emu, d, n, new_nf)
            assert e is None
            b = a.copy()
            emu.emu_cmd_apply(_p(b), _p(ms), _p(ext), _p(m), len(m))
            layer, _ = recount(b, max(new_nf, nflocks))
            want_ok = (layer < nlayers)[np.unique(m["uid"][(m["mask"] & (capi.DELTA_FLOCK | capi.DELTA_FLAGS | capi.DELTA_RADIUS)) != 0])].all() \
                and (b["flock"] < new_nf).all()
            rc = emu.emu_mirror_batch(h, _p(m), len(m), new_nf, nlayers, err)
            assert (rc == 0) == bool(want_ok), err.value
            if rc == 0:
                a, nflocks = b, new_nf
            else:
                refused += 1
            check(a, nflocks)
        assert 0 < refused < 40
    finally:
        emu.emu_mirror_delete(h)


def test_flock_emptied_and_dropped_in_one_batch(emu):
    """a batch moves every member of the last flocks into surviving ones and the table drops them: the mirror follows;
    the same table with one member left behind is refused and changes nothing"""
    n, nflocks = 12, 4
    a = np.zeros(n, capi.AGENT)
    a["radius"] = 1.5
    a["flock"] = np.arange(n) % nflocks
    a["flags"][::5] = WATER
    h = emu.emu_mirror_new(_p(a), n, nflocks)
    err = C.create_string_buffer(256)

    def state(nf):
        fl, ly, us = np.zeros(n, np.int32), np.zeros(n, np.uint8), np.zeros((nf, 12), np.uint8)
        emu.emu_mirror_state(h, _p(fl), _p(ly), _p(us))
        return fl, ly, us

    try:
        tail = np.nonzero(a["flock"] >= 2)[0]
        d = np.zeros(len(tail), D)
        d["uid"], d["mask"], d["flock"] = tail, capi.DELTA_FLOCK, a["flock"][tail] - 2
        m, e = merge(emu, d[1:], n, 2)
        assert e is None
        assert emu.emu_mirror_batch(h, _p(m), len(m), 2, 8, err) == -1 and b"shorter" in err.value
        assert (state(nflocks)[0] == a["flock"]).all()
        m, e = merge(emu, d, n, 2)
        assert e is None
        assert emu.emu_mirror_batch(h, _p(m), len(m), 2, 8, err) == 0, err.value
        fl, ly, us = state(2)
        assert (fl == np.arange(n) % 2).all()
        want = np.zeros((2, 12), np.uint8)
        for f, w in zip(fl, a["flags"]):
            want[f, 4 if w & WATER else 0] = 1
        assert (us == want).all()
        # and growing again after the shrink
        m, e = merge(emu, d[:1], n, 5)
        assert e is None and emu.emu_mirror_batch(h, _p(m), len(m), 5, 8, err) == 0
        assert state(5)[2].shape == (5, 12) and not state(5)[2][2:].any()
    finally:
        emu.emu_mirror_delete(h)
