"""The checkpoint segment of pfnav_agents_save / pfnav_agents_restore on the CPU (csrc/pfnav_checkpoint_host.h through
tests/emu/checkpoint_emu.cpp): the device's row pack run on CPU threads, then a restore's validation, range choice and
record gather, and the incref ops of the restored blocking rows.

- Round trip: a population saved by 1..8 members restores onto 1..8 members; each member takes
  pfnav_mgpu_shard_range(n_total, rank, world), and the members' records joined equal the saved tables; the ops are the
  blocking rows' recorded circles in uid order.
- Refusals: truncated and padded segments, bad magic / version / record sizes / table bits / hz, overlapping, gapped and
  mismatched segments, and every out-of-range record; a refusal writes nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from test_agent_population_emu import agents

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
MS, EXT, FORM, BLK = 1, 2, 4, 8
LAYERS = 12
HDR = 64


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libcheckpoint_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-D_GLIBCXX_ASSERTIONS", "-fPIC", "-shared", "-pthread",
                    os.path.join(HERE, "emu", "checkpoint_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    p, sz = C.c_void_p, C.c_size_t
    L.emu_ckpt_size.restype = sz
    L.emu_ckpt_size.argtypes = [C.c_uint32, sz, sz]
    L.emu_ckpt_save.restype = sz
    L.emu_ckpt_save.argtypes = [C.c_uint32, sz, sz, sz, C.c_int, p, sz, p, p, p, p, p, C.c_int, p]
    L.emu_ckpt_restore.argtypes = [p, p, sz, C.c_int, C.c_int, C.c_int, p, p, p, p, p, p, C.c_int, p, C.c_char_p]
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def ranges(n, world):
    base, rem = divmod(n, world)
    return [r * base + min(r, rem) for r in range(world + 1)]


def population(rng, n, nf, tables):
    """random tables of n entities with every float finite and every record valid"""
    a = agents(rng, n, nf)
    a["velocity"] = rng.standard_normal((n, 2)); a["max_speed"] = 8.0; a["speed"] = 6.0
    a["aux_dest1"] = rng.integers(0, 5, n)
    fl = np.zeros(nf, capi.FLOCK)
    fl["target"] = rng.random((nf, 2)) * 100; fl["dest"] = np.arange(nf); fl["layer"] = rng.integers(0, 4, nf)
    T = {"agents": a, "flocks": fl}
    if tables & MS:
        m = np.zeros(n, capi.MOVESTATE)
        m["next_pos"] = rng.random((n, 3)); m["vel_hist"] = rng.standard_normal((n, 14, 2)); m["left"] = rng.integers(0, 9, n)
        T["ms"] = m
    if tables & EXT:
        e = np.zeros(n, capi.MOVESTATE_EXT)
        e["surround_target_uid"] = np.where(rng.random(n) < 0.5, capi.NULL_UID, rng.integers(0, max(n, 1), n))
        e["target_range"] = rng.random(n); e["rot"] = rng.random((n, 4)); e["wait_ticks_left"] = rng.integers(0, 9, n)
        T["ext"] = e
    if tables & FORM:
        f = np.zeros(n, capi.FORMATION_IN)
        f["cell_pos"] = rng.random((n, 2)); f["flags"] = rng.integers(0, 32, n)
        T["form"] = f
    if tables & BLK:
        b = np.zeros(n, capi.BLOCKING)
        b["blocking"] = rng.integers(0, 2, n); b["faction_id"] = rng.integers(0, 16, n)
        b["stop_x"] = rng.random(n) * 100; b["stop_z"] = rng.random(n) * 100; b["stop_radius"] = rng.choice([1.5, 60.0], n)
        T["blk"] = b
    return T


def save(L, T, tables, lo, hi, hz=20, nthreads=3):
    n = len(T["agents"])
    out = np.zeros(L.emu_ckpt_size(tables, len(T["flocks"]), hi - lo), np.uint8)
    got = L.emu_ckpt_save(tables, n, lo, hi, hz, _p(T["flocks"]), len(T["flocks"]), _p(T["agents"]), _p(T.get("ms")),
                          _p(T.get("ext")), _p(T.get("form")), _p(T.get("blk")), nthreads, _p(out))
    assert got == len(out)
    return out.tobytes()


def save_job(L, T, tables, world, hz=20):
    lo = ranges(len(T["agents"]), world)
    return [save(L, T, tables, lo[r], lo[r + 1], hz) for r in range(world)]


def restore(L, segs, world=1, rank=0, nlayers=LAYERS, room=None):
    """-> (info dict, records dict) or (None, error text); on a refusal the output buffers must be untouched"""
    bufs = [np.frombuffer(s, np.uint8) for s in segs]
    ptrs = (C.c_void_p * max(len(bufs), 1))(*[b.ctypes.data for b in bufs])
    sizes = (C.c_size_t * max(len(bufs), 1))(*[len(b) for b in bufs])
    m = room if room is not None else max([C.cast(ptrs[i], C.POINTER(C.c_uint64))[4] for i in range(len(bufs))] + [1])
    out = {"agents": np.full(m * 64, 0xAB, np.uint8).view(capi.AGENT), "ms": np.zeros(m, capi.MOVESTATE),
           "ext": np.zeros(m, capi.MOVESTATE_EXT), "form": np.zeros(m, capi.FORMATION_IN), "blk": np.zeros(m, capi.BLOCKING)}
    ops = np.zeros(m, OP)
    before = {k: v.tobytes() for k, v in out.items()}
    info = np.zeros(7, np.int64)
    err = C.create_string_buffer(256)
    rc = L.emu_ckpt_restore(ptrs, sizes, len(bufs), nlayers, world, rank, _p(out["agents"]), _p(out["ms"]), _p(out["ext"]),
                            _p(out["form"]), _p(out["blk"]), _p(ops), 2, _p(info), err)
    if rc != 0:
        assert all(out[k].tobytes() == before[k] for k in out), "a refusal wrote records"
        return None, err.value.decode()
    n_total, lo, hi, hz, nflocks, tables, nops = (int(v) for v in info)
    rec = {k: v[:hi - lo] for k, v in out.items()}
    rec["ops"] = ops[:nops]
    return dict(n_total=n_total, lo=lo, hi=hi, hz=hz, nflocks=nflocks, tables=tables), rec


OP = np.dtype([("x", "<f4"), ("z", "<f4"), ("range", "<f4"), ("faction_id", "<i4"), ("flags", "<u4"), ("delta", "<i4")])
KEYS = (("ms", MS), ("ext", EXT), ("form", FORM), ("blk", BLK))


@pytest.mark.parametrize("tables", [0, MS, MS | EXT | FORM | BLK, MS | BLK, EXT | FORM])
def test_round_trip_every_world_size(emu, tables):
    rng = np.random.default_rng(tables + 1)
    for n in (0, 1, 5, 257):
        T = population(rng, n, 4, tables)
        for w_save in range(1, 9):
            segs = save_job(emu, T, tables, w_save, hz=10)
            order = rng.permutation(len(segs))
            segs = [segs[i] for i in order]                             # any order
            for w_new in range(1, 9):
                parts = []
                for r in range(w_new):
                    info, rec = restore(emu, segs, w_new, r)
                    assert info is not None, rec
                    lo = ranges(n, w_new)
                    assert (info["lo"], info["hi"]) == (lo[r], lo[r + 1])
                    assert info["n_total"] == n and info["hz"] == 10 and info["nflocks"] == 4 and info["tables"] == tables
                    parts.append(rec)
                got = np.concatenate([p["agents"] for p in parts])
                assert got.tobytes() == T["agents"].tobytes()
                for k, bit in KEYS:
                    if tables & bit:
                        assert np.concatenate([p[k] for p in parts]).tobytes() == T[k].tobytes(), k
                if tables & BLK:
                    ops = np.concatenate([p["ops"] for p in parts])
                    held = np.nonzero(T["blk"]["blocking"] == 1)[0]       # uid order
                    b, a = T["blk"][held], T["agents"][held]
                    assert len(ops) == len(held)
                    assert (ops["x"] == b["stop_x"]).all() and (ops["z"] == b["stop_z"]).all()
                    assert (ops["range"] == b["stop_radius"]).all() and (ops["faction_id"] == b["faction_id"]).all()
                    assert (ops["flags"] == a["flags"]).all() and (ops["delta"] == 1).all()


def test_segment_layout(emu):
    """header fields at their offsets, the flock table after it, then one row per uid: agent, movestate, ext, formation,
    blocking"""
    rng = np.random.default_rng(3)
    tables = MS | EXT | FORM | BLK
    T = population(rng, 10, 3, tables)
    s = save(emu, T, tables, 2, 7, hz=5)
    h = np.frombuffer(s[:HDR], np.uint32)
    assert h[0] == 0x4B434650 and h[1] == 1 and list(h[2:7]) == [64, 176, 64, 64, 32] and h[7] == tables
    assert list(np.frombuffer(s[32:56], np.uint64)) == [10, 2, 7]
    assert np.frombuffer(s[56:60], np.int32)[0] == 5 and h[15] == 3
    assert s[HDR:HDR + 48] == T["flocks"].tobytes()
    row = 64 + 176 + 64 + 64 + 32
    rows = s[HDR + 48:]
    assert len(rows) == 5 * row
    for i in range(5):
        r = rows[i * row:(i + 1) * row]
        u = 2 + i
        assert r[:64] == T["agents"][u].tobytes() and r[64:240] == T["ms"][u].tobytes()
        assert r[240:304] == T["ext"][u].tobytes() and r[304:368] == T["form"][u].tobytes() and r[368:] == T["blk"][u].tobytes()


def _patch(seg, off, dtype, value):
    b = bytearray(seg)
    b[off:off + np.dtype(dtype).itemsize] = np.array([value], dtype).tobytes()
    return bytes(b)


def test_refused_headers_and_sets(emu):
    rng = np.random.default_rng(5)
    tables = MS | EXT | BLK
    T = population(rng, 60, 3, tables)
    segs = save_job(emu, T, tables, 3)
    assert restore(emu, segs)[0] is not None
    U = population(rng, 60, 3, tables)
    other = save_job(emu, U, tables, 3)
    bad = {
        "no segment": [],
        "truncated": [segs[0][:-1]] + segs[1:],
        "padded": [segs[0] + b"\0"] + segs[1:],
        "shorter than the header": [segs[0][:40]] + segs[1:],
        "magic": [_patch(segs[0], 0, np.uint32, 0x12345678)] + segs[1:],
        "version": [_patch(segs[0], 4, np.uint32, 2)] + segs[1:],
        "record size": [_patch(segs[0], 12, np.uint32, 160)] + segs[1:],
        "table bit": [_patch(segs[0], 28, np.uint32, tables | 16)] + segs[1:],
        "hz": [_patch(segs[0], 56, np.int32, 30)] + segs[1:],
        "overlap": segs + [segs[1]],
        "gap": [segs[0], segs[2]],
        "n_total": [_patch(segs[0], 32, np.uint64, 61)] + segs[1:],
        "range": [_patch(segs[2], 48, np.uint64, 61)] + segs[:2],
        "hz mismatch": [save_job(emu, T, tables, 3, hz=10)[0]] + segs[1:],
        "flock table": [other[0]] + segs[1:],
        "tables": [save(emu, T, MS | EXT, 0, 20)] + segs[1:],
        "nflocks": [save(emu, dict(T, flocks=T["flocks"][:2]), tables, 0, 20)] + segs[1:],
        "split from another world size overlapping": save_job(emu, T, tables, 2)[:1] + segs[1:],
    }
    for name, s in bad.items():
        info, err = restore(emu, s, room=64)
        assert info is None, name
        assert err, name
    # records of another save with the same header facts and flock table complete the population: accepted
    V = dict(U, flocks=T["flocks"])
    assert restore(emu, [segs[0]] + save_job(emu, V, tables, 3)[1:])[0] is not None


def test_refused_records(emu):
    rng = np.random.default_rng(9)
    tables = MS | EXT | FORM | BLK
    T = population(rng, 40, 3, tables)
    T["agents"]["radius"] = 1.5; T["agents"]["flags"] = capi.FLAG_MOVABLE        # layer 0 for everyone

    def spoiled(key, field, value, idx=None):
        U = {k: v.copy() for k, v in T.items()}
        if idx is None:
            U[key][field][17] = value
        else:
            U[key][field][17][idx] = value
        return save_job(emu, U, tables, 2)

    cases_ = [
        ("agents", "flock", 3, None),
        ("agents", "pos", np.nan, 1), ("agents", "speed", np.inf, None),
        ("ms", "vel_hist", np.nan, (3, 1)), ("ms", "step", np.inf, None),
        ("ext", "surround_target_uid", 40, None), ("ext", "target_dir", np.nan, 2), ("ext", "rot", np.inf, 3),
        ("form", "cell_pos", np.nan, 0), ("form", "target_orientation", np.nan, 3),
        ("blk", "blocking", 2, None), ("blk", "faction_id", 16, None), ("blk", "faction_id", -1, None),
        ("blk", "stop_radius", np.nan, None), ("flocks", "target", np.nan, 0),
    ]
    for key, field, value, idx in cases_:
        if key == "flocks":
            U = {k: v.copy() for k, v in T.items()}
            U["flocks"]["target"][1][0] = value
            s = save_job(emu, U, tables, 2)
        else:
            s = spoiled(key, field, value, idx)
        info, err = restore(emu, s, room=64)
        assert info is None, (key, field, value)
    ok = {k: v.copy() for k, v in T.items()}
    ok["agents"]["radius"][17] = 6.0                                           # layer 1: needs two layers
    assert restore(emu, save_job(emu, ok, tables, 2), nlayers=1, room=64)[0] is None
    assert restore(emu, save_job(emu, ok, tables, 2), nlayers=2)[0] is not None
    ok["ext"]["surround_target_uid"][17] = 39                                  # the last uid: inside the population
    assert restore(emu, save_job(emu, ok, tables, 2))[0] is not None
    # what the uploads accept restores: a flock index below -1 (no flock) and a state the uploads do not check
    ok["agents"]["flock"][3] = -7; ok["agents"]["state"][4] = 12
    info, rec = restore(emu, save_job(emu, ok, tables, 1))
    assert info is not None and rec["agents"].tobytes() == ok["agents"].tobytes()


@pytest.mark.parametrize("world", range(1, 9))
def test_empty_member_ranges(emu, world):
    """a population smaller than the world: members with empty ranges save empty segments and restore empty ranges"""
    rng = np.random.default_rng(world)
    T = population(rng, 3, 2, MS | BLK)
    segs = save_job(emu, T, MS | BLK, world)
    for w in range(1, 9):
        got = []
        for r in range(w):
            info, rec = restore(emu, segs, w, r)
            got.append(rec["agents"])
        assert np.concatenate(got).tobytes() == T["agents"].tobytes()
