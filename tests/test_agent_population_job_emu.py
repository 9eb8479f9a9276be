"""The job form of a population change on the CPU (csrc/pfnav_commands_host.h through tests/emu/population_job_emu.cpp):
a population split into the balanced ranges of 1-8 members, every member given the job's whole batch. For random
batches: the segments and appended runs tile every member's new range exactly once, each segment's rows come from the
sender's old range, at most R + A rows cross any member boundary, the members' mirrors concatenated equal the solo
compaction + append, and the members' verdicts combined equal the solo verdict -- including a stranded flock index that
only one member can see."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from test_agent_population_emu import agents

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
LAYERS = 12
MS, BLK = 1, 8


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libpopulation_job_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-D_GLIBCXX_ASSERTIONS", "-fPIC", "-shared",
                    os.path.join(HERE, "emu", "population_job_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    p, i = C.c_void_p, C.c_int
    L.emu_mirror_new.restype = p
    L.emu_mirror_new.argtypes = [p, i, i]
    L.emu_mirror_delete.argtypes = [p]
    L.emu_mirror_state.argtypes = [p, p, p, p]
    L.emu_solo.argtypes = [p, i, i, p, i, p, p, p, p, p, i, i, C.c_char_p]
    L.emu_job_member.argtypes = [p, i, i, i, i, i, p, i, p, p, p, p, p, i, i, p, p, p, i, p, p, p, C.c_char_p]
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def ranges(n, world):
    base, rem = divmod(n, world)
    lo = [r * base + min(r, rem) for r in range(world + 1)]
    return lo


def mirror_state(L, h, n, nflocks):
    fl, ly, us = np.zeros(n, np.int32), np.zeros(n, np.uint8), np.zeros((nflocks, LAYERS), np.uint8)
    L.emu_mirror_state(h, _p(fl), _p(ly), _p(us))
    return fl, ly, us


def columns(a):
    """the flock column, radii and state << 24 | flags of the neighbour records, as every member holds them"""
    return (a["flock"].astype(np.int32), a["radius"].astype(np.float32),
            (a["state"].astype(np.uint32) << 24) | (a["flags"] & np.uint32(0xFFFFFF)))


def run(L, a, world, rm, add, nflocks, nflocks_new, nlayers=LAYERS, tables=0, ms=None, blk=None):
    """the solo call and every member's; -> (solo n_new or None, list of member results), the checks made"""
    n = len(a)
    rm = np.ascontiguousarray(rm, np.uint32)
    add = np.ascontiguousarray(add, capi.AGENT)
    err = C.create_string_buffer(256)
    hs = L.emu_mirror_new(_p(a), n, nflocks)
    try:
        n_solo = L.emu_solo(hs, nlayers, tables, _p(rm), len(rm), _p(add), _p(ms), None, None, _p(blk), len(add), nflocks_new, err)
        solo = mirror_state(L, hs, n_solo, nflocks_new) if n_solo >= 0 else None
    finally:
        L.emu_mirror_delete(hs)
    old = ranges(n, world)
    removed = np.unique(rm[rm < n]) if n_solo >= 0 else None
    keep = np.delete(np.arange(n), removed.astype(np.int64)) if n_solo >= 0 else None
    cols = None
    if n_solo >= 0:
        cf, cr, cs = columns(np.concatenate([a[keep], add]))
        cols = (np.ascontiguousarray(cf), np.ascontiguousarray(cr), np.ascontiguousarray(cs))
    verdicts, parts, plans = [], [], []
    for r in range(world):
        sub = np.ascontiguousarray(a[old[r]:old[r + 1]])
        h = L.emu_mirror_new(_p(sub), len(sub), nflocks)
        try:
            bounds = np.zeros(3 * (world + 1), np.int64)
            seg = np.zeros(2 * world * world, np.int64)
            app = np.zeros(2 * world, np.int64)
            c = cols if cols is not None else (np.zeros(1, np.int32), np.zeros(1, np.float32), np.zeros(1, np.uint32))
            rc = L.emu_job_member(h, n, world, r, nlayers, tables, _p(rm), len(rm), _p(add), _p(ms), None, None, _p(blk), len(add),
                                  nflocks_new, _p(c[0]), _p(c[1]), _p(c[2]), 1 if cols is not None else 0, _p(bounds), _p(seg),
                                  _p(app), err)
            verdicts.append(rc)
            if rc == 0 and cols is not None:
                nlo = bounds[world + 1:2 * (world + 1)]
                parts.append(mirror_state(L, h, int(nlo[r + 1] - nlo[r]), nflocks_new))
                plans.append((bounds, seg.reshape(world, world, 2), app.reshape(world, 2)))
        finally:
            L.emu_mirror_delete(h)
    # the combined verdict is the solo verdict
    assert (n_solo >= 0) == all(v == 0 for v in verdicts), (n_solo, verdicts)
    if n_solo < 0:
        return None, verdicts
    n_new = n_solo
    new = ranges(n_new, world)
    R, A = len(removed), len(add)
    for bounds, seg, app in plans:                  # every member derives the same plan
        assert (bounds == plans[0][0]).all() and (seg == plans[0][1]).all() and (app == plans[0][2]).all()
    bounds, seg, app = plans[0]
    assert list(bounds[:world + 1]) == old and list(bounds[world + 1:2 * (world + 1)]) == new
    src = np.concatenate([keep, np.full(A, -1)])    # the old uid of every new row, -1 for appended
    for r in range(world):
        cover = np.zeros(new[r + 1] - new[r], np.int64)
        for s in range(world):
            lo, hi = seg[s, r]
            assert new[r] <= lo <= hi <= new[r + 1]
            cover[lo - new[r]:hi - new[r]] += 1
            if hi > lo:
                assert hi <= n_new - A and (src[lo:hi] >= old[s]).all() and (src[lo:hi] < old[s + 1]).all(), (s, r)
        lo, hi = app[r]
        assert hi == lo or (new[r] <= lo <= hi <= new[r + 1] and lo >= n_new - A)
        cover[lo - new[r]:hi - new[r]] += 1
        assert (cover == 1).all(), (r, cover)
    for b in range(1, world):
        crossing = sum(int(seg[s, r, 1] - seg[s, r, 0]) for s in range(world) for r in range(world) if (s < b) != (r < b))
        assert crossing <= R + A, (b, crossing, R, A)
    got = tuple(np.concatenate([p[k] for p in parts]) for k in range(2))
    assert np.array_equal(got[0], solo[0]) and np.array_equal(got[1], solo[1])
    used = np.zeros_like(solo[2])
    for p in parts:
        used |= p[2]
    assert np.array_equal(used, solo[2])
    return n_new, verdicts


@pytest.mark.parametrize("world", range(1, 9))
def test_random_batches(emu, world):
    rng = np.random.default_rng(100 + world)
    for t in range(60):
        n = int(rng.integers(0, 300))
        nf = int(rng.integers(1, 6))
        a = agents(rng, n, nf)
        kind = t % 4
        R = int(rng.integers(0, n + 1)) if n else 0
        if kind == 0:
            rm = rng.choice(n, R, replace=False) if R else []
        elif kind == 1:                                  # only the first member's range: every boundary shifts down
            rm = np.arange(min(R, ranges(n, world)[1]))
        elif kind == 2:                                  # a member's whole old range
            lo = ranges(n, world)
            r = int(rng.integers(0, world))
            rm = np.arange(lo[r], lo[r + 1])
        else:
            rm = rng.integers(0, max(n, 1), int(rng.integers(0, 20))) if n else []    # repeats
        A = int(rng.integers(0, 300)) if t % 3 else 0
        add = agents(rng, A, nf)
        run(emu, a, world, np.asarray(rm, np.int64), add, nf, nf)


@pytest.mark.parametrize("world", [1, 2, 3, 5, 8])
def test_population_below_world_then_empty_then_refilled(emu, world):
    rng = np.random.default_rng(7)
    a = agents(rng, 40, 3)
    n1, _ = run(emu, a, world, np.arange(40 - max(world - 1, 1) + 1), np.zeros(0, capi.AGENT), 3, 3)
    assert n1 < world or world == 1
    b = agents(rng, n1, 3)
    n2, _ = run(emu, b, world, np.arange(n1), np.zeros(0, capi.AGENT), 3, 3)
    assert n2 == 0
    n3, _ = run(emu, np.zeros(0, capi.AGENT), world, [], agents(rng, 25, 3), 3, 3)
    assert n3 == 25


@pytest.mark.parametrize("world", [2, 3, 4, 7])
def test_stranded_flock_index_one_member_sees(emu, world):
    """the new table drops the last flock; one survivor of it sits in the last member's range: only that member refuses,
    and the combined verdict is the solo refusal. Removing that survivor in the same batch makes every member pass."""
    rng = np.random.default_rng(world)
    n, nf = 200, 4
    a = agents(rng, n, nf)
    a["flock"][a["flock"] == nf - 1] = 0
    lo = ranges(n, world)
    u = lo[world - 1] + 3
    a["flock"][u] = nf - 1
    res, verdicts = run(emu, a, world, [5], np.zeros(0, capi.AGENT), nf, nf - 1)
    assert res is None and verdicts[:-1] == [0] * (world - 1) and verdicts[-1] == -1
    res, verdicts = run(emu, a, world, [5, u], np.zeros(0, capi.AGENT), nf, nf - 1)
    assert res == n - 2


@pytest.mark.parametrize("world", [1, 2, 3, 6])
def test_refusals_every_member_sees(emu, world):
    """batch checks that do not depend on the member: a removal outside the population, an appended record with a
    layer that was not created, a flock index beyond the new table, and records missing for a table that exists"""
    rng = np.random.default_rng(11)
    n, nf = 90, 3
    a = agents(rng, n, nf)
    add = agents(rng, 4, nf)
    res, v = run(emu, a, world, [n], add, nf, nf)
    assert res is None and v == [-1] * world
    bad = add.copy(); bad["radius"][0] = 16.0
    res, v = run(emu, a, world, [], bad, nf, nf, nlayers=1)
    assert res is None and v == [-1] * world
    bad = add.copy(); bad["flock"][1] = nf
    res, v = run(emu, a, world, [], bad, nf, nf)
    assert res is None and v == [-1] * world
    res, v = run(emu, a, world, [], add, nf, nf, tables=MS | BLK, blk=np.zeros(4, capi.BLOCKING))
    assert res is None and v == [-1] * world
    ms = np.zeros(4, capi.MOVESTATE)
    blk = np.zeros(4, capi.BLOCKING); blk["faction_id"] = 15
    res, v = run(emu, a, world, [1, 2], add, nf, nf, tables=MS | BLK, ms=ms, blk=blk)
    assert res == n - 2 + 4
