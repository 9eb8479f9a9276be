"""The per-item rule of pfnav_agents_collect_events (csrc/pfnav_events_kernel.cuh) run on CPU threads
(tests/emu/events_emu.cpp) over random patch and agent arrays, against the numpy restatement of the selection,
state_after and pos (tests/events_ref.py): equal byte for byte. Test infrastructure, not a product path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from events_ref import SET_DEST, SET_MOVING, SET_POSITION, SET_STATE, expected_events

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
GARR = capi.FLAG_GARRISONED


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libevents_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fno-strict-aliasing", "-fPIC", "-shared", "-pthread",
                    os.path.join(HERE, "emu", "events_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_events.restype = C.c_size_t
    L.emu_events.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def _case(seed, n_agents, n_work, p_garr=0.1):
    """random patches over a random work list: a mix of the flag bits the rule looks at and the ones it ignores"""
    rng = np.random.default_rng(seed)
    agents = np.zeros(n_agents, capi.AGENT)
    agents["pos"] = rng.normal(scale=300.0, size=(n_agents, 2))
    agents["state"] = rng.integers(0, 9, n_agents)
    agents["flags"] = np.where(rng.random(n_agents) < p_garr, GARR, 0) | capi.FLAG_MOVABLE | \
        np.where(rng.random(n_agents) < 0.2, capi.FLAG_COMBAT_HELD, 0)
    work = rng.choice(n_agents, n_work, replace=False).astype(np.uint32)
    p = np.zeros(n_work, capi.PATCH)
    for name in p.dtype.names:
        if p.dtype[name].base.kind == "f":
            p[name] = rng.normal(scale=100.0, size=p[name].shape)
    p["next_state"] = rng.integers(-1, 9, n_work)
    p["next_block"] = rng.integers(0, 2, n_work)
    p["next_attack"] = rng.integers(-1, 3, n_work)
    p["wait_ticks_left"] = rng.integers(0, 60, n_work)
    # the bits the rule ignores (velocity, rotation, steps ...) on most items; the ones it reads on some
    other = rng.integers(0, 1 << 15, n_work).astype(np.uint32) & ~np.uint32(SET_STATE | SET_MOVING | SET_DEST)
    kind = rng.integers(0, 6, n_work)
    f = other.copy()
    f[kind == 1] |= SET_STATE
    f[kind == 2] |= SET_MOVING
    f[kind == 3] |= SET_STATE | SET_MOVING
    f[kind == 4] |= SET_DEST
    p["flags"] = f
    todo = np.where(rng.random(n_work) < 0.15, rng.integers(1, 8, n_work), 0).astype(np.uint32)
    p["engine_todo"] = todo
    return p, agents, work


def _run(emu, p, agents, work, nthreads):
    out = np.zeros(max(len(work), 1), capi.EVENT)
    k = emu.emu_events(_p(p), _p(agents), _p(work), len(work), nthreads, _p(out))
    return out[:k]


@pytest.mark.parametrize("seed,n_agents,n_work,nthreads", [(1, 5000, 4000, 8), (2, 700, 700, 3), (3, 40000, 33333, 32),
                                                           (4, 64, 1, 1)])
def test_rule_matches_numpy(emu, seed, n_agents, n_work, nthreads):
    p, agents, work = _case(seed, n_agents, n_work)
    got = _run(emu, p, agents, work, nthreads)
    want = expected_events(p, agents, work)
    assert got.tobytes() == want.tobytes(), (len(got), len(want))
    if n_work < 100:
        return
    # every family the rule distinguishes is present, and garrisoned items with qualifying patches are dropped
    garr = (agents["flags"][work] & GARR) != 0
    f, todo = p["flags"], p["engine_todo"]
    qual = ((f & (SET_STATE | SET_MOVING | SET_DEST)) != 0) | (todo != 0)
    assert (garr & qual).sum() > 5
    assert (~qual).sum() > 5
    assert (((f & (SET_STATE | SET_MOVING | SET_DEST)) == 0) & (todo != 0) & ~garr).sum() > 5
    both = ((f & SET_STATE) != 0) & ((f & SET_MOVING) != 0) & ~garr
    assert both.sum() > 5
    assert ((f & SET_POSITION) != 0).any() and ((f & SET_POSITION) == 0).any()
    assert len(got) == int((qual & ~garr).sum())
    assert set(got["uid"].tolist()) <= set(work.tolist())


def test_state_after_and_pos_rules(emu):
    """hand-built items: SET_STATE then SET_MOVING writes next_state once; SET_POSITION takes next_pos x, z; neither
    keeps the entity's own values; a todo-only item and a SET_DEST item keep the state"""
    agents = np.zeros(6, capi.AGENT)
    agents["state"] = [0, 2, 4, 5, 6, 0]
    agents["pos"] = np.arange(12, dtype=np.float32).reshape(6, 2)
    agents["flags"][5] = GARR
    p = np.zeros(6, capi.PATCH)
    p["flags"] = [SET_STATE | SET_MOVING | SET_POSITION, SET_STATE, 0, SET_DEST, SET_MOVING | SET_POSITION, SET_STATE]
    p["engine_todo"] = [0, 0, capi.TODO_SURROUND_QUERY, 0, 0, 0]
    p["next_state"] = [1, 2, -1, -1, 7, 2]
    p["next_pos"] = np.arange(18, dtype=np.float32).reshape(6, 3) + 100
    p["next_dest"] = [[1, 2], [3, 4], [5, 6], [7, 8], [9, 10], [11, 12]]
    p["next_attack"] = [0, 0, 0, 1, 0, 0]
    work = np.arange(6, dtype=np.uint32)
    got = _run(emu, p, agents, work, 2)
    assert got["uid"].tolist() == [0, 1, 2, 3, 4]                      # 5 is garrisoned
    assert got["state_before"].tolist() == [0, 2, 4, 5, 6]
    assert got["state_after"].tolist() == [1, 2, 4, 5, 7]
    assert got["pos"].tolist() == [[100, 102], [2, 3], [4, 5], [6, 7], [112, 114]]
    assert got["attack"].tolist() == [0, 0, 0, 1, 0] and got["todo"].tolist() == [0, 0, 1, 0, 0]
    assert got["dest"][3].tolist() == [7, 8]
    assert got.tobytes() == expected_events(p, agents, work).tobytes()


def test_empty_and_nothing_selected(emu):
    p, agents, work = _case(9, 100, 50)
    p["flags"] &= ~np.uint32(SET_STATE | SET_MOVING | SET_DEST)
    p["engine_todo"] = 0
    assert len(_run(emu, p, agents, work, 4)) == 0
    assert len(_run(emu, p[:0], agents, work[:0], 4)) == 0
