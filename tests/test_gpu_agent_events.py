"""GPU suite: pfnav_agents_collect_events / pfnav_agents_read_events.

Derivation: the population read before the collect, the patches, the apply, and the population read after it. The
expected list is the numpy filter of tests/events_ref.py over the patches and the state before; the device's list must
equal it field for field, bit for bit, and state_after / pos must be what the apply left. Cases: the all-states scenario
of test_gpu_states.py (with live surround targets and garrisoned work items) at 20 and 10 Hz, an empty work list, resident
ticks of the C2 population with PFNAV_APPLY_BLOCKERS, and a population grown from 1 000 to 1 000 000 between ticks.
The collect has no side effect: a context that collects leaves every table equal to one that does not. Then the call
contract, and groups of 2 and 3 members whose lists joined in rank order equal one context's."""
import importlib
import os
import sys

import numpy as np
import pytest

import cases
import commands_ref as cr
from events_ref import SET_DEST, SET_MOVING, SET_STATE, expected_events
from test_gpu_mgpu_population import _blk, _c2_job, _spawn
from test_gpu_states import ST_ARRIVED, ST_ENTER, ST_SURROUND, ST_WAITING, _scenario

pytestmark = pytest.mark.gpu
capi = cases.capi
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GARR = capi.FLAG_GARRISONED
ST_MOVING = 0


def _check(ev, patches, before, after, work):
    """ev against the numpy filter, and state_after / pos against what the apply left"""
    want = expected_events(patches, before, work)
    assert ev.dtype == capi.EVENT and len(ev) == len(want), (len(ev), len(want))
    assert ev.tobytes() == want.tobytes(), np.nonzero(ev != want)[0][:10]
    assert (ev["state_after"] == after["state"][ev["uid"]]).all()
    assert ev["pos"].tobytes() == np.ascontiguousarray(after["pos"][ev["uid"]]).tobytes()


def _derived_tick(X, n, work, apply=lambda X: X.agents_apply_updates(), tick_flags=0):
    """tick -> compute_updates -> read_state -> collect -> read_patches -> apply -> read_events (late, after the
    apply) -> read_state; checks the list and returns (events, patches)"""
    X.agents_tick(tick_flags)
    X.agents_compute_updates()
    before, _ = X.agents_read_state(n, movestate=False)
    X.agents_collect_events()
    p = X.agents_read_patches(len(work))
    apply(X)
    X.agents_rebuild_index()
    ev = X.agents_read_events()
    after, _ = X.agents_read_state(n, movestate=False)
    _check(ev, p, before, after, work)
    return ev, p, before


@pytest.mark.parametrize("hz", [20, 10])
def test_all_states(nav, hz):
    """every movement state, SET_DEST from moving enter-range targets, WAITING expiry, surround TODOs (live targets),
    garrisoned work items that carry patches; three ticks"""
    p, cost, a, ms, form, ext = _scenario(5151, hz)
    n = len(a["radius"])
    rng = np.random.default_rng(hz)
    sur = np.nonzero(a["state"] == ST_SURROUND)[0]
    ext["surround_target_uid"][sur[::2]] = rng.integers(0, n, len(sur[::2]))
    work = np.nonzero(a["state"] != ST_ARRIVED)[0].astype(np.uint32)
    garr = rng.choice(work, len(work) // 20, replace=False)
    a["flags"][garr] |= GARR
    vdes = rng.normal(size=(len(work), 2)).astype(np.float32)
    vdes /= np.linalg.norm(vdes, axis=1, keepdims=True)
    aa = dict(a)
    aa["vdes"] = np.zeros((n, 2), np.float32); aa["vdes"][work] = vdes
    aa["has_los"] = np.zeros(n, np.uint32)
    rec, fl = capi.pack_agents(aa)
    nav.map_create(3, 3, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.agents_upload(rec, fl, hz)
    nav.agents_upload_movestate(ms)
    nav.agents_upload_formation(form)
    nav.agents_upload_movestate_ext(ext)
    nav.agents_set_work(work)
    seen = []
    for t in range(3):
        ev, pt, before = _derived_tick(nav, n, work)
        seen.append((ev, pt, before))
    ev = np.concatenate([s[0] for s in seen])
    assert (ev["flags"] & SET_DEST).any()
    assert ((ev["flags"] & SET_STATE) != 0).any() and ((ev["flags"] & SET_MOVING) != 0).any()
    assert (ev["todo"] & capi.TODO_SURROUND_QUERY).any()
    assert ((ev["state_before"] == ST_WAITING) & (ev["state_after"] != ST_WAITING)).any()      # WAITING expiry
    assert (ev["state_before"] == ST_ENTER).any()
    # garrisoned work items carry qualifying patches and give no event
    ev0, pt0, before0 = seen[0]
    g = (before0["flags"][work] & GARR) != 0
    qual = ((pt0["flags"] & (SET_STATE | SET_MOVING | SET_DEST)) != 0) | (pt0["engine_todo"] != 0)
    assert (g & qual).sum() > 5 and not np.isin(ev0["uid"], work[g]).any()


def test_empty_work_list(nav):
    _, cost, a, ms = cases.update_case(77, 20)
    rec, fl = capi.pack_agents(a)
    n = len(rec)
    nav.map_create(3, 3, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.agents_upload(rec, fl, 20)
    nav.agents_upload_movestate(ms)
    nav.agents_set_work(np.arange(n, dtype=np.uint32))
    ev, _, _ = _derived_tick(nav, n, np.arange(n, dtype=np.uint32))
    assert len(ev) > 0
    nav.agents_set_work(np.zeros(0, np.uint32))
    nav.agents_compute_updates()
    nav.agents_collect_events()
    nav.agents_apply_updates()
    assert len(nav.agents_read_events()) == 0 and len(nav.agents_read_events(cap=0)) == 0


def _crowd(pf, workload):
    """the benchmark's population with every flock's target at the flock's own centre and a desired velocity towards it,
    so that the crowd arrives (the adjacent-arrived cascade spreads) while the rest keeps moving"""
    sys.path.insert(0, ROOT)
    bench = importlib.import_module("bench")
    bench.set_workload(workload)
    try:
        W = bench.build_workload(pf, 1, 0)
        chunks = bench.CHUNKS
    finally:
        bench.set_workload("C2")
    a = W["agents"]
    for f in range(len(a["flock_target"])):
        a["flock_target"][f] = a["pos"][a["flock_of"] == f].mean(axis=0)
    d = a["flock_target"][a["flock_of"]] - a["pos"]
    a["vdes"] = (d / np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-6)).astype(np.float32)
    a["has_los"] = np.ones(len(d), np.uint32)
    a["state"][:] = 0
    rec, fl = capi.pack_agents(a)
    ms = np.zeros(len(rec), capi.MOVESTATE)
    ms["next_pos"][:, 0], ms["next_pos"][:, 2] = a["pos"][:, 0], a["pos"][:, 1]
    ms["step"] = 1.0
    ms["next_rot"] = cases.dir_quat(a["vdes"]); ms["combat_facing"] = ms["next_rot"]
    return chunks, W["cost"], rec, fl, ms


def _context(cw, cost, rec, fl, ms):
    X = capi.Nav(0)
    X.map_create(cw, cw, 1); X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
    X.agents_upload(rec, fl, 20)
    X.agents_upload_movestate(ms)
    b = np.zeros(len(rec), capi.BLOCKING); b["faction_id"] = capi.FACTION_ID_NONE
    X.agents_upload_blocking(b)
    return X


def _blockers_apply(X):
    X.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
    X.map_commit()


@pytest.fixture(scope="module")
def c2(pf):
    return _crowd(pf, "C2")


def test_c2_resident_ticks_and_no_side_effects(c2):
    """8 resident ticks of the C2 crowd with PFNAV_APPLY_BLOCKERS: every list derived; a twin context that never collects
    ends every tick with the same tables byte for byte"""
    cw, cost, rec, fl, ms = c2
    n = len(rec)
    A, B = _context(cw, cost, rec, fl, ms), _context(cw, cost, rec, fl, ms)
    try:
        total = 0
        for t in range(8):
            nw = A.agents_set_work_dev()
            assert B.agents_set_work_dev() == nw
            work = A.agents_read_work()
            ev, _, _ = _derived_tick(A, n, work, apply=_blockers_apply)
            B.agents_tick(0); B.agents_compute_updates(); _blockers_apply(B); B.agents_rebuild_index()
            total += len(ev)
            sa, ma = A.agents_read_state(n); sb, mb = B.agents_read_state(n)
            assert sa.tobytes() == sb.tobytes() and ma.tobytes() == mb.tobytes(), t
            assert A.agents_read_blocking(n).tobytes() == B.agents_read_blocking(n).tobytes(), t
            assert (A.blockers(0) == B.blockers(0)).all(), t
            assert A.agents_read_work().tobytes() == B.agents_read_work().tobytes()
        assert total > 0
    finally:
        A.close(); B.close()


def test_growth_to_a_million(pf):
    """1 000 entities, a tick, then 999 000 appended: the list regrows from 1 000 records to the million's"""
    cw, cost, rec, fl, ms = _crowd(pf, "C3")
    n = len(rec)
    assert n == 1_000_000
    X = _context(cw, cost, rec[:1000], fl, ms[:1000])
    try:
        w = X.agents_set_work_dev()
        _derived_tick(X, 1000, X.agents_read_work(), apply=_blockers_apply)
        b = np.zeros(n - 1000, capi.BLOCKING); b["faction_id"] = capi.FACTION_ID_NONE
        X.agents_change_population([], rec[1000:], ms=ms[1000:], blocking=b)
        with pytest.raises(capi.PfnavError, match="error -4"):
            X.agents_read_events()                                   # renumbered since the collect
        assert X.agents_set_work_dev() > 900_000 > w
        ev, _, _ = _derived_tick(X, n, X.agents_read_work(), apply=_blockers_apply)
        assert len(ev) > 0
    finally:
        X.close()


def _small(nav):
    _, cost, a, ms = cases.update_case(31, 20)
    rec, fl = capi.pack_agents(a)
    nav.map_create(3, 3, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.agents_upload(rec, fl, 20)
    nav.agents_upload_movestate(ms)
    nav.agents_set_work(np.arange(len(rec), dtype=np.uint32))
    return rec, fl, ms


def test_contract(pf):
    import ctypes as C
    L = capi.load()
    nav = capi.Nav(0)
    try:
        rec, fl, ms = _small(nav)
        n = len(rec)
        nout = C.c_size_t(12345)
        assert L.pfnav_agents_read_events(nav.h, None, 0, C.byref(nout)) == capi.ERR_STATE        # before any collect
        assert L.pfnav_agents_collect_events(nav.h, None) == capi.ERR_ARG                         # no update pass has run
        nav.agents_tick(0)
        nav.agents_compute_updates()
        nav.agents_collect_events()
        # null pointers
        out = np.zeros(4, capi.EVENT)
        assert L.pfnav_agents_read_events(nav.h, out.ctypes.data_as(C.c_void_p), 4, None) == capi.ERR_ARG
        assert L.pfnav_agents_read_events(nav.h, None, 4, C.byref(nout)) == capi.ERR_ARG
        # NOMEM: out untouched, out_n set; the list stays readable
        full = nav.agents_read_events()
        k = len(full)
        assert k > 2
        out = np.frombuffer(bytearray(b"\xa5" * ((k - 1) * capi.EVENT.itemsize)), capi.EVENT)
        assert L.pfnav_agents_read_events(nav.h, out.ctypes.data_as(C.c_void_p), k - 1, C.byref(nout)) == capi.ERR_NOMEM
        assert nout.value == k and out.tobytes() == b"\xa5" * len(out.tobytes())
        assert L.pfnav_agents_read_events(nav.h, None, 0, C.byref(nout)) == capi.ERR_NOMEM and nout.value == k
        big = np.zeros(k + 3, capi.EVENT)
        assert L.pfnav_agents_read_events(nav.h, big.ctypes.data_as(C.c_void_p), k + 3, C.byref(nout)) == 0
        assert nout.value == k and big[:k].tobytes() == full.tobytes() and not big[k:].tobytes().strip(b"\0")
        # the Python wrapper grows its buffer once
        assert nav.agents_read_events(cap=1).tobytes() == full.tobytes()
        # reading twice gives the same list, also after the apply
        nav.agents_apply_updates()
        assert nav.agents_read_events().tobytes() == full.tobytes()
        # collect after the apply
        with pytest.raises(capi.PfnavError, match="error -4"):
            nav.agents_collect_events()
        assert nav.agents_read_events().tobytes() == full.tobytes()                               # the refusal kept it
        # a new pass, then a population change: the list is refused until the next collect
        nav.agents_rebuild_index(); nav.agents_tick(0); nav.agents_compute_updates(); nav.agents_collect_events()
        nav.agents_apply_updates()
        assert len(nav.agents_read_events()) >= 0
        nav.agents_change_population([0, 1], np.zeros(0, capi.AGENT), ms=np.zeros(0, capi.MOVESTATE))
        with pytest.raises(capi.PfnavError, match="error -4"):
            nav.agents_read_events()
        # a re-upload renumbers too
        nav.agents_set_work(np.arange(n - 2, dtype=np.uint32))
        nav.agents_tick(0); nav.agents_compute_updates(); nav.agents_collect_events()
        nav.agents_read_events()
        nav.agents_upload(rec, fl, 20)
        with pytest.raises(capi.PfnavError, match="error -4"):
            nav.agents_read_events()
    finally:
        nav.close()
    host = capi.Nav(0, hostonly=True)
    try:
        nout = C.c_size_t(0)
        assert L.pfnav_agents_collect_events(host.h, None) == capi.ERR_NO_DEVICE
        assert L.pfnav_agents_read_events(host.h, None, 0, C.byref(nout)) == capi.ERR_NO_DEVICE
    finally:
        host.close()


def test_other_stream(pf):
    """collect on a caller's stream, read without a device synchronise"""
    import torch
    nav = capi.Nav(0)
    try:
        rec, fl, ms = _small(nav)
        n = len(rec)
        s = torch.cuda.Stream()
        nav.agents_tick(0)
        nav.agents_compute_updates()
        before, _ = nav.agents_read_state(n, movestate=False)
        p = nav.agents_read_patches(n)
        nav.agents_collect_events(stream=s.cuda_stream)
        nav.agents_apply_updates(stream=s.cuda_stream)
        ev = nav.agents_read_events()
        s.synchronize()
        after, _ = nav.agents_read_state(n, movestate=False)
        _check(ev, p, before, after, np.arange(n, dtype=np.uint32))
    finally:
        nav.close()


@pytest.mark.parametrize("world", [2, 3])
def test_group_members_joined_equal_one_context(pf, world):
    """the C2 population in a group of `world` members and in one context, 8 resident ticks with device blockers; flock
    targets moved onto the flocks' centres by a command batch at tick 2 (arrivals), a population change at tick 5. Every
    tick the members' lists joined in rank order equal the single context's byte for byte"""
    J = _c2_job(pf, world)
    J.events = {}

    def tick_one(X, nw, passes):
        X.agents_tick(capi.TICK_VDES_FROM_POOL)
        X.agents_compute_updates()
        X.agents_collect_events()
        out = (X.agents_read_velocities(nw),) + X.agents_read_debug(nw) + (X.agents_read_patches(nw),)
        X.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
        J.events[id(X)] = X.agents_read_events(cap=nw)
        return out
    J._tick_one = tick_one
    rng = np.random.default_rng(world)
    total = 0
    try:
        for t in range(8):
            J.events = {}
            s = J.tick()
            none = np.zeros(0, capi.EVENT)
            one = J.events.get(id(J.one), none)
            joined = np.concatenate([J.events.get(id(nv), none) for nv in J.navs])
            assert joined.tobytes() == one.tobytes(), (t, len(joined), len(one))
            total += len(one)
            if t == 2:
                fl = J.fl.copy()
                for f in range(len(fl)):
                    fl["target"][f] = s["pos"][s["flock"] == f].mean(axis=0)
                who = rng.choice(J.n, 200, replace=False)
                J.commands(cr.deltas(who[s["state"][who] == ST_ARRIVED], state=ST_MOVING, clear_hist=True), fl)
            if t == 5:
                k = J.n // 100
                a, m = _spawn(J, rng.choice(J.n, k, replace=False), shift=0.25)
                a["state"] = ST_MOVING
                J.change(rng.choice(J.n, k, replace=False), a, m, blk=_blk(k))
        assert total > 0
    finally:
        J.close()
