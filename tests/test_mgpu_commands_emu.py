"""The job form of the command batch on the CPU (csrc/pfnav_commands_host.h through tests/emu/commands_job_emu.cpp): a
population split into 1-3 contiguous ranges, every member given the whole batch. The members' verdicts together must
equal the solo verdict on the whole population -- including refusals only one range can see (a layer that was not
created, a flock index the new table drops) -- each member's own records must give its range the mirror and
flock_layer_used the solo call gives that range, and the foreign records must leave every member's flock column, radii
and flag bits equal to the solo call's."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from test_agent_commands_emu import population, random_deltas

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
D = capi.AGENT_DELTA
FOREIGN = np.dtype([("uid", np.uint32), ("mask", np.uint32), ("flock", np.int32), ("radius", np.float32), ("flags", np.uint32)])
AIR, WATER = capi.FLAG_AIR, capi.FLAG_WATER
FOREIGN_BITS = capi.DELTA_FLOCK | capi.DELTA_RADIUS | capi.DELTA_FLAGS


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libcommands_job_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-D_GLIBCXX_ASSERTIONS", "-fPIC", "-shared", os.path.join(HERE, "emu", "commands_job_emu.cpp"),
                    "-o", so], check=True)
    L = C.CDLL(so)
    p, i = C.c_void_p, C.c_int
    L.emu_mirror_new.restype = p
    L.emu_mirror_new.argtypes = [p, i, i]
    L.emu_mirror_delete.argtypes = [p]
    L.emu_mirror_state.argtypes = [p, p, p, p]
    L.emu_solo.argtypes = [p, i, i, i, i, i, p, i, i, p, C.c_char_p]
    L.emu_job_member.argtypes = [p, i, i, i, i, i, i, i, p, i, i, p, p, p, p, C.c_char_p]
    L.emu_apply_own.argtypes = [p, p, p, p, i, p, p, p]
    L.emu_apply_foreign.argtypes = [p, i, p, p, p]
    assert L.emu_foreign_size() == FOREIGN.itemsize
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def ranges(n, world):
    base, rem = divmod(n, world)
    lo = [r * base + min(r, rem) for r in range(world)]
    return [(l, l + base + (1 if r < rem else 0)) for r, l in enumerate(lo)]


class Side:
    """one context: its agent tables (meaningful on [lo, hi)), the neighbour-record columns and flock column of the
    whole population, and the (flock, layer) mirror of [lo, hi)"""

    def __init__(self, L, a, ms, ext, lo, hi, nflocks):
        self.L, self.lo, self.hi = L, lo, hi
        self.a, self.ms, self.ext = a.copy(), ms.copy(), ext.copy()
        self.flock_of = a["flock"].astype(np.int32)
        self.radius = a["radius"].astype(np.float32)
        self.sf = (a["state"].astype(np.uint32) << 24) | (a["flags"] & np.uint32(0xFFFFFF))
        sub = np.ascontiguousarray(a[lo:hi])
        self.h = L.emu_mirror_new(_p(sub), hi - lo, nflocks)

    def close(self):
        self.L.emu_mirror_delete(self.h)

    def mirror(self, nflocks):
        k = self.hi - self.lo
        fl, ly, us = np.zeros(k, np.int32), np.zeros(k, np.uint8), np.zeros((nflocks, 12), np.uint8)
        self.L.emu_mirror_state(self.h, _p(fl), _p(ly), _p(us))
        return fl, ly, us

    def apply_own(self, recs):
        self.L.emu_apply_own(_p(self.a), _p(self.ms), _p(self.ext), _p(recs), len(recs), _p(self.flock_of), _p(self.radius), _p(self.sf))

    def apply_foreign(self, f):
        self.L.emu_apply_foreign(_p(f), len(f), _p(self.flock_of), _p(self.radius), _p(self.sf))


def solo(L, side, d, n, nf, nlayers, commit):
    d = np.ascontiguousarray(d, D)
    out = np.zeros(max(len(d), 1), D)
    err = C.create_string_buffer(256)
    k = L.emu_solo(_p(d), len(d), n, nf, 1, 1, side.h, nlayers, int(commit), _p(out), err)
    return (None, err.value.decode()) if k < 0 else (out[:k].copy(), None)


def member(L, side, d, n, nf, nlayers, commit, have_ms=True):
    d = np.ascontiguousarray(d, D)
    own, foreign = np.zeros(max(len(d), 1), D), np.zeros(max(len(d), 1), FOREIGN)
    no, nfo = C.c_int(0), C.c_int(0)
    err = C.create_string_buffer(256)
    rc = L.emu_job_member(_p(d), len(d), n, nf, int(have_ms), 1, side.lo, side.hi, side.h, nlayers, int(commit), _p(own),
                          C.byref(no), _p(foreign), C.byref(nfo), err)
    return (None, None, err.value.decode()) if rc < 0 else (own[:no.value].copy(), foreign[:nfo.value].copy(), None)


def used_of(a, nflocks):
    used = np.zeros((nflocks, 12), np.uint8)
    for f, fl, r in zip(a["flock"], a["flags"], a["radius"]):
        if f >= 0:
            used[f, (4 if fl & WATER else 8 if fl & AIR else 0) + (3 if r >= 15 else 2 if r >= 10 else 1 if r >= 5 else 0)] = 1
    return used


@pytest.mark.parametrize("world", [1, 2, 3])
@pytest.mark.parametrize("seed", range(4))
def test_members_agree_with_the_solo_call(emu, world, seed):
    """random batches with a growing and shrinking flock table on 61 entities: the members' verdicts together are the solo
    verdict; after an accepted batch every member's own range (agents, movestate, ext, mirror, used table) equals the
    solo call's, and every member's whole flock column, radii and low flag bits equal the solo call's. Between batches a
    gather brings every member the owners' records; the flock column is not gathered."""
    rng = np.random.default_rng(1000 * world + seed)
    n, nflocks, nlayers = 61, 4, 8                # ground and water layers exist, air does not
    a, ms, ext = population(rng, n, nflocks)
    a["flags"] &= ~np.uint32(AIR)
    one = Side(emu, a, ms, ext, 0, n, nflocks)
    mem = [Side(emu, a, ms, ext, lo, hi, nflocks) for lo, hi in ranges(n, world)]
    try:
        accepted = refused = 0
        for it in range(40):
            new_nf = max(1, nflocks + int(rng.integers(-1, 3)))
            d = random_deltas(rng, int(rng.integers(0, 25)), n, new_nf)
            if it % 3:
                d["flags"] &= ~np.uint32(AIR)
            if it % 4 == 0:
                d["mask"] &= FOREIGN_BITS | capi.DELTA_STATE
            m, e1 = solo(emu, one, d, n, new_nf, nlayers, False)
            verdicts = [member(emu, s, d, n, new_nf, nlayers, False) for s in mem]
            assert (e1 is None) == all(v[2] is None for v in verdicts), (e1, [v[2] for v in verdicts])
            if e1 is not None:
                refused += 1
                continue
            accepted += 1
            solo(emu, one, d, n, new_nf, nlayers, True)
            one.apply_own(m)
            nflocks = new_nf
            for s, (own, foreign, _) in zip(mem, verdicts):
                member(emu, s, d, n, new_nf, nlayers, True)
                lo, hi = s.lo, s.hi
                assert list(own["uid"]) == [u for u in m["uid"] if lo <= u < hi]
                assert own.tobytes() == m[(m["uid"] >= lo) & (m["uid"] < hi)].tobytes()
                outside = m[((m["uid"] < lo) | (m["uid"] >= hi)) & ((m["mask"] & FOREIGN_BITS) != 0)]
                assert list(foreign["uid"]) == list(outside["uid"]) and (foreign["mask"] == outside["mask"] & FOREIGN_BITS).all()
                s.apply_own(own)
                s.apply_foreign(foreign)
                assert s.a[lo:hi].tobytes() == one.a[lo:hi].tobytes()
                assert s.ms[lo:hi].tobytes() == one.ms[lo:hi].tobytes() and s.ext[lo:hi].tobytes() == one.ext[lo:hi].tobytes()
                assert (s.flock_of == one.flock_of).all()
                assert s.radius.tobytes() == one.radius.tobytes()
                assert ((s.sf ^ one.sf) & 0xFFFFFF == 0).all() and (s.sf[lo:hi] == one.sf[lo:hi]).all()
                fl, ly, us = s.mirror(nflocks)
                ofl, oly, _ = one.mirror(nflocks)
                assert (fl == ofl[lo:hi]).all() and (ly == oly[lo:hi]).all()
                assert (us == used_of(one.a[lo:hi], nflocks)).all()
            for s in mem:                             # the gather: the owners' neighbour records
                s.radius[:], s.sf[:] = one.radius, one.sf
        assert accepted >= 5 and refused >= 3, (accepted, refused)
    finally:
        for s in [one] + mem:
            s.close()


def _fixed(emu, world):
    n, nflocks = 30, 4
    a = np.zeros(n, capi.AGENT)
    a["radius"] = 1.5
    a["flock"] = np.arange(n) % nflocks
    ms = np.zeros(n, capi.MOVESTATE)
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    return n, nflocks, a, Side(emu, a, ms, ext, 0, n, nflocks), [Side(emu, a, ms, ext, lo, hi, nflocks) for lo, hi in ranges(n, world)]


def test_refusals_only_one_range_can_see(emu):
    """a layer that was not created and a flock index the new table drops, each on one range's entity: only the owner
    refuses, so the job refuses as the solo call does; a POSITION delta refused by the one member without movestate"""
    n, nflocks, a, one, mem = _fixed(emu, 3)
    try:
        def verdicts(d, nf, nlayers=1, ms=(True, True, True)):
            return [member(emu, s, d, n, nf, nlayers, False, have_ms=h)[2] for s, h in zip(mem, ms)]
        d = np.zeros(2, D)
        d["uid"], d["mask"], d["radius"] = [1, 25], capi.DELTA_RADIUS, [2.0, 6.0]          # uid 25: layer 1 (not created)
        v = verdicts(d, nflocks)
        assert v[0] is None and v[1] is None and "layer" in v[2]
        assert "layer" in solo(emu, one, d, n, nflocks, 1, False)[1]
        # the table drops flock 3; every entity of flock 3 moves but uid 15 (range 1)
        tail = np.nonzero(a["flock"] == 3)[0]
        d = np.zeros(len(tail), D)
        d["uid"], d["mask"], d["flock"] = tail, capi.DELTA_FLOCK, 0
        d = d[d["uid"] != 15]
        v = verdicts(d, 3)
        assert v[0] is None and "shorter" in v[1] and v[2] is None
        assert "shorter" in solo(emu, one, d, n, 3, 1, False)[1]
        d = np.zeros(1, D)
        d["uid"], d["mask"] = 12, capi.DELTA_POSITION
        v = verdicts(d, nflocks, ms=(True, False, True))
        assert v[0] is None and "movestate" in v[1] and v[2] is None
        # a delta outside the population refuses everywhere; one inside any range is accepted everywhere
        d["uid"], d["mask"] = n, capi.DELTA_STATE
        assert all(e and "outside" in e for e in verdicts(d, nflocks))
        d["uid"] = n - 1
        assert verdicts(d, nflocks) == [None] * 3
    finally:
        for s in [one] + mem:
            s.close()


def test_batch_on_one_range_only(emu):
    """a batch whose uids all sit on the last range: the other members get no own record and only the foreign part
    (flock, radius, flags; not state or velocity)"""
    n, nflocks, a, one, mem = _fixed(emu, 3)
    try:
        lo = mem[2].lo
        d = np.zeros(4, D)
        d["uid"] = [lo, lo + 1, lo + 2, lo + 2]
        d["mask"] = [capi.DELTA_STATE | capi.DELTA_VELOCITY, capi.DELTA_FLOCK | capi.DELTA_STATE, capi.DELTA_RADIUS, capi.DELTA_FLAGS]
        d["flock"], d["radius"], d["flags"] = 2, 3.0, (1 << 24) | capi.FLAG_GARRISONED | capi.FLAG_MOVABLE
        for s in mem[:2]:
            own, foreign, e = member(emu, s, d, n, nflocks, 1, False)
            assert e is None and len(own) == 0
            assert list(foreign["uid"]) == [lo + 1, lo + 2]
            assert list(foreign["mask"]) == [capi.DELTA_FLOCK, capi.DELTA_RADIUS | capi.DELTA_FLAGS]
            assert foreign["flags"][1] == capi.FLAG_GARRISONED | capi.FLAG_MOVABLE     # merged: only the low 24 bits
        own, foreign, e = member(emu, mem[2], d, n, nflocks, 1, False)
        assert e is None and list(own["uid"]) == [lo, lo + 1, lo + 2] and len(foreign) == 0
    finally:
        for s in [one] + mem:
            s.close()
