"""The host side of pfnav_agents_change_population (csrc/pfnav_commands_host.h, compiled with g++ through
tests/emu/population_emu.cpp): validation of a batch with the reason of every refusal, the numbering rule the device
gather runs per row (stable compaction, then append) against np.delete + concatenate, the (flock, layer) mirror after
compaction + append against a fresh mirror of the resulting population, and the stranding rule of a shorter flock table."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
WATER, AIR, GARR = capi.FLAG_WATER, capi.FLAG_AIR, capi.FLAG_GARRISONED
LAYERS = 12                      # PFNAV_NAV_LAYER_MAX
MS, EXT, FORM, BLK = 1, 2, 4, 8


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libpopulation_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-D_GLIBCXX_ASSERTIONS", "-fPIC", "-shared", os.path.join(HERE, "emu", "population_emu.cpp"),
                    "-o", so], check=True)
    L = C.CDLL(so)
    p = C.c_void_p
    L.emu_mirror_new.restype = p
    L.emu_mirror_new.argtypes = [p, C.c_int, C.c_int]
    L.emu_mirror_delete.argtypes = [p]
    L.emu_pop_batch.argtypes = [p, C.c_int, C.c_int, p, C.c_int, p, p, p, p, p, C.c_int, C.c_int, C.c_int, p, p, p, C.c_char_p]
    L.emu_mirror_state.argtypes = [p, p, p, p, p]
    L.emu_mirror_size.argtypes = [p, p]
    return L


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def agents(rng, n, nflocks):
    a = np.zeros(n, capi.AGENT)
    a["pos"] = rng.random((n, 2)) * 100
    a["prev_pos"] = a["pos"]
    a["radius"] = rng.choice([1.5, 5.0, 12.0, 16.0], n)
    a["flags"] = rng.choice([0, WATER, AIR, AIR | GARR], n).astype(np.uint32) | capi.FLAG_MOVABLE
    a["flock"] = rng.integers(-1, nflocks, n) if nflocks else -1
    a["state"] = rng.integers(0, 9, n)
    return a


class Mirror:
    def __init__(self, L, a, nflocks):
        self.L, self.h = L, L.emu_mirror_new(_p(a), len(a), nflocks)

    def close(self):
        self.L.emu_mirror_delete(self.h)

    def batch(self, rm, add, nflocks_new, tables=0, ms=None, ext=None, form=None, blk=None, nlayers=LAYERS, commit=True):
        """-> (n_new, src, renum, any_fac, None) or (None, .., reason)"""
        nf = C.c_int(0)
        n_old = self.L.emu_mirror_size(self.h, C.byref(nf))
        rm = np.ascontiguousarray(rm, np.uint32)
        add = np.ascontiguousarray(add, capi.AGENT)
        src = np.zeros(n_old + 1, np.uint32)
        renum = np.zeros(n_old + 1, np.uint32)
        fac = C.c_int(0)
        err = C.create_string_buffer(256)
        k = self.L.emu_pop_batch(self.h, nlayers, tables, _p(rm), len(rm), _p(add), _p(ms), _p(ext), _p(form), _p(blk), len(add),
                                 nflocks_new, int(commit), _p(src), _p(renum), C.byref(fac), err)
        if k < 0:
            return None, None, None, None, err.value.decode()
        return k, src[:n_old - len(np.unique(rm))], renum, bool(fac.value), None

    def state(self):
        nf = C.c_int(0)
        n = self.L.emu_mirror_size(self.h, C.byref(nf))
        flock, layer = np.zeros(n, np.int32), np.zeros(n, np.uint8)
        used, count = np.zeros(nf.value * LAYERS, np.uint8), np.zeros(nf.value * LAYERS, np.uint32)
        self.L.emu_mirror_state(self.h, _p(flock), _p(layer), _p(used), _p(count))
        return flock, layer, used, count


@pytest.mark.parametrize("seed", range(8))
def test_numbering_rule_is_delete_then_append(emu, seed):
    """random removal lists with repeats: survivor rows come from np.delete's order, every old uid maps to its row there
    (removed ones and PFNAV_NULL_UID to PFNAV_NULL_UID), appended entities follow"""
    rng = np.random.default_rng(seed)
    n = int(rng.integers(1, 400))
    a = agents(rng, n, 4)
    M = Mirror(emu, a, 4)
    try:
        rm = rng.integers(0, n, int(rng.integers(0, n + 40)))
        if seed == 0:
            rm = np.arange(n)                           # everything
        add = agents(rng, int(rng.integers(0, 50)), 4)
        n_new, src, renum, _, err = M.batch(rm, add, 4)
        assert err is None
        keep = np.delete(np.arange(n), rm)
        assert n_new == len(keep) + len(add)
        assert np.array_equal(src, keep)
        want = np.full(n + 1, capi.NULL_UID, np.uint32)
        want[keep] = np.arange(len(keep))
        assert np.array_equal(renum, want)
        # the rule the header states: u - |{removed r < u}|
        r = np.unique(rm)
        assert all(want[u] == u - np.searchsorted(r, u) for u in keep)
    finally:
        M.close()


@pytest.mark.parametrize("seed", range(8))
def test_mirror_after_compaction_and_append_equals_a_fresh_mirror(emu, seed):
    """several flocks and layers, removals with repeats, appends into old flocks and into flocks the new table adds, a
    table that grows or drops empty flocks; several batches in a row"""
    rng = np.random.default_rng(100 + seed)
    nf = int(rng.integers(1, 7))
    pop = agents(rng, int(rng.integers(0, 300)), nf)
    M = Mirror(emu, pop, nf)
    try:
        for _ in range(4):
            nf_new = nf + int(rng.integers(-1, 3))
            rm = rng.integers(0, max(len(pop), 1), int(rng.integers(0, len(pop) + 1))) if len(pop) else np.zeros(0, np.int64)
            keep = np.delete(pop, rm)
            if nf_new < nf:                                # drop the last flock: its survivors move, or are removed
                gone = np.nonzero(pop["flock"] >= nf_new)[0]
                rm = np.concatenate([rm, gone])
                keep = np.delete(pop, rm)
            add = agents(rng, int(rng.integers(0, 60)), max(nf_new, 0))
            n_new, _, _, _, err = M.batch(rm, add, max(nf_new, 0))
            assert err is None, err
            nf = max(nf_new, 0)
            pop = np.concatenate([keep, add])
            assert n_new == len(pop)
            F = Mirror(emu, pop, nf)
            try:
                for x, y in zip(M.state(), F.state()):
                    assert np.array_equal(x, y)
            finally:
                F.close()
    finally:
        M.close()


def test_stranding_rule(emu):
    """a table shorter than a flock some survivor or appended entity keeps is refused; removing the last members of the
    dropped flock, or appending into kept flocks only, passes"""
    a = np.zeros(6, capi.AGENT)
    a["radius"], a["flock"] = 1.0, [0, 1, 2, 2, -1, 1]
    M = Mirror(emu, a, 3)
    try:
        add = np.zeros(1, capi.AGENT); add["radius"] = 1.0; add["flock"] = 1
        assert "shorter" in M.batch([2], add, 2, commit=False)[4]        # uid 3 stays in flock 2
        assert M.batch([2, 3, 3], add, 2, commit=False)[4] is None
        add["flock"] = 2
        assert "flock index out of range" in M.batch([2, 3], add, 2, commit=False)[4]
        assert "shorter" in M.batch([], np.zeros(0, capi.AGENT), 1, commit=False)[4]
        n_new, _, _, _, err = M.batch([1, 2, 3, 5], np.zeros(0, capi.AGENT), 1)
        assert err is None and n_new == 2
        flock, _, used, _ = M.state()
        assert list(flock) == [0, -1] and used.reshape(1, LAYERS)[0, 0] == 1
    finally:
        M.close()


def test_validation_names_every_reason(emu):
    rng = np.random.default_rng(3)
    a = agents(rng, 20, 2)
    a["radius"], a["flags"] = 1.0, capi.FLAG_MOVABLE
    add = np.zeros(2, capi.AGENT); add["radius"] = 1.0
    ms, ext = np.zeros(2, capi.MOVESTATE), np.zeros(2, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID
    form, blk = np.zeros(2, capi.FORMATION_IN), np.zeros(2, capi.BLOCKING)
    blk["faction_id"] = 15
    all_t = MS | EXT | FORM | BLK
    M = Mirror(emu, a, 2)

    def why(rm=(), ad=add, tables=all_t, nl=1, nf=2, **kw):
        kw.setdefault("ms", ms); kw.setdefault("blk", blk)
        return M.batch(np.asarray(rm, np.int64), ad, nf, tables=tables, nlayers=nl, commit=False, **kw)[4]

    try:
        assert why() is None
        assert why(ext=ext, form=form) is None
        assert "remove uid outside" in why(rm=[20])
        assert why(rm=[19, 19, 0]) is None
        assert "movestate records for a table" in why(tables=all_t & ~MS)
        assert "movestate_ext records" in why(tables=all_t & ~EXT, ext=ext)
        assert "formation records" in why(tables=all_t & ~FORM, form=form)
        assert "blocking records without" in why(tables=all_t & ~BLK)
        assert "need movestate records" in why(ms=None)
        assert "need blocking records" in why(blk=None)
        assert why(ms=None, blk=None, tables=EXT | FORM) is None
        assert why(ad=np.zeros(0, capi.AGENT), ms=None, blk=None) is None     # nothing appended: no records needed
        bad = add.copy(); bad["flock"][1] = 2
        assert "flock index out of range" in why(ad=bad)
        bad = add.copy(); bad["radius"][0] = 6.0
        assert "navigation layer" in why(ad=bad)
        assert why(ad=bad, nl=2) is None
        bad = add.copy(); bad["flags"][0] = AIR
        assert "navigation layer" in why(ad=bad, nl=8)
        for field, v in (("pos", np.nan), ("velocity", np.inf), ("speed", np.nan), ("vdes", -np.inf)):
            bad = add.copy(); bad[field][0] = v
            assert "agent with a float that is not finite" in why(ad=bad)
        b = ms.copy(); b["vel_hist"][1, 3, 1] = np.nan
        assert "movestate with a float" in why(ms=b)
        e = ext.copy(); e["surround_target_uid"][0] = 22               # 20 - 0 + 2 entities after the call: 0 .. 21
        assert "target outside" in why(ext=e)
        e["surround_target_uid"][0] = 21
        assert why(ext=e) is None
        assert "target outside" in why(ext=e, rm=[0])
        e = ext.copy(); e["rot"][1, 3] = np.nan
        assert "movestate_ext with a float" in why(ext=e)
        f = form.copy(); f["target_orientation"][0, 0] = np.inf
        assert "formation record with a float" in why(form=f)
        b = blk.copy(); b["blocking"][0] = 2
        assert "blocking must be 0 or 1" in why(blk=b)
        b = blk.copy(); b["faction_id"][1] = 16
        assert "faction_id" in why(blk=b)
        b = blk.copy(); b["stop_radius"][1] = np.nan
        assert "blocking record with a float" in why(blk=b)
        # nothing changed by the refusals
        flock, _, _, _ = M.state()
        assert np.array_equal(flock, np.maximum(a["flock"], -1))
    finally:
        M.close()


def test_appended_faction_flag(emu):
    a = np.zeros(3, capi.AGENT); a["radius"] = 1.0; a["flock"] = -1
    M = Mirror(emu, a, 0)
    try:
        add = np.zeros(2, capi.AGENT); add["radius"] = 1.0; add["flock"] = -1
        blk = np.zeros(2, capi.BLOCKING); blk["faction_id"] = 15
        assert M.batch([], add, 0, tables=BLK, blk=blk, commit=False)[3] is False
        blk["faction_id"][1] = 3
        assert M.batch([], add, 0, tables=BLK, blk=blk, commit=False)[3] is True
    finally:
        M.close()
