"""The device source of pfnav_ents_in_circles (csrc/pfnav_ents_query_kernel.cuh: the index walk, the count pass and the
write pass) run as one warp on CPU threads (tests/emu/ents_query_emu.cpp) against the plain-C port's pfo_ents_in_circle
(oracle/pf_oracle.c, pinned to the reference's golden q10 / q30 lists by tests/test_oracle.py): every query's uids, in
the same order, for point and uid centres, every walk (off the grid, wide, the int32 "small" path up to 46.875 wu, the
int64 path above it), the cut at maxout and filter_garrisoned's swap-remove. Each family asserts that the branch it targets
was taken. Test infrastructure, not a product path."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
NULL = capi.NULL_UID
NO_WALK, WALK_OFF, WALK_WIDE, WALK_SMALL, WALK_LARGE = -1, 0, 1, 2, 3
SMALL_MAX = 46.875                                  # ir = 12000: the last range of the int32 path


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libents_query_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-strict-aliasing", "-fPIC", "-shared", "-pthread",
                    os.path.join(HERE, "emu", "ents_query_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_ents_query.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_int, C.c_int, C.c_float, C.c_float, C.c_void_p,
                                 C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p, C.c_void_p]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class World:
    """a population on a cw x cw map, in the port and as the records the device holds"""

    def __init__(self, pforacle, cw, n, seed, garrisoned=0.0, spacing=2.6):
        _, cost, a = cases.agent_case(cw, n, 3, seed, 0.03, spacing)
        rng = np.random.default_rng(seed + 17)
        if garrisoned:
            a["flags"] = a["flags"] | np.where(rng.random(len(a["radius"])) < garrisoned, capi.FLAG_GARRISONED, 0).astype(a["flags"].dtype)
        self.rec, fl = capi.pack_agents(a)
        self.cw, self.n = cw, len(self.rec)
        self.pos = np.ascontiguousarray(self.rec["pos"], np.float32)
        self.sf = ((self.rec["state"].astype(np.uint32) << 24) | (self.rec["flags"].astype(np.uint32) & 0xFFFFFF)).astype(np.uint32)
        self.garr = bool((self.rec["flags"] & capi.FLAG_GARRISONED).any())
        self.port = pforacle.OracleWorld(pforacle.OracleMap(cw, cw, cost), self.rec, fl, 20)

    def close(self):
        self.port.close()

    def run(self, emu, q, filter_garr=None):
        """filter_garr=0: the raw cut, without filter_garrisoned"""
        q = np.ascontiguousarray(q, capi.ENTS_QUERY)
        nq = len(q)
        cap = int(np.minimum(np.maximum(q["maxout"], 0), self.n).sum()) + 1
        off, ids = np.zeros(nq + 1, np.uint32), np.zeros(cap, np.uint32)
        raw, walk, scr = np.zeros(nq, np.uint32), np.zeros(nq, np.int32), np.zeros(nq, np.uint32)
        assert emu.emu_ents_query(_p(self.pos), _p(self.sf), self.n, self.cw, self.cw, 0.0, 0.0, _p(q), nq,
                                  int(self.garr if filter_garr is None else filter_garr),
                                  _p(off), _p(ids), cap, _p(raw), _p(walk), _p(scr)) == 0
        return [ids[off[i]:off[i + 1]] for i in range(nq)], raw, walk, scr

    def expected(self, q):
        out = []
        for r in q:
            x, z = (float(r["x"]), float(r["z"])) if r["uid"] == NULL else map(float, self.pos[r["uid"]])
            out.append(self.port.ents_in_circle(x, z, float(r["range"]), int(r["maxout"])))
        return out

    def check(self, emu, q):
        got, raw, walk, scr = self.run(emu, q)
        want = self.expected(q)
        bad = [(i, tuple(q[i]), got[i][:8], want[i][:8]) for i in range(len(q))
               if len(got[i]) != len(want[i]) or (got[i] != want[i]).any()]
        assert not bad, (len(bad), bad[:3])
        return got, raw, walk, scr


def queries(rows):
    q = np.zeros(len(rows), capi.ENTS_QUERY)
    for i, (x, z, r, uid, maxout) in enumerate(rows):
        q[i] = (x, z, r, uid, maxout, 0)
    return q


@pytest.fixture(scope="module")
def worlds(pforacle):
    ws = {"plain": World(pforacle, 3, 1500, 3131), "dense": World(pforacle, 1, 600, 77, spacing=2.1),
          "garrisoned": World(pforacle, 3, 1500, 4242, garrisoned=0.15)}
    yield ws
    for w in ws.values():
        w.close()


RANGES = (0.0, 1.5, 10.0, 30.0, SMALL_MAX, SMALL_MAX + 1.0 / 256, 47.0)


@pytest.mark.parametrize("name", ["plain", "dense", "garrisoned"])
def test_point_and_uid_centres_every_range(emu, worlds, name):
    """an entity's own position as a point and as a uid, random points, every range family; maxout 512"""
    w = worlds[name]
    rng = np.random.default_rng(5)
    rows = []
    for u in rng.choice(w.n, 60, replace=False):
        for r in RANGES:
            rows.append((w.pos[u, 0], w.pos[u, 1], r, NULL, 512))
            rows.append((0.0, 0.0, r, int(u), 512))
    span = w.cw * 256.0
    for x, z in zip(-rng.uniform(0, span, 40), rng.uniform(0, span, 40)):
        for r in (10.0, 30.0):
            rows.append((x, z, r, NULL, 512))
    q = queries(rows)
    got, raw, walk, _ = w.check(emu, q)
    small = q["range"] <= SMALL_MAX
    assert (walk[small] == WALK_SMALL).all() and (walk[~small] == WALK_LARGE).all()
    at_ent = np.arange(len(q)) < 60 * len(RANGES) * 2
    assert (raw[at_ent] >= 1).all(), "a query centred on an entity finds at least that entity"
    assert (raw[at_ent & (q["range"] >= 10.0)] > 1).mean() > 0.9
    uidq = q["uid"] != NULL
    assert all((got[i] == got[i - 1]).all() for i in np.nonzero(uidq)[0]), "a uid centre is that entity's point"


def test_wide_queries(emu, worlds):
    """extents covering at least 3/4 of the cells take the pool-order path: the whole index in cell order"""
    w = worlds["plain"]
    span = w.cw * 256.0
    rows = [(-span / 2, span / 2, r, NULL, m) for r in (0.45 * span, 0.75 * span, 2.0 * span) for m in (32, 512, 5000)]
    rows += [(0.0, 0.0, 0.8 * span, u, 512) for u in (0, 7, w.n - 1)]
    q = queries(rows)
    got, raw, walk, _ = w.check(emu, q)
    assert (walk == WALK_WIDE).all()
    assert len(got[8]) == w.n, "a 5000-uid cut of a query covering the map holds everybody"


def test_off_grid_negative_range_maxout_zero(emu, worlds):
    w = worlds["plain"]
    span = w.cw * 256.0
    rows = [(300.0, 300.0, 10.0, NULL, 512),                 # east of the map (x decreases across it)
            (-span / 2, -200.0, 30.0, NULL, 512),            # south of it
            (-span - 100.0, span + 100.0, 46.0, NULL, 512),  # beyond the far corner
            (20.0, w.pos[0, 1] + 0.0, 30.0, NULL, 512),      # off the grid, but the circle reaches into it
            (w.pos[0, 0], w.pos[0, 1], -1.0, NULL, 512), (0.0, 0.0, -0.001, 3, 512),
            (w.pos[0, 0], w.pos[0, 1], 30.0, NULL, 0), (0.0, 0.0, 30.0, 3, 0)]
    q = queries(rows)
    got, raw, walk, _ = w.check(emu, q)
    assert list(walk[:3]) == [WALK_OFF] * 3 and walk[3] == WALK_SMALL
    assert list(walk[4:]) == [NO_WALK] * 4
    assert all(len(g) == 0 for i, g in enumerate(got) if i != 3)


@pytest.mark.parametrize("name", ["dense", "garrisoned"])
def test_cut_at_maxout(emu, worlds, name):
    """maxout 0, 1, 32, 512, and below the raw hit count: the raw list is cut there, in walk order"""
    w = worlds[name]
    rng = np.random.default_rng(9)
    rows = [(0.0, 0.0, r, int(u), m) for u in rng.choice(w.n, 50, replace=False) for r in (10.0, 30.0, 60.0)
            for m in (0, 1, 3, 32, 512)]
    q = queries(rows)
    got, raw, walk, _ = w.check(emu, q)
    full = w.run(emu, queries([(0.0, 0.0, float(r["range"]), int(r["uid"]), 1 << 20) for r in q]))[1]
    cut = (q["maxout"] > 0) & (full > q["maxout"])
    assert cut.sum() > 100 and (raw[cut] == q["maxout"][cut]).all()
    assert (raw[~cut] == np.minimum(full[~cut], q["maxout"][~cut])).all()


def test_garrisoned_swap_remove(emu, worlds):
    """GARRISONED entities inside the cut: the write pass builds the raw cut in its scratch and filter_garrisoned
    reorders the survivors; queries without one inside the cut write straight to their answer"""
    w = worlds["garrisoned"]
    rng = np.random.default_rng(13)
    rows = [(0.0, 0.0, r, int(u), m) for u in rng.choice(w.n, 150, replace=False) for r in (10.0, 30.0) for m in (8, 32, 512)]
    q = queries(rows)
    got, raw, walk, scr = w.check(emu, q)
    used = scr > 0
    assert used.sum() > 50 and (~used).sum() > 10
    assert (scr[used] == raw[used]).all() and all(len(got[i]) < raw[i] for i in np.nonzero(used)[0])
    # the swap-remove moved survivors: the answer is not the in-order filtered cut
    raw_lists = w.run(emu, q, filter_garr=0)[0]
    garr = (w.sf & capi.FLAG_GARRISONED) != 0
    assert all(len(raw_lists[i]) == raw[i] for i in range(len(q)))
    reordered = sum(1 for i in np.nonzero(used)[0] if not np.array_equal(got[i], raw_lists[i][~garr[raw_lists[i]]]))
    assert reordered > 20
