"""The device source of ClearPath (csrc/pfnav_clearpath_kernel.cuh) run as one warp on CPU threads
(tests/emu/clearpath_emu.cpp) against the plain-C port's clearpath() + vec2_truncate, bit for bit: float32 values compared
with ==, both the single pass (k_agent_velocity<0>) and the two-phase split (phase A's clearpath_collect, phase B's
clearpath_finish, as k_agent_velocity<1> / <2> run them). Each case family asserts that the branch it aims at was taken:
first solves without an admissible velocity, the literal removal schedule on equal distances, the order-dependent tie
replay, the phase-A overflow, a neighbour at the entity's position, the schedule ending after one removal. The inside-VO
test (vo_contains), quot_lt0 and line_isect_s are checked on their own at the edges their shortcuts argue about.
Test infrastructure, not a product path."""
import ctypes as C
import os
import subprocess
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

import clearpath_cases as cc

HERE = os.path.dirname(os.path.abspath(__file__))
F = np.float32
EPS = cc.EPS


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def build_emu(tmp, defines=()):
    so = str(tmp / "libclearpath_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-ffp-contract=off", "-fno-strict-aliasing", "-fPIC", "-shared", "-pthread",
                    *defines, os.path.join(HERE, "emu", "clearpath_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    L.emu_clearpath_batch.argtypes = [C.c_int] + [C.c_void_p] * 6 + [C.c_int] + [C.c_void_p] * 4
    L.emu_clearpath.argtypes = [C.c_void_p] * 3 + [C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_float, C.c_void_p, C.c_void_p,
                                                   C.c_void_p]
    L.emu_vo_contains.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p]
    L.emu_quot_lt0.argtypes = [C.c_void_p, C.c_void_p, C.c_long, C.c_void_p]
    L.emu_line_isect_s.argtypes = [C.c_void_p, C.c_long, C.c_void_p]
    L.emu_retry_better.argtypes = [C.c_int, C.c_float, C.c_float, C.c_float, C.c_int, C.c_float, C.c_int, C.c_float, C.c_float,
                                   C.c_void_p]
    return L


@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    return build_emu(tmp_path_factory.mktemp("clearpath_emu"))


def run_emu(L, cs, mode, workers=8, chunk=16):
    """-> (vel [n][2], stats [n][4], info [n][4]) of every case; chunks of cases run as concurrent warps"""
    n = len(cs)
    out = np.zeros((n, 2), F)
    stats = np.zeros((n, 4), np.uint64)
    info = np.zeros((n, 4), np.int32)
    arrs = [np.ascontiguousarray(a) for a in (cs.self5, cs.vpref, cs.dyn, cs.ndyn, cs.stat, cs.nstat, cs.max_len)]

    def one(lo):
        hi = min(n, lo + chunk)
        s5, vp, dy, nd, st, ns, ml = (a[lo:hi] for a in arrs)
        r = L.emu_clearpath_batch(hi - lo, _p(s5), _p(vp), _p(dy), _p(nd), _p(st), _p(ns), mode, _p(ml), _p(out[lo:hi]),
                                  _p(stats[lo:hi]), _p(info[lo:hi]))
        assert r == 0

    with ThreadPoolExecutor(workers) as ex:
        list(ex.map(one, range(0, n, chunk)))
    return out, stats, info


def run_port(pforacle, cs):
    return np.stack([pforacle.clearpath(*cs.case(i)[:4], cs.max_len[i]) for i in range(len(cs))]) if len(cs) else np.zeros((0, 2), F)


def bits_equal(a, b):
    """float32 arrays equal value for value, no NaN anywhere (+0 == -0 as the kernel's == would have it)"""
    a, b = np.asarray(a, F), np.asarray(b, F)
    return not np.isnan(a).any() and not np.isnan(b).any() and bool((a == b).all())


def compare_family(emu, pforacle, name, n, seed):
    """runs family `name` in both modes against the port; -> (cases, stats, info) of mode 0 and the counts to report"""
    rng = np.random.default_rng(seed)
    cs = cc.FAMILIES[name](rng, n)
    t0 = time.time()
    want = run_port(pforacle, cs)
    v0, s0, i0 = run_emu(emu, cs, 0)
    v2, s2, i2 = run_emu(emu, cs, 2)
    bad0 = [i for i in range(n) if not bits_equal(v0[i], want[i])]
    bad2 = [i for i in range(n) if not bits_equal(v2[i], want[i])]
    assert not bad0, "%s mode 0: %d of %d differ, first %d: emu %r port %r" % (name, len(bad0), n, bad0[0], v0[bad0[0]], want[bad0[0]])
    assert not bad2, "%s mode 2: %d of %d differ, first %d: emu %r port %r" % (name, len(bad2), n, bad2[0], v2[bad2[0]], want[bad2[0]])
    # phase B reaches the same first-solve outcome; it takes the retry path exactly where the single pass does
    assert (s0[:, :2] == s2[:, :2]).all()
    counts = branch_counts(cs, s0, i0, i2)
    print("\n[clearpath %s] %d cases, %.1f s: %s" % (name, n, time.time() - t0, counts))
    return cs, s0, i0, i2, counts


def branch_counts(cs, s0, i0, i2):
    n = len(cs)
    fail = s0[:, 0] > 0
    both = s0[:, 1] > 0
    return {
        "first_solve_failed": int(fail.sum()),
        "both_lists": int(both.sum()),
        "literal_schedule": int(sum(1 for i in range(n) if both[i] and cc.has_distance_tie(cs, i)
                                    and not cc.ends_after_first_removal(cs, i))),
        "tie_replay": int((s0[:, 2] > 0).sum()),
        "replay_solves": int(s0[:, 3].sum()),
        "overflow": int((i2[:, 3] > 64).sum()),
        "same_position": int(sum(1 for i in range(n) if cc.same_position(cs, i))),
        "ends_after_first_removal": int(sum(1 for i in range(n) if fail[i] and cc.ends_after_first_removal(cs, i))),
    }


def test_clearpath_random_sets(emu, pforacle):
    """every (ndyn, nstat) pair of {0, 1, 2, 5, 31, 32}, map-sized coordinates"""
    _, _, _, _, c = compare_family(emu, pforacle, "random", 36 * 60, 0xC1EA0)
    assert c["first_solve_failed"] > 0 and c["both_lists"] > 0


def test_clearpath_forced_retries(emu, pforacle):
    cs, s0, _, _, c = compare_family(emu, pforacle, "forced_retries", 600, 0xC1EA1)
    assert c["both_lists"] > 0.5 * len(cs)              # most first solves fail with both lists non-empty


def test_clearpath_equal_distances(emu, pforacle):
    """bit-equal float distances: retry_schedule_fast falls back to the literal schedule"""
    cs, _, _, _, c = compare_family(emu, pforacle, "equal_distances", 600, 0xC1EA2)
    assert c["literal_schedule"] > 0.1 * len(cs)


def test_clearpath_point_ties(emu, pforacle):
    """mirror-symmetric cases: two different points at the same (time, distance) -> exact = false, literal replay"""
    _, _, _, _, c = compare_family(emu, pforacle, "point_ties", 800, 0xC1EA3)
    assert c["tie_replay"] > 0 and c["replay_solves"] > 0


def test_clearpath_degenerate_neighbours(emu, pforacle):
    cs, s0, i0, _, c = compare_family(emu, pforacle, "degenerate_neighbours", 400, 0xC1EA4)
    assert c["same_position"] == len(cs)
    # the neighbours closer than EPS build no obstacle, yet keep their place in the removal schedule
    assert (i0[:, 2] < 2 * (cs.ndyn + cs.nstat)).all()
    assert c["both_lists"] > 0.15 * len(cs)


def test_clearpath_early_end(emu, pforacle):
    cs, s0, _, _, c = compare_family(emu, pforacle, "early_end", 450, 0xC1EA5)
    fail = s0[:, 0] > 0
    one_empty = (cs.ndyn == 0) | (cs.nstat == 0)
    assert (fail & one_empty).sum() > 10                                 # no second solve at all
    assert (fail & ~one_empty).sum() > 0 and c["ends_after_first_removal"] >= (fail & one_empty).sum() + 1


def test_clearpath_degenerate_geometry(emu, pforacle):
    cs, _, _, _, c = compare_family(emu, pforacle, "degenerate_geometry", 1000, 0xC1EA6)
    assert c["first_solve_failed"] > 0
    assert (cs.self5[:, 2:4] == 0).all(axis=1).sum() > 0 and (cs.vpref == 0).all(axis=1).sum() > 0
    # near-vertical edges: some ray of the cases has |dir.x| < EPS (line_slope's NaN)
    assert _vertical_edges(cs) > 0


def _vertical_edges(cs):
    k = 0
    for i in range(len(cs)):
        p = cs.self5[i, :2]
        r = cs.self5[i, 4]
        for nb in np.concatenate([cs.dyn[i, :cs.ndyn[i]], cs.stat[i, :cs.nstat[i]]]):
            d = (nb[:2] - p).astype(F)
            ln = np.sqrt(F(d[0] * d[0] + d[1] * d[1]))
            if ln < EPS:
                continue
            e = (d / ln).astype(F)
            rr = (np.array([-e[1], e[0]], F) * F(nb[4] + r + F(0))).astype(F)
            for t in ((nb[:2] + rr).astype(F), (nb[:2] - rr).astype(F)):
                q = (t - p).astype(F)
                ql = np.sqrt(F(q[0] * q[0] + q[1] * q[1]))
                k += abs(F(q[0] / ql)) < EPS
    return k


def test_clearpath_overflow(emu, pforacle):
    """32 + 32 neighbours: phase A keeps at most 64 admissible intersections; beyond that phase B solves in full"""
    cs, _, _, i2, c = compare_family(emu, pforacle, "overflow", 160, 0xC1EA7)
    assert c["overflow"] > 0 and c["overflow"] < len(cs)


def test_clearpath_single_case_entry(emu, pforacle):
    """emu_clearpath (one case, the counters accumulated) agrees with the batch entry"""
    cs = cc.FAMILIES["forced_retries"](np.random.default_rng(5), 8)
    vb, sb, ib = run_emu(emu, cs, 0)
    acc = np.zeros(8, np.uint64)
    for i in range(len(cs)):
        s5, vp, dy, st, ml = cs.case(i)
        out = np.zeros(2, F)
        info = np.zeros(4, np.int32)
        dy, st = np.ascontiguousarray(dy), np.ascontiguousarray(st)
        assert emu.emu_clearpath(_p(s5), _p(vp), _p(dy), len(dy), _p(st), len(st), 0, float(ml), _p(out), _p(acc), _p(info)) == 0
        assert bits_equal(out, vb[i]) and (info == ib[i]).all()
    assert (acc[:4] == sb.sum(axis=0)).all()


# ---- the pieces on their own ----
def _cone(rng):
    """one obstacle: apex and two unit edge directions 10-120 degrees apart"""
    apex = np.array([-rng.uniform(10, 4000), rng.uniform(10, 4000)])
    a = rng.uniform(0, 2 * np.pi)
    w = rng.uniform(np.radians(10), np.radians(120))
    right = np.array([np.cos(a), np.sin(a)])
    left = np.array([np.cos(a + w), np.sin(a + w)])
    return (apex, left, right) if rng.random() < 0.5 else (apex, right, left)     # either orientation


def _rot(d, s):
    """d rotated so that the normalised cross (n.z d.x - n.x d.z) is -s; i.e. by angle -asin(s)"""
    c = np.sqrt(1 - s * s)
    return np.stack([d[0] * c + d[1] * s, -d[0] * s + d[1] * c], axis=-1)


def test_vo_contains_thresholds(emu, pforacle):
    """points whose normalised determinant against either edge lies in [0.98, 1.02] * EPS (both signs), and points at
    |p - apex| in [0.98, 1.02] * EPS: the fast path's 1 % margins must never decide differently from inside_pcr"""
    rng = np.random.default_rng(0x70C)
    total = inside = 0
    for _ in range(200):
        apex, left, right = _cone(rng)
        rays = np.array([[apex[0], apex[1], *left], [apex[0], apex[1], *right]], F)
        rays[:, 2:] = rays[:, 2:] / np.sqrt((rays[:, 2:] ** 2).sum(axis=1, keepdims=True))
        m = 4000
        # half of them within 3e-4 of the threshold, where the unnormalised cross product's cancellation error matters
        band = np.where(rng.random(m) < 0.5, rng.uniform(0.98, 1.02, m), 1.0 + rng.uniform(-3e-4, 3e-4, m))
        s = band * float(EPS) * rng.choice([-1.0, 1.0], m)
        dist = np.exp(rng.uniform(np.log(2e-3), np.log(30.0), m))
        pts = []
        for d in (left, right):          # near each edge, at the threshold angle
            pts.append(apex + _rot(d, s) * dist[:, None])
        u = rng.uniform(0, 2 * np.pi, m)  # near the apex, at the threshold distance
        pts.append(apex + np.stack([np.cos(u), np.sin(u)], 1) * (rng.uniform(0.98, 1.02, m) * float(EPS))[:, None])
        mid = (left + right) / np.linalg.norm(left + right)  # and along the centreline, close to the apex
        pts.append(apex + mid * (rng.uniform(0.98, 1.02, m) * float(EPS))[:, None])
        pts = np.ascontiguousarray(np.concatenate(pts), F)
        got = np.zeros(len(pts), np.uint8)
        emu.emu_vo_contains(_p(np.ascontiguousarray(rays)), _p(pts), len(pts), _p(got))
        want = pforacle.inside_pcr(rays, pts)
        bad = np.nonzero(got.astype(bool) != want)[0]
        assert not len(bad), "vo_contains differs from inside_pcr at %r (rays %r)" % (pts[bad[0]], rays)
        total += len(pts)
        inside += int(want.sum())
    print("\n[vo_contains] %d points, %d inside" % (total, inside))
    assert total >= 2_000_000 and 0.02 * total < inside < 0.98 * total


def test_retry_better_order(emu):
    """retry_better: strict (time, distance) order; an equal (time, distance) never replaces the best, and flags a tie only
    between two different points when a best exists"""
    cases_ = [  # (T, dist, px, pz, best T, dist, id, px, pz) -> (better, tie)
        ((1, 2.0, 0.0, 0.0, 2, 1.0, 5, 0.0, 0.0), (1, 0)),
        ((3, 0.5, 0.0, 0.0, 2, 1.0, 5, 0.0, 0.0), (0, 0)),
        ((2, 0.5, 0.0, 0.0, 2, 1.0, 5, 0.0, 0.0), (1, 0)),
        ((2, 1.5, 0.0, 0.0, 2, 1.0, 5, 0.0, 0.0), (0, 0)),
        ((2, 1.0, 0.25, 0.0, 2, 1.0, 5, 0.0, 0.0), (0, 1)),       # same time and distance, another point: tie
        ((2, 1.0, 0.0, 0.0, 2, 1.0, 5, 0.0, 0.0), (0, 0)),        # the same point again: no tie
        ((2, 1.0, 0.25, 0.0, 2, 1.0, -1, 0.0, 0.0), (0, 0)),      # no best yet
    ]
    for args, want in cases_:
        out = np.zeros(2, np.int32)
        emu.emu_retry_better(*[C.c_int(int(v)) if k in (0, 4, 6) else C.c_float(v) for k, v in enumerate(args)], _p(out))
        assert tuple(out) == want, (args, tuple(out), want)


def _specials():
    dmin = np.array([1], np.uint32).view(F)[0]
    v = [0.0, -0.0, dmin, -dmin, np.float32(1e-40), np.float32(-1e-40), np.finfo(F).tiny, -np.finfo(F).tiny, 1.0, -1.0,
         np.nextafter(F(1), F(2)), -np.nextafter(F(1), F(2)), np.float32(0.5), np.float32(-0.5), np.inf, -np.inf, np.nan,
         -np.nan, np.finfo(F).max, -np.finfo(F).max]
    return np.array(v, F)


def test_quot_lt0_vs_division(emu):
    """quot_lt0(a, b) == (a / b < 0.0f) for |b| <= 1 + 4 ulp: signed zeros, denormals, infinities, NaN, dense values"""
    rng = np.random.default_rng(0x9107)
    sp = _specials()
    bsp = sp[(np.abs(sp) <= np.nextafter(F(1), F(2)) * F(1 + 4 * 2 ** -23)) | np.isnan(sp)]
    a1, b1 = np.meshgrid(sp, bsp)
    n = 2_000_000
    a_bits = rng.integers(0, 2 ** 32, n, dtype=np.uint64).astype(np.uint32).view(F)          # every float class
    b = rng.uniform(-1.0, 1.0, n).astype(F) * np.where(rng.random(n) < 0.3, F(2 ** -100), F(1)).astype(F)
    b = np.where(rng.random(n) < 0.05, np.array([1], np.uint32).view(F)[0] * rng.integers(1, 9, n).astype(F), b).astype(F)
    ulp = np.array([0x3F800000 + k for k in range(5)], np.uint32).view(F)
    b_edge = np.concatenate([ulp, -ulp])
    a = np.ascontiguousarray(np.concatenate([a1.ravel(), a_bits, rng.standard_normal(len(b_edge) * 1000).astype(F)]), F)
    b = np.ascontiguousarray(np.concatenate([b1.ravel(), b, np.repeat(b_edge, 1000)]), F)
    got = np.zeros(len(a), np.uint8)
    emu.emu_quot_lt0(_p(a), _p(b), len(a), _p(got))
    with np.errstate(all="ignore"):
        want = (a / b) < F(0)
    bad = np.nonzero(got.astype(bool) != want)[0]
    assert not len(bad), "quot_lt0(%r, %r) = %d, a / b = %r" % (a[bad[0]], b[bad[0]], got[bad[0]], a[bad[0]] / b[bad[0]])
    assert want.sum() > 0.3 * len(a)


def test_line_isect_s_vs_port(emu, pforacle):
    """line_isect_s (slopes precomputed by line_slope) against C_InfiniteLineIntersection: random lines, (near-)vertical
    ones on either side (the preserved l2.point expression), parallel and identical slopes"""
    rng = np.random.default_rng(0x11E)
    n = 200_000
    pts = np.stack([-rng.uniform(10, 4000, (n, 2)), rng.uniform(10, 4000, (n, 2))], axis=-1)
    ang = rng.uniform(0, 2 * np.pi, (n, 2))
    kind = rng.integers(0, 5, n)
    ang[kind == 1, 0] = np.pi / 2 + rng.uniform(-1.5, 1.5, (kind == 1).sum()) * float(EPS)     # l1 near-vertical
    ang[kind == 2, 1] = -np.pi / 2 + rng.uniform(-1.5, 1.5, (kind == 2).sum()) * float(EPS)    # l2 near-vertical
    ang[kind == 3, 1] = ang[kind == 3, 0] + rng.uniform(-2e-3, 2e-3, (kind == 3).sum())         # (near-)parallel
    ang[kind == 4, 1] = ang[kind == 4, 0] + np.pi
    lines = np.zeros((n, 2, 4), F)
    lines[:, :, :2] = pts
    lines[:, :, 2] = np.cos(ang)
    lines[:, :, 3] = np.sin(ang)
    lines = np.ascontiguousarray(lines)
    got = np.zeros((n, 3), F)
    emu.emu_line_isect_s(_p(lines), n, _p(got))
    want = pforacle.line_isect(lines)
    ok = want[:, 0] == 1
    assert (got[:, 0] == want[:, 0]).all()
    with np.errstate(invalid="ignore"):
        same = (got[ok, 1:] == want[ok, 1:]) | (np.isnan(got[ok, 1:]) & np.isnan(want[ok, 1:]))
    assert same.all()
    assert 0 < (~ok).sum() < n and ok[kind == 1].any() and ok[kind == 2].any()
