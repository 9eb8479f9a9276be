"""GPU suite: pfnav_pool_request_paths_resident, pfnav_map_query_resident and pfnav_group_arrival_velocity_resident, the
path requests, map queries and group-arrival velocities whose positions name resident entities by uid.

Twin contexts: twin A reads the records back (pfnav_agents_read_state), substitutes the named positions in numpy and
calls the plain entry point; twin B makes the resident call. Both must end with the same outputs, return code and ndone,
the same pool entries (has bits, ff_id, flow and LOS bytes), and for paths the same vdes and velocities after a tick, bit
for bit. The resident loop (stale records refused until the index is rebuilt) and group members resolving uids owned by
another member are checked the same way."""
import ctypes as C

import numpy as np
import pytest

import cases
from test_gpu_mgpu_commands import Job, _population
from test_gpu_request_paths import _blocker_ops, _map, _nav, _pool, _requests

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
NULL = capi.NULL_UID
OFF = np.float32(1e9)           # a given value at a named entry: off the map, so a missed substitution cannot pass


def _agents(points, dest, target):
    """one MOVING flock at the given positions, heading for `target` through pool destination `dest`"""
    n = len(points)
    rec = np.zeros(n, capi.AGENT)
    rec["pos"] = points; rec["prev_pos"] = points
    rec["radius"] = 1.0; rec["max_speed"] = 20.0; rec["speed"] = 20.0
    rec["flags"] = capi.FLAG_MOVABLE; rec["flock"] = 0
    fl = np.zeros(1, capi.FLOCK); fl["target"] = target; fl["dest"] = dest
    return rec, fl


def _substitute(nav, n, uids, given):
    """twin A: the named entries' positions from the records read back, the rest as given"""
    pos = nav.agents_read_state(n, False)[0]["pos"]
    out = np.zeros((len(uids), 2), np.float32) if given is None else np.array(given, np.float32).reshape(-1, 2)
    named = uids != NULL
    out[named] = pos[uids[named]]
    return out


def _masked(given, uids):
    """twin B's given array: OFF wherever the entry names a uid"""
    g = np.array(given, np.float32).reshape(-1, 2)
    g[uids != NULL] = OFF
    return g


def _paths_raw(nav, dests, su, sx, du, dx):
    """the resident call without exceptions -> rc, ok, did, nf, nl, ndone"""
    n = len(dests)
    outs = [np.full(n, 77, np.int32), np.full(n, 77, np.uint32), np.full(n, 77, np.int32), np.full(n, 77, np.int32)]
    nd = C.c_int(-1)
    ptr = lambda a: None if a is None or not len(a) else capi._p(np.ascontiguousarray(a))
    rc = nav.L.pfnav_pool_request_paths_resident(nav.h, n, ptr(dests), 0, ptr(su), ptr(sx), ptr(du), ptr(dx), None,
                                                 capi._p(outs[1]), capi._p(outs[0]), capi._p(outs[2]), capi._p(outs[3]),
                                                 C.byref(nd))
    return (rc,) + tuple(outs) + (nd.value,)


def _tick_compare(navs, nwork):
    out = []
    for nav in navs:
        nav.agents_set_work(np.arange(nwork, dtype=np.uint32))
        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        out.append((nav.agents_read_debug(nwork)[1], nav.agents_read_velocities(nwork)))
    assert out[0][0].tobytes() == out[1][0].tobytes(), "vdes"
    assert out[0][1].tobytes() == out[1][1].tobytes(), "velocities"


def _paths_twins(cw, ch, seed, nblockers, n, ndests, pool_max, faction=None, c2=False, npop=3000, p_src=0.6, p_dst=0.3,
                 all_src=False, expect_nomem=False, warm=8):
    cost = _map(cw, ch, seed, c2)
    ops = _blocker_ops(cw, ch, nblockers, seed + 1) if nblockers else None
    navs = [_nav(cost, cw, ch, ops, ndests, pool_max) for _ in range(2)]
    try:
        dests, src, dst = _requests(cost, cw, ch, n + warm + npop, ndests, seed + 2)
        rng = np.random.default_rng(seed + 3)
        # the population stands on request endpoints of all kinds (blocked tiles and other islands included)
        points = np.concatenate([src[n + warm:], dst[n + warm:]])[rng.permutation(2 * npop)[:npop]]
        rec, fl = _agents(points, int(dests[0]), dst[0])
        for nav in navs:
            if faction is not None:                   # attacking requests: blockers of factions 0 and 5 are enemies
                nav.set_enemy_factions(faction, (1 << 0) | (1 << 5))
                nav.request_faction(faction)
            for i in range(warm):
                nav.pool_request_path(int(dests[i]), tuple(src[i]), tuple(dst[i]))
            nav.agents_upload(rec, fl, 20)
        dests, src, dst = dests[warm:warm + n], src[warm:warm + n], dst[warm:warm + n]
        su = rng.integers(0, npop, n).astype(np.uint32)
        if not all_src:
            su[rng.random(n) >= p_src] = NULL
        du = rng.integers(0, npop, n).astype(np.uint32)
        du[rng.random(n) >= p_dst] = NULL          # attack / follow targets by uid, the rest at points
        a = navs[0].pool_request_paths(dests, _substitute(navs[0], npop, su, None if all_src else src),
                                       _substitute(navs[0], npop, du, dst))
        b = navs[1].pool_request_paths_resident(dests, su, None if all_src else _masked(src, su), du, _masked(dst, du))
        assert a[4] == b[4] and (a[4] < n) == expect_nomem, (a[4], b[4], n)
        for x, y in zip(a[:4], b[:4]):
            assert np.array_equal(x, y)
        assert _pool(navs[0], ndests, cw * ch) == _pool(navs[1], ndests, cw * ch)
        if not expect_nomem:
            assert a[0].any() and a[2].sum() > 0
        _tick_compare(navs, npop)
    finally:
        for nav in navs:
            nav.close()


@pytest.mark.parametrize("cw,ch,seed,nblockers,n,ndests,pool_max,faction", [
    (4, 4, 12, 300, 96, 12, 12 * 16, 3),      # an attacking faction, repeated dests
    (8, 8, 31, 200, 120, 12, 40, None),       # a pool far smaller than the batch: evictions inside it
    (8, 8, 13, 800, 300, 16, 16 * 64, None),  # blockers on a larger map, 300 requests
])
def test_paths_resident_vs_plain(cw, ch, seed, nblockers, n, ndests, pool_max, faction):
    _paths_twins(cw, ch, seed, nblockers, n, ndests, pool_max, faction=faction)


def test_paths_nomem_stop():
    """a request needing more fields than the pool holds stops both twins at the same request, pools equal"""
    _paths_twins(8, 8, 41, 0, 80, 6, 6, expect_nomem=True, warm=0)


def test_paths_c2_sized():
    """4096 requests whose sources are random uids of a C2-sized population (100 000 entities), with NULL src_xz: search
    rounds large enough for the portal-graph searches to run on the device"""
    _paths_twins(16, 16, 21, 800, 4096, 48, 48 * 256, c2=True, npop=100000, all_src=True, p_dst=0.5)


def test_paths_arguments():
    """argument errors and an endpoint resolved off the map change nothing; n == 0 and no uid arrays are the plain call"""
    cw = ch = 4
    ndests = 4
    cost = _map(cw, ch, 51)
    nav = _nav(cost, cw, ch, None, ndests, 64)
    try:
        dests, src, dst = _requests(cost, cw, ch, 16, ndests, 52)
        pts = src.copy()
        pts[3] = (1.0, -5.0)                                  # an entity off the map box
        rec, fl = _agents(pts, 0, dst[0])
        nav.agents_upload(rec, fl, 20)
        before, launches = _pool(nav, ndests, 16), nav.launch_count()
        u = np.arange(16, dtype=np.uint32)
        bad = [(u, None, None, None),                         # dst_xz NULL, no dst uids
               (np.where(u == 5, NULL, u).astype(np.uint32), None, None, dst),   # src_xz NULL, an entry unnamed
               (np.where(u == 5, 16, u).astype(np.uint32), src, None, dst),      # uid == population
               (u, src, np.where(u == 2, 1 << 30, u).astype(np.uint32), dst),    # dst uid far outside
               (np.where(u == 3, 3, NULL).astype(np.uint32), src, None, dst)]    # resolves off the map
        for i, (su, sx, du, dx) in enumerate(bad):
            r = _paths_raw(nav, dests, su, sx, du, dx)
            assert r[0] == capi.ERR_ARG and r[5] == 0, i
            assert all((o == 77).all() for o in r[1:5]), i
            assert nav.launch_count() == launches + (i == 4), i     # only the last one resolves its uids
        assert _pool(nav, ndests, 16) == before
        assert _paths_raw(nav, dests[:0], None, None, None, None)[0] == 0
        assert nav.L.pfnav_pool_request_paths_resident(nav.h, -1, None, 0, None, None, None, None, None, None, None, None,
                                                       None, None) == capi.ERR_ARG
        # no uid arrays: the plain call
        r = _paths_raw(nav, dests, None, src, None, dst)
        assert r[0] == 0 and r[5] == 16
    finally:
        nav.close()
    host = capi.Nav(hostonly=True)
    try:
        assert _paths_raw(host, dests[:1], np.zeros(1, np.uint32), None, None, dst[:1])[0] == capi.ERR_ARG
    finally:
        host.close()


# ---- map queries

def _queries(rng, n, nlayers, cw, ch):
    """all six kinds on random layers and points over (and a little beyond) the map; DEST_ID plain and attacking"""
    W, H = cw * 256.0, ch * 256.0
    q = np.zeros(n, capi.MAP_QUERY)
    q["kind"] = rng.integers(0, 6, n)
    q["layer"] = rng.integers(0, nlayers, n)
    q["x"], q["z"] = rng.uniform(-W - 4, 4, n), rng.uniform(-4, H + 4, n)
    q["dst_x"], q["dst_z"] = rng.uniform(-W, 0, n), rng.uniform(0, H, n)
    q["tolerance"] = rng.choice([0.0, 2.0, 6.0, 40.0], n)
    q["faction_id"] = np.where(q["kind"] == capi.QUERY_DEST_ID, rng.choice([capi.FACTION_ID_NONE, 0, 3], n), 0)
    return q


def _query_twin(nav, npop, q, pu, du):
    """twin A: the plain call on the queries with the named positions substituted from the read-back"""
    qa = q.copy()
    xz = _substitute(nav, npop, pu, np.stack([q["x"], q["z"]], 1))
    qa["x"], qa["z"] = xz[:, 0], xz[:, 1]
    xz = _substitute(nav, npop, du, np.stack([q["dst_x"], q["dst_z"]], 1))
    qa["dst_x"], qa["dst_z"] = xz[:, 0], xz[:, 1]
    return nav.map_query(qa)


def _named_queries(q, pu, du):
    """twin B's records: OFF at every named position"""
    qb = q.copy()
    qb["x"][pu != NULL] = OFF; qb["z"][pu != NULL] = OFF
    qb["dst_x"][du != NULL] = OFF; qb["dst_z"][du != NULL] = OFF
    return qb


def test_map_queries_c2():
    """4096 queries of all six kinds on two layers of the C2 map, positions and destinations named by uid or given"""
    from test_gpu_map_query import _c2_nav
    nav, _ = _c2_nav(2)
    try:
        rng = np.random.default_rng(71)
        npop = 100000
        pts = np.stack([rng.uniform(-16 * 256.0, 0, npop), rng.uniform(0, 16 * 256.0, npop)], 1).astype(np.float32)
        pts[:50] = (2.0, 5.0)                                # a few entities off the map: ok = 0
        rec, fl = _agents(pts, 0, pts[0])
        nav.agents_upload(rec, fl, 20)
        q = _queries(rng, 4096, 2, 16, 16)
        pu = rng.integers(0, npop, len(q)).astype(np.uint32); pu[rng.random(len(q)) < 0.4] = NULL
        du = rng.integers(0, npop, len(q)).astype(np.uint32); du[rng.random(len(q)) < 0.5] = NULL
        pu[:8] = np.arange(8)                               # off the map
        a = _query_twin(nav, npop, q, pu, du)
        b = nav.map_query_resident(_named_queries(q, pu, du), pu, du)
        assert a.tobytes() == b.tobytes()
        for k in range(6):
            assert (q["kind"] == k).any()
        assert a["ok"].any() and not a["ok"][:8].any()
        # one uid array only, and none
        none = np.full(len(q), NULL, np.uint32)
        assert nav.map_query_resident(_named_queries(q, pu, none), pu, None).tobytes() == \
            _query_twin(nav, npop, q, pu, none).tobytes()
        assert nav.map_query_resident(q).tobytes() == nav.map_query(q).tobytes()
    finally:
        nav.close()


def test_map_queries_host_finish():
    """searches that leave the kernel's window are finished on the host with the substituted positions"""
    import map_query_cases as mq
    img = np.ones((256, 256), np.uint8)
    img[28:228, 28:228] = 0xFF
    img[60, 128] = 1
    nav = capi.Nav(0)
    try:
        nav.map_create(4, 4, 1)
        nav.map_upload_layer(0, synth.image_to_blocked(img, 4, 4))
        nav.map_build_nav(0)
        nav.route_build(0)
        cx, cz = mq.tile_xz(128, 128)
        ix, iz = mq.tile_xz(60, 128)
        px, pz = mq.tile_xz(10, 10)
        pts = np.array([(px, pz), (cx, cz), (ix, iz), (cx + 1.0, cz - 1.0)], np.float32)
        rec, fl = _agents(pts, 0, pts[0])
        nav.agents_upload(rec, fl, 20)
        q = np.array([(capi.QUERY_PATHABLE, 0, px, pz, 0, 0, 0, 0),
                      (capi.QUERY_CLOSEST_PATHABLE, 0, px, pz, 0, 0, 0, 0),
                      (capi.QUERY_MAXIMALLY_CLOSE, 0, px, pz, px, pz, 100.0, 0),
                      (capi.QUERY_CLOSEST_PATHABLE, 0, px, pz, 0, 0, 0, 0),
                      (capi.QUERY_MAXIMALLY_CLOSE, 0, px, pz, px, pz, 0.0, 0)], capi.MAP_QUERY)
        pu = np.array([1, 1, 2, 3, NULL], np.uint32)
        du = np.array([NULL, NULL, 2, NULL, 1], np.uint32)
        a = _query_twin(nav, 4, q, pu, du)
        b = nav.map_query_resident(_named_queries(q, pu, du), pu, du)
        assert a.tobytes() == b.tobytes()
        assert a["ok"][0] == 0 and a["ok"][1] == 1 and a["ok"][3] == 1
        # the given values at the named entries are never read: the same answers with other values there
        assert nav.map_query_resident(q, pu, du).tobytes() == b.tobytes()
    finally:
        nav.close()


# ---- group arrival

def test_group_arrival_flock():
    """a flock of 12 000 uids against a zone dest: out_vel and out_flags equal the plain call on the read-back"""
    cw = ch = 8
    nav = capi.Nav(0)
    try:
        cost = synth.cost_from_pathable(synth.make_map(cw, ch, 0x5EED1B00, rivers=True), cw, ch)
        nav.map_create(cw, ch, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
        nav.pool_create(4, 4 * cw * ch)
        centre = np.array([-4.5 * 256, 4.5 * 256], np.float32)
        nav.pool_request_zone(2, centre, 12)
        rng = np.random.default_rng(81)
        npop = 15000
        pts = np.stack([rng.uniform(-cw * 256.0 - 8, 8, npop), rng.uniform(-8, ch * 256.0 + 8, npop)], 1).astype(np.float32)
        pts[: npop // 2] = centre + rng.normal(0, 200.0, (npop // 2, 2)).astype(np.float32)
        rec, fl = _agents(pts, 2, centre)
        nav.agents_upload(rec, fl, 20)
        uids = rng.permutation(npop)[:12000].astype(np.uint32)
        va, fa = nav.group_arrival_velocity(2, centre, 12, _substitute(nav, npop, uids, None))
        vb, fb = nav.group_arrival_velocity_resident(2, centre, 12, uids)
        assert va.tobytes() == vb.tobytes() and fa.tobytes() == fb.tobytes()
        assert (fa & 1).any() and not (fa & 1).all()
        vel, fl8 = np.full((3, 2), 7, np.float32), np.full(3, 7, np.uint8)
        for u in (np.array([0, npop, 1], np.uint32), np.array([0, NULL, 1], np.uint32)):
            rc = nav.L.pfnav_group_arrival_velocity_resident(nav.h, 2, capi._p(centre), 12, capi._p(u), 3, capi._p(vel),
                                                             capi._p(fl8))
            assert rc == capi.ERR_ARG and (vel == 7).all() and (fl8 == 7).all()
        rc = nav.L.pfnav_group_arrival_velocity_resident(nav.h, 2, capi._p(centre), 12, None, 3, capi._p(vel), capi._p(fl8))
        assert rc == capi.ERR_ARG
        assert nav.L.pfnav_group_arrival_velocity_resident(nav.h, 2, capi._p(centre), 12, None, 0, None, None) == 0
    finally:
        nav.close()


# ---- the resident loop and groups

def _job_case(world):
    cost, rec, fl, ms = _population(4242, 20)
    return Job(3, cost, rec, fl, ms, 20, world, ndests=len(fl) + 10), cost


def _twin(cost, ndests, max_fields):
    X = capi.Nav(0)
    X.map_create(3, 3, 1)
    X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
    X.pool_create(ndests, max_fields)
    return X


def _calls(n, nd, seed):
    """one set of the three calls' arguments over a population of n: 40 paths, 200 queries, a flock of 300"""
    rng = np.random.default_rng(seed)
    dests = rng.integers(0, nd, 40).astype(np.int32)
    su = rng.integers(0, n, 40).astype(np.uint32)
    du = rng.integers(0, n, 40).astype(np.uint32); du[::3] = NULL
    dxz = np.stack([rng.uniform(-3 * 256.0, 0, 40), rng.uniform(0, 3 * 256.0, 40)], 1).astype(np.float32)
    q = _queries(rng, 200, 1, 3, 3)
    pu = rng.integers(0, n, 200).astype(np.uint32); pu[::4] = NULL
    qu = rng.integers(0, n, 200).astype(np.uint32); qu[1::4] = NULL
    flock = rng.choice(n, 300, replace=False).astype(np.uint32)
    return dests, su, du, dxz, q, pu, qu, flock


def _resident_all(X, a, nd, centre):
    """the three resident calls on X -> their outputs and X's pool"""
    dests, su, du, dxz, q, pu, qu, flock = a
    p = X.pool_request_paths_resident(dests, su, None, du, _masked(dxz, du))
    mqr = X.map_query_resident(_named_queries(q, pu, qu), pu, qu)
    X.pool_request_zone(nd - 1, centre, 10)
    g = X.group_arrival_velocity_resident(nd - 1, centre, 10, flock)
    return p, mqr.tobytes(), g, _pool(X, nd, 9)


def _plain_all(A, X, n, a, nd, centre):
    """the plain calls on A with the positions read back from X"""
    dests, su, du, dxz, q, pu, qu, flock = a
    p = A.pool_request_paths(dests, _substitute(X, n, su, None), _substitute(X, n, du, dxz))
    mqr = _query_twin_on(A, X, n, q, pu, qu)
    A.pool_request_zone(nd - 1, centre, 10)
    g = A.group_arrival_velocity(nd - 1, centre, 10, _substitute(X, n, flock, None))
    return p, mqr.tobytes(), g, _pool(A, nd, 9)


def _query_twin_on(A, X, n, q, pu, du):
    qa = q.copy()
    xz = _substitute(X, n, pu, np.stack([q["x"], q["z"]], 1)); qa["x"], qa["z"] = xz[:, 0], xz[:, 1]
    xz = _substitute(X, n, du, np.stack([q["dst_x"], q["dst_z"]], 1)); qa["dst_x"], qa["dst_z"] = xz[:, 0], xz[:, 1]
    return A.map_query(qa)


def _same(r1, r2):
    (p1, m1, g1, pool1), (p2, m2, g2, pool2) = r1, r2
    assert all(np.array_equal(x, y) for x, y in zip(p1[:4], p2[:4])) and p1[4] == p2[4]
    assert m1 == m2
    assert g1[0].tobytes() == g2[0].tobytes() and g1[1].tobytes() == g2[1].tobytes()
    assert pool1 == pool2


def test_resident_loop_stale_then_rebuilt():
    """positions moved only on the device (compute_updates -> apply_updates): each call refuses with PFNAV_ERR_STATE and
    changes nothing; after pfnav_agents_rebuild_index the calls equal twin A built from the read-back"""
    J, cost = _job_case(2)
    nd = len(J.fl) + 10
    A = _twin(cost, nd, nd * 9)
    centre = np.array([-1.5 * 256, 1.5 * 256], np.float32)
    try:
        one = J.one
        nw = len(one.agents_read_work())
        assert nw > 0
        for step in range(2):
            a = _calls(J.n, nd, 90 + step)
            dests, su, du, dxz, q, pu, qu, flock = a
            J._tick_one(one, nw, 1)                             # ... compute_updates, apply_updates: records moved
            before = _pool(one, nd, 9)
            r = _paths_raw(one, dests, su, None, du, _masked(dxz, du))
            assert r[0] == capi.ERR_STATE and r[5] == 0 and all((o == 77).all() for o in r[1:5])
            out = np.full(len(q), 7, capi.MAP_QUERY_RESULT)
            out0 = out.copy()
            qb = _named_queries(q, pu, qu)
            assert one.L.pfnav_map_query_resident(one.h, capi._p(qb), capi._p(pu), capi._p(qu), len(q), capi._p(out),
                                                  None) == capi.ERR_STATE
            assert out.tobytes() == out0.tobytes()
            vel, fl8 = np.full((len(flock), 2), 7, np.float32), np.full(len(flock), 7, np.uint8)
            assert one.L.pfnav_group_arrival_velocity_resident(one.h, 0, capi._p(centre), 10, capi._p(flock), len(flock),
                                                               capi._p(vel), capi._p(fl8)) == capi.ERR_STATE
            assert (vel == 7).all() and (fl8 == 7).all()
            assert _pool(one, nd, 9) == before
            # a uid outside the population: PFNAV_ERR_ARG first
            bad = flock.copy(); bad[7] = J.n
            assert one.L.pfnav_group_arrival_velocity_resident(one.h, 0, capi._p(centre), 10, capi._p(bad), len(bad),
                                                               capi._p(vel), capi._p(fl8)) == capi.ERR_ARG
            one.agents_rebuild_index()
            one.pool_clear(); A.pool_clear()                    # the tick's repairs wrote the pool: compare from empty
            _same(_resident_all(one, a, nd, centre), _plain_all(A, one, J.n, a, nd, centre))
            r = _paths_raw(one, dests, np.where(su == su[0], J.n, su).astype(np.uint32), None, du, _masked(dxz, du))
            assert r[0] == capi.ERR_ARG and r[5] == 0
    finally:
        A.close()
        J.close()


@pytest.mark.parametrize("world", [2, 3])
def test_group_members_vs_single_context(world):
    """every member of a group, resolving uids that other members own, equals the single context given the same calls"""
    J, cost = _job_case(world)
    nd = len(J.fl) + 10
    centre = np.array([-1.5 * 256, 1.5 * 256], np.float32)
    try:
        for step in range(2):
            a = _calls(J.n, nd, 100 + step)
            for lo, hi in J.ranges:                             # every member resolves uids of every range
                assert ((a[1] >= lo) & (a[1] < hi)).any() and ((a[7] >= lo) & (a[7] < hi)).any()
            for X in J.all():
                X.pool_clear()
            ref = _resident_all(J.one, a, nd, centre)
            for nv in J.navs:
                _same(_resident_all(nv, a, nd, centre), ref)
            J.tick()                                            # records move on every context; the gather makes them whole
    finally:
        J.close()
