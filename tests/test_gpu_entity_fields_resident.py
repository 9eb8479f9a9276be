"""GPU suite: pfnav_pool_request_entity_fields_resident and its group form, the enemy-seek and surround field batch with
the moving entities and the seekers named by uid and resolved from the resident records.

Twin contexts: twin A reads the records back (pfnav_agents_read_state), builds the footprints and each request's
de-duplicated seeker chunks in numpy and calls pfnav_pool_request_entity_fields_batch; twin B makes the resident call.
Both must end with the same ndone and the same (dest, chunk) entries (has bits, ff_id, flow bytes), and after
tick -> pfnav_pool_repair -> tick with the same repair counts, vdes and velocities, bit for bit. Group members are
compared with solo twins the same way, as in test_gpu_mgpu_aux_fields.py."""
import ctypes as C

import numpy as np
import pytest

import cases
from test_gpu_entity_field_batch import _agents_on, _building, _ctx, _pool, _req, _tick
from test_gpu_mgpu_commands import Job, _population

pytestmark = pytest.mark.gpu
capi = cases.capi
NULL = capi.NULL_UID


def chunk_of(pos, cw, ch, map_x=0.0, map_z=0.0):
    """M_Tile_DescForPoint2D's chunk in the tick's arithmetic (pfnav_map_view.cuh): r * cw + c, -1 off the map"""
    px, pz = pos[:, 0].astype(np.float32), pos[:, 1].astype(np.float32)
    mx, mz = np.float32(map_x), np.float32(map_z)
    on = ~((px > mx) | (px < mx - np.float32(cw * 256)) | (pz < mz) | (pz > mz + np.float32(ch * 256)))
    r = np.clip((np.abs((mz - pz).astype(np.float64)) / 256.0).astype(np.int64), 0, ch - 1)
    c = np.clip((np.abs((mx - px).astype(np.float64)) / 256.0).astype(np.int64), 0, cw - 1)
    return np.where(on, r * cw + c, -1)


def resolve(nav, n, reqs, fp, uids, seekers, cw, ch):
    """twin A's inputs: the contract of include/pfnav.h on the records read back"""
    a, _ = nav.agents_read_state(n, False)
    ents = np.zeros(len(uids), capi.FOOTPRINT) if fp is None else fp.copy()
    named = uids != NULL
    ents[named] = np.zeros(1, capi.FOOTPRINT)
    ents["x"][named], ents["z"][named] = a["pos"][uids[named], 0], a["pos"][uids[named], 1]
    ents["sel_radius"][named] = a["radius"][uids[named]]
    sc = chunk_of(a["pos"][seekers], cw, ch)
    assert (sc >= 0).all()
    out, chunks = reqs.copy(), []
    for i, q in enumerate(reqs):
        s = sc[int(q["chunk_off"]):int(q["chunk_off"]) + int(q["chunk_n"])]
        _, first = np.unique(s, return_index=True)
        seen = s[np.sort(first)]
        out["chunk_off"][i], out["chunk_n"][i] = len(chunks), len(seen)
        chunks += [divmod(int(c), cw) for c in seen]
    return out, ents, np.array(chunks, np.int32).reshape(-1, 2)


def raw(nav, reqs, fp, uids, seekers, stream=0):
    """the resident call's return code and ndone (no exception)"""
    a = capi._resident_args(reqs, fp, uids, seekers)
    nd = C.c_int(-1)
    rc = nav.L.pfnav_pool_request_entity_fields_resident(nav.h, *a[:7], C.c_void_p(stream), C.byref(nd))
    return rc, nd.value


def batch_case(cw, ch, n, nreq, ndests, seed, buildings=6):
    """an enemy list of uids mixed with building footprints, TARGET_ENTITY by uid, overlapping ranges, repeated dests,
    repeated seekers (repeated (dest, chunk) keys), every reference layer, radii on both sides of the device / host
    rasterisation bound"""
    rng = np.random.default_rng(seed)
    W, H = cw * 256.0, ch * 256.0
    nb = buildings
    fp = np.zeros(nb, capi.FOOTPRINT)
    for i in range(nb):
        cx, cz = -rng.uniform(24, W - 24), rng.uniform(24, H - 24)
        fp["is_building"][i] = 1; fp["x"][i], fp["z"][i] = cx, cz
        fp["corners_xz"][i] = _building(cx, cz, rng.uniform(2, 10), rng.uniform(2, 10), rng.uniform(0, np.pi))
    nu = min(n, 400)
    uids = np.concatenate([np.full(nb, NULL, np.uint32), rng.choice(n, nu, replace=False).astype(np.uint32)])
    perm = rng.permutation(len(uids))
    uids = uids[perm]
    fpa = np.zeros(len(uids), capi.FOOTPRINT)
    fpa[np.nonzero(uids == NULL)[0]] = fp
    seekers = rng.integers(0, n, 600).astype(np.uint32)
    seekers[50:80] = seekers[10]
    reqs = []
    for i in range(nreq):
        kind = int(rng.integers(0, 2))
        if kind == capi.TARGET_ENTITY:
            ent = (int(rng.integers(0, len(uids))), 1)
        else:
            a = int(rng.integers(0, len(uids) - 1)); ent = (a, int(rng.integers(1, len(uids) - a + 1)))
        s0 = int(rng.integers(0, len(seekers) - 1))
        sk = (s0, int(min(rng.integers(0, 40), len(seekers) - s0)))
        reqs.append(_req(int(rng.integers(0, ndests)), kind, ent, sk, 0, int(rng.integers(0, 12))))
    reqs.append(_req(0, capi.TARGET_ENEMIES, (0, len(uids)), (0, len(seekers)), 0, 11))
    return np.concatenate(reqs), fpa, uids, seekers


NLAYERS = 4                 # radii up to 60: the size classes of layers 0 .. 3 (Entity_NavLayerWithRadius)


def radii(rec, rng):
    rec["radius"] = rng.choice(np.array([0.5, 1.0, 3.0, 8.0, 16.0, 28.0, 28.5, 40.0, 40.5, 60.0], np.float32), len(rec))


def twins_compare(navs, rec, fl, ext, ndests, cw, ch):
    out = []
    for nav in navs:
        _tick(nav, rec, fl, ext)
        rep = nav.pool_repair()
        _tick(nav, rec, fl, ext)
        _, vdes, _ = nav.agents_read_debug(len(rec))
        out.append((rep, vdes, nav.agents_read_velocities(len(rec)), _pool(nav, ndests, cw, ch)))
    assert out[0][0] == out[1][0]
    assert (out[0][1] == out[1][1]).all() and (out[0][2] == out[1][2]).all()
    assert out[0][3] == out[1][3]


@pytest.mark.parametrize("pool_max", [4096, 40])
def test_resident_vs_batch(pool_max):
    """twin A (read-back + numpy + batch) == twin B (resident call); pool_max 40 evicts inside the batch"""
    cw = ch = 4
    ndests = 24
    navs = [_ctx(cw, ch, 0x5EED1A00, NLAYERS) for _ in range(2)]
    try:
        rec, fl, ext = _agents_on(navs[0], cw, ch, ndests, 3000, 31)
        radii(rec, np.random.default_rng(3))
        reqs, fp, uids, seekers = batch_case(cw, ch, len(rec), 120, ndests, 7)
        for nav in navs:
            nav.pool_create(ndests, pool_max)
            nav.agents_upload(rec, fl, 20)
        ra, fa, ca = resolve(navs[0], len(rec), reqs, fp, uids, seekers, cw, ch)
        nd_a = navs[0].pool_request_entity_fields_batch(ra, fa, ca)
        nd_b = navs[1].pool_request_entity_fields_resident(reqs, fp, uids, seekers)
        assert nd_a == nd_b == len(reqs)
        assert _pool(navs[0], ndests, cw, ch) == _pool(navs[1], ndests, cw, ch)
        twins_compare(navs, rec, fl, ext, ndests, cw, ch)
    finally:
        for nav in navs:
            nav.close()


def test_target_entity_by_uid_every_layer():
    """TARGET_ENTITY fields whose one footprint names a uid (ents NULL), on all 12 reference layers"""
    cw = ch = 4
    navs = [_ctx(cw, ch, 0x5EED1A10, NLAYERS) for _ in range(2)]
    try:
        rec, fl, ext = _agents_on(navs[0], cw, ch, 12, 2000, 33)
        radii(rec, np.random.default_rng(4))
        rng = np.random.default_rng(5)
        uids = rng.choice(len(rec), 12, replace=False).astype(np.uint32)
        seekers = rng.integers(0, len(rec), 240).astype(np.uint32)
        reqs = np.concatenate([_req(L, capi.TARGET_ENTITY, (L, 1), (20 * L, 20), 0, L) for L in range(12)])
        for nav in navs:
            nav.pool_create(12, 12 * 16)
            nav.agents_upload(rec, fl, 20)
        ra, fa, ca = resolve(navs[0], len(rec), reqs, None, uids, seekers, cw, ch)
        assert navs[0].pool_request_entity_fields_batch(ra, fa, ca) == 12
        assert navs[1].pool_request_entity_fields_resident(reqs, None, uids, seekers) == 12
        assert _pool(navs[0], 12, cw, ch) == _pool(navs[1], 12, cw, ch)
        twins_compare(navs, rec, fl, ext, 12, cw, ch)
    finally:
        for nav in navs:
            nav.close()


def test_nomem_stop_and_errors():
    """a request the pool cannot hold stops both twins at the same request; every argument error, the host-only context
    and m == 0 change nothing"""
    cw = ch = 4
    navs = [_ctx(cw, ch, 0x5EED1A20) for _ in range(2)]
    try:
        rec, fl, ext = _agents_on(navs[0], cw, ch, 8, 2000, 35)
        reqs, fp, uids, seekers = batch_case(cw, ch, len(rec), 30, 8, 9)
        # a seeker on every chunk that holds one: more distinct chunks than a pool of 12 holds
        cpos = chunk_of(rec["pos"], cw, ch)
        every = np.array([int(np.nonzero(cpos == c)[0][0]) for c in range(cw * ch) if (cpos == c).any()], np.uint32)
        assert len(every) > 12
        seekers = np.concatenate([seekers, every])
        reqs = np.concatenate([reqs[:12], _req(3, capi.TARGET_ENEMIES, (0, 50), (len(seekers) - len(every), len(every))),
                               reqs[12:]])
        for nav in navs:
            nav.pool_create(8, 12)
            nav.agents_upload(rec, fl, 20)
        ra, fa, ca = resolve(navs[0], len(rec), reqs, fp, uids, seekers, cw, ch)
        nd_a = navs[0].pool_request_entity_fields_batch(ra, fa, ca)
        nd_b = navs[1].pool_request_entity_fields_resident(reqs, fp, uids, seekers)
        assert nd_a == nd_b and nd_a < len(reqs)
        assert _pool(navs[0], 8, cw, ch) == _pool(navs[1], 8, cw, ch)
        nav = navs[1]
        before = _pool(nav, 8, cw, ch)
        n = len(rec)
        ok = _req(0, capi.TARGET_ENEMIES, (0, 10), (0, 5))
        u10, s10 = uids[:10].copy(), seekers[:10].copy()
        half = u10.copy(); half[0] = 5
        bad = [(ok, fp[:10], np.where(np.arange(10) == 3, n, u10).astype(np.uint32), s10),     # uid outside the population
               (ok, fp[:10], u10, np.append(s10[:9], n).astype(np.uint32)),                  # seeker outside
               (ok, None, np.where(np.arange(10) == 3, NULL, half).astype(np.uint32), s10),  # ents NULL, an entry unnamed
               (_req(0, capi.TARGET_ENEMIES, (5, 6), (0, 5)), fp[:10], u10, s10),            # footprint range
               (_req(0, capi.TARGET_ENEMIES, (0, 10), (8, 5)), fp[:10], u10, s10),           # seeker range
               (_req(8, capi.TARGET_ENEMIES, (0, 10), (0, 5)), fp[:10], u10, s10),           # dest (the batch's check)
               (_req(0, capi.TARGET_ENTITY, (0, 2), (0, 5)), fp[:10], u10, s10)]             # TARGET_ENTITY takes one
        for i, (r, f, u, s) in enumerate(bad):
            rc, nd = raw(nav, np.concatenate([ok, r]), f, u, s)
            assert rc == capi.ERR_ARG and nd == 0, i
            assert _pool(nav, 8, cw, ch) == before, i
        assert raw(nav, np.zeros(0, capi.ENTITY_FIELD_REQ), None, np.array([n + 5], np.uint32), s10) == (capi.ERR_ARG, 0)
        assert raw(nav, np.zeros(0, capi.ENTITY_FIELD_REQ), fp[:10], u10, s10) == (0, 0)
        assert _pool(nav, 8, cw, ch) == before
    finally:
        for nav in navs:
            nav.close()
    host = capi.Nav(hostonly=True)
    try:
        rc, _ = raw(host, _req(0, capi.TARGET_ENEMIES, (0, 1), (0, 1)), None, np.array([0], np.uint32), np.array([0], np.uint32))
        assert rc == capi.ERR_NO_DEVICE
    finally:
        host.close()


def test_c2_sized():
    """100 000 entities on 16 x 16 chunks: four enemy lists of 30 000 uids plus buildings, 10 000 seekers"""
    cw = ch = 16
    ndests = 4
    navs = [_ctx(cw, ch, 0x5EED1A30, NLAYERS) for _ in range(2)]
    try:
        rec, fl, ext = _agents_on(navs[0], cw, ch, ndests, 100000, 37)
        radii(rec, np.random.default_rng(6))
        rng = np.random.default_rng(8)
        _, fpb, ub, _ = batch_case(cw, ch, len(rec), 1, ndests, 10, buildings=40)
        bmask = ub == NULL
        lists, reqs, off = [], [], 0
        seekers = rng.integers(0, len(rec), 10000).astype(np.uint32)
        for f in range(4):
            u = np.concatenate([rng.choice(len(rec), 30000, replace=False).astype(np.uint32), np.full(int(bmask.sum()), NULL, np.uint32)])
            lists.append(u)
            reqs.append(_req(f, capi.TARGET_ENEMIES, (off, len(u)), (2500 * f, 2500), 0, f))
            off += len(u)
        uids = np.concatenate(lists)
        fp = np.zeros(len(uids), capi.FOOTPRINT)
        fp[uids == NULL] = np.tile(fpb[bmask], 4)
        reqs = np.concatenate(reqs)
        for nav in navs:
            nav.pool_create(ndests, ndests * cw * ch)
            nav.agents_upload(rec, fl, 20)
        ra, fa, ca = resolve(navs[0], len(rec), reqs, fp, uids, seekers, cw, ch)
        assert navs[0].pool_request_entity_fields_batch(ra, fa, ca) == 4
        assert navs[1].pool_request_entity_fields_resident(reqs, fp, uids, seekers) == 4
        assert _pool(navs[0], ndests, cw, ch) == _pool(navs[1], ndests, cw, ch)
    finally:
        for nav in navs:
            nav.close()


def _job_case(world):
    cost, rec, fl, ms = _population(4242, 20)
    return Job(3, cost, rec, fl, ms, 20, world, ndests=len(fl) + 10), cost, rec


def _twin(cost, ndests, max_fields):
    X = capi.Nav(0)
    X.map_create(3, 3, 1)
    X.map_upload_layer(0, cost); X.map_build_nav(0); X.route_build(0)
    X.pool_create(ndests, max_fields)
    return X


def test_resident_loop_stale_then_rebuilt():
    """positions moved only on the device (compute_updates -> apply_updates): before the rebuild the call refuses and
    leaves the pool as it was; after it the call equals twin A built from the read-back"""
    J, cost, rec = _job_case(2)
    nd = len(J.fl) + 10
    A = _twin(cost, nd, nd * 9)
    try:
        one = J.one
        rng = np.random.default_rng(11)
        reqs, fp, uids, seekers = batch_case(3, 3, J.n, 16, nd, 12)
        nw = len(one.agents_read_work())
        assert nw > 0
        for step in range(2):
            J._tick_one(one, nw, 1)                             # ... compute_updates, apply_updates: records moved
            before = _pool(one, nd, 3, 3)
            assert raw(one, reqs, fp, uids, seekers) == (capi.ERR_STATE, 0)
            assert _pool(one, nd, 3, 3) == before
            one.agents_rebuild_index()
            one.pool_clear(); A.pool_clear()                    # the tick's repairs wrote the pool: compare from empty
            ra, fa, ca = resolve(one, J.n, reqs, fp, uids, seekers, 3, 3)
            assert A.pool_request_entity_fields_batch(ra, fa, ca) == one.pool_request_entity_fields_resident(reqs, fp, uids, seekers)
            assert _pool(A, nd, 3, 3) == _pool(one, nd, 3, 3)
    finally:
        A.close()
        J.close()


@pytest.mark.parametrize("world", [2, 3])
def test_group_vs_solo_twins(world):
    """every member of a group equals a solo twin taking the batch built from the read-back: every entry, later
    evictions, the remembered footprints through pfnav_pool_repair_batch; one stale member makes the group call refuse
    with PFNAV_ERR_STATE and no pool changes"""
    J, cost, rec = _job_case(world)
    nd = len(J.fl) + 10
    reqs, fp, uids, seekers = batch_case(3, 3, J.n, 24, nd, 13)
    ra, fa, ca = resolve(J.one, J.n, reqs, fp, uids, seekers, 3, 3)
    keys = {(int(q["dest"]), int(r) * 3 + int(c)) for q in ra
            for r, c in ca[int(q["chunk_off"]):int(q["chunk_off"]) + int(q["chunk_n"])]}
    small = len(keys) + 4                                   # the batch fits; filling every dest evicts
    assert small < nd * 9
    twins = [_twin(cost, nd, small) for _ in range(world)]
    try:
        for nv in J.navs:
            nv.pool_create(nd, small)
        J.grp.request_entity_fields_resident(reqs, fp, uids, seekers)
        for T in twins:
            assert T.pool_request_entity_fields_batch(ra, fa, ca) == len(reqs)
        for nv, T in zip(J.navs, twins):
            assert _pool(nv, nd, 3, 3) == _pool(T, nd, 3, 3)
        # later evictions: solo batches that fill the pools evict by each pool's own history
        allc = np.array([divmod(c, 3) for c in range(9)], np.int32)
        for d in range(nd):
            for X in J.navs + twins:
                X.pool_request_entity_fields_batch(_req(d, capi.TARGET_ENEMIES, (0, 20), (0, 9)), fa, allc)
        for nv, T in zip(J.navs, twins):
            assert _pool(nv, nd, 3, 3) == _pool(T, nd, 3, 3)
        J.grp.request_entity_fields_resident(reqs, fp, uids, seekers)
        for T in twins:
            T.pool_request_entity_fields_batch(ra, fa, ca)
        # one stale member: every member refuses, no pool changes
        lo, hi = J.ranges[world - 1]
        state = J.one.agents_read_state(J.n, False)[0]
        J.navs[-1].agents_upload_shard(state[lo:hi], lo, hi, J.n, J.fl, 20, capi.UPLOAD_SAME_FLOCKS)
        before = [_pool(nv, nd, 3, 3) for nv in J.navs]
        a = capi._resident_args(reqs, fp, uids, seekers)
        assert capi.load().pfnav_group_request_entity_fields_resident(J.grp.g, *a[:7]) == capi.ERR_STATE
        assert [_pool(nv, nd, 3, 3) for nv in J.navs] == before
        J.grp.gather()
        # the remembered footprints: a repair batch on members and twins after the group is gone
        J.grp.close(); J.grp = None
        rec2, fl2, ext2 = _agents_on(J.navs[0], 3, 3, nd - 1, 1500, 17)
        for nv, T in zip(J.navs, twins):
            out = []
            for X in (nv, T):
                _tick(X, rec2, fl2, ext2)
                out.append(X.pool_repair_batch())
            assert out[0] == out[1]
            assert _pool(nv, nd, 3, 3) == _pool(T, nd, 3, 3)
    finally:
        for T in twins:
            T.close()
        J.close()
