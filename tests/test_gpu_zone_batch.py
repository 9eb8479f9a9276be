"""GPU suite: pfnav_pool_request_zones, the batched N_RequestAsyncGroupArrivalField + N_AwaitAsyncFields
(nav.c:3921, 3958) with its seed floods (field_zone_initial_frontier, field.c:1683) replayed on the device.

- one batch reproduces the compiled reference's zone fields and group-arrival velocities (region.npz);
- the device flood equals the host flood (pfnav_zone_fields: host seeds + the same integration kernel) byte for byte on
  1 x 1, 4 x 4 and C2 maps, including phase one through blocked areas, the budget cap and windows without the centre;
- the batch leaves the pool (flow bytes, has, ffid, remaining capacity) exactly as the serial loop of
  pfnav_pool_request_zone does, at a NOMEM stop too; bad arguments change nothing;
- launches are ordered on the caller's stream, after pfnav_pool_clear and the goal batch's forked field work."""
import ctypes as C
import importlib
import os

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
C2_SEED = 0x5EED0001            # bench.py's C2 map


def _map(cw, ch, seed, square=True):
    """a synthetic cost layer (chunk-blocked) with a large blocked square; -> (cost, centre of the square)"""
    rng = np.random.default_rng(seed)
    img = synth.blocked_to_image(synth.cost_from_pathable(synth.make_map(cw, ch, seed, rivers=cw > 1 and ch > 1), cw, ch), cw, ch).copy()
    side = min(40, 64 * min(cw, ch) - 8)
    r0, c0 = int(rng.integers(0, ch * 64 - side + 1)), int(rng.integers(0, cw * 64 - side + 1))
    if square:
        img[r0:r0 + side, c0:c0 + side] = 0xFF
    return synth.image_to_blocked(img, cw, ch), (r0 + side // 2, c0 + side // 2)


def _ctx(cw, ch, cost, route=False):
    nav = capi.Nav(0)
    nav.map_create(cw, ch, 1)
    nav.map_upload_layer(0, cost)
    nav.map_build_nav(0)
    if route:
        nav.route_build(0)
    return nav


def _xz(tile):
    """world centre of an absolute nav tile (map at the origin)"""
    r, c = int(tile[0]), int(tile[1])
    return synth.tile_center_xz(r // 64, c // 64, r % 64, c % 64)


def _reqs(rows):
    """rows: (dest, (x, z), radius) -> ZONE_REQ records"""
    out = np.zeros(len(rows), capi.ZONE_REQ)
    for i, (d, xz, rad) in enumerate(rows):
        out[i]["dest"], out[i]["centre_x"], out[i]["centre_z"], out[i]["radius"] = d, xz[0], xz[1], rad
    return out


def _reach(tile, radius, cw, ch):
    """the chunks N_RequestAsyncGroupArrivalField requests (nav.c:3945-3951; C division truncates toward zero)"""
    cl = lambda v, hi: min(max(v, 0), hi)
    tdiv = lambda a: int(a / 64)
    r, c, k = int(tile[0]), int(tile[1]), 2 * radius
    return [(cr, cc) for cr in range(cl(tdiv(r - k), ch - 1), cl(tdiv(r + k), ch - 1) + 1)
            for cc in range(cl(tdiv(c - k), cw - 1), cl(tdiv(c + k), cw - 1) + 1)]


def _raw(nav, reqs, stream=0, nfields=True):
    """-> (rc, ndone, nfields) without raising"""
    reqs = np.ascontiguousarray(reqs, capi.ZONE_REQ)
    nf = np.full(max(len(reqs), 1), -7, np.int32); nd = C.c_int(-1)
    rc = nav.L.pfnav_pool_request_zones(nav.h, capi._p(reqs) if len(reqs) else None, len(reqs), C.c_void_p(stream),
                                        capi._p(nf) if nfields else None, C.byref(nd))
    return rc, nd.value, nf[:len(reqs)]


def _serial(nav, reqs):
    """the serial loop of pfnav_pool_request_zone; -> (rc, ndone, nfields)"""
    nf = np.zeros(len(reqs), np.int32)
    for i, q in enumerate(reqs):
        c = np.array([q["centre_x"], q["centre_z"]], np.float32); n = C.c_int(-7)
        rc = nav.L.pfnav_pool_request_zone(nav.h, int(q["dest"]), int(q["layer"]), capi._p(c), int(q["radius"]), None, C.byref(n))
        if rc:
            return rc, i, nf
        nf[i] = n.value
    return 0, len(reqs), nf


def _pool(nav, ndests, cw, ch):
    """every (dest, chunk) entry: has bits, ffid, flow bytes"""
    out = []
    for d in range(ndests):
        for c in range(cw * ch):
            f, l, ffid = nav.pool_get(d, divmod(c, cw))
            out.append((f is not None, l is not None, ffid, None if f is None else f.tobytes()))
    return out


def test_batch_region_golden():
    """one batch of every gv_* request of region.npz (each its own dest): field counts and N_DesiredGroupArrivalVelocity
    bit for bit; one batch of every zc / zrad zone at its tile's world centre: the fields of the chunks in reach == zexp"""
    g = np.load(os.path.join(GOLD, "region.npz"))
    cw = ch = 3
    nav = capi.Nav(0)
    try:
        nav.map_create(cw, ch, 1)
        nav.map_upload_layer(0, g["cost"], g["blk"])
        ngv, nzc = len(g["gv_radius"]), len(g["zc"])
        nav.pool_create(ngv + nzc, (ngv + nzc) * 9)
        reqs = _reqs([(k, g["gv_centre"][k], int(g["gv_radius"][k])) for k in range(ngv)])
        nd, nf = nav.pool_request_zones(reqs)
        assert nd == ngv and (nf == g["gv_nfields"]).all()
        for k in range(ngv):
            v, f = nav.group_arrival_velocity(k, g["gv_centre"][k], int(g["gv_radius"][k]), g["gv_pos"][k])
            assert (f == g["gv_flags"][k]).all() and (v == g["gv_vel"][k]).all(), k
        reqs = _reqs([(ngv + k, _xz(g["zc"][k]), int(g["zrad"][k])) for k in range(nzc)])
        nd, nf = nav.pool_request_zones(reqs)
        assert nd == nzc
        for k in range(nzc):
            chunks = _reach(g["zc"][k], int(g["zrad"][k]), cw, ch)
            assert nf[k] == len(chunks)
            for cr, cc in chunks:
                f, _, _ = nav.pool_get(ngv + k, (cr, cc))
                assert f is not None and (f == g["zexp"][k, cr * cw + cc]).all(), (k, cr, cc)
    finally:
        nav.close()


def _centres(cw, ch, cost, inside, rng, n):
    """open and blocked tiles, the middle of the blocked square, chunk borders, map edges and corners"""
    H, W = ch * 64, cw * 64
    img = synth.blocked_to_image(cost, cw, ch)
    open_, blocked = np.argwhere(img != 0xFF), np.argwhere(img == 0xFF)
    out = [tuple(open_[i]) for i in rng.integers(0, len(open_), n)]
    out += [tuple(blocked[i]) for i in rng.integers(0, len(blocked), n // 2)]
    out += [inside, (0, 0), (H - 1, W - 1), (0, W - 1), (H - 1, 0), (H // 2, W - 1)]
    for _ in range(n // 2):
        out.append((64 * int(rng.integers(0, ch)) + int(rng.choice([0, 31, 32, 63])), int(rng.integers(0, W))))
        out.append((int(rng.integers(0, H)), 64 * int(rng.integers(0, cw)) + int(rng.choice([0, 31, 32, 63]))))
    return [(int(a), int(b)) for a, b in out]


@pytest.mark.parametrize("cw,seed", [(1, 0x5EED0400), (4, 0x5EED0404), (16, C2_SEED)])
def test_device_flood_vs_host_flood(cw, seed):
    """pool fields of one batch == pfnav_zone_fields (host flood, same integration kernel) for every chunk in reach"""
    ch = cw
    if cw == 16:
        cost = synth.cost_from_pathable(synth.make_map(cw, ch, seed, rivers=True), cw, ch)
        inside = tuple(int(v) for v in np.argwhere(synth.blocked_to_image(cost, cw, ch) == 0xFF)[0])
    else:
        cost, inside = _map(cw, ch, seed)
    nav = _ctx(cw, ch, cost)
    try:
        rng = np.random.default_rng(seed)
        centres = _centres(cw, ch, cost, inside, rng, 12 if cw == 16 else 16)
        radii = [0, 1, 73, 80, 2, 5, 13, 32, 90]
        rows = [(i, _xz(t), radii[i % len(radii)]) for i, t in enumerate(centres)]
        nav.pool_create(len(rows), 8192)
        nd, nf = nav.pool_request_zones(_reqs(rows))
        assert nd == len(rows)
        nonzero = 0
        for i, (t, (_, _, rad)) in enumerate(zip(centres, rows)):
            chunks = _reach(t, rad, cw, ch)
            assert nf[i] == len(chunks), i
            host = nav.zone_fields(t, rad, chunks)
            for j, c in enumerate(chunks):
                f, _, _ = nav.pool_get(i, c)
                assert f is not None and (f == host[j]).all(), (t, rad, c)
                nonzero += int(host[j].any())
        assert nonzero > len(rows) // 4                         # the floods did seed fields
    finally:
        nav.close()


@pytest.mark.parametrize("nbig,nsmall", [(1, 0), (2, 3), (12, 40)])
def test_host_and_device_floods(nbig, nsmall):
    """a batch whose floods' budgets add up to little more than its largest flood floods on the host (two launches: the
    pool-entry scatter and the integration); a larger one on the device (k_zone_seed_bits in between). Both leave the pool as the serial loop
    and as the host flood (pfnav_zone_fields)"""
    cw = ch = 16
    cost = synth.cost_from_pathable(synth.make_map(cw, ch, C2_SEED, rivers=True), cw, ch)
    navs = [_ctx(cw, ch, cost) for _ in range(2)]
    try:
        rng = np.random.default_rng(nbig)
        open_ = np.argwhere(synth.blocked_to_image(cost, cw, ch) != 0xFF)
        tiles = [tuple(int(v) for v in open_[i]) for i in rng.integers(0, len(open_), nbig + nsmall)]
        rows = [(i, _xz(t), 80 if i < nbig else int(rng.choice([2, 4, 8]))) for i, t in enumerate(tiles)]
        reqs = _reqs(rows)
        for nav in navs:
            nav.pool_create(len(rows), 4096)
        a = _serial(navs[0], reqs)
        l0 = navs[1].launch_count()
        b = _raw(navs[1], reqs)
        launches = navs[1].launch_count() - l0
        assert launches == (3 if nbig + nsmall > 8 else 2)
        assert a[0] == b[0] == 0 and (a[2] == b[2]).all()
        assert _pool(navs[0], len(rows), cw, ch) == _pool(navs[1], len(rows), cw, ch)
        for i, (t, (_, _, rad)) in enumerate(zip(tiles, rows)):
            chunks = _reach(t, rad, cw, ch)
            host = navs[1].zone_fields(t, rad, chunks)
            for j, c in enumerate(chunks):
                assert (navs[1].pool_get(i, c)[0] == host[j]).all(), (t, rad, c)
    finally:
        for nav in navs:
            nav.close()


def _path(nav, cw, ch, rng):
    """a path request between two open tiles (world xz)"""
    cost, _, _ = nav.map_get_layer(0)
    t = np.argwhere(synth.blocked_to_image(cost, cw, ch) != 0xFF)
    a, b = t[rng.integers(0, len(t), 2)]
    return _xz(a), _xz(b)


def test_batch_vs_serial_loop():
    """repeated dests with different centres, a dest holding path fields, centres off the map, and zones after a
    blocker batch and a commit: the batch leaves the pool exactly as the serial loop; after the commit both equal the
    host flood"""
    cw = ch = 4
    ndests = 12
    cost, inside = _map(cw, ch, 0x5EED0410)
    navs = [_ctx(cw, ch, cost, route=True) for _ in range(2)]
    try:
        rng = np.random.default_rng(3)
        centres = _centres(cw, ch, cost, inside, rng, 10)
        rows = [(int(rng.integers(0, ndests)), _xz(t), int(rng.choice([0, 1, 4, 8, 16, 32, 80]))) for t in centres]
        rows += [(3, (10.0, 100.0), 5), (4, (-100.0, -3.0), 5), (5, (-100.0, 4 * 256.0 + 1.0), 5)]      # off the map
        rows += [(0, _xz(centres[0]), 8), (0, _xz(centres[1]), 16), (0, _xz(centres[0]), 8)]          # dest 0 again
        order = rng.permutation(len(rows))
        reqs = _reqs([rows[i] for i in order])
        src, dst = _path(navs[0], cw, ch, rng)
        for nav in navs:
            nav.pool_create(ndests, 4096)
            ok, _, nfl, _ = nav.pool_request_path(7, src, dst)          # dest 7 holds path fields first
            assert ok and nfl > 0
        a = _serial(navs[0], reqs)
        b = _raw(navs[1], reqs)
        assert a[0] == b[0] == 0 and a[1] == b[1] == len(reqs) and (a[2] == b[2]).all()
        assert (b[2][[i for i, q in enumerate(reqs) if q["centre_x"] > 0 or q["centre_z"] < 0 or q["centre_z"] > 1024]] == 0).all()
        assert _pool(navs[0], ndests, cw, ch) == _pool(navs[1], ndests, cw, ch)
        # blocker churn, committed, then more zones on the same dests
        ops = np.zeros(60, capi.BLOCKER_OP)
        ops["x"] = -rng.uniform(0, cw * 256, 60); ops["z"] = rng.uniform(0, ch * 256, 60)
        ops["range"] = rng.uniform(2, 30, 60); ops["flags"] = capi.FLAG_MOVABLE; ops["delta"] = 1
        for nav in navs:
            nav.blockers_batch(ops)
            nav.map_commit()
        rows2 = [(int(rng.integers(0, ndests)), (float(o["x"]), float(o["z"])), int(rng.choice([1, 8, 24]))) for o in ops[:16]]
        reqs2 = _reqs(rows2)
        a = _serial(navs[0], reqs2)
        b = _raw(navs[1], reqs2)
        assert a[0] == b[0] == 0 and (a[2] == b[2]).all()
        assert _pool(navs[0], ndests, cw, ch) == _pool(navs[1], ndests, cw, ch)
        # the last request of each (dest, chunk) is what the pool holds: compare with the host flood on the new blockers
        last = {}
        for q in reqs2:
            x, z = float(q["centre_x"]), float(q["centre_z"])
            t = (min(int(z / 4), ch * 64 - 1), min(int(-x / 4), cw * 64 - 1))
            for c in _reach(t, int(q["radius"]), cw, ch):
                last[(int(q["dest"]), c)] = (t, int(q["radius"]))
        for (d, c), (t, rad) in last.items():
            f, _, _ = navs[1].pool_get(d, c)
            assert (f == navs[1].zone_fields(t, rad, [c])[0]).all(), (d, c)
    finally:
        for nav in navs:
            nav.close()


def test_nomem_stop():
    """a request that does not fit stops the batch where the serial loop stops, with the same partial reservations and
    remaining capacity"""
    cw = ch = 4
    cost, inside = _map(cw, ch, 0x5EED0420)
    navs = [_ctx(cw, ch, cost) for _ in range(2)]
    try:
        rng = np.random.default_rng(4)
        centres = _centres(cw, ch, cost, inside, rng, 6)[:9]
        rows = [(i, _xz(t), 20) for i, t in enumerate(centres)]
        need = [len(_reach(t, 20, cw, ch)) for t in centres]
        k = 6
        pool_max = sum(need[:k]) + need[k] - 1                  # request k's last chunk does not fit
        assert need[k] > 1
        reqs = _reqs(rows)
        for nav in navs:
            nav.pool_create(len(rows) + 1, pool_max)
        a = _serial(navs[0], reqs)
        b = _raw(navs[1], reqs)
        assert a[0] == b[0] == capi.ERR_NOMEM and a[1] == b[1] == k
        assert (a[2][:k] == b[2][:k]).all() and (b[2][k:] == 0).all()
        assert _pool(navs[0], len(rows) + 1, cw, ch) == _pool(navs[1], len(rows) + 1, cw, ch)
        # one more single-chunk request: a new (dest, chunk) does not fit on either side; the first chunk request k
        # reserved does, and gets its field
        cr, cc = _reach(centres[k], 20, cw, ch)[0]
        new, held = _reqs([(len(rows), _xz(centres[0]), 0)]), _reqs([(k, _xz((cr * 64 + 32, cc * 64 + 32)), 0)])
        for q, rc in ((new, capi.ERR_NOMEM), (held, 0)):
            assert _serial(navs[0], q)[0] == _raw(navs[1], q)[0] == rc
            assert _pool(navs[0], len(rows) + 1, cw, ch) == _pool(navs[1], len(rows) + 1, cw, ch)
        assert navs[1].pool_get(k, (cr, cc))[0] is not None
    finally:
        for nav in navs:
            nav.close()


def test_bad_arguments_change_nothing():
    """dest, layer, radius, null pointers and a 4 x 1 map: PFNAV_ERR_ARG, ndone == 0, the pool unchanged"""
    cw = ch = 4
    cost, _ = _map(cw, ch, 0x5EED0430)
    nav = _ctx(cw, ch, cost)
    try:
        nav.pool_create(4, 256)
        ok = _reqs([(1, _xz((100, 100)), 8)])
        assert _raw(nav, ok)[:2] == (0, 1)
        before = _pool(nav, 4, cw, ch)
        bad = [_reqs([(4, _xz((10, 10)), 3)]), _reqs([(-1, _xz((10, 10)), 3)]), _reqs([(0, _xz((10, 10)), 3)]),
               _reqs([(0, _xz((10, 10)), -1)]), _reqs([(0, _xz((10, 10)), 0x10000)])]
        bad[2]["layer"] = 1                                             # the map has one layer
        for i, r in enumerate(bad):
            rc, nd, _ = _raw(nav, np.concatenate([ok, r]))
            assert rc == capi.ERR_ARG and nd == 0, i
            assert _pool(nav, 4, cw, ch) == before, i
        nd = C.c_int(-1)
        assert nav.L.pfnav_pool_request_zones(nav.h, None, 2, None, None, C.byref(nd)) == capi.ERR_ARG and nd.value == 0
        assert _raw(nav, ok, nfields=False)[:2] == (0, 1)                # out_nfields may be NULL
        assert _raw(nav, ok[:0])[:2] == (0, 0)
    finally:
        nav.close()
    cost, _ = _map(4, 1, 0x5EED0431, square=False)
    nav = _ctx(4, 1, cost)
    try:
        nav.pool_create(2, 64)
        rc, nd, _ = _raw(nav, _reqs([(0, (-900.0, 100.0), 1), (1, _xz((10, 10)), 3)]))
        assert rc == capi.ERR_ARG and nd == 0 and nav.pool_get(1, (0, 0))[0] is None
        rc, nd, nf = _raw(nav, _reqs([(0, (10.0, 100.0), 1)]))            # off the map only: nothing is requested
        assert (rc, nd, int(nf[0])) == (0, 1, 0)
    finally:
        nav.close()


def test_stream_order_and_hostonly():
    """a clear then a batch on a user stream with no host wait: the batch sees an empty pool. Goal batch, zone batch and
    tick back to back on one stream == the same steps synchronised after each. Host-only context: PFNAV_ERR_NO_DEVICE."""
    import torch
    pf = importlib.import_module("permafrost-engine_b200")
    bench = importlib.import_module("bench")
    bench.set_workload("C2")
    W = bench.build_workload(pf, 1, 0)
    cw = bench.CHUNKS
    ngoals = W["g_hi"] - W["g_lo"]
    dests = np.arange(ngoals, dtype=np.int32)
    targets = np.array([tuple(int(v) for v in W["agents"]["flock_target_tile"][f]) for f in range(W["g_lo"], W["g_hi"])], np.int32)
    rng = np.random.default_rng(6)
    img = synth.blocked_to_image(W["cost"], cw, cw)
    open_ = np.argwhere(img != 0xFF)
    steps = []
    for s in range(3):
        t = open_[rng.integers(0, len(open_), 24)]
        steps.append(_reqs([(int(rng.integers(0, ngoals + 8)), _xz(x), int(rng.choice([4, 8, 16, 32, 80]))) for x in t]))
    results = []
    for sync in (False, True):
        nav = capi.Nav(0)
        try:
            nav.map_create(cw, cw, 1); nav.map_upload_layer(0, W["cost"]); nav.map_build_nav(0)
            nav.pool_create(ngoals + 8, 8192)
            nav.agents_upload_shard(W["rec"][W["lo"]:W["hi"]], W["lo"], W["hi"], W["n_total"], W["flocks"], bench.HZ, 0)
            nav.agents_set_work(np.arange(W["lo"], W["hi"], dtype=np.uint32))
            nav.set_two_phase(2)
            stream = torch.cuda.Stream()
            sp = stream.cuda_stream
            for reqs in steps:
                nav.pool_clear()
                nav.pool_request_goals(dests, targets, 0, sp)
                if sync:
                    torch.cuda.synchronize()
                assert nav.pool_request_zones(reqs, sp)[0] == len(reqs)
                if sync:
                    torch.cuda.synchronize()
                nav.agents_rebuild_index(sp)
                nav.agents_tick(capi.TICK_VDES_FROM_POOL, sp)
                if sync:
                    torch.cuda.synchronize()
            torch.cuda.synchronize()
            nwork = W["hi"] - W["lo"]
            _, vdes, los = nav.agents_read_debug(nwork)
            results.append((_pool(nav, ngoals + 8, cw, cw), vdes, los, nav.agents_read_velocities(nwork)))
            # clear, then a batch on the user stream with no host wait: only this batch's fields are in the pool
            nav.pool_request_zones(steps[0], sp)
            nav.pool_clear()
            nav.pool_request_zones(steps[1], sp)
            stream.synchronize()
            after = _pool(nav, ngoals + 8, cw, cw)
        finally:
            nav.close()
        fresh = capi.Nav(0)
        try:
            fresh.map_create(cw, cw, 1); fresh.map_upload_layer(0, W["cost"]); fresh.map_build_nav(0)
            fresh.pool_create(ngoals + 8, 8192)
            fresh.pool_request_zones(steps[1])
            torch.cuda.synchronize()
            assert _pool(fresh, ngoals + 8, cw, cw) == after
        finally:
            fresh.close()
    (pa, da, la, va), (pb, db, lb, vb) = results
    assert pa == pb
    assert np.array_equal(da, db) and np.array_equal(la, lb) and np.array_equal(va, vb)
    assert (np.abs(da).sum(axis=1) > 0).mean() > 0.5
    host = capi.Nav(hostonly=True)
    try:
        assert _raw(host, _reqs([(0, (-10.0, 10.0), 1)]))[0] == capi.ERR_NO_DEVICE
    finally:
        host.close()
