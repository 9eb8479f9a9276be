"""pfnav_pool_request_paths (a batch of N_RequestPath calls against the field pool) against the same requests issued one
by one through pfnav_pool_request_path on a second context with the same map. The serial path is pinned to the
reference's field cache by test_pool_request_path_golden and test_c2_desired_velocity_from_pool_vs_reference.
Per request: ok, dest_id, n_flow and n_los identical; per (dest, chunk): has bits, ff_id, flow and LOS bytes identical.
Also the warp-per-search portal-graph kernel at C2 scale against the host routine, and the argument checks (CPU)."""
import ctypes as C

import numpy as np
import pytest

import cases

capi, synth = cases.capi, cases.synth


def _world(gr, gc):
    """centre of global tile (row, column) as (x, z) on a map at (0, 0)"""
    return (-(gc * 4.0 + 2.0), gr * 4.0 + 2.0)


def _map(cw, ch, seed, c2=False):
    if c2:
        import bench
        bench.set_workload("C2")
        return synth.cost_from_pathable(synth.make_map(bench.CHUNKS, bench.CHUNKS, bench.MAP_SEED, rivers=True),
                                        bench.CHUNKS, bench.CHUNKS)
    return synth.cost_from_pathable(cases.noise_map(cw, ch, seed, 0.0), cw, ch)


def _blocker_ops(cw, ch, n, seed):
    rng = np.random.default_rng(seed)
    ops = np.zeros(n, capi.BLOCKER_OP)
    ops["x"] = -rng.uniform(4, cw * 256 - 4, n); ops["z"] = rng.uniform(4, ch * 256 - 4, n)
    ops["range"] = rng.choice([3.0, 6.0, 10.0], n); ops["flags"] = capi.FLAG_MOVABLE; ops["delta"] = 1
    ops["faction_id"] = rng.choice([0, 2, 5], n)
    return ops


def _nav(cost, cw, ch, ops, ndests, pool_max):
    nav = capi.Nav(0)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    if ops is not None and len(ops):
        nav.blockers_batch(ops)
        assert nav.map_commit() > 0
    nav.pool_create(ndests, pool_max)
    return nav


def _requests(cost, cw, ch, n, ndests, seed):
    """dest d has one target tile; each request names a dest and a source. Sources: any tile (blocked ones, other global
    islands included), a quarter of them in the target's own chunk."""
    rng = np.random.default_rng(seed)
    H, W = ch * 64, cw * 64
    g = cost.reshape(ch, cw, 64, 64).transpose(0, 2, 1, 3).reshape(H, W)
    passable = np.argwhere(g != 255)
    targets = [tuple(passable[rng.integers(len(passable))]) if rng.random() < 0.85 else (int(rng.integers(H)), int(rng.integers(W)))
               for _ in range(ndests)]
    dests = rng.integers(0, ndests, n).astype(np.int32)
    src, dst = np.zeros((n, 2), np.float32), np.zeros((n, 2), np.float32)
    for i in range(n):
        tr, tc = targets[dests[i]]
        dst[i] = _world(tr, tc)
        u = rng.random()
        if u < 0.25:                      # same chunk as the target
            sr, sc = (tr // 64) * 64 + int(rng.integers(64)), (tc // 64) * 64 + int(rng.integers(64))
        elif u < 0.85:
            sr, sc = passable[rng.integers(len(passable))]
        else:                             # anywhere, blocked tiles included
            sr, sc = int(rng.integers(H)), int(rng.integers(W))
        src[i] = _world(sr, sc)
    return dests, src, dst


def _serial(nav, dests, src, dst):
    """pool_request_path in a loop, stopped at the first PFNAV_ERR_NOMEM -> (ok, dest_id, n_flow, n_los, ndone)"""
    n = len(dests)
    ok, nf, nl, did = np.zeros(n, bool), np.zeros(n, np.int32), np.zeros(n, np.int32), np.zeros(n, np.uint32)
    for i in range(n):
        try:
            ok[i], did[i], nf[i], nl[i] = nav.pool_request_path(int(dests[i]), tuple(src[i]), tuple(dst[i]))
        except capi.PfnavError as e:
            assert "pool full" in str(e), e
            return ok, did, nf, nl, i
    return ok, did, nf, nl, n


def _pool(nav, ndests, chunks):
    """every (dest, chunk) entry: has bits, ff_id, flow and LOS bytes"""
    out = []
    for d in range(ndests):
        for c in range(chunks):
            f, l, ffid = nav.pool_get(d, divmod(c, nav.cw))
            out.append(((f is not None) | ((l is not None) << 1), ffid, None if f is None else f.tobytes(), None if l is None else l.tobytes()))
    return out


def _compare(batch_nav, serial_nav, dests, src, dst, ndests, chunks, expect_nomem=False):
    ok_s, did_s, nf_s, nl_s, done_s = _serial(serial_nav, dests, src, dst)
    ok_b, did_b, nf_b, nl_b, done_b = batch_nav.pool_request_paths(dests, src, dst)
    assert done_b == done_s
    assert (done_s < len(dests)) == expect_nomem, (done_s, len(dests))
    k = done_s
    assert np.array_equal(ok_b[:k], ok_s[:k]) and np.array_equal(did_b[:k], did_s[:k])
    assert np.array_equal(nf_b[:k], nf_s[:k]) and np.array_equal(nl_b[:k], nl_s[:k])
    pb, ps = _pool(batch_nav, ndests, chunks), _pool(serial_nav, ndests, chunks)
    bad = [i for i in range(len(pb)) if pb[i] != ps[i]]
    assert not bad, [(divmod(i, chunks), pb[i][:2], ps[i][:2]) for i in bad[:5]]
    return ok_s[:k], nf_s[:k], nl_s[:k]


def _case(cw, ch, seed, nblockers, n, ndests, pool_max, warm=8, faction=None, c2=False):
    cost = _map(cw, ch, seed, c2)
    ops = _blocker_ops(cw, ch, nblockers, seed + 1) if nblockers else None
    navs = [_nav(cost, cw, ch, ops, ndests, pool_max) for _ in range(2)]
    dests, src, dst = _requests(cost, cw, ch, n + warm, ndests, seed + 2)
    for nav in navs:                                   # part of the pool is warm before the batch
        if faction is not None:                        # attacking requests: blockers of factions 0 and 5 are enemies
            nav.set_enemy_factions(faction, (1 << 0) | (1 << 5))
            nav.request_faction(faction)
        for i in range(warm):
            nav.pool_request_path(int(dests[i]), tuple(src[i]), tuple(dst[i]))
    return navs, cost, (dests[warm:], src[warm:], dst[warm:])


def _close(navs):
    for nav in navs:
        nav.close()


def _assert_coverage(ok, nf, nl, dests):
    assert ok.any() and not ok.all()                   # paths found, and requests across global islands
    assert nf.sum() > 0 and nl.sum() > 0
    assert len(np.unique(dests)) < len(dests)          # dests shared between requests


@pytest.mark.gpu
@pytest.mark.parametrize("cw,ch,seed,nblockers,n,ndests,faction", [
    (4, 4, 11, 0, 96, 12, None),
    (4, 4, 12, 300, 96, 12, 3),
    (8, 8, 13, 800, 160, 16, None),
])
def test_batch_equals_serial(cw, ch, seed, nblockers, n, ndests, faction):
    navs, _, (dests, src, dst) = _case(cw, ch, seed, nblockers, n, ndests, ndests * cw * ch, faction=faction)
    ok, nf, nl = _compare(navs[0], navs[1], dests, src, dst, ndests, cw * ch)
    _assert_coverage(ok, nf, nl, dests)
    _close(navs)


@pytest.mark.gpu
def test_batch_equals_serial_c2():
    navs, _, (dests, src, dst) = _case(16, 16, 21, 800, 1024, 48, 48 * 256, warm=16, c2=True)
    ok, nf, nl = _compare(navs[0], navs[1], dests, src, dst, 48, 256)
    _assert_coverage(ok, nf, nl, dests)
    _close(navs)


@pytest.mark.gpu
def test_batch_pool_pressure():
    """a pool far smaller than the batch's fields: slots are evicted and handed out again inside the batch"""
    ndests = 12
    navs, _, (dests, src, dst) = _case(8, 8, 31, 200, 120, ndests, 40)
    _compare(navs[0], navs[1], dests, src, dst, ndests, 64)
    _close(navs)


@pytest.mark.gpu
def test_batch_nomem_stops_like_serial():
    """a request needing more fields than the pool holds: ndone, the return code and the pool equal the serial loop
    stopped at its first failure"""
    ndests = 6
    navs, _, (dests, src, dst) = _case(8, 8, 41, 0, 80, ndests, 6, warm=0)
    _compare(navs[0], navs[1], dests, src, dst, ndests, 64, expect_nomem=True)
    rc = navs[0].L.pfnav_pool_request_paths(navs[0].h, len(dests), capi._p(dests), 0, capi._p(src), capi._p(dst), None,
                                            None, None, None, None, C.byref(C.c_int(0)))
    assert rc == capi.ERR_NOMEM
    _close(navs)


@pytest.mark.gpu
def test_batch_bad_arguments_change_nothing():
    ndests = 4
    navs, _, (dests, src, dst) = _case(4, 4, 51, 0, 16, ndests, 64)
    nav = navs[0]
    before, launches = _pool(nav, ndests, 16), nav.launch_count()
    for d, s in ((np.where(np.arange(16) == 7, ndests, dests), src), (dests, np.where(np.arange(16)[:, None] == 9, 50.0, src))):
        d, s = np.ascontiguousarray(d, np.int32), np.ascontiguousarray(s, np.float32)
        rc = nav.L.pfnav_pool_request_paths(nav.h, 16, capi._p(d), 0, capi._p(s), capi._p(dst), None, None, None, None, None, None)
        assert rc == capi.ERR_ARG
    assert nav.L.pfnav_pool_request_paths(nav.h, -1, None, 0, None, None, None, None, None, None, None, None) == capi.ERR_ARG
    assert _pool(nav, ndests, 16) == before and nav.launch_count() == launches
    _close(navs)


@pytest.mark.gpu
@pytest.mark.parametrize("n,device", [(4, False), (1024, True)])
def test_batch_search_side_of_k(n, device):
    """a batch whose search round holds fewer searches than the device threshold searches on the host; a large one on
    the device. Every request has a destination of its own; re-issued, the requests whose fields are all pooled (a path
    that merges twice into one chunk is not among them) launch nothing but their searches."""
    cost = _map(16, 16, 0, c2=True)
    navs = [_nav(cost, 16, 16, None, n, 40000) for _ in range(2)]
    _, src, dst = _requests(cost, 16, 16, n, n, 62)
    dests = np.arange(n, dtype=np.int32)
    ok_s, did_s, nf_s, nl_s, done_s = _serial(navs[1], dests, src, dst)
    ok, did, nf, nl, done = navs[0].pool_request_paths(dests, src, dst)
    assert done == done_s == n and np.array_equal(ok, ok_s) and np.array_equal(did, did_s)
    assert np.array_equal(nf, nf_s) and np.array_equal(nl, nl_s) and nf.sum() > 0
    _, _, nf_r, nl_r, _ = _serial(navs[1], dests, src, dst)          # what a re-issue emits, request by request
    keep = (nf_r == 0) & (nl_r == 0)
    assert keep.sum() >= 0.75 * n
    nav = navs[0]
    l0 = nav.launch_count()
    ok2, _, nf2, nl2, done = nav.pool_request_paths(dests[keep], src[keep], dst[keep])
    assert done == keep.sum() and np.array_equal(ok2, ok[keep]) and nf2.sum() == 0 and nl2.sum() == 0
    assert (nav.launch_count() > l0) == device
    _close(navs)


@pytest.mark.gpu
def test_portal_graph_paths_device_equals_host_c2():
    """k_portal_graph_path_warp: 4096 searches on the C2 map with committed blockers, identical to the host routine"""
    import test_gpu_route_dev as rd
    cost = _map(16, 16, 0, c2=True)
    nav = _nav(cost, 16, 16, _blocker_ops(16, 16, 800, 71), 1, 1)
    ports = nav.portals(0)
    nav.portals_of = lambda c: ports[(ports[:, 0] * 16 + ports[:, 1]) == c]
    req = rd._searches(nav, cost, 16, 16, np.random.default_rng(72), 4096)
    st_d, cost_d, hops_d = nav.route_graph_paths(req, 512, True)
    st_h, cost_h, hops_h = nav.route_graph_paths(req, 512, False)
    assert (st_h >= 0).all() and (st_d == st_h).all(), np.nonzero(st_d != st_h)[0][:10]
    assert (cost_d.view(np.uint32) == cost_h.view(np.uint32)).all()
    for i in range(len(req)):
        assert np.array_equal(hops_d[i], hops_h[i]), (i, req[i])
    assert int((st_h == 1).sum()) >= 1000
    nav.close()


def test_request_paths_host_only_and_bad_arguments():
    """on a host-only context: malformed arguments are PFNAV_ERR_ARG, a well-formed batch PFNAV_ERR_NO_DEVICE"""
    cw = ch = 2
    cost = _map(cw, ch, 81)
    nav = capi.Nav(hostonly=True)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    dests, src, dst = _requests(cost, cw, ch, 8, 2, 82)
    call = lambda n, d, s, t, layer=0: nav.L.pfnav_pool_request_paths(
        nav.h, n, capi._p(d), layer, capi._p(s), capi._p(t), None, None, None, None, None, None)
    assert call(8, dests, src, dst) == capi.ERR_NO_DEVICE
    assert call(-1, dests, src, dst) == capi.ERR_ARG
    assert call(8, np.where(np.arange(8) == 3, -1, dests).astype(np.int32), src, dst) == capi.ERR_ARG
    outside = src.copy(); outside[5] = (10.0, 10.0)
    assert call(8, dests, outside, dst) == capi.ERR_ARG
    assert call(8, dests, src, outside) == capi.ERR_ARG
    assert call(8, dests, src, dst, layer=1) == capi.ERR_ARG
    assert call(8, None, src, dst) == capi.ERR_ARG
    nav.close()
