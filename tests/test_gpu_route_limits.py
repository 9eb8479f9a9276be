"""The device portal-graph search (k_portal_graph_path_warp) where it gives up, and what the product path does then, on
two 32 x 32-chunk maps:
  S  cases.serpentine_cost: every route forced through one gap per chunk-row boundary, up to 1 984 hops and LOS chains
     1 024 chunks deep (its host plans are pinned by tests/test_route_limits_host.py);
  P  cases.portal_grid_cost: 15 808 portals (16 per interior chunk) and a walled-off 2 x 2-chunk region with portals of
     its own, so a search toward the region exhausts the whole graph.
The kernel returns status -1 when a search outgrows its scratch (GP_PQ heap entries, GP_HT * 3 / 4 table keys) or its
path has more than max_hops hops; a search round of pfnav_pool_request_paths then runs the host routine for it. Checked:
the -1 contract against the host routine, a >= 256-request batch (the device search tier, fallbacks included) against
the same requests one at a time, and the longest route's and goal batch's pool fields against the plain-C port."""
import numpy as np
import pytest

import cases
import test_gpu_request_paths as rp
import test_gpu_route_dev as rd

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
CW = CH = 32
REGION = ((14, 14), (2, 2))
FULL_HOPS = 4096                    # longer than any path on these maps: the host routine's whole path


def _nav(cost, cw=CW, ch=CH, ndests=1, pool_max=1):
    nav = rp._nav(cost, cw, ch, None, ndests, pool_max)
    ports = nav.portals(0)
    nav.portals_of = lambda c: ports[(ports[:, 0] * cw + ports[:, 1]) == c]
    return nav


def _in_region(chunk):
    (r0, c0), (nr, nc) = REGION
    return r0 <= chunk // CW < r0 + nr and c0 <= chunk % CW < c0 + nc


def _contract(nav, req, max_hops, outgrow):
    """route_graph_paths on the device against the host routine. A device -1 is accepted when the host's whole path has
    more than max_hops hops, or for a search marked in `outgrow` (one that may explore more nodes than the scratch
    holds); every other search equals the host's at max_hops (status, cost bits, every hop).
    -> (# -1 by hop count, device -1 without a too-long path, per search)"""
    st_d, cost_d, hops_d = nav.route_graph_paths(req, max_hops, True)
    st_h, cost_h, hops_h = nav.route_graph_paths(req, max_hops, False)
    st_f, _, hops_f = nav.route_graph_paths(req, FULL_HOPS, False)
    assert (st_f >= 0).all()
    too_long = (st_f == 1) & np.array([len(h) > max_hops for h in hops_f])
    assert np.array_equal(st_h == -1, too_long)                 # the host routine keeps the same limit
    neg = st_d == -1
    bad = np.nonzero(neg & ~too_long & ~outgrow)[0]
    assert len(bad) == 0, ("device -1 without cause", bad[:10], req[bad[:3]])
    same = ~neg
    assert np.array_equal(st_d[same], st_h[same]), np.nonzero(same & (st_d != st_h))[0][:10]
    assert np.array_equal(cost_d.view(np.uint32)[same], cost_h.view(np.uint32)[same])
    for i in np.nonzero(same)[0]:
        assert np.array_equal(hops_d[i], hops_h[i]), (i, req[i])
    assert (st_h[same] == 1).sum() > 0
    return int((neg & too_long).sum()), neg & ~too_long


@pytest.mark.parametrize("which,max_hops", [("S", 512), ("C2", 16), ("P", 512)])
def test_graph_paths_minus_one_contract(which, max_hops):
    rng = np.random.default_rng({"S": 1, "C2": 2, "P": 3}[which])
    if which == "S":
        nav = _nav(cases.serpentine_cost(CW, CH))
        req = rd._searches(nav, None, CW, CH, rng, 600)
        exhausting = np.zeros(len(req), bool)
    elif which == "C2":
        nav = _nav(rp._map(16, 16, 0, c2=True), 16, 16)
        req = rd._searches(nav, None, 16, 16, rng, 600)
        exhausting = np.zeros(len(req), bool)
    else:
        nav = _nav(cases.portal_grid_cost(CW, CH, region=REGION))
        # searches to chunks at most two chunks away (a few hundred nodes explored) ...
        req = []
        while len(req) < 500:
            s = int(rng.integers(CW * CH))
            er, ec = s // CW + int(rng.integers(-2, 3)), s % CW + int(rng.integers(-2, 3))
            if not (0 <= er < CH and 0 <= ec < CW) or _in_region(s) != _in_region(er * CW + ec):
                continue
            e = er * CW + ec
            req.append([s, int(rng.integers(64)), int(rng.integers(64)), e, int(rng.integers(64)), int(rng.integers(64)), e,
                        int(rng.integers(len(nav.portals_of(e))))])
        req = np.array(req, np.int32)
        # ... and from outside the walled-off region to portals inside it: no path, the search exhausts the graph
        inside = [c for c in range(CW * CH) if _in_region(c)]
        ex = []
        while len(ex) < 24:
            s = int(rng.integers(CW * CH))
            if _in_region(s):
                continue
            e = inside[len(ex) % len(inside)]
            ex.append([s, int(rng.integers(64)), int(rng.integers(64)), e, 32, 32, e, int(rng.integers(len(nav.portals_of(e))))])
        # ... and reachable searches 10 to 62 chunks long: the longer ones explore more nodes than the scratch holds
        far = []
        while len(far) < 48:
            s, e = int(rng.integers(CW * CH)), int(rng.integers(CW * CH))
            dist = abs(s // CW - e // CW) + abs(s % CW - e % CW)
            if _in_region(s) or _in_region(e) or dist < 10 + len(far):
                continue
            far.append([s, int(rng.integers(64)), int(rng.integers(64)), e, int(rng.integers(64)), int(rng.integers(64)), e,
                        int(rng.integers(len(nav.portals_of(e))))])
        req = np.concatenate([req, np.array(ex, np.int32), np.array(far, np.int32)])
        exhausting = np.zeros(len(req), bool); exhausting[len(req) - len(far) - len(ex):len(req) - len(far)] = True
        is_far = np.zeros(len(req), bool); is_far[len(req) - len(far):] = True
    try:
        by_hops, scratch = _contract(nav, req, max_hops, exhausting | (is_far if which == "P" else False))
        print(f"{which} max_hops={max_hops}: {len(req)} searches, device -1 by hop count {by_hops}, by scratch "
              f"{int(scratch.sum())}")
        if which == "P":
            print(f"P: toward the walled-off region {int(scratch[exhausting].sum())} of {int(exhausting.sum())} -1; "
                  f"far reachable searches {int(scratch[is_far].sum())} of {int(is_far.sum())} -1, the rest identical")
            assert scratch[exhausting].sum() >= 1
            assert (~scratch[is_far]).sum() >= 10       # far searches the device answered, compared hop by hop
        else:
            assert by_hops >= 1 and not scratch.any()
    finally:
        nav.close()


def _far_requests(cost, n, targets, rng, opposite=False):
    """n requests, round robin over the dests of `targets` ((chunk, r, c) each): sources on passable tiles outside the
    target's chunk; opposite=True: every other source in the chunk diagonally opposite the target's"""
    pas = np.argwhere(cost != 255)
    dests = np.arange(n, dtype=np.int32) % len(targets)
    src, dst = np.zeros((n, 2), np.float32), np.zeros((n, 2), np.float32)
    for i in range(n):
        c, r, cc = targets[dests[i]]
        dst[i] = synth.tile_center_xz(c // CW, c % CW, r, cc)
        while True:
            s = pas[rng.integers(len(pas))]
            if opposite and i % 2:
                s = (CH - 1 - c // CW) * CW + CW - 1 - c % CW, int(rng.integers(8, 56)), int(rng.integers(8, 56))
            if s[0] != c:
                break
        src[i] = synth.tile_center_xz(int(s[0]) // CW, int(s[0]) % CW, int(s[1]), int(s[2]))
    return dests, src, dst


def _fell_back(nav, dests, src, dst, max_hops=512):
    """requests whose search the device certainly gives up: -1 toward every portal of the target chunk (the search round
    sends the device one of them). Requests into or out of the walled-off region of P are not searched at all (the
    global-island test comes first) and are not counted."""
    req, owner = [], []
    for i in range(len(dests)):
        sr, sc = synth.tile_for_xz(np.float32(src[i, 0]), np.float32(src[i, 1]), CW, CH)
        tr, tc = synth.tile_for_xz(np.float32(dst[i, 0]), np.float32(dst[i, 1]), CW, CH)
        s, e = int(sr // 64) * CW + int(sc // 64), int(tr // 64) * CW + int(tc // 64)
        if _in_region(s) != _in_region(e):
            continue
        for p in range(len(nav.portals_of(e))):
            req.append([s, int(sr % 64), int(sc % 64), e, int(tr % 64), int(tc % 64), e, p]); owner.append(i)
    st, _, _ = nav.route_graph_paths(np.array(req, np.int32), max_hops, True)
    owner = np.array(owner)
    return int(sum(((st[owner == i] == -1).all()) for i in np.unique(owner)))


def _port_route(om, nav_host, src, dst):
    """the host plan of one request on an empty dest, executed by the port -> (expected pool entries by chunk, LOS depth)"""
    ok, _, fr, fid, fc, lr, lc = nav_host.route_request_path(src, dst)
    fields, los = cases.execute_route(lambda r, io: om.flow_fields_update(r, inout=io), om.los_fields_create, fr, fc, lr, lc)
    last_id = {int(fc[i]): int(fid[i]) for i in range(len(fr))}
    return ok, fields, los, last_id, int(cases.los_depths(lr).max())


@pytest.mark.parametrize("which", ["S", "P"])
def test_request_paths_fallback_equals_serial(which, pforacle):
    """320 requests in one pfnav_pool_request_paths batch (its search round runs on the device, the searches it gives up
    on the host) against the same requests issued one at a time on a twin context: ok, dest_id, flow and LOS counts,
    and every pool entry (has bits, ff_id, flow and LOS bytes) identical. On S, dest 0 holds the corner-to-corner route
    alone: its flow fields and its 993-deep LOS chain equal the host plan executed by the plain-C port."""
    cost = cases.serpentine_cost(CW, CH) if which == "S" else cases.portal_grid_cost(CW, CH, region=REGION)
    rng = np.random.default_rng(17 if which == "S" else 18)
    pas = np.argwhere(cost != 255)
    ndests, n = 6, 320
    targets = [tuple(int(v) for v in pas[rng.integers(len(pas))]) for _ in range(ndests)]
    if which == "P":
        r0, c0 = REGION[0]
        targets[-1] = (r0 * CW + c0, 30, 30)               # inside the walled-off region: unreachable from outside
    dests, src, dst = _far_requests(cost, n, targets, rng, opposite=which == "P")
    if which == "S":                                         # dest 0: only the corner-to-corner request
        corner = np.array([synth.tile_center_xz(0, 0, 10, 10)], np.float32), np.array([synth.tile_center_xz(31, 31, 50, 50)], np.float32)
        keep = dests != 0
        dests = np.concatenate([[0], dests[keep]]).astype(np.int32)
        src, dst = np.concatenate([corner[0], src[keep]]), np.concatenate([corner[1], dst[keep]])
    navs = [_nav(cost, ndests=ndests, pool_max=ndests * CW * CH) for _ in range(2)]
    try:
        nfb = _fell_back(navs[0], dests, src, dst)
        ok, nf, nl = rp._compare(navs[0], navs[1], dests, src, dst, ndests, CW * CH)
        assert len(dests) >= 256 and ok.any() and nf.sum() > 0 and nl.sum() > 0
        if which == "P":
            assert not ok.all()                              # the region's requests
        print(f"{which}: {len(dests)} requests, {nfb} certainly fell back to the host search, {int(nf.sum())} flow and "
              f"{int(nl.sum())} LOS fields built")
        assert nfb >= 10
        if which == "S":
            host = capi.Nav(hostonly=True)
            host.map_create(CW, CH, 1); host.map_upload_layer(0, cost); host.map_build_nav(0); host.route_build(0)
            om = pforacle.OracleMap(CW, CH, cost, None, navs[0].local_islands(0))
            try:
                ok0, fields, los, last_id, depth = _port_route(om, host, tuple(src[0]), tuple(dst[0]))
            finally:
                host.close()
            assert ok0 and depth == 993 and len(fields) == 993
            for c in range(CW * CH):
                f, l, ffid = navs[0].pool_get(0, divmod(c, CW))
                assert (f is not None) == (c in fields) and (l is not None) == (c in los), c
                if f is not None:
                    assert np.array_equal(f, fields[c]) and ffid == last_id[c], c
                    assert np.array_equal(l, los[c]), c
            print(f"S corner-to-corner: {len(fields)} flow and {len(los)} LOS fields equal the port, LOS chain depth {depth}")
    finally:
        rp._close(navs)


def test_goal_batch_longest_chain_vs_port(pforacle):
    """a cold pfnav_pool_request_goals on S, three goals (one of them in the top-left chunk: a single LOS chain through
    all 1 024 chunks), against the port running plan_goal's waves; then the same batch again (the resident-plan path),
    which must launch its waves again and leave the same pool. Every host write to the pool drops the resident plan, so
    the relaunch can only be checked over the bytes the cold call left."""
    cost = cases.serpentine_cost(CW, CH)
    targets = np.array([[0, 0, 10, 10], [31, 31, 50, 50], [15, 16, 30, 30]], np.int32)
    ng = len(targets)
    nav = _nav(cost, ndests=ng, pool_max=ng * CW * CH)
    try:
        om = pforacle.OracleMap(CW, CH, cost, None, nav.local_islands(0))
        exp = [cases.port_goal_fields(nav, om, t) for t in targets]
        depth = max(int(cases.los_depths(e[2]).max()) for e in exp)
        assert depth == CW * CH
        for call in range(2):                              # cold, then the resident plan
            l0 = nav.launch_count()
            nf, nl = nav.pool_request_goals(np.arange(ng, dtype=np.int32), targets)
            assert nav.launch_count() > l0, call           # the resident plan is relaunched, not skipped
            assert nf == sum(e[3] for e in exp) and nl == sum(len(e[1]) for e in exp), (call, nf, nl)
            ncmp = cases.check_goal_pool(nav, exp, CW, CW * CH)
            print(f"S goal batch call {call}: {ncmp} fields equal the port, longest LOS chain {depth}")
    finally:
        nav.close()
