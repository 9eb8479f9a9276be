"""GPU suite: arrived()'s constants built on the device per used (flock, layer) pair (pfnav_agents_read_arrival_consts)
against the host routine pfnav_route_arrival_consts, after upload and after blocker commits that move the map epoch;
pfnav_agents_compute_updates returning while its stream is still busy; and pfnav_map_query searches that leave the
128 x 128 window, finished on the device by the whole-layer tier, against the host routine."""
import numpy as np
import pytest

import cases
import map_query_cases as mq

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth


def _expect_table(nav, fl, table):
    assert len(table) > 0
    for r in table:
        ok, nearest, mc = nav.route_arrival_consts(fl["target"][r["flock"]], int(r["layer"]))
        assert r["nearest_ok"] == ok, (r["flock"], r["layer"])
        if ok:
            assert tuple(r["nearest"]) == tuple(nearest), (r["flock"], r["nearest"], nearest)
        assert r["mc_n"] == len(mc) and (r["mc"][:len(mc)] == mc).all(), (r["flock"], r["mc_n"], len(mc))


def _setup(nav, seed=4242, hz=20):
    p, cost, a, ms = cases.update_case(seed, hz)
    rec, fl = capi.pack_agents(a)
    img = synth.blocked_to_image(cost, 3, 3)
    imp = np.argwhere(img == 255)
    # flock 2 aims at an impassable tile too: with flock 1, the window tiers and their blocked-target path
    if len(imp):
        r, c = imp[len(imp) // 2]
        fl["target"][2] = mq.tile_xz(int(r), int(c))
    nav.map_create(3, 3, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    nav.agents_upload(rec, fl, hz)
    nav.agents_upload_movestate(ms)
    work = np.arange(len(a["radius"]), dtype=np.uint32)
    nav.agents_set_work(work)
    return a, fl, img


def test_arrival_table_vs_host(nav):
    a, fl, img = _setup(nav)
    nav.agents_tick(0)
    nav.agents_compute_updates()
    _expect_table(nav, fl, nav.agents_read_arrival_consts())
    # blockers next to the targets, committed: the epoch moves and the table is rebuilt from the new blocker counts
    for k in range(len(fl)):
        x, z = fl["target"][k]
        nav.blockers_incref(float(x) - 4.0, float(z) + 4.0, 6.0)
    nav.map_commit()
    nav.agents_tick(0)
    nav.agents_compute_updates()
    _expect_table(nav, fl, nav.agents_read_arrival_consts())


def _far_case(nav):
    """update_case's agents on the top-left 3 x 3 chunks of an 8 x 8 map whose lower right holds a 200 x 200 impassable
    blob, with four more flocks (members taken from the first three) whose targets need the later tiers:
      3  70 tiles from the nearest pathable tile: N_ClosestPathable leaves the 128 x 128 window (whole-layer tier)
      4  a one-tile island in the blob: its island list is empty, so the search leaves every window (whole-layer tier)
      5  20 tiles from the nearest pathable tile: N_ClosestPathable leaves the 32 x 32 window only (128 tier)
      6  the end of a corridor that blockers cover for 90 tiles: the blockers move its list to the blob's edge
    -> agents dict, flock table, the corridor blockers"""
    p, cost, a, ms = cases.update_case(4243, 20)
    img = np.ones((512, 512), np.uint8)
    img[:192, :192] = synth.blocked_to_image(cost, 3, 3)
    img[250:450, 250:450] = 0xFF
    img[265, 300] = 1
    img[260, 340:451] = 1
    n = len(a["radius"])
    rng = np.random.default_rng(7)
    a["flock_target"] = np.concatenate([a["flock_target"], np.array([mq.tile_xz(380, 350), mq.tile_xz(265, 300),
                                        mq.tile_xz(280, 350), mq.tile_xz(260, 340)], np.float32)]).astype(np.float32)
    movers = rng.permutation(np.nonzero(a["flock_of"] >= 0)[0])
    for k, f in enumerate((3, 4, 5, 6)):
        a["flock_of"][movers[8 * k:8 * k + 8]] = f
    rec, fl = capi.pack_agents(a)
    fl["dest"] = np.minimum(fl["dest"], 2)           # the new flocks share the first three goals
    nav.map_create(8, 8, 1); nav.map_upload_layer(0, synth.image_to_blocked(img, 8, 8)); nav.map_build_nav(0); nav.route_build(0)
    nav.agents_upload(rec, fl, 20)
    nav.agents_upload_movestate(ms)
    nav.agents_set_work(np.arange(n, dtype=np.uint32))
    blockers = [(*mq.tile_xz(260, c), 6.0) for c in range(341, 432, 2)]
    return a, fl, blockers


def test_arrival_table_later_tiers(nav):
    """flock targets that take the 128 and whole-layer tiers, before and after blocker commits that move the map epoch
    (a rebuild that skipped a dirtied epoch would keep the corridor's old list)"""
    a, fl, blockers = _far_case(nav)
    nav.agents_tick(0)
    nav.agents_compute_updates()
    t0 = nav.agents_read_arrival_consts()
    _expect_table(nav, fl, t0)
    assert {3, 4, 5, 6} <= set(t0["flock"].tolist())
    for b in blockers:
        nav.blockers_incref(*b)
    nav.map_commit()
    with pytest.raises(capi.PfnavError):
        nav.agents_read_arrival_consts()         # the committed map changed: the table is not current
    nav.agents_tick(0)
    nav.agents_compute_updates()
    t1 = nav.agents_read_arrival_consts()
    _expect_table(nav, fl, t1)
    c0, c1 = (t[t["flock"] == 6][0] for t in (t0, t1))
    assert c0["mc_n"] > 0 and c1["mc_n"] > 0 and (c0["mc"][0] != c1["mc"][0]).any(), "the blockers move the corridor's list"
    ok, nearest, mc = nav.route_arrival_consts(fl["target"][3])
    assert ok == 1 and abs(float(nearest[1]) - float(fl["target"][3][1])) > 64 * 4, "flock 3 needs the whole layer"
    for b in blockers[::2]:
        nav.blockers_decref(*b)
    nav.map_commit()
    nav.agents_tick(0)
    nav.agents_compute_updates()
    _expect_table(nav, fl, nav.agents_read_arrival_consts())


def test_compute_updates_does_not_wait(nav):
    torch = pytest.importorskip("torch")
    a, fl, img = _setup(nav)
    st = torch.cuda.current_stream()
    nav.agents_tick(0, stream=st.cuda_stream)
    nav.agents_compute_updates(stream=st.cuda_stream)
    torch.cuda.synchronize()
    x, z = fl["target"][0]
    nav.blockers_incref(float(x), float(z), 5.0)
    nav.map_commit()
    torch.cuda._sleep(200_000_000)              # a bounded spin on the stream, about 0.1 s
    nav.agents_compute_updates(stream=st.cuda_stream)
    busy = not st.query()
    torch.cuda.synchronize()
    assert busy, "compute_updates waited for its stream"
    _expect_table(nav, fl, nav.agents_read_arrival_consts())


def test_map_query_whole_layer_tier(nav):
    """the window-overflow blob of the CPU tests, on the device: both flagged searches and more inside the blob"""
    cw = ch = 4
    img = np.zeros((256, 256), np.uint8) + 1
    img[28:228, 28:228] = 0xFF
    img[60, 128] = 1
    img[200, 40] = 1
    cost_c = synth.image_to_blocked(img, cw, ch)
    nav.map_create(cw, ch, 1); nav.map_upload_layer(0, cost_c); nav.map_build_nav(0); nav.route_build(0)
    tiles = [(128, 128), (60, 128), (200, 40), (100, 200), (227, 28), (150, 60)]
    q = []
    for r, c in tiles:
        x, z = mq.tile_xz(r, c)
        q.append((capi.QUERY_CLOSEST_PATHABLE, 0, x, z, 0, 0, 0, 0))
        for tol in (0.0, 6.0, 300.0):
            q.append((capi.QUERY_MAXIMALLY_CLOSE, 0, x + 3.0, z - 250.0, x, z, tol, 0))
    q = np.array(q, capi.MAP_QUERY)
    got = nav.map_query(q)
    for i, e in enumerate(q):
        if e["kind"] == capi.QUERY_CLOSEST_PATHABLE:
            ok, nearest, _ = nav.route_arrival_consts((e["x"], e["z"]))
            assert got[i]["ok"] == ok and (not ok or (got[i]["x"], got[i]["z"]) == tuple(nearest)), (i, got[i], nearest)
        else:
            _, _, mc = nav.route_arrival_consts((e["dst_x"], e["dst_z"]))
            d = np.sqrt(((mc - np.array([e["x"], e["z"]], np.float32)) ** 2).sum(axis=1)).astype(np.float32)
            assert got[i]["ok"] == int(bool(len(mc)) and bool((d <= e["tolerance"]).any())), (i, got[i], len(mc))
