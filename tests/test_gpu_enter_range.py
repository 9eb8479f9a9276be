"""GPU suite: STATE_ENTER_ENTITY_RANGE's maximally-close stop (movement.c:2583-2584) decided on the device.

k_entity_update appends the items whose stop depends on N_IsMaximallyClose(new_pos, target, 0); k_enter_window and
k_enter_layer search the target's tile list and finish their patches. These tests build every branch by construction on
a 4 x 4-chunk map with test_map_query_whole_layer_tier's blob, and compare with the plain-C port fed the host lists
(pfnav_route_arrival_consts), the rule the host used to apply:
  - units standing exactly on a listed tile position next to impassable terrain (stop through the list), the same
    position one float off (no stop), and a listed position away from impassable terrain (not a candidate);
  - a target on a blocked tile, and a target at the end of a blocker-covered corridor into the blob, whose list lies more
    than 64 tiles away (the whole-layer tier);
  - a target on a one-tile island (empty list, whole-layer tier), NULL and self targets, and the re-issued order.
Units have no desired velocity, so nothing moves and every patch is compared bit for bit."""
import numpy as np
import pytest

import cases
import map_query_cases as mq

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
ST_ARRIVED, ST_WAITING, ST_ENTER = 2, 4, 6
UPDATE_SET_DEST = 1 << 10             # PFNAV_UPDATE_SET_DEST
CW = CH = 4
NLAYERS = 9
LAYER_FLAGS = {0: 0, 4: capi.FLAG_WATER, 8: capi.FLAG_AIR}
OFFSET = (130.3, -61.7)              # not a multiple of the 4 wu tile


def _image():
    img = np.ones((256, 256), np.uint8)
    img[28:228, 28:228] = 0xFF
    img[60, 128] = 1                 # a one-tile island: its list is empty and leaves every window
    img[200, 40] = 1
    img[128, 28:128] = 1             # a corridor from the blob's left edge to its centre
    return img


def _blockers(map_xz):
    """the corridor covered from column 40 to its end, and a blocker on the blocked target's tile"""
    out = [(*mq.tile_xz(128, c, map_xz), 6.0) for c in range(40, 128, 2)]
    out.append((*mq.tile_xz(26, 160, map_xz), 3.0))
    return out


def _map(nav, cost, map_xz, layer):
    """every layer the same terrain and routed; the blockers on the group of layers `layer` belongs to (air blockers
    block layers 8-11 only)"""
    nav.map_create(CW, CH, NLAYERS, *map_xz)
    for L in range(NLAYERS):
        nav.map_upload_layer(L, cost); nav.map_build_nav(L); nav.route_build(L)
    flags = capi.FLAG_MOVABLE | (capi.FLAG_AIR if layer >= 8 else 0)
    for b in _blockers(map_xz):
        nav.blockers_incref(*b, 0, flags)
    nav.map_commit()


def _tile_of(xz, map_xz):
    return int(round((float(xz[1]) - map_xz[1]) / 4.0)), int(round((map_xz[0] - float(xz[0])) / 4.0))


def _blocked_image(img, blk):
    """impassable or under a blocker, per absolute tile (blk: blocker counts as Nav.blockers returns them)"""
    b = blk.reshape(CH, CW, 64, 64).transpose(0, 2, 1, 3).reshape(CH * 64, CW * 64)
    return (img == 0xFF) | (b > 0)


def _next_to_blocked(bimg, r, c):
    return any(0 <= r + dr < 256 and 0 <= c + dc < 256 and bimg[r + dr, c + dc]
               for dr, dc in ((-1, 0), (1, 0), (0, -1), (0, 1)))


def scene(layer, map_xz):
    """-> dict(cost, img, rec, fl, ms, ext, work, kinds): targets (ARRIVED, outside the work list) first, then the
    ENTER_ENTITY_RANGE units; kinds names each unit's construction"""
    img = _image()
    cost = synth.image_to_blocked(img, CW, CH)
    host = capi.Nav(hostonly=True)
    try:
        _map(host, cost, map_xz, layer)
        targets = {"edge": (26, 100), "blocked": (26, 160), "far": (128, 127), "island": (60, 128)}
        pos, kinds, tgt_of, rng_of, prev_of = [], [], [], [], []
        tpos = {}
        for name, (r, c) in targets.items():
            tpos[name] = np.array(mq.tile_xz(r, c, map_xz), np.float32)
            pos.append(tpos[name]); kinds.append("target_" + name); tgt_of.append(-1); rng_of.append(0.0); prev_of.append(tpos[name])
        tuid = {name: k for k, name in enumerate(targets)}

        def unit(kind, p, target, rng=0.0, moved=False):
            t = tpos[target] if target in tpos else np.array(p, np.float32)
            pos.append(np.array(p, np.float32)); kinds.append(kind)
            tgt_of.append(tuid.get(target, -2 if target == "self" else -1)); rng_of.append(rng)
            prev_of.append(t + np.float32(10.0) if moved else t)

        bimg = _blocked_image(img, host.blockers(layer))
        mc_n = {}
        for name in ("edge", "blocked", "far"):
            ok, _, mc = host.route_arrival_consts(tpos[name], layer)
            mc_n[name] = mc
            adj = [p for p in mc if _next_to_blocked(bimg, *_tile_of(p, map_xz))]
            assert adj, name
            for moved in (False, True):
                unit("hit_" + name, adj[0], name, moved=moved)
                off = adj[-1].copy(); off[0] = np.nextafter(off[0], np.float32(np.inf))
                unit("off_" + name, off, name, moved=moved)
            if name == "edge":
                free = [p for p in mc if not _next_to_blocked(bimg, *_tile_of(p, map_xz))]
                unit("noadj_edge", free[0], name)
        far_tiles = np.array([_tile_of(p, map_xz) for p in mc_n["far"]])
        assert np.abs(far_tiles - np.array(targets["far"])).sum(axis=1).min() > 64, "the far list must leave the window"
        # the one-tile island's empty list, from a unit next to the blob's top edge
        unit("island", mq.tile_xz(27, 128, map_xz), "island", moved=True)
        unit("null", mq.tile_xz(27, 60, map_xz), None)
        unit("self_range", mq.tile_xz(27, 62, map_xz), "self", rng=0.0)
        unit("self_adjacent", mq.tile_xz(27, 64, map_xz), "self", rng=-1.0)
    finally:
        host.close()
    n = len(pos)
    pos = np.array(pos, np.float32)
    a = {"pos": pos, "prev_pos": pos.copy(), "vel": np.zeros((n, 2), np.float32), "radius": np.full(n, 1.0, np.float32),
         "max_speed": np.zeros(n, np.float32), "speed": np.zeros(n, np.float32),
         "state": np.where(np.arange(n) < len(targets), ST_ARRIVED, ST_ENTER).astype(np.int32),
         "flags": np.full(n, LAYER_FLAGS[layer], np.uint32), "flock_of": np.full(n, -1, np.int32),
         "flock_target": np.array([tpos["edge"]], np.float32), "vdes": np.zeros((n, 2), np.float32),
         "has_los": np.zeros(n, np.uint32)}
    rec, fl = capi.pack_agents(a)
    ms = np.zeros(n, capi.MOVESTATE)
    ms["next_pos"][:, 0] = pos[:, 0]; ms["next_pos"][:, 2] = pos[:, 1]
    ms["step"] = 1.0; ms["next_rot"][:, 3] = 1.0; ms["combat_facing"][:, 3] = 1.0
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["rot"][:, 3] = 1.0; ext["target_dir"][:, 3] = 1.0
    tg = np.array(tgt_of, np.int64)
    tg = np.where(tg == -2, np.arange(n), tg)
    ext["surround_target_uid"] = np.where(tg < 0, capi.NULL_UID, tg).astype(np.uint32)
    ext["target_range"] = np.array(rng_of, np.float32)
    ext["target_prev_pos"] = np.array(prev_of, np.float32)
    form = np.zeros(n, capi.FORMATION_IN)
    work = np.nonzero(rec["state"] != ST_ARRIVED)[0].astype(np.uint32)
    return dict(cost=cost, img=img, rec=rec, fl=fl, ms=ms, ext=ext, form=form, work=work, kinds=np.array(kinds),
                layer=layer, map_xz=map_xz)


def _setup(nav, S):
    _map(nav, S["cost"], S["map_xz"], S["layer"])
    nav.agents_upload(S["rec"], S["fl"], 20)
    nav.agents_upload_movestate(S["ms"])
    nav.agents_upload_movestate_ext(S["ext"])


def _port(S, rec, ms, ext, work):
    host = capi.Nav(hostonly=True)
    try:
        _map(host, S["cost"], S["map_xz"], S["layer"])
        import pforacle
        L = S["layer"]
        omaps = {L: pforacle.OracleMap(CW, CH, S["cost"], host.blockers(L), None, *S["map_xz"])}
        lou = np.full(len(rec), L, np.int32)
        return cases.states_port_tick(host, omaps, rec, S["fl"], ms, S["form"], ext, work, 20, lou)
    finally:
        host.close()


def _same_bits(tag, got, exp):
    for k in got.dtype.names:
        g, e = np.ascontiguousarray(got[k]), np.ascontiguousarray(exp[k])
        bad = np.nonzero((g.view(np.uint8).reshape(len(g), -1) != e.view(np.uint8).reshape(len(e), -1)).any(axis=1))[0]
        assert len(bad) == 0, (tag, k, bad[:10], g[bad[:3]], e[bad[:3]])


def _port_stopped_through_list(S, tarr_items, exp_patches):
    """the work items the port stopped through the list: WAITING although farther than target_range"""
    out = []
    for i, u in enumerate(S["work"]):
        t = S["ext"]["surround_target_uid"][u]
        if S["rec"]["state"][u] != ST_ENTER or t == capi.NULL_UID:
            continue
        d = np.float32(np.sqrt(np.float32(((S["rec"]["pos"][t] - S["rec"]["pos"][u]) ** 2).sum())))
        if d > S["ext"]["target_range"][u] and exp_patches["next_state"][i] == ST_WAITING:
            out.append(S["kinds"][u])
    return out


@pytest.mark.parametrize("layer", [0, 4, 8])
@pytest.mark.parametrize("offset", [False, True], ids=["origin", "offset"])
def test_enter_range_vs_port(nav, layer, offset):
    """one tick, then 8 resident ticks, every patch bit for bit with the port fed the host lists"""
    S = scene(layer, OFFSET if offset else (0.0, 0.0))
    _setup(nav, S)
    n = len(S["rec"])
    rec, ms, ext = S["rec"], S["ms"], S["ext"]
    for tick in range(9):
        work = np.nonzero(rec["state"] != ST_ARRIVED)[0].astype(np.uint32)
        exp = _port(S, rec, ms, ext, work)
        nav.agents_set_work(work)
        nav.agents_tick(0)
        nav.agents_compute_updates()
        got = nav.agents_read_patches(len(work))
        _same_bits("tick %d" % tick, got, exp["patches"])
        if tick == 0:
            stopped = _port_stopped_through_list(S, None, exp["patches"])
            assert {"hit_edge", "hit_blocked", "hit_far"} <= set(stopped), stopped
            kinds = S["kinds"][work]
            ns = exp["patches"]["next_state"]
            assert (ns[kinds == "hit_far"] == ST_WAITING).all() and (ns[kinds == "off_far"] != ST_WAITING).all()
            assert (ns[np.isin(kinds, ["off_edge", "off_blocked", "noadj_edge", "island"])] != ST_WAITING).all()
            flags = exp["patches"]["flags"]
            assert (flags[kinds == "off_far"] & UPDATE_SET_DEST).any() and not (flags[kinds == "off_far"] & UPDATE_SET_DEST).all()
        nav.agents_apply_updates()
        nav.agents_rebuild_index()
        rec, ms = nav.agents_read_state(n)
        ext = nav.agents_read_movestate_ext(n)
        assert (rec["state"] == exp["agents"]["state"]).all(), tick
        for k in ("wait_prev", "wait_ticks_left"):
            assert (ext[k] == exp["ext"][k]).all(), (tick, k)


def test_compute_updates_does_not_wait_with_candidates(nav):
    torch = pytest.importorskip("torch")
    S = scene(0, (0.0, 0.0))
    _setup(nav, S)
    st = torch.cuda.current_stream()
    nav.agents_set_work(S["work"])
    nav.agents_tick(0, stream=st.cuda_stream)
    nav.agents_compute_updates(stream=st.cuda_stream)          # sizes the buffers
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)                              # a bounded spin on the stream, about 0.1 s
    nav.agents_compute_updates(stream=st.cuda_stream)
    busy = not st.query()
    torch.cuda.synchronize()
    assert busy, "compute_updates waited for its stream"
    exp = _port(S, S["rec"], S["ms"], S["ext"], S["work"])
    _same_bits("no wait", nav.agents_read_patches(len(S["work"])), exp["patches"])


def _route_case(nav, unit_layer_flags, radius):
    """two layers, only layer 0 routed; one ENTER_ENTITY_RANGE unit aimed at one ARRIVED target"""
    img = _image()
    cost = synth.image_to_blocked(img, CW, CH)
    nav.map_create(CW, CH, 2)
    for L in range(2):
        nav.map_upload_layer(L, cost); nav.map_build_nav(L)
    nav.route_build(0)
    pos = np.array([mq.tile_xz(26, 100), mq.tile_xz(27, 90)], np.float32)
    a = {"pos": pos, "prev_pos": pos.copy(), "vel": np.zeros((2, 2), np.float32), "radius": np.array([1.0, radius], np.float32),
         "max_speed": np.zeros(2, np.float32), "speed": np.zeros(2, np.float32), "state": np.array([ST_ARRIVED, ST_ENTER], np.int32),
         "flags": np.array([0, unit_layer_flags], np.uint32), "flock_of": np.full(2, -1, np.int32),
         "flock_target": pos[:1].copy()}
    rec, fl = capi.pack_agents(a)
    ms = np.zeros(2, capi.MOVESTATE)
    ms["next_pos"][:, 0] = pos[:, 0]; ms["next_pos"][:, 2] = pos[:, 1]; ms["step"] = 1.0; ms["next_rot"][:, 3] = 1.0
    ext = np.zeros(2, capi.MOVESTATE_EXT)
    ext["rot"][:, 3] = 1.0; ext["surround_target_uid"] = [capi.NULL_UID, 0]; ext["target_prev_pos"] = pos[0]
    nav.agents_upload(rec, fl, 20)
    nav.agents_upload_movestate(ms)
    nav.agents_upload_movestate_ext(ext)
    nav.agents_set_work(np.array([1], np.uint32))


def test_unrouted_layer_refuses(nav):
    _route_case(nav, 0, 6.0)                 # radius 6: layer 1, not routed
    nav.agents_tick(0)
    with pytest.raises(capi.PfnavError, match=r"pfnav_route_build\(layer 1\) is needed"):
        nav.agents_compute_updates()


def test_routed_layers_do_not_wait(nav):
    torch = pytest.importorskip("torch")
    _route_case(nav, 0, 1.0)                 # every entity on layer 0; layer 1 has no routing structure
    st = torch.cuda.current_stream()
    nav.agents_tick(0, stream=st.cuda_stream)
    nav.agents_compute_updates(stream=st.cuda_stream)
    torch.cuda.synchronize()
    torch.cuda._sleep(200_000_000)
    nav.agents_compute_updates(stream=st.cuda_stream)
    busy = not st.query()
    torch.cuda.synchronize()
    assert busy, "compute_updates waited for its stream"
    nav.agents_read_patches(1)


def _job_ticks(S, world, nticks=8):
    """nticks ticks of the scene on one context (world 1) or a group of `world` members on device 0 -> per tick the
    joined patches, events and state tables as bytes"""
    n = len(S["rec"])
    navs = [capi.Nav(0) for _ in range(world)]
    grp = capi.Group(navs) if world > 1 else None
    out = []
    try:
        rg = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
        for nv in navs:
            _map(nv, S["cost"], S["map_xz"], S["layer"])
        if grp is None:
            navs[0].agents_upload(S["rec"], S["fl"], 20)
        else:
            for nv, (lo, hi) in zip(navs, rg):
                nv.agents_upload_shard(S["rec"][lo:hi].copy(), lo, hi, n, S["fl"], 20)
            grp.gather()
        for nv, (lo, hi) in zip(navs, rg):
            nv.agents_upload_movestate(S["ms"][lo:hi].copy()); nv.agents_upload_movestate_ext(S["ext"][lo:hi].copy())
        for tick in range(nticks):
            pat, ev, tabs = [], [], []
            for nv, (lo, hi) in zip(navs, rg):
                a, _ = nv.agents_read_state(hi - lo)
                w = (lo + np.nonzero(a["state"] != ST_ARRIVED)[0]).astype(np.uint32)
                nv.agents_set_work(w)
                if not len(w):
                    continue
                nv.agents_tick(0)
                nv.agents_compute_updates()
                nv.agents_collect_events()
                pat.append(nv.agents_read_patches(len(w))); ev.append(nv.agents_read_events(len(w)))
                nv.agents_apply_updates()
            if grp is not None:
                grp.gather()
            else:
                navs[0].agents_rebuild_index()
            for nv, (lo, hi) in zip(navs, rg):
                a, m = nv.agents_read_state(hi - lo)
                tabs.append((a, m, nv.agents_read_movestate_ext(hi - lo)))
            out.append((np.concatenate(pat).tobytes(), np.concatenate(ev).tobytes(),
                        *(np.concatenate([t[k] for t in tabs]).tobytes() for k in range(3))))
    finally:
        if grp is not None:
            grp.close()
        for nv in navs:
            nv.close()
    return out


@pytest.mark.parametrize("world", [2, 3])
def test_enter_range_jobs(pf, world):
    """a group of 2 or 3 members ticks the scene like one context, with targets owned by another member"""
    S = scene(0, OFFSET)
    n = len(S["rec"])
    own = [capi.mgpu_shard_range(n, r, world) for r in range(world)]
    member = lambda u: next(r for r, (lo, hi) in enumerate(own) if lo <= u < hi)
    cross = [u for u in S["work"] if S["ext"]["surround_target_uid"][u] != capi.NULL_UID
             and member(int(S["ext"]["surround_target_uid"][u])) != member(int(u)) and S["kinds"][u].startswith("hit")]
    assert cross, "no candidate aims at another member's entity"
    one, job = _job_ticks(S, 1), _job_ticks(S, world)
    for t, (a, b) in enumerate(zip(one, job)):
        for k, name in enumerate(("patches", "events", "agents", "movestate", "ext")):
            assert a[k] == b[k], (world, t, name)
