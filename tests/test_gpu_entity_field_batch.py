"""GPU suite: pfnav_pool_request_entity_fields_batch, the batched N_RequestAsyncEnemySeekField /
N_RequestAsyncSurroundField + N_AwaitAsyncFields (nav.c:3769-3960) with its seed frontiers rasterised on the device.

- the batch reproduces the compiled reference's TARGET_ENTITY / TARGET_ENEMIES fields (targets.npz);
- device seeding equals host seeding (pfnav_entity_fields, the same integration kernel) byte for byte, on both sides of
  the 512-tile cap, for all 12 reference layers, both kinds and 1 x 1, 4 x 4 and 16 x 16 maps;
- the batch leaves the pool (flow bytes, has, ffid), the repairs and the consumers' velocities exactly as the serial
  loop of pfnav_pool_request_entity_fields does, under pool pressure and at a NOMEM stop;
- launches are ordered on the caller's stream, after pfnav_pool_clear."""
import ctypes as C
import os

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
ST_SEEK, ST_SURROUND = 3, 5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _ctx(cw, ch, seed, nlayers=1):
    nav = capi.Nav(0)
    p = synth.make_map(cw, ch, seed, rivers=cw > 1 and ch > 1)
    cost = synth.cost_from_pathable(p, cw, ch)
    nav.map_create(cw, ch, nlayers)
    for layer in range(nlayers):
        nav.map_upload_layer(layer, cost)
        nav.map_build_nav(layer)
        nav.route_build(layer)                            # pfnav_pool_repair needs the global islands
    return nav


def _req(dest, kind, ent, chunk, layer=0, ref_layer=0):
    r = np.zeros(1, capi.ENTITY_FIELD_REQ)
    r["dest"], r["layer"], r["ref_layer"], r["target_kind"] = dest, layer, ref_layer, kind
    r["ent_off"], r["ent_n"], r["chunk_off"], r["chunk_n"] = ent[0], ent[1], chunk[0], chunk[1]
    return r


def _raw(nav, reqs, fp, chunks, stream=0):
    """the return code of the batch (no exception)"""
    reqs = np.ascontiguousarray(reqs, capi.ENTITY_FIELD_REQ)
    fp = np.ascontiguousarray(fp, capi.FOOTPRINT)
    ch = np.ascontiguousarray(chunks, np.int32).reshape(-1, 2)
    nd = C.c_int(-1)
    rc = nav.L.pfnav_pool_request_entity_fields_batch(nav.h, capi._p(reqs) if len(reqs) else None, len(reqs),
                                                      capi._p(fp) if len(fp) else None, len(fp), capi._p(ch) if len(ch) else None,
                                                      len(ch), C.c_void_p(stream), C.byref(nd))
    return rc, nd.value


def _serial(nav, reqs, fp, chunks):
    """the serial loop: pool_request_entity_fields per request; -> ndone (stops at the first NOMEM)"""
    ch = np.asarray(chunks, np.int32).reshape(-1, 2)
    for i, r in enumerate(reqs):
        e0, en, c0, cn = int(r["ent_off"]), int(r["ent_n"]), int(r["chunk_off"]), int(r["chunk_n"])
        rc = nav.L.pfnav_pool_request_entity_fields(nav.h, int(r["dest"]), int(r["layer"]), int(r["ref_layer"]), int(r["target_kind"]),
                                                    capi._p(np.ascontiguousarray(fp[e0:e0 + en])) if en else None, en,
                                                    capi._p(np.ascontiguousarray(ch[c0:c0 + cn])) if cn else None, cn, None)
        if rc == capi.ERR_NOMEM:
            return i
        assert rc == 0, (i, rc)
    return len(reqs)


def _pool(nav, ndests, cw, ch):
    """every pool entry: (has flow, ffid, flow bytes)"""
    out = []
    for d in range(ndests):
        for c in range(cw * ch):
            f, _, ffid = nav.pool_get(d, divmod(c, cw))
            out.append((f is not None, ffid, None if f is None else f.tobytes()))
    return out


def _building(cx, cz, hx, hz, ang):
    c, s = np.cos(ang), np.sin(ang)
    pts = [(-hx, -hz), (hx, -hz), (hx, hz), (-hx, hz)]
    return np.array([(cx + c * a - s * b, cz + s * a + c * b) for a, b in pts], np.float32).reshape(-1)


def _footprints(cw, ch, n, seed):
    """circles of radius 0 .. past the device / host bound and buildings, on chunk borders, map edges and exactly on the
    scaled bounds of the TARGET_ENEMIES search rectangles (chunk +- 144 units, field.c:1229-1243)"""
    rng = np.random.default_rng(seed)
    W, H = cw * 256.0, ch * 256.0
    x = -rng.uniform(0, W, n).astype(np.float32)
    z = rng.uniform(0, H, n).astype(np.float32)
    k = n // 8
    x[:k] = -256.0 * rng.integers(0, cw + 1, k)                                      # chunk borders / map edges
    z[k:2 * k] = 256.0 * rng.integers(0, ch + 1, k)
    bx = np.concatenate([-(256.0 * np.arange(cw) + 400.0), -(256.0 * np.arange(cw)) + 144.0])
    bz = np.concatenate([256.0 * np.arange(ch) - 144.0, 256.0 * np.arange(ch) + 400.0])
    eps = np.array([0.0, 0.5 / 256, -0.5 / 256, 1.0 / 256, -1.0 / 256])
    x[2 * k:3 * k] = (rng.choice(bx, k) + rng.choice(eps, k)).astype(np.float32)     # on a rectangle's scaled bound
    z[3 * k:4 * k] = (rng.choice(bz, k) + rng.choice(eps, k)).astype(np.float32)
    x[4 * k:4 * k + 4] = [0.0, -W, -W / 2, 1.0]                                       # map edges, one just outside
    z[4 * k:4 * k + 4] = [H / 2, 0.0, H, 3.0]
    fp = capi.Nav.footprints(np.stack([x, z], 1), 0.0)
    r = rng.uniform(0.0, 46.0, n).astype(np.float32)
    r[::7] = rng.choice(np.array([0.0, 4.0, 16.0, 20.0, 24.0, 28.0, 28.5, 36.0, 40.0, 40.5, 60.0], np.float32), len(r[::7]))
    fp["sel_radius"] = r
    for i in range(5 * k, 5 * k + max(2, k // 2)):                                    # buildings, corners inside the map
        hx, hz = rng.uniform(2, 20, 2)
        cx = -rng.uniform(24, W - 24) if W > 48 else -W / 2
        cz = rng.uniform(24, H - 24) if H > 48 else H / 2
        fp["is_building"][i] = 1
        fp["corners_xz"][i] = _building(cx, cz, min(hx, 10), min(hz, 10), rng.uniform(0, np.pi))
        fp["x"][i], fp["z"][i] = cx, cz
    return fp


def test_batch_targets_golden(nav):
    """one batch reproduces every TARGET_ENTITY / TARGET_ENEMIES field of targets.npz on reference layers 0 and 2"""
    g = np.load(os.path.join(GOLDEN, "targets.npz"))
    cw = ch = 3
    wars = [tuple(w) for w in g["wars"]]
    nav.map_create(cw, ch, 2)
    for slot, L in enumerate((0, 2)):
        nav.map_upload_layer(slot, g["cost_%d" % L], g["blk_%d" % L])
    fp_all = nav.footprints(g["pos"], g["radius"])
    allchunks = np.array([(c // cw, c % cw) for c in range(cw * ch)], np.int32)
    fps, reqs, dests = [fp_all], [], []
    for f in range(4):
        sel = np.nonzero(cases.enemies_of(f, wars, g["factions"], g["flags"]))[0]
        fps.append(fp_all[sel])
    off = np.cumsum([0] + [len(x) for x in fps])
    fp = np.concatenate(fps)
    for slot, L in enumerate((0, 2)):
        for k, u in enumerate(g["uids"]):
            reqs.append(_req(len(dests), capi.TARGET_ENTITY, (int(u), 1), (0, 9), slot, L)); dests.append(("ent_%d" % L, k))
        for f in range(4):
            reqs.append(_req(len(dests), capi.TARGET_ENEMIES, (off[f + 1], off[f + 2] - off[f + 1]), (0, 9), slot, L))
            dests.append(("foe_%d" % L, f))
    nav.pool_create(len(dests), len(dests) * 9)
    assert nav.pool_request_entity_fields_batch(np.concatenate(reqs), fp, allchunks) == len(reqs)
    for d, (key, k) in enumerate(dests):
        for c in range(9):
            f, _, _ = nav.pool_get(d, divmod(c, cw))
            assert f is not None and (f == g[key][k][c]).all(), (key, k, c)


@pytest.mark.parametrize("cw,ch", [(1, 1), (4, 4), (16, 16)])
def test_device_seeds_vs_host_seeds(cw, ch):
    """pool fields from the batch == pfnav_entity_fields (host entity_seeds + the same kernel), every reference layer,
    both kinds, circles on both sides of the device / host bound, buildings, borders and scaled bounds"""
    nav = _ctx(cw, ch, 0x5EED00A0 + cw)
    try:
        fp = _footprints(cw, ch, 400 if cw > 1 else 120, 17 + cw)
        rng = np.random.default_rng(cw)
        nchk = cw * ch
        chunks = np.array([divmod(c, cw) for c in (range(nchk) if nchk <= 16 else rng.choice(nchk, 24, replace=False))], np.int32)
        ents = [int(i) for i in np.nonzero(fp["is_building"])[0][:2]] + \
               [int(i) for i in np.argsort(-fp["sel_radius"])[:2]] + [int(i) for i in rng.choice(len(fp), 3, replace=False)] + [0, 4 * (len(fp) // 8)]
        nav.pool_create(1 + len(ents), (1 + len(ents)) * len(chunks))
        for L in range(12):
            nav.pool_clear()
            reqs = [_req(0, capi.TARGET_ENEMIES, (0, len(fp)), (0, len(chunks)), 0, L)]
            reqs += [_req(1 + i, capi.TARGET_ENTITY, (e, 1), (0, len(chunks)), 0, L) for i, e in enumerate(ents)]
            assert nav.pool_request_entity_fields_batch(np.concatenate(reqs), fp, chunks) == len(reqs)
            host = [nav.entity_fields(capi.TARGET_ENEMIES, fp, chunks, 0, L)]
            host += [nav.entity_fields(capi.TARGET_ENTITY, fp[e:e + 1], chunks, 0, L) for e in ents]
            for d in range(len(host)):
                for j, c in enumerate(chunks):
                    f, _, _ = nav.pool_get(d, tuple(c))
                    assert f is not None and (f == host[d][j]).all(), (L, d, tuple(c))
    finally:
        nav.close()


def test_one_by_n_map_is_an_argument_error():
    nav = _ctx(4, 1, 0x5EED00B0)
    try:
        nav.pool_create(1, 8)
        fp = capi.Nav.footprints(np.array([[-100.0, 100.0]], np.float32), 3.0)
        rc, nd = _raw(nav, _req(0, capi.TARGET_ENEMIES, (0, 1), (0, 1)), fp, [(0, 1)])
        assert rc == capi.ERR_ARG and nd == 0
    finally:
        nav.close()


def _mixed(cw, ch, nfp, nreq, ndests, seed):
    """a shared footprint array, overlapping ranges, duplicate dests and repeated (dest, chunk) pairs"""
    rng = np.random.default_rng(seed)
    fp = _footprints(cw, ch, nfp, seed)
    chunks, reqs = [], []
    for i in range(nreq):
        kind = int(rng.integers(0, 2))
        if kind == capi.TARGET_ENTITY:
            ent = (int(rng.integers(0, nfp)), 1)
        else:
            a = int(rng.integers(0, nfp - 1)); ent = (a, int(rng.integers(1, nfp - a + 1)))
        n = int(rng.integers(0, 6))
        cs = [divmod(int(c), cw) for c in rng.integers(0, cw * ch, n)]
        if n and rng.random() < 0.2:
            cs.append(cs[0])                                # the same chunk twice in one request
        reqs.append(_req(int(rng.integers(0, ndests)), kind, ent, (len(chunks), len(cs)), 0, int(rng.integers(0, 12))))
        chunks += cs
    return fp, np.concatenate(reqs), np.array(chunks, np.int32).reshape(-1, 2)


def _agents_on(nav, cw, ch, ndests, n, seed):
    """SEEK_ENEMIES / SURROUND_ENTITY agents on passable tiles, naming the destinations through aux_dest1"""
    rng = np.random.default_rng(seed)
    cost, blk, _ = nav.map_get_layer(0)
    img = synth.blocked_to_image(cost, cw, ch)
    t = np.argwhere(img != 255)
    t = t[rng.integers(0, len(t), n)]
    pos = np.stack([-(t[:, 1] + rng.uniform(0.05, 0.95, n)) * 4.0, (t[:, 0] + rng.uniform(0.05, 0.95, n)) * 4.0], 1).astype(np.float32)
    rec = np.zeros(n, capi.AGENT)
    rec["pos"] = pos; rec["prev_pos"] = pos; rec["radius"] = 1.0; rec["max_speed"] = 20.0; rec["speed"] = 20.0
    rec["flags"] = capi.FLAG_MOVABLE
    rec["aux_dest1"] = rng.integers(1, ndests + 1, n)
    rec["state"][: n // 2] = ST_SEEK; rec["flock"][: n // 2] = -1
    rec["state"][n // 2:] = ST_SURROUND; rec["flock"][n // 2:] = 0
    fl = np.zeros(1, capi.FLOCK); fl["target"] = pos[0]; fl["dest"] = -1
    ext = np.zeros(n, capi.MOVESTATE_EXT)
    ext["surround_target_uid"] = capi.NULL_UID
    ext["surround_target_uid"][n // 2:] = 0; ext["using_surround_field"][n // 2:] = 1
    return rec, fl, ext


def _tick(nav, rec, fl, ext, stream=0):
    nav.agents_upload(rec, fl, 20)
    nav.agents_upload_movestate_ext(ext)
    nav.agents_set_work(np.arange(len(rec), dtype=np.uint32))
    nav.agents_tick(capi.TICK_VDES_FROM_POOL, stream)


@pytest.mark.parametrize("pool_max", [4096, 48])
def test_batch_vs_serial_loop(pool_max):
    """hundreds of mixed requests in one batch vs the serial loop: every pool entry, then the repairs of those
    destinations and the consumers' velocities; pool_max 48 evicts inside the batch"""
    cw = ch = 4
    ndests = 40
    navs = [_ctx(cw, ch, 0x5EED00C0) for _ in range(2)]
    try:
        fp, reqs, chunks = _mixed(cw, ch, 300, 400, ndests, 5)
        for nav in navs:
            nav.pool_create(ndests, pool_max)
        nd_serial = _serial(navs[0], reqs, fp, chunks)
        nd_batch = navs[1].pool_request_entity_fields_batch(reqs, fp, chunks)
        assert nd_serial == nd_batch == len(reqs)
        assert _pool(navs[0], ndests, cw, ch) == _pool(navs[1], ndests, cw, ch)
        rec, fl, ext = _agents_on(navs[0], cw, ch, ndests, 3000, 9)
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
    finally:
        for nav in navs:
            nav.close()


def test_nomem_stop_and_bad_arguments():
    """a request the pool cannot hold stops the batch where the serial loop stops; malformed batches change nothing"""
    cw = ch = 4
    navs = [_ctx(cw, ch, 0x5EED00D0) for _ in range(2)]
    try:
        fp, reqs, chunks = _mixed(cw, ch, 120, 60, 8, 11)
        big = np.array([divmod(c, cw) for c in range(cw * ch)], np.int32)
        reqs = np.concatenate([reqs[:30], _req(3, capi.TARGET_ENEMIES, (0, 50), (len(chunks), 16)), reqs[30:]])
        chunks = np.concatenate([chunks, big])
        for nav in navs:
            nav.pool_create(8, 12)                          # 16 distinct chunks never fit
        nd_serial = _serial(navs[0], reqs, fp, chunks)
        nd_batch = navs[1].pool_request_entity_fields_batch(reqs, fp, chunks)
        assert nd_serial == nd_batch == 30
        assert _pool(navs[0], 8, cw, ch) == _pool(navs[1], 8, cw, ch)
        nav = navs[1]
        before = _pool(nav, 8, cw, ch)
        outside = fp.copy()
        outside["is_building"][0] = 1
        outside["corners_xz"][0] = _building(10.0, 100.0, 4.0, 4.0, 0.3)            # x > 0: outside the map
        outside["x"][0], outside["z"][0] = -100.0, 100.0
        ok = _req(0, capi.TARGET_ENEMIES, (0, 10), (0, 1))
        bad = [(_req(0, capi.TARGET_ENEMIES, (100, 30), (0, 2)), fp, chunks),         # footprint range
               (_req(0, capi.TARGET_ENEMIES, (0, 10), (len(chunks) - 1, 2)), fp, chunks),   # chunk range
               (_req(8, capi.TARGET_ENEMIES, (0, 10), (0, 2)), fp, chunks),           # dest
               (_req(0, capi.TARGET_ENEMIES, (0, 10), (0, 2), layer=1), fp, chunks),  # layer
               (_req(0, capi.TARGET_ENEMIES, (0, 10), (0, 2), ref_layer=12), fp, chunks),
               (_req(0, 2, (0, 10), (0, 2)), fp, chunks),                              # target kind
               (_req(0, capi.TARGET_ENTITY, (0, 2), (0, 2)), fp, chunks),              # TARGET_ENTITY takes one footprint
               (_req(0, capi.TARGET_ENTITY, (0, 1), (0, 2)), outside, chunks),         # building corner outside the map
               (_req(0, capi.TARGET_ENEMIES, (0, 1), (0, 1)), outside, [(0, 0)]),
               (_req(0, capi.TARGET_ENEMIES, (0, 10), (0, 1)), fp, [(4, 0)])]          # chunk outside the map
        for i, (r, f, c) in enumerate(bad):
            rc, nd = _raw(nav, np.concatenate([ok, r]), f, c)
            assert rc == capi.ERR_ARG and nd == 0, i
            assert _pool(nav, 8, cw, ch) == before, i
        # an ENEMIES building outside the map but far from every requested chunk is not used: not an error (as before)
        far = _req(0, capi.TARGET_ENEMIES, (0, 1), (0, 1))
        assert _raw(nav, far, outside, [(3, 3)])[0] == 0
    finally:
        for nav in navs:
            nav.close()


def test_consumers_match_serial_fill():
    """SEEK_ENEMIES / SURROUND_ENTITY agents on the targets map get the same vdes and velocities whether the pool was
    filled by one batch or by the serial loop"""
    g = np.load(os.path.join(GOLDEN, "targets.npz"))
    cw = ch = 3
    wars = [tuple(w) for w in g["wars"]]
    navs = []
    for _ in range(2):
        nav = capi.Nav(0)
        nav.map_create(cw, ch, 1)
        nav.map_upload_layer(0, g["cost_0"], g["blk_0"]); nav.map_build_nav(0); nav.route_build(0)
        navs.append(nav)
    try:
        fp_all = navs[0].footprints(g["pos"], g["radius"])
        fps = [fp_all] + [fp_all[cases.enemies_of(f, wars, g["factions"], g["flags"])] for f in range(4)]
        off = np.cumsum([0] + [len(x) for x in fps])
        fp = np.concatenate(fps)
        allchunks = np.array([(c // cw, c % cw) for c in range(9)], np.int32)
        reqs = [_req(f, capi.TARGET_ENEMIES, (off[f + 1], off[f + 2] - off[f + 1]), (0, 9)) for f in range(4)]
        reqs += [_req(4 + k, capi.TARGET_ENTITY, (int(u), 1), (0, 9)) for k, u in enumerate(g["uids"])]
        reqs = np.concatenate(reqs)
        nd = 4 + len(g["uids"])
        for nav in navs:
            nav.pool_create(nd, nd * 9)
        _serial(navs[0], reqs, fp, allchunks)
        navs[1].pool_request_entity_fields_batch(reqs, fp, allchunks)
        rec, fl, ext = _agents_on(navs[0], cw, ch, nd, 6000, 21)
        res = []
        for nav in navs:
            _tick(nav, rec, fl, ext)
            _, vdes, _ = nav.agents_read_debug(len(rec))
            res.append((vdes, nav.agents_read_velocities(len(rec))))
        assert (res[0][0] == res[1][0]).all() and (res[0][1] == res[1][1]).all()
        assert (np.abs(res[0][0]).sum(axis=1) > 0).mean() > 0.5
    finally:
        for nav in navs:
            nav.close()


def test_stream_order_clear_and_hostonly():
    """back-to-back batch + tick steps on one stream without host synchronisation == the same steps synchronised after
    each; a batch right after pool_clear sees an empty pool; a host-only context has no device path"""
    import torch
    cw = ch = 4
    ndests = 16
    navs = [_ctx(cw, ch, 0x5EED00E0) for _ in range(2)]
    try:
        steps = [_mixed(cw, ch, 200, 60, ndests, 100 + s) for s in range(3)]
        rec, fl, ext = _agents_on(navs[0], cw, ch, ndests, 2000, 4)
        s = torch.cuda.Stream()
        out = []
        for k, nav in enumerate(navs):
            nav.pool_create(ndests, 4096)
            for i, (fp, reqs, chunks) in enumerate(steps):
                if i == 1:
                    nav.pool_clear()                        # the next batch must see an empty pool
                nav.pool_request_entity_fields_batch(reqs, fp, chunks, stream=s.cuda_stream if k == 0 else 0)
                if k == 0:
                    _tick(nav, rec, fl, ext, s.cuda_stream)
                else:
                    torch.cuda.synchronize()
                    _tick(nav, rec, fl, ext)
                    torch.cuda.synchronize()
            s.synchronize()
            _, vdes, _ = nav.agents_read_debug(len(rec))
            out.append((vdes, nav.agents_read_velocities(len(rec)), _pool(nav, ndests, cw, ch)))
        assert (out[0][0] == out[1][0]).all() and (out[0][1] == out[1][1]).all() and out[0][2] == out[1][2]
        # the pool after clear holds only what steps 1 and 2 requested: compare with a fresh context
        fresh = _ctx(cw, ch, 0x5EED00E0)
        try:
            fresh.pool_create(ndests, 4096)
            for fp, reqs, chunks in steps[1:]:
                fresh.pool_request_entity_fields_batch(reqs, fp, chunks)
            assert _pool(fresh, ndests, cw, ch) == out[1][2]
        finally:
            fresh.close()
    finally:
        for nav in navs:
            nav.close()
    host = capi.Nav(hostonly=True)
    try:
        fp = capi.Nav.footprints(np.array([[-100.0, 100.0]], np.float32), 3.0)
        assert _raw(host, _req(0, capi.TARGET_ENEMIES, (0, 1), (0, 1)), fp, [(0, 0)])[0] == capi.ERR_NO_DEVICE
    finally:
        host.close()
