"""Seeded scenario builders shared by the golden-vector generator, the CPU tests and the GPU tests.
Everything is a pure function of its seed (numpy + the package's synth module)."""
import hashlib
import importlib
import os

import numpy as np

pf = importlib.import_module("permafrost-engine_b200")
capi, synth = pf.capi, pf.synth
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def digests(fields):
    """SHA-256 of every array along the first axis -> uint8 [n, 32]: bit-exact comparisons of large fields keep a stored
    expectation small"""
    fields = np.asarray(fields)
    return np.array([np.frombuffer(hashlib.sha256(np.ascontiguousarray(f).tobytes()).digest(), np.uint8) for f in fields],
                    np.uint8).reshape(len(fields), 32)


class Expected:
    """Expected values of a GPU test whose comparison needs the compiled reference. With the reference (`ref` not None)
    every value comes from it. Without it the values stored in tests/golden/<name>.npz are used; see
    tests/golden/README.md for where each such file came from (its "source" entry says it too): a file recorded from the
    CUDA path itself is a regression baseline, not a reference comparison.

    PFNAV_RECORD_GOLDEN=<dir> writes <dir>/<name>.npz while the test runs: the reference's values where it is built.
    Without the reference it refuses, unless PFNAV_RECORD_GOLDEN_SELF=1 asks for a regression baseline recorded from
    the CUDA path's own values."""

    def __init__(self, name, ref):
        self.name, self.ref, self.store = name, ref, {}
        self.record = os.environ.get("PFNAV_RECORD_GOLDEN")
        if self.record and ref is None and os.environ.get("PFNAV_RECORD_GOLDEN_SELF") != "1":
            raise RuntimeError("PFNAV_RECORD_GOLDEN without the compiled reference would record the CUDA path's own values; "
                               "set PFNAV_RECORD_GOLDEN_SELF=1 to record such a regression baseline on purpose")
        self.g = None if (ref is not None or self.record) else np.load(os.path.join(GOLD, name + ".npz"))

    def __call__(self, key, from_ref, got=None):
        """the expected value `key`: from_ref() with the reference, else the stored one; while recording a regression
        baseline without the reference, `got` (the CUDA path's value) is what is stored and returned"""
        if self.ref is not None:
            v = from_ref()
        elif self.record:
            v = got
        else:
            return self.g[key]
        if self.record:
            self.store[key] = np.asarray(v)
        return v

    def save(self):
        if self.record:
            os.makedirs(self.record, exist_ok=True)
            self.store["source"] = np.array("reference" if self.ref is not None else "cuda-path regression baseline")
            np.savez_compressed(os.path.join(self.record, self.name + ".npz"), **self.store)


def noise_map(cw, ch, seed, density):
    rng = np.random.default_rng(seed)
    p = synth.make_map(cw, ch, seed, frac_blocked=0.12, rivers=(cw * ch > 1))
    if density > 0:
        p[rng.random(p.shape) < density] = 0
    return p


def local_islands_np(cost, blockers=None):
    """numpy/python restatement of n_update_local_islands (nav.c:967) for test inputs: ids from 1 in
    row-major discovery order."""
    out = np.full(cost.shape, 0xFFFF, np.uint16)
    for ch in range(cost.shape[0]):
        nxt = 0
        free = cost[ch] != 0xFF
        if blockers is not None:
            free &= blockers[ch] == 0
        lab = out[ch]
        for r, c in np.argwhere(free):
            if lab[r, c] != 0xFFFF:
                continue
            nxt += 1
            stack = [(r, c)]
            lab[r, c] = nxt
            while stack:
                y, x = stack.pop()
                for yy, xx in ((y, x - 1), (y, x + 1), (y - 1, x), (y + 1, x)):
                    if 0 <= yy < 64 and 0 <= xx < 64 and free[yy, xx] and lab[yy, xx] == 0xFFFF:
                        lab[yy, xx] = nxt
                        stack.append((yy, xx))
    return out


def serpentine_cost(cw=32, ch=32, gap=40):
    """A map whose every route is forced: a 2-tile wall on every chunk-row boundary (the last nav-tile row of the upper
    chunk row and the first of the lower one), open only over `gap` tiles at the right end of odd boundaries and at the
    left end of even ones. A route from the top-left chunk crosses chunk row 0 to the right, goes down at the right end,
    crosses row 1 to the left, and so on (boustrophedon). -> cost [ch * cw][64][64]"""
    img = np.ones((ch * 64, cw * 64), np.uint8)
    for k in range(1, ch):
        img[64 * k - 1:64 * k + 1, :] = 0xFF
        if k % 2:
            img[64 * k - 1:64 * k + 1, cw * 64 - gap:] = 1
        else:
            img[64 * k - 1:64 * k + 1, :gap] = 1
    return synth.image_to_blocked(img, cw, ch)


def serpentine_order(cw, ch):
    """the chunk indices of serpentine_cost's forced route from the top-left chunk, row by row, in travel order"""
    return [r * cw + (c if r % 2 == 0 else cw - 1 - c) for r in range(ch) for c in range(cw)]


PORTAL_GRID_GAPS = (6, 22, 38, 54)


def portal_grid_cost(cw=32, ch=32, gaps=PORTAL_GRID_GAPS, region=((14, 14), (2, 2))):
    """A map of many portals: a 2-tile wall on every chunk border, opened by a 3-tile gap at each offset of `gaps` per
    side, so an interior chunk has 4 * len(gaps) portals. region ((chunk row, chunk column), (rows, columns)): a block of
    chunks whose outer border has no gaps; inside it the borders keep theirs, so it holds portals of its own that
    nothing outside it reaches. -> cost [ch * cw][64][64]"""
    img = np.ones((ch * 64, cw * 64), np.uint8)
    for k in range(1, ch):
        img[64 * k - 1:64 * k + 1, :] = 0xFF
    for k in range(1, cw):
        img[:, 64 * k - 1:64 * k + 1] = 0xFF
    for k in range(1, ch):                  # gaps in the walls between chunk rows
        for c in range(cw):
            for g in gaps:
                img[64 * k - 1:64 * k + 1, 64 * c + g:64 * c + g + 3] = 1
    for k in range(1, cw):                  # and between chunk columns
        for r in range(ch):
            for g in gaps:
                img[64 * r + g:64 * r + g + 3, 64 * k - 1:64 * k + 1] = 1
    if region is not None:
        (r0, c0), (nr, nc) = region
        R0, R1, C0, C1 = 64 * r0, 64 * (r0 + nr), 64 * c0, 64 * (c0 + nc)
        img[R0 - 1:R0 + 1, C0 - 1:C1 + 1] = 0xFF
        img[R1 - 1:R1 + 1, C0 - 1:C1 + 1] = 0xFF
        img[R0 - 1:R1 + 1, C0 - 1:C0 + 1] = 0xFF
        img[R0 - 1:R1 + 1, C1 - 1:C1 + 1] = 0xFF
    return synth.image_to_blocked(img, cw, ch)


def flow_tile_case(seed, dens, n=8):
    """-> cost[1,64,64], reqs"""
    p = noise_map(1, 1, seed, dens)
    cost = synth.cost_from_pathable(p, 1, 1)
    rng = np.random.default_rng(seed)
    tiles = np.argwhere(cost[0] != 255)
    sel = tiles[rng.integers(0, len(tiles), n)]
    if (cost[0] == 255).any():
        sel = np.concatenate([sel, np.argwhere(cost[0] == 255)[:1]])      # impassable target: empty frontier
    reqs = np.concatenate([capi.tile_req((0, 0), (int(r), int(c))) for r, c in sel])
    return p, cost, reqs


def portal_specs(portals, liid, cw, limit=None):
    """TARGET_PORTAL request specs for every portal: (chunk, idx, ep, next_chunk, next_ep, port_iid, next_iid)"""
    out = []
    key = portals[:, 0] * cw + portals[:, 1]
    for row in portals:
        cr, cc, idx, r0, c0, r1, c1, conn_chunk, conn_idx = [int(v) for v in row[:9]]
        nrow = portals[(key == conn_chunk) & (portals[:, 2] == conn_idx)][0]
        ncr, ncc = int(nrow[0]), int(nrow[1])
        nr0, nc0, nr1, nc1 = [int(v) for v in nrow[3:7]]
        piids = np.unique(liid[cr * cw + cc][r0:r1 + 1, c0:c1 + 1]); piids = piids[piids != 0xFFFF]
        niids = np.unique(liid[ncr * cw + ncc][nr0:nr1 + 1, nc0:nc1 + 1]); niids = niids[niids != 0xFFFF]
        for pi in list(piids[:2]) + [0xFFFF]:
            for ni in niids[:2]:
                out.append(((cr, cc), idx, (r0, c0, r1, c1), (ncr, ncc), (nr0, nc0, nr1, nc1), int(pi), int(ni)))
    return out[:limit] if limit else out


def portal_reqs(specs, init=1):
    return np.concatenate([capi.portal_req(s[0], s[2], s[3], s[4], s[5], s[6], init=init) for s in specs])


def los_case(cost, cw, ch, seed, ntargets=4):
    """LOS request batch: destination chunk + chained neighbours (+ one more hop). -> reqs"""
    rng = np.random.default_rng(seed)
    reqs = []
    for t in range(ntargets):
        chunk = (int(rng.integers(0, ch)), int(rng.integers(0, cw)))
        tiles = np.argwhere(cost[chunk[0] * cw + chunk[1]] != 255)
        tr, tc = [int(v) for v in tiles[rng.integers(0, len(tiles))]]
        td = (chunk[0], chunk[1], tr, tc)
        i0 = len(reqs)
        reqs.append(capi.los_req(chunk, td))
        for nb in ((chunk[0] + 1, chunk[1]), (chunk[0] - 1, chunk[1]), (chunk[0], chunk[1] + 1), (chunk[0], chunk[1] - 1)):
            if not (0 <= nb[0] < ch and 0 <= nb[1] < cw):
                continue
            i1 = len(reqs)
            reqs.append(capi.los_req(nb, td, prev_index=i0, prev_chunk=chunk))
            for nb2 in ((nb[0] + 1, nb[1]), (nb[0], nb[1] + 1), (nb[0] - 1, nb[1]), (nb[0], nb[1] - 1)):
                if not (0 <= nb2[0] < ch and 0 <= nb2[1] < cw) or nb2 == chunk:
                    continue
                reqs.append(capi.los_req(nb2, td, prev_index=i1, prev_chunk=nb))
    return np.concatenate(reqs)


def ref_los_batch(ref, reqs):
    """run a LOS request batch through the compiled reference"""
    out = np.zeros((len(reqs), 64, 64), np.uint8)
    for i, q in enumerate(reqs):
        td = (int(q["tgt_chunk_r"]), int(q["tgt_chunk_c"]), int(q["tgt_tile_r"]), int(q["tgt_tile_c"]))
        chunk = (int(q["chunk_r"]), int(q["chunk_c"]))
        if q["prev_index"] < 0:
            out[i] = ref.los(chunk, td)
        else:
            out[i] = ref.los(chunk, td, prev=out[int(q["prev_index"])], prev_chunk=(int(q["prev_chunk_r"]), int(q["prev_chunk_c"])))
    return out


def agent_case(cw, n, nflocks, seed, dens, spacing):
    """-> pathable, cost, agents dict (with ~10% ARRIVED and ~10% slow movers)"""
    p = noise_map(cw, cw, seed, dens)
    cost = synth.cost_from_pathable(p, cw, cw)
    a = synth.make_agents(cost, cw, cw, n, nflocks, seed, radius=1.0, spacing=spacing)
    rng = np.random.default_rng(seed)
    st = a["state"].copy(); st[rng.random(n) < 0.1] = 2
    a["state"] = st
    slow = rng.random(n) < 0.1
    a["vel"][slow] *= np.float32(0.05)
    a["prev_pos"] = (a["pos"] - a["vel"]).astype(np.float32)
    return p, cost, a


def relerr(g, e):
    d = np.abs(g - e).max(axis=1)
    return d / np.maximum(np.abs(e).max(axis=1), 1e-3)


def route_pairs(cost, cw, ch, seed, n):
    """n seeded (src_xz, dst_xz) pairs on passable tile centres"""
    rng = np.random.default_rng(seed)
    img = synth.blocked_to_image(cost, cw, ch)
    pas = np.argwhere(img != 255)
    out = []
    for _ in range(n):
        (sr, sc), (dr, dc) = pas[rng.integers(0, len(pas), 2)]
        out.append(((float(-(sc + 0.5) * 4), float((sr + 0.5) * 4)), (float(-(dc + 0.5) * 4), float((dr + 0.5) * 4))))
    return out


def execute_route(flow_exec, los_exec, fr, fc, lr, lc):
    """run a route's requests in order (flow merges in place per chunk; LOS as one chained batch)
    -> {chunk: flow}, {chunk: los}"""
    fields = {}
    for k in range(len(fr)):
        base = fields.get(int(fc[k]))
        out = flow_exec(fr[k:k + 1], None if fr[k]["init"] else base[None])
        fields[int(fc[k])] = out[0]
    los = los_exec(lr) if len(lr) else np.zeros((0, 64, 64), np.uint8)
    return fields, {int(lc[k]): los[k] for k in range(len(lr))}


def los_depths(lr):
    """depth of every LOS request of a batch: 1 without a parent, else its parent's + 1 (parents come first)"""
    depth = np.zeros(len(lr), np.int64)
    for i, q in enumerate(lr):
        p = int(q["prev_index"])
        depth[i] = 1 if p < 0 else depth[p] + 1
    return depth


def port_goal_fields(nav, om, target_td):
    """N_RequestGoal's plan for target_td (nav.plan_goal: flow waves, chained LOS requests) executed by the port `om`
    -> ({chunk: flow}, {chunk: los}, the plan's LOS requests, its number of flow requests)"""
    fr, fc, fw, lr, lc = nav.plan_goal(tuple(int(v) for v in target_td))
    fields = {}
    for w in range(int(fw.max()) + 1):
        sel = np.nonzero(fw == w)[0]
        base = np.stack([fields.get(int(fc[i]), np.zeros((64, 64), np.uint8)) for i in sel])
        out = om.flow_fields_update(fr[sel], inout=base)
        for k, i in enumerate(sel):
            fields[int(fc[i])] = out[k]
    los = om.los_fields_create(lr)
    return fields, {int(lc[k]): los[k] for k in range(len(lr))}, lr, len(fr)


def check_goal_pool(nav, expected, cw, nchunks):
    """every (dest, chunk) entry of the pool against port_goal_fields' results per dest: presence and bytes
    -> the number of fields compared"""
    n = 0
    for d, (flows, los) in enumerate(e[:2] for e in expected):
        for c in range(nchunks):
            f, l, _ = nav.pool_get(d, divmod(c, cw))
            assert (f is not None) == (c in flows) and (l is not None) == (c in los), (d, c)
            if f is not None:
                assert np.array_equal(f, flows[c]), (d, c)
                n += 1
            if l is not None:
                assert np.array_equal(l, los[c]), (d, c)
                n += 1
    return n


def tile_attr_case(cw, ch, seed, terrain=False):
    """int32[H32][W32][4] = {pathable, type, base_height, ramp_height} (struct tile, tile.h:101).
    terrain=False: every tile type / height combination at random (stress for n_set_cost_for_tile and
    the cliff rule); terrain=True: plateaus of different heights joined by ramps and corner tiles,
    mostly pathable, so that portals / islands downstream are non-trivial."""
    rng = np.random.default_rng(seed)
    H, W = ch * 32, cw * 32
    t = np.zeros((H, W, 4), np.int32)
    if not terrain:
        t[..., 0] = rng.random((H, W)) < 0.9
        t[..., 1] = np.where(rng.random((H, W)) < 0.6, 0, rng.integers(0, 13, (H, W)))
        t[..., 2] = rng.integers(-3, 4, (H, W))
        t[..., 3] = rng.integers(0, 4, (H, W))
        return t
    t[..., 0] = 1
    for _ in range(3 * cw * ch):                       # plateaus (cliffs all around) and lakes
        h, w = rng.integers(4, 14, 2)
        r, c = rng.integers(0, H - h), rng.integers(0, W - w)
        t[r:r + h, c:c + w, 2] = rng.integers(-2, 3)
    for _ in range(6 * cw * ch):                       # ramps / corner tiles sprinkled on the borders
        r, c = rng.integers(0, H), rng.integers(0, W)
        t[r, c, 1] = rng.integers(1, 13)
        t[r, c, 3] = rng.integers(1, 3)
    t[..., 0] &= (rng.random((H, W)) > 0.03).astype(np.int32)
    return t


def dir_quat(v):
    """dir_quat_from_velocity (movement.c:1411), float64 maths is fine for INPUT generation"""
    ang = np.arctan2(v[..., 1], v[..., 0]) - np.pi / 2
    q = np.zeros(v.shape[:-1] + (4,), np.float32)
    q[..., 1] = np.sin(ang / 2); q[..., 3] = np.cos(ang / 2)
    return q


def update_case(seed, hz):
    """Agents + movestate for the state-update pass (entity_compute_update, movement.c:2303):
    flock 0 aims at its own centre (arrivals, adjacent-arrived cascade, closest-pathable clause),
    flock 1 aims into an obstacle, random facings trip the heading gate, some histories are empty,
    a few agents are combat-held / garrisoned / have no desired velocity."""
    cw = 3
    p, cost, a = agent_case(cw, 1500, 3, seed, 0.03, 2.6)
    rng = np.random.default_rng(seed + 1000)
    n = len(a["radius"])
    img = synth.blocked_to_image(cost, cw, cw)
    # flock 0 -> centre of its own disc; flock 1 -> the impassable tile nearest to its disc centre
    c0 = a["pos"][a["flock_of"] == 0].mean(axis=0)
    a["flock_target"][0] = c0
    c1 = a["pos"][a["flock_of"] == 1].mean(axis=0)
    imp = np.argwhere(img == 255)
    if len(imp):
        xz = np.stack([-(imp[:, 1] + 0.5) * 4.0, (imp[:, 0] + 0.5) * 4.0], axis=1)
        a["flock_target"][1] = xz[np.argmin(((xz - c1) ** 2).sum(axis=1))]
    tgt = a["flock_target"][a["flock_of"]]
    d = tgt - a["pos"]
    dist = np.maximum(np.linalg.norm(d, axis=1, keepdims=True), 1e-3)
    a["vel"] = (d / dist * (0.5 * a["max_speed"][:, None] / hz)).astype(np.float32)
    a["vel"][rng.random(n) < 0.1] *= np.float32(0.05)
    a["vel"][rng.random(n) < 0.05] = 0.0
    a["prev_pos"] = (a["pos"] - a["vel"]).astype(np.float32)
    # ARRIVED members start the adjacent-arrived cascade (movement.c:2457): many in flock 0, none in 1, few in 2
    st = np.zeros(n, np.int32)
    u = rng.random(n)
    st[(a["flock_of"] == 0) & (u < 0.05)] = 2
    st[(a["flock_of"] == 2) & (u < 0.004)] = 2
    a["state"] = st
    fl = a["flags"].copy()
    fl[rng.random(n) < 0.03] |= capi.FLAG_COMBAT_HELD
    fl[rng.random(n) < 0.01] |= capi.FLAG_GARRISONED
    a["flags"] = fl
    ms = np.zeros(n, capi.MOVESTATE)
    ms["next_pos"][:, 0] = a["pos"][:, 0]; ms["next_pos"][:, 2] = a["pos"][:, 1]
    ms["step"] = 1.0 / (20 // hz)
    ms["left"] = 0 if hz == 20 else (rng.random(n) < 0.3).astype(np.int32)
    face = np.where(np.linalg.norm(a["vel"], axis=1, keepdims=True) > 1e-3, a["vel"], d / dist)
    ang = rng.uniform(-2.4, 2.4, n) * (rng.random(n) < 0.5)
    rot = np.stack([face[:, 0] * np.cos(ang) - face[:, 1] * np.sin(ang), face[:, 0] * np.sin(ang) + face[:, 1] * np.cos(ang)], axis=1)
    ms["next_rot"] = dir_quat(rot)
    ms["combat_facing"] = dir_quat(rng.normal(size=(n, 2)))
    hist = np.repeat(a["vel"][:, None, :], 14, axis=1) + rng.normal(scale=0.02, size=(n, 14, 2))
    hist[rng.random(n) < 0.3] = 0.0
    ms["vel_hist"] = hist.astype(np.float32)
    ms["vel_hist_idx"] = rng.integers(0, 14, n)
    return p, cost, a, ms


def pool_fields(nav, ndests, nchunks):
    """the device field pool read back with pool_get -> (slot[ndests * nchunks], flow[n, 64, 64], los[n, 64, 64]) as
    pfo_desired_velocity takes it: one slot per (dest, chunk) that holds a flow or a LOS field, the absent half zero
    (FD_NONE / no LOS, which is what the device reads for a missing field too)"""
    slot = np.full(ndests * nchunks, -1, np.int32)
    flow, los = [], []
    for d in range(ndests):
        for c in range(nchunks):
            f, l, _ = nav.pool_get(d, divmod(c, nav.cw))
            if f is None and l is None:
                continue
            slot[d * nchunks + c] = len(flow)
            flow.append(f if f is not None else np.zeros((64, 64), np.uint8))
            los.append(l if l is not None else np.zeros((64, 64), np.uint8))
    return slot, np.array(flow, np.uint8).reshape(-1, 64, 64), np.array(los, np.uint8).reshape(-1, 64, 64)


def port_tick(omap, agents, flocks, movestate, work, hz, arrival, pool=None, vdes=None, los=None, formation=None, ext=None,
              target_arrival=None):
    """One tick in the plain-C port (oracle/pf_oracle.c): desired velocity and LOS bit (pfo_desired_velocity over `pool`,
    else the given `vdes` / `los`), the velocity pass on them (pfo_velocity_work, every steering variant), entity_compute_update
    on the new velocities (pfo_entity_updates, all nine states) and the movestate part of entity_apply_update
    (pfo_entity_apply).
    agents / movestate: AGENT / MOVESTATE records of the whole population (not modified); flocks: FLOCK records;
    work: the uids of this tick; arrival: route_arrival_consts of every flock target; pool: pool_fields().
    formation / ext: FORMATION_IN / MOVESTATE_EXT records of the whole population (not modified) or None;
    target_arrival: per work item route_arrival_consts of an ENTER_ENTITY_RANGE item's target (None elsewhere), or None.
    -> dict(vdes, los, vel, vpref, patches, agents, movestate[, ext]), the last ones after the apply."""
    import pforacle
    work = np.ascontiguousarray(work, np.uint32)
    rec = np.array(agents, capi.AGENT)
    if pool is not None:
        vdes, los = omap.desired_velocity(rec, flocks, work, *pool)
    rec["vdes"][work] = vdes
    rec["has_dest_los"][work] = los
    world = pforacle.OracleWorld(omap, rec, flocks, hz, formation, ext)
    try:
        vel, vpref = world.velocity_work(work)
        patches = world.entity_updates(movestate, arrival, work, vel, vdes, capi.PATCH, target_arrival)
    finally:
        world.close()
    out = dict(vdes=vdes, los=los, vel=vel, vpref=vpref, patches=patches)
    if ext is None:
        out["agents"], out["movestate"] = pforacle.entity_apply(rec, movestate, work, patches)
    else:
        out["agents"], out["movestate"], out["ext"] = pforacle.entity_apply(rec, movestate, work, patches, ext)
    return out


def nav_layer(flags, radius):
    """Entity_NavLayerWithRadius (entity.c:554) for arrays: ground 0-3, water 4-7, air 8-11 by radius class
    (< 5, < 10, < 15, >= 15 wu)"""
    flags = np.asarray(flags, np.uint32); radius = np.asarray(radius, np.float32)
    base = np.where(flags & capi.FLAG_WATER, 4, np.where(flags & capi.FLAG_AIR, 8, 0))
    return (base + (radius >= 5.0) + (radius >= 10.0) + (radius >= 15.0)).astype(np.int32)


def port_tick_layers(omaps, agents, flocks, movestate, work, hz, arrivals, layer_of_unit, pool, formation=None, ext=None,
                     target_arrival=None):
    """port_tick for a population on several navigation layers. The port's world holds one layer, and a unit's layer
    only changes its own tile probes and arrival constants (neighbours are the whole population on every layer), so
    the port runs once per layer in use and every unit's results come from the run of its own layer.
    omaps / arrivals: per layer (OracleMap, route_arrival_consts of every flock target on that layer). pool=None: the
    desired velocities and LOS bits of the agent records. formation / ext / target_arrival: as port_tick (target_arrival
    per work item of `work`, each computed on its unit's layer)."""
    work = np.ascontiguousarray(work, np.uint32)
    lw = np.asarray(layer_of_unit)[work]
    out = None
    for L in np.unique(lw):
        sel = np.nonzero(lw == L)[0]
        own = {} if pool is not None else dict(vdes=agents["vdes"][work[sel]], los=agents["has_dest_los"][work[sel]])
        ta = None if target_arrival is None else [target_arrival[i] for i in sel]
        r = port_tick(omaps[L], agents, flocks, movestate, work[sel], hz, arrivals[L], pool=pool, formation=formation, ext=ext,
                      target_arrival=ta, **own)
        whole = ("agents", "movestate", "ext")
        if out is None:
            out = {k: v.copy() if k in whole else np.zeros((len(work),) + v.shape[1:], v.dtype) for k, v in r.items()}
        for k in ("vdes", "los", "vel", "vpref", "patches"):
            out[k][sel] = r[k]
        for k in whole:
            if k in r:
                out[k][work[sel]] = r[k][work[sel]]
    return out


def pforacle_map(cw, ch, cost, map_xz=(0.0, 0.0)):
    """the port's map of one layer without blockers"""
    import pforacle
    return pforacle.OracleMap(cw, ch, cost, None, None, *map_xz)


def target_arrivals(host, rec, ext, work, layer_of_unit=None):
    """per work item: N_IsMaximallyClose's tiles around the target's position of an ENTER_ENTITY_RANGE item, on the unit's
    own layer (route_arrival_consts), as pfnav_agents_compute_updates computes them; None for the other items"""
    lou = np.zeros(len(rec), np.int32) if layer_of_unit is None else np.asarray(layer_of_unit, np.int32)
    tarr = [None] * len(work)
    for i, u in enumerate(work):
        t = ext["surround_target_uid"][u]
        if rec["state"][u] == 6 and t != capi.NULL_UID:
            tarr[i] = host.route_arrival_consts(rec["pos"][t], int(lou[u]))
    return tarr


def states_port_tick(host, omaps, rec, fl, ms, form, ext, work, hz, layer_of_unit=None):
    """One tick of every movement state in the port, with the arrival constants the device computes: arrived()'s per
    (flock, layer) and, for each ENTER_ENTITY_RANGE item with a target, N_IsMaximallyClose's tiles around the target's
    position on the unit's own layer (pfnav_agents_compute_updates). host: a host-only Nav holding the same map;
    omaps: {layer: OracleMap}; rec / fl / ms / form / ext: AGENT (vdes and has_dest_los set for the work items) / FLOCK
    / MOVESTATE / FORMATION_IN / MOVESTATE_EXT records of the whole population. -> port_tick_layers' dict"""
    work = np.ascontiguousarray(work, np.uint32)
    lou = np.zeros(len(rec), np.int32) if layer_of_unit is None else np.asarray(layer_of_unit, np.int32)
    arrivals = {int(L): [host.route_arrival_consts(t, int(L)) for t in fl["target"]] for L in np.unique(lou[work])}
    tarr = target_arrivals(host, rec, ext, work, lou)
    return port_tick_layers({int(L): omaps[int(L)] for L in arrivals}, rec, fl, ms, work, hz, arrivals, lou, None,
                            formation=form, ext=ext, target_arrival=tarr)


VEL_RTOL = 1e-4


def vel_ok(vel, evel, pos, cohesion_floor=0.0):
    """north_star's 1e-4 relative -- or ONE float spacing of the entity's position, the reference's own noise floor:
    G_ClearPath_NewVelocity works in absolute map coordinates and returns `chosen point - position` (clearpath.c:694-715),
    so its result is quantised at ulp(|pos|) (3e-5 wu at |pos| = 256..512) whatever the velocity's own magnitude; a
    1e-7 relative difference in a preferred velocity (cohesion summation order) can move the chosen point by that one
    step. cohesion_floor=c widens the floor to c * |pos|: cohesion_force (movement.c:1653) divides the weighted sum of
    the member positions by the member count, not by the weights, so where that sum nearly cancels the position the
    term keeps an absolute error proportional to |pos| (the float summation of both sides, and the device's 1e-6
    relative weights), whatever the preferred velocity's own size.
    Returns (all within bounds, number of entities that needed the floor)."""
    d = np.abs(vel - evel).max(axis=1)
    rel_ok = d <= VEL_RTOL * np.maximum(np.abs(evel).max(axis=1), 1e-3)
    apos = np.abs(pos).max(axis=1).astype(np.float32)
    floor_ok = d <= np.maximum(np.spacing(apos), cohesion_floor * apos)
    return bool((rel_ok | floor_ok).all()), int((~rel_ok & floor_ok).sum())


def settle_pool(nav, passes=8, pool=None):
    """agents_tick with desired velocities from the pool, pool_repair serving the misses, until a pass requests nothing
    (nreq + nrep == 0); then the compared tick. A pool that has not settled after `passes` fails the test.
    pool=(ndests, nchunks): a pass without path requests whose repairs leave every pool byte as it was also counts as
    settled. An entity on a tile that keeps no direction after the repair (its goal tile) is repaired again every
    tick, as the reference does inline (nav.c:3508-3554), without changing the field."""
    for _ in range(passes):
        before = pool_fields(nav, *pool) if pool else None
        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        nreq, nrep = nav.pool_repair()
        if nreq + nrep == 0:
            break
        if pool and nreq == 0 and all(np.array_equal(x, y) for x, y in zip(before, pool_fields(nav, *pool))):
            break
    else:
        raise AssertionError("the field pool did not settle in %d passes: %d requests, %d repairs outstanding" % (passes, nreq, nrep))
    nav.agents_tick(capi.TICK_VDES_FROM_POOL)


def run_trajectory(nav, ref, pforacle, a, ms, cw, cost, hz, nticks, with_blockers, follow=False, ch=None,
                   map_xz=(0.0, 0.0), nlayers=1, layer_of_unit=None, tiles=None, requests=(), cohesion_modes=(), log=None, cohesion_floor=0.0):
    """tick -> entity_compute_update -> entity_apply_update -> next snapshot, `nticks` times, on both sides; the engine's
    share of the apply (entity_block: N_BlockersIncref for patches with next_block, then N_Update) is done by the test
    on our side. The device state is uploaded once and never touched again.
    With the compiled reference (ref not None) the reference runs the same ticks. follow=True: before every tick after
    the first the REFERENCE is re-seeded with the device's state (positions, velocities, movestates), so that every
    tick is compared on identical inputs; free-running, the two sides are two chaotic trajectories that separate by one
    position ulp per tick from the first ClearPath rounding step on (tests/tools/diag_traj.py prints both).
    Without it (ref None) every tick's expectation comes from the plain-C port (port_tick_layers), re-seeded before
    every tick with the device's state read back: desired velocities and LOS over the device pool's fields read back
    (both sides consume identical bytes) bit-exact, preferred velocities and velocities (vel_ok), patches (flags, states
    and blocking identical, floats within 1e-4 of max(|x|, 1)), and the state after the apply; blocker refcounts of
    every layer from a host-only context and local islands from the numpy restatement, bit-exact. Positions are
    compared within 1e-4 * max(1, max_speed / hz): 1e-4 of the largest per-tick displacement (at least one float
    spacing of the map's largest coordinate).
    The map: cw x ch chunks (ch defaults to cw) placed at map_xz, `nlayers` layers. cost: the cost grid of the one
    layer, or [nlayers][chunks][64][64]. tiles (int32[H32][W32][4]): the device builds every layer from them
    (map_cost_from_tiles) and its cost must equal `cost`; the host-only context takes `cost`. layer_of_unit: the
    navigation layer of every unit (nav_layer); a["flock_layer"], when present, the layer of every flock's fields.
    requests: (flock, src_xz) path requests (pool_request_path on the flock's layer) made before the first tick.
    cohesion_modes: every tick's velocity pass is run and compared once per mode (set_cohesion_mode) after the pool
    has settled. log: a list that receives one dict(work, layers, patches, nfloor) per tick. cohesion_floor: vel_ok's
    for preferred velocities and velocities.
    Returns the per-tick (work items, maximum position deviation, maximum velocity deviation)."""
    ch = cw if ch is None else ch
    nchunks = cw * ch
    costs = [cost] if nlayers == 1 else list(cost)
    assert len(costs) == nlayers
    assert ref is None or (nlayers == 1 and ch == cw and tuple(map_xz) == (0.0, 0.0)), "the compiled reference runs square maps at the origin, one layer"
    n = len(a["radius"])
    nflocks = len(a["flock_target"])
    lou = np.zeros(n, np.int32) if layer_of_unit is None else np.asarray(layer_of_unit, np.int32)
    if ref is not None:
        dest_ids = np.array([ref.dest_id((float(t[0]), float(t[1]))) for t in a["flock_target"]], np.uint32)
        ref.agents_set(a["pos"], a["prev_pos"], a["vel"], a["radius"], a["max_speed"], a["state"], a["flags"],
                       a["flock_of"], a["flock_target"], dest_ids, hz=hz)
        ref.movestate_set(ms["next_pos"][:, [0, 2]], ms["next_rot"], ms["step"], ms["left"], ms["vel_hist"], ms["vel_hist_idx"],
                          np.zeros(n, np.int32), np.zeros(n, np.int32), ms["combat_facing"])
    nav.map_create(cw, ch, nlayers, *map_xz)
    for L in range(nlayers):
        if tiles is not None:
            nav.map_cost_from_tiles(L, L, tiles)
            assert (nav.map_get_layer(L)[0] == costs[L]).all(), L
        else:
            nav.map_upload_layer(L, costs[L])
        nav.map_build_nav(L); nav.route_build(L)
    nav.pool_create(nflocks, nflocks * nchunks)
    aa = dict(a); aa["flock_dest_index"] = np.arange(nflocks, dtype=np.int32)
    rec, fl = capi.pack_agents(aa)
    if "flock_layer" in a:
        fl["layer"] = a["flock_layer"]
    for f, src in requests:
        nav.pool_request_path(int(f), (float(src[0]), float(src[1])), (float(fl["target"][f][0]), float(fl["target"][f][1])),
                              layer=int(fl["layer"][f]))
    nav.agents_upload(rec, fl, hz)
    nav.agents_upload_movestate(ms)
    host = None
    blk, liid = [None] * nlayers, [None] * nlayers
    if ref is None:         # blockers and the arrived() constants: the host code on a host-only copy of the map
        host = capi.Nav(hostonly=True)
        host.map_create(cw, ch, nlayers, *map_xz)
        for L in range(nlayers):
            host.map_upload_layer(L, costs[L]); host.map_build_nav(L); host.route_build(L)
    state = a["state"].copy()
    snapshot = a["pos"].copy()              # gamestate.positions of the current tick (what entity_block reads, movement.c:583)
    # 1e-4 of the largest per-tick displacement, and at least one float spacing of the map's largest coordinate
    extent = max(abs(map_xz[0]), abs(map_xz[0] - cw * 256.0), abs(map_xz[1]), abs(map_xz[1] + ch * 256.0))
    pos_tol = np.maximum(1e-4 * np.maximum(1.0, a["max_speed"] / hz), np.spacing(np.float32(extent)))
    out = []
    # settle both field caches before the first compared tick (the reference fills its cache inline while it walks the
    # entities, see test_c2_desired_velocity_from_pool_vs_reference)
    work = np.nonzero((state != 2) & (state != 4))[0].astype(np.uint32)
    if ref is not None:
        ref.work_set(work, np.zeros((len(work), 2), np.float32), np.zeros(len(work), np.uint8), a["speed"][work])
        ref.desired_from_cache()
    nfloor = 0
    try:
        for tick in range(nticks):
            work = np.nonzero((state != 2) & (state != 4))[0].astype(np.uint32)
            if len(work) == 0:
                break
            # reference
            if ref is not None:
                if follow and tick:
                    ref.agents_set(got["pos"], got["prev_pos"], got["velocity"], a["radius"], a["max_speed"], got["state"], a["flags"],
                                   a["flock_of"], a["flock_target"], dest_ids, hz=hz)
                    ref.movestate_set(gms["next_pos"][:, [0, 2]], gms["next_rot"], gms["step"], gms["left"], gms["vel_hist"],
                                      gms["vel_hist_idx"], np.zeros(n, np.int32), np.zeros(n, np.int32), gms["combat_facing"])
                ref.work_set(work, np.zeros((len(work), 2), np.float32), np.zeros(len(work), np.uint8), a["speed"][work])
                evdes, elos = ref.desired_from_cache()
                evel, _ = ref.velocity_work(os.cpu_count())
                ref.update_and_apply()
                est = ref.state_get(n)
            else:
                seed_a, seed_ms = nav.agents_read_state(n)
            # device
            nav.agents_set_work(work)
            settle_pool(nav, pool=(nflocks, nchunks))
            if ref is None:
                layers = np.unique(lou[work])
                omaps = {L: pforacle.OracleMap(cw, ch, costs[L], blk[L], liid[L], *map_xz) for L in layers}
                arrivals = {L: [host.route_arrival_consts(t, int(L)) for t in a["flock_target"]] for L in layers}
                exp = port_tick_layers(omaps, seed_a, fl, seed_ms, work, hz, arrivals, lou, pool_fields(nav, nflocks, nchunks))
                evdes, elos, evel = exp["vdes"], exp["los"], exp["vel"]
            try:
                for mode in tuple(cohesion_modes) or (None,):
                    if mode is not None:
                        nav.set_cohesion_mode(mode)
                        nav.agents_tick(capi.TICK_VDES_FROM_POOL)
                    vel = nav.agents_read_velocities(len(work))
                    vpref, vdes, los = nav.agents_read_debug(len(work))
                    assert (los == elos).all(), (tick, mode, np.nonzero(los != elos)[0][:10])
                    if ref is None or tick == 0:
                        assert (vdes == evdes).all(), (tick, mode, np.nonzero((vdes != evdes).any(axis=1))[0][:10])
                    else:   # positions carry the <= 1e-6 relative deviation of the previous ticks' velocities into the blend weights
                        assert np.abs(vdes - evdes).max() <= VEL_RTOL, (tick, np.abs(vdes - evdes).max(), np.nonzero(np.abs(vdes - evdes).max(axis=1) > VEL_RTOL)[0][:10])
                    if ref is None:
                        ok, _ = vel_ok(vpref, exp["vpref"], snapshot[work], cohesion_floor)
                        assert ok, (tick, mode, "vpref", relerr(vpref, exp["vpref"]).max(), work[np.argmax(relerr(vpref, exp["vpref"]))])
                    ok, nf = vel_ok(vel, evel, snapshot[work], cohesion_floor)
                    assert ok, (tick, mode, relerr(vel, evel).max(), work[np.argmax(relerr(vel, evel))])
                    nfloor += nf
            finally:
                if cohesion_modes:
                    nav.set_cohesion_mode(0)
            nav.agents_compute_updates()
            patches = nav.agents_read_patches(len(work))
            nav.agents_apply_updates()
            nav.agents_rebuild_index()
            got, gms = nav.agents_read_state(n)
            if log is not None:
                log.append(dict(work=work, layers=lou[work], patches=patches, nfloor=nfloor))
            if ref is None:
                ep = exp["patches"]
                same = (patches["flags"] == ep["flags"]) & (patches["next_state"] == ep["next_state"]) & (patches["next_block"] == ep["next_block"])
                assert same.all(), (tick, work[np.nonzero(~same)[0][:10]])
                pg, pe = patch_floats(patches), patch_floats(ep)
                perr = np.abs(pg - pe) / np.maximum(np.abs(pe), 1.0)
                assert perr.max() <= 1e-4, (tick, perr.max(), np.unravel_index(perr.argmax(), perr.shape))
                ea, ems = exp["agents"], exp["movestate"]
                est = dict(state=ea["state"], pos=ea["pos"], prev_pos=ea["prev_pos"], vel=ea["velocity"])
                for k in ("vel_hist_idx", "left", "step"):
                    assert (gms[k] == ems[k]).all(), (tick, k, np.nonzero(gms[k] != ems[k])[0][:10])
                herr = np.abs(gms["vel_hist"] - ems["vel_hist"]) / np.maximum(np.abs(ems["vel_hist"]), 1.0)
                assert herr.max() <= 1e-4, (tick, herr.max())
                e_next = np.abs(gms["next_pos"] - ems["next_pos"]).max(axis=1)
                assert (e_next <= pos_tol).all(), (tick, e_next.max(), np.nonzero(e_next > pos_tol)[0][:10])
            assert (got["state"] == est["state"]).all(), (tick, np.nonzero(got["state"] != est["state"])[0][:10])
            e_pos = np.abs(got["pos"] - est["pos"]).max(axis=1); e_prev = np.abs(got["prev_pos"] - est["prev_pos"]).max(axis=1)
            e_vel = relerr(got["velocity"], est["vel"]).max()
            # 1e-4 of the largest per-tick displacement (max_speed / hz wu, at least 1)
            assert (e_pos <= pos_tol).all() and (e_prev <= pos_tol).all() and vel_ok(got["velocity"], est["vel"], snapshot, cohesion_floor)[0], \
                (tick, e_pos.max(), e_prev.max(), e_vel)
            out.append((len(work), float(e_pos.max()), float(e_vel)))
            if with_blockers:
                # the engine side of entity_apply_update: entity_finish_moving -> entity_block (movement.c:685, 580)
                stopped = np.nonzero(((patches["flags"] & 1) != 0) & (patches["next_block"] != 0) &
                                     ((a["flags"][work] & capi.FLAG_GARRISONED) == 0))[0]
                for w in stopped:
                    u = work[w]
                    # G_Pos_GetXZFrom(gamestate.positions): the snapshot position of this tick, not the new one (movement.c:583)
                    for nv in (nav, host) if host is not None else (nav,):
                        nv.blockers_incref(float(snapshot[u, 0]), float(snapshot[u, 1]), float(a["radius"][u]), 0, int(a["flags"][u]))
                nav.map_commit()
                if ref is not None:
                    eblk, eliid = [ref.blockers()], [ref.local_islands()]
                else:
                    host.map_commit()
                    eblk = [host.blockers(L) for L in range(nlayers)]
                    eliid = [local_islands_np(costs[L], eblk[L]) for L in range(nlayers)]
                    blk, liid = eblk, eliid         # the port's maps of the next tick
                for L in range(nlayers):
                    assert (nav.blockers(L) == eblk[L]).all(), (tick, L)
                    assert (nav.local_islands(L) == eliid[L]).all(), (tick, L)
            state = got["state"]
            snapshot = got["pos"].copy()
    finally:
        if host is not None:
            host.close()
    # the position-ulp floor is a rare event (a rounding step of ClearPath's absolute-coordinate result), not a blanket
    if not cohesion_floor:          # with the cohesion floor the count includes that term's noise: not a rare event
        assert nfloor <= max(2, nticks // 2) * max(1, len(tuple(cohesion_modes))), nfloor
    return out


PATCH_FLOATS = ("next_velocity", "next_pos", "next_rot", "next_ppos", "next_npos", "next_step", "next_left", "next_nrot",
                "next_prot")


def patch_floats(p):
    """the 25 floats of a patch (port or device layout) -> float32[n, 25]"""
    return np.concatenate([p[k].reshape(len(p), -1) for k in PATCH_FLOATS], axis=1)


def repair_case(ref, cw, ch, seed, per_chunk=4):
    """Requests for the repair chain of N_DesiredPointSeekVelocity (nav.c:3508-3554) on a map with blockers.
    ref: a pfref.RefMap that already holds the blockers (after update()). Returns (targets FIELD_REQ[n],
    kinds, args, base fields[n,64,64], expected[n,64,64])."""
    rng = np.random.default_rng(seed)
    cost, blk, liid = ref.cost_base(), ref.blockers(), ref.local_islands()
    ports = ref.portals()
    T, K, A, B, E = [], [], [], [], []
    for chunk in range(cw * ch):
        cr, cc = chunk // cw, chunk % cw
        npass = np.argwhere((cost[chunk] != 255) & (blk[chunk] == 0))
        nonp = np.argwhere((cost[chunk] == 255) | (blk[chunk] > 0))
        if len(npass) == 0:
            continue
        bases = []
        t = npass[rng.integers(len(npass))]
        bases.append((capi.tile_req((cr, cc), (int(t[0]), int(t[1]))), ref.flow_tile((cr, cc), (int(t[0]), int(t[1]))),
                      dict(tile=(int(t[0]), int(t[1])))))
        # a blocked target tile: the frontier is empty until `ignoreblock` (field.c:2367)
        bt = np.argwhere((cost[chunk] != 255) & (blk[chunk] > 0))
        if len(bt):
            t = bt[rng.integers(len(bt))]
            bases.append((capi.tile_req((cr, cc), (int(t[0]), int(t[1]))), ref.flow_tile((cr, cc), (int(t[0]), int(t[1]))),
                          dict(tile=(int(t[0]), int(t[1])))))
        specs = portal_specs(ports[(ports[:, 0] == cr) & (ports[:, 1] == cc)][:2] if False else ports, liid, cw)
        specs = [s for s in specs if s[0] == (cr, cc)][:3]
        for s in specs:
            bases.append((portal_reqs([s]), ref.flow_portal(s[0], s[1], s[5], s[6]), dict(portal=(s[1], s[5], s[6]))))
        iids = [int(i) for i in np.unique(liid[chunk]) if i != 0xFFFF]
        for req, base, kw in bases:
            for s in (nonp[rng.integers(0, len(nonp), per_chunk)] if len(nonp) else []):
                T.append(req); K.append(0); A.append((int(s[0]) << 8) | int(s[1])); B.append(base)
                E.append(ref.flow_nearest_pathable((cr, cc), (int(s[0]), int(s[1])), base))
            for iid in iids[:per_chunk + 2]:
                T.append(req); K.append(1); A.append(iid); B.append(base)
                E.append(ref.flow_island_to_nearest((cr, cc), iid, base, **kw))
    return (np.concatenate(T), np.array(K, np.int32), np.array(A, np.int32), np.stack(B), np.stack(E))


def region_case(seed, cw=3, ch=3, n=40, dim=96):
    """Region-field scenario ("cell arrival" fields, field.c:2445-2711) on a map with faction blockers.
    -> (pathable, blockers[(x, z, radius, faction)], wars, reqs) where reqs is a list of dicts
    {center, target, enemies, overlay, start} in absolute tile coordinates (start = None: no fixup pass).
    Covers: interior regions, regions hanging over every map edge (incl. the rows < columns clamp whose visited
    array aliases, field.c:1431), a target one past the far edge (base shift, field.c:2477), overlay tiles,
    enemy masks and blocked / impassable fixup starts."""
    rng = np.random.default_rng(seed)
    p = noise_map(cw, ch, seed, 0.10)
    H, W = ch * 64, cw * 64
    blockers = [(float(-rng.uniform(10, cw * 256 - 10)), float(rng.uniform(10, ch * 256 - 10)), float(rng.uniform(2, 12)),
                 int(rng.integers(0, 4))) for _ in range(80)]
    wars = [(0, 1), (0, 2), (3, 1)]
    half = dim // 2
    reqs = []
    for i in range(n):
        kind = i % 8
        if kind in (0, 1, 2):      # interior
            cr_, cc_ = int(rng.integers(half, H - half)), int(rng.integers(half, W - half))
        elif kind == 3:            # top edge (rows clamped, columns not: aliasing flood)
            cr_, cc_ = int(rng.integers(0, half - 4)), int(rng.integers(half, W - half))
        elif kind == 4:            # left / bottom
            cr_, cc_ = int(rng.integers(H - half + 2, H)), int(rng.integers(0, half))
        elif kind == 5:            # right edge
            cr_, cc_ = int(rng.integers(half, H - half)), int(rng.integers(W - half + 1, W))
        elif kind == 6:            # corner
            cr_, cc_ = int(rng.integers(0, 20)), int(rng.integers(W - 20, W))
        else:
            cr_, cc_ = int(rng.integers(0, H)), int(rng.integers(0, W))
        lo_r, hi_r = max(cr_ - half, 0), min(cr_ + half - 1, H - 1)
        lo_c, hi_c = max(cr_ * 0 + cc_ - half, 0), min(cc_ + half - 1, W - 1)
        tr, tc = int(rng.integers(lo_r, hi_r + 1)), int(rng.integers(lo_c, hi_c + 1))
        if i % 11 == 5 and cr_ + half < H and cc_ + half < W:
            tr, tc = cr_ + half, cc_ + half          # one past the far edge: the base shifts
        ov = None
        if i % 3 == 1:
            k = int(rng.integers(1, 40))
            ov = np.stack([rng.integers(cr_ - half - 3, cr_ + half + 3, k), rng.integers(cc_ - half - 3, cc_ + half + 3, k)], 1)
            ov = ov[(ov[:, 0] >= 0) & (ov[:, 0] < H) & (ov[:, 1] >= 0) & (ov[:, 1] < W)].astype(np.int32)
        enemies = [0, 0, 0b0010, 0b0110, 0b1111][i % 5]
        reqs.append(dict(center=(cr_, cc_), target=(tr, tc), enemies=enemies, overlay=ov, start=None, want_fixup=(i % 2 == 0)))
    return p, blockers, wars, reqs


def region_pick_starts(reqs, cost, blk, cw, ch, seed, dim=96):
    """choose the fixup start of every request that wants one: a non-passable tile inside the clamped region
    (clamped_region, field.c:1892), nearest to the centre in a seeded scan order"""
    rng = np.random.default_rng(seed)
    H, W = ch * 64, cw * 64
    half = dim // 2
    img_c = cost.reshape(ch, cw, 64, 64).transpose(0, 2, 1, 3).reshape(H, W)
    img_b = blk.reshape(ch, cw, 64, 64).transpose(0, 2, 1, 3).reshape(H, W)
    nonp = (img_c == 255) | (img_b > 0)
    for q in reqs:
        if not q["want_fixup"]:
            continue
        cr_, cc_ = q["center"]
        b_r = cr_ - half if cr_ - half >= 0 else 0
        b_c = cc_ - half if cc_ - half >= 0 else 0
        e_r = cr_ + half if cr_ + half < H else H - 1
        e_c = cc_ + half if cc_ + half < W else W - 1
        cand = np.argwhere(nonp[b_r:e_r, b_c:e_c])
        if len(cand) == 0:
            continue
        s = cand[rng.integers(len(cand))]
        q["start"] = (int(s[0]) + b_r, int(s[1]) + b_c)
    return reqs


def region_reqs_from_golden(rec, ov):
    """inverse of make_golden.pack_region_reqs"""
    out, o = [], 0
    for row in rec:
        n = int(row[7])
        out.append(dict(center=(int(row[0]), int(row[1])), target=(int(row[2]), int(row[3])), enemies=int(row[4]),
                        start=None if row[5] < 0 else (int(row[5]), int(row[6])), overlay=ov[o:o + n] if n else None))
        o += n
    return out


def target_case(seed, cw=3, ch=3, n=120):
    """entities for the TARGET_ENTITY / TARGET_ENEMIES fields: positions, selection radii, factions, flags
    (all MOVABLE, ~85 % COMBATABLE) -> dict"""
    rng = np.random.default_rng(seed)
    pos = np.stack([-rng.uniform(4, cw * 256 - 4, n), rng.uniform(4, ch * 256 - 4, n)], 1).astype(np.float32)
    radius = rng.uniform(0.5, 9.0, n).astype(np.float32)
    factions = rng.integers(0, 4, n).astype(np.int32)
    flags = np.full(n, (1 << 3) | (1 << 4), np.uint32)
    flags[rng.random(n) < 0.15] &= ~np.uint32(1 << 4)
    return dict(pos=pos, radius=radius, factions=factions, flags=flags)


def enemies_of(faction, wars, factions, flags):
    """field_enemy_ent (field.c:963) with fog disabled: other faction, COMBATABLE, at war"""
    foes = [b if a == faction else a for a, b in wars if faction in (a, b)]
    return np.isin(factions, foes) & ((flags & (1 << 4)) != 0)


def stress_layout(army=256, spacing=12.0):
    """the unit layout of the reference's own stress test (scripts/test_stress.py:73-121): two armies of `army` units in
    4 rows on the 4 x 4-chunk plain map centred at the origin, red (selection radius 3.25) attacking (-100, 0), blue
    (3.00) attacking (+100, 0). -> pos[2 * army, 2], radius, flock_of, targets[2, 2]"""
    import math
    nrows = 4; ncols = math.ceil(army / nrows)
    red, blue = [], []
    for r in range(int(-nrows // 2), int(nrows // 2 + nrows % 2)):
        for c in range(int(-ncols // 2), int(ncols // 2 + ncols % 2)):
            red.append((-(r * spacing) + 35.0, c * spacing))
            blue.append(((r * spacing) - 35.0, c * spacing))
    pos = np.array(red + blue, np.float32)
    radius = np.concatenate([np.full(len(red), 3.25, np.float32), np.full(len(blue), 3.0, np.float32)])
    flock_of = np.concatenate([np.zeros(len(red), np.int32), np.ones(len(blue), np.int32)])
    return pos, radius, flock_of, np.array([[-100.0, 0.0], [100.0, 0.0]], np.float32)
