"""GPU suite: the field calls that take DEVICE buffers and queue on the caller's stream, against the plain-C port
(oracle/pf_oracle.c), byte for byte.

- (1) pfnav_flow_fields_update_dev (k_flow_unit, TMA on and off, then k_flow_general on non-unit chunks and attacking
  requests): the goal plans of pfnav_plan_goal, launched wave by wave as the planner defines them -- wave 0 with init = 1,
  wave k > 0 with init = 0 merging into the same chunk's field -- the fields gathered into the request-indexed buffer
  before each launch and scattered back after it. Maps: 1 x 1, 3 x 3 with rivers, 5 x 2, two layers with the requests on
  layer 1, bench.py's C2 map, non-unit costs (transient 0 and weights 2..254 on some chunks), blockers of four factions
  at war with attacking requests.
- (2) pfnav_flow_fields_update_general_dev (k_flow_general on every request): the same plans, and TARGET_PORTAL requests
  of every portal with PFNAV_ISLAND_NONE and with explicit island ids, then init = 0 merges of other portals into those
  fields. Equal to the port and to k_flow_unit.
- (3) pfnav_los_fields_create_dev for every LOS variant: requests in the order the caller builds them (several goals'
  pfnav_plan_goal chains concatenated, prev_index shifted, so not sorted by depth), parents named by raw request index
  (no slot table), chains 15 deep on a 1 x 16 strip, about 4 096 requests on the C2 map (more than the persistent grid's
  warps, so warps loop and wait on parents other warps are building), attacking requests and layer 1. Equal to the port
  and to the host call pfnav_los_fields_create.
- (4) pfnav_region_fields_dev: CREATE (many seeds), CREATE | CELL, CREATE | CELL | FIXUP, and FIXUP alone in place on a
  caller-held field with null seed and overlay pointers, at dims 96 and 128.
- (5) Streams: the calls return while the caller's stream is busy; stream NULL is the context's own stream; LOS batches
  on two streams, one of which grows the LOS scheduler buffer; LOS and flow batches on two streams of one context.
- (6) The argument contract, host side: n = 0, null buffers, bad wave offsets, bad region dims, host-only contexts. Each
  returns its status and queues no launch."""
import ctypes as C

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
C2_SEED = 0x5EED0001            # bench.py's C2 map
WARS = [(0, 1), (0, 2), (3, 1)]
LOS_WARPS_PER_CTA = 4           # pfnav_los_kernel.cuh
LOS_BLOCKED = 2                 # LOS field byte: bit 0 visible, bit 1 wavefront_blocked


def _enemies():
    en = np.zeros(16, np.uint16)
    for a, b in WARS:
        en[a] |= 1 << b; en[b] |= 1 << a
    return en


def _weighted(cost, seed, chunks):
    """non-unit costs on `chunks`: the transient 0 of n_clear_cost_for_tile (nav.c:359) and weights 2..254"""
    rng = np.random.default_rng(seed)
    out = cost.copy()
    for c in chunks:
        w = np.where(rng.random((64, 64)) < 0.1, 0, rng.integers(2, 255, (64, 64))).astype(np.uint8)
        out[c] = np.where(cost[c] == 255, 255, np.where(rng.random((64, 64)) < 0.4, w, 1))
    return out


def _map_spec(name):
    """-> (chunk_w, chunk_h, [cost of each layer], blockers [(x, z, radius, faction)], whether the factions are at war)"""
    if name == "1x1":
        return 1, 1, [synth.cost_from_pathable(cases.noise_map(1, 1, 0x5EED0D01, 0.05), 1, 1)], [], False
    if name in ("3x3", "weighted", "faction", "blocked"):
        cost = synth.cost_from_pathable(cases.noise_map(3, 3, 0x5EED0D03, 0.05), 3, 3)
        if name == "weighted":
            cost = _weighted(cost, 0x5EED0D03, (0, 4, 5, 7))
        blk = []
        if name in ("faction", "blocked"):      # discs of four factions; they cut portals into several local islands
            rng = np.random.default_rng(0x5EED0D03 + (name == "blocked"))
            blk = [(float(-rng.uniform(10, 3 * 256 - 10)), float(rng.uniform(10, 3 * 256 - 10)), float(rng.uniform(2, 12)),
                    int(rng.integers(0, 4))) for _ in range(120 if name == "faction" else 400)]
        return 3, 3, [cost], blk, name == "faction"
    if name == "5x2":
        return 5, 2, [synth.cost_from_pathable(cases.noise_map(5, 2, 0x5EED0D05, 0.05), 5, 2)], [], False
    if name == "layer1":        # layer 1 differs from layer 0: a kernel reading the wrong layer gives other fields
        return 2, 2, [synth.cost_from_pathable(cases.noise_map(2, 2, s, 0.05), 2, 2) for s in (0x5EED0D06, 0x5EED0D07)], [], False
    if name == "strip":
        return 16, 1, [synth.cost_from_pathable(synth.make_map(16, 1, 0x5EED0D08, frac_blocked=0.08, rivers=False), 16, 1)], [], False
    if name == "c2":
        return 16, 16, [synth.cost_from_pathable(synth.make_map(16, 16, C2_SEED, rivers=True), 16, 16)], [], False
    raise KeyError(name)


class Map:
    """one map on a context (a device context, or a host-only one to plan on), the port's map of every layer, and the
    goal plans of a seeded set of targets"""

    def __init__(self, name, pforacle, nav):
        cw, ch, costs, blockers, wars = _map_spec(name)
        self.name, self.cw, self.ch, self.costs, self.nav = name, cw, ch, costs, nav
        nav.map_create(cw, ch, len(costs))
        for L, c in enumerate(costs):
            nav.map_upload_layer(L, c); nav.map_build_nav(L)
        en = _enemies() if wars else None
        if wars:
            for f in range(15):
                nav.set_enemy_factions(f, int(en[f]))
        if blockers:
            for x, z, r, f in blockers:
                nav.blockers_incref(x, z, r, f)
            nav.map_commit()
        self.om = []
        for L, c in enumerate(costs):
            blk, liid = nav.blockers(L), nav.local_islands(L)
            fac = nav.faction_counts(L) if wars else None
            self.om.append(pforacle.OracleMap(cw, ch, c, blk, liid, factions=fac, enemies=en))
        self.liid0 = nav.local_islands(0)

    def targets(self, k, seed, layer=0):
        """k goal tiles (chunk_r, chunk_c, r, c), open and unblocked; on the strip, its two end chunks"""
        rng = np.random.default_rng(seed)
        free = (self.costs[layer] != 255) & (self.nav.blockers(layer) == 0)
        if self.name == "strip":
            free[1:self.cw - 1] = False
        idx = np.argwhere(free)
        sel = idx[rng.choice(len(idx), k, replace=False)]
        return [(int(c) // self.cw, int(c) % self.cw, int(r), int(cc)) for c, r, cc in sel]

    def plans(self, targets, layer=0, attack=()):
        """the goals' plans as one batch: flow requests, their waves and field keys (goal, chunk), and the LOS requests
        concatenated in goal order with prev_index shifted. Goals whose index is in `attack` get faction 0's requests."""
        fr_, fw_, key_, lr_ = [], [], [], []
        for g, t in enumerate(targets):
            fr, fc, fw, lr, lc = self.nav.plan_goal(t, layer)
            if g in attack:
                fr["faction_id"] = 0; lr["faction_id"] = 0
            base = sum(len(x) for x in lr_)
            lr["prev_index"] = np.where(lr["prev_index"] >= 0, lr["prev_index"] + base, lr["prev_index"])
            fr_.append(fr); fw_.append(fw); key_.append(g * self.cw * self.ch + fc); lr_.append(lr)
        return np.concatenate(fr_), np.concatenate(fw_), np.concatenate(key_), np.concatenate(lr_)


def _map_case(name, pforacle, nav):
    """the flow plan and LOS batch of each map: targets, layer, attacking goals"""
    m = Map(name, pforacle, nav)
    layer = 1 if name == "layer1" else 0
    k = {"c2": 16, "strip": 2, "1x1": 3}.get(name, 4)
    attack = (1, 3) if name == "faction" else ()
    t = m.targets(k, sum(map(ord, name)), layer)
    m.layer = layer
    m.fr, m.fw, m.fkey, m.lr = m.plans(t, layer, attack)
    if name == "c2":            # the flow fields of a few goals; the LOS batch of all 16
        m.fr, m.fw, m.fkey, _ = m.plans(t[:3], layer, attack)
    return m


def flow_port(om, reqs, wave, key):
    """the port run wave by wave -> the fields of the sorted unique keys"""
    keys = np.unique(key)
    slot = np.searchsorted(keys, key)
    F = np.zeros((len(keys), 64, 64), np.uint8)
    for w in range(int(wave.max()) + 1):
        sel = np.nonzero(wave == w)[0]
        F[slot[sel]] = om.flow_fields_update(reqs[sel], F[slot[sel]])
    return F


def los_depth(reqs):
    d = np.zeros(len(reqs), np.int64)
    for i, q in enumerate(reqs):
        d[i] = 0 if q["prev_index"] < 0 else d[int(q["prev_index"])] + 1
    return d


# ------------------------------------------------------------------------------------------------------ fixtures
@pytest.fixture(scope="module")
def torch():
    import torch as t
    return t


@pytest.fixture
def stream(torch):
    """a caller stream, current for torch too: the gathers, scatters and copies are ordered with the calls on it"""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        yield s
    torch.cuda.synchronize()


@pytest.fixture(scope="module")
def maps(pforacle):
    """Map cases by name, built once per module on contexts of their own"""
    made = {}

    def get(name):
        if name not in made:
            made[name] = _map_case(name, pforacle, capi.Nav(0))
        return made[name]
    yield get
    for m in made.values():
        m.nav.close()


def _dev(torch, a):
    return torch.from_numpy(np.ascontiguousarray(a).view(np.uint8).reshape(-1)).cuda()


def flow_dev(torch, nav, reqs, wave, key, st, general=False):
    """the plan wave by wave through the device call: gather the wave's chunk fields into a request-indexed buffer,
    launch, scatter them back"""
    keys = np.unique(key)
    slot = np.searchsorted(keys, key)
    F = torch.zeros((len(keys), 4096), dtype=torch.uint8, device="cuda")
    keep = []
    for w in range(int(wave.max()) + 1):
        sel = np.nonzero(wave == w)[0]
        assert len(np.unique(slot[sel])) == len(sel), "a wave names a chunk's field twice"
        idx = torch.from_numpy(slot[sel]).cuda()
        d_req, buf = _dev(torch, reqs[sel]), F.index_select(0, idx)
        nav.flow_fields_update_dev(d_req.data_ptr(), len(sel), buf.data_ptr(), st.cuda_stream, general)
        F.index_copy_(0, idx, buf)
        keep += [d_req, buf]
    return F.cpu().numpy().reshape(-1, 64, 64)


def los_dev(torch, nav, reqs, st):
    d_req = _dev(torch, reqs)
    out = torch.full((len(reqs), 4096), 0xA5, dtype=torch.uint8, device="cuda")     # every byte must be written
    nav.los_fields_create_dev(d_req.data_ptr(), len(reqs), out.data_ptr(), [0, len(reqs)], st.cuda_stream)
    return out.cpu().numpy().reshape(-1, 64, 64)


def _same(got, exp, what):
    bad = np.nonzero((got != exp).reshape(len(exp), -1).any(axis=1))[0]
    assert len(bad) == 0, "%s: %d of %d fields differ, first %s" % (what, len(bad), len(exp), bad[:8])


# ------------------------------------------------------------------------------------------------------ (1), (2) flow
FLOW_MAPS = ["1x1", "3x3", "5x2", "layer1", "c2", "weighted", "faction", "blocked"]


@pytest.mark.parametrize("name", FLOW_MAPS)
def test_flow_plan_waves(torch, maps, stream, name):
    """a goal plan's flow waves: k_flow_unit with TMA off and on (followed by k_flow_general where the map has non-unit
    chunks or attacking requests), and the forced general kernel, all equal to the port run in the same wave order"""
    m = maps(name)
    exp = flow_port(m.om[m.layer], m.fr, m.fw, m.fkey)
    nz = int((exp.reshape(len(exp), -1) != 0).any(axis=1).sum())
    assert nz == len(exp), (nz, len(exp))                  # a plan's fields all lead somewhere
    if name != "1x1":
        assert (m.fr["target_type"] == capi.TARGET_PORTAL).sum() > 0
    if name not in ("1x1", "layer1"):
        assert (m.fw > 0).sum() > 0                        # init = 0 merges into a field of an earlier wave
    if name == "layer1":
        assert (m.fr["layer"] == 1).all()
        assert (flow_port(m.om[0], m.fr, m.fw, m.fkey) != exp).any(), "layer 0 gives the same fields"
    if name == "faction":
        assert (m.fr["faction_id"] == 0).sum() > 0 and (m.fr["faction_id"] == capi.FACTION_ID_NONE).sum() > 0
    for tma in (0, 1):
        m.nav.set_tma(tma)
        unit = flow_dev(torch, m.nav, m.fr, m.fw, m.fkey, stream)
        _same(unit, exp, "flow_fields_update_dev tma=%d" % tma)
    general = flow_dev(torch, m.nav, m.fr, m.fw, m.fkey, stream, general=True)
    _same(general, exp, "flow_fields_update_general_dev")
    _same(general, unit, "flow_fields_update_general_dev vs flow_fields_update_dev")


@pytest.mark.parametrize("name", ["5x2", "blocked"])
def test_general_portal_seeds(torch, maps, stream, name):
    """TARGET_PORTAL requests of every portal (border chunks included) with PFNAV_ISLAND_NONE and explicit island ids on
    maps with cut-off islands, then init = 0 merges of another portal of the same chunk into each field: the general
    kernel and k_flow_unit equal the port"""
    m = maps(name)
    specs = cases.portal_specs(m.nav.portals(0), m.liid0, m.cw)
    reqs = cases.portal_reqs(specs)
    assert (reqs["port_iid"] == capi.ISLAND_NONE).sum() > 0 and (reqs["port_iid"] != capi.ISLAND_NONE).sum() > 0
    # the port_iid filter decides: portals whose tiles belong to more than one local island
    multi = sum(1 for s in specs if s[5] != capi.ISLAND_NONE and len(np.unique(
        m.liid0[s[0][0] * m.cw + s[0][1]][s[2][0]:s[2][2] + 1, s[2][1]:s[2][3] + 1])) > 1)
    assert multi > 0 or name != "blocked"
    # merges: request i's field is updated by the next spec of the same chunk
    chunk = reqs["chunk_r"] * m.cw + reqs["chunk_c"]
    nxt = np.arange(len(reqs))
    for c in np.unique(chunk):
        idx = np.nonzero(chunk == c)[0]
        nxt[idx] = np.roll(idx, -1)
    merge = reqs[nxt].copy()
    merge["init"] = 0
    om = m.om[0]
    exp1 = om.flow_fields_update(reqs)
    exp2 = om.flow_fields_update(merge, exp1)
    assert (exp2 != exp1).reshape(len(reqs), -1).any(axis=1).sum() > len(reqs) // 4
    d1, d2 = _dev(torch, reqs), _dev(torch, merge)
    for general in (True, False):
        out = torch.zeros((len(reqs), 4096), dtype=torch.uint8, device="cuda")
        m.nav.flow_fields_update_dev(d1.data_ptr(), len(reqs), out.data_ptr(), stream.cuda_stream, general)
        _same(out.cpu().numpy().reshape(-1, 64, 64), exp1, "portal seeds, general=%s" % general)
        m.nav.flow_fields_update_dev(d2.data_ptr(), len(reqs), out.data_ptr(), stream.cuda_stream, general)
        _same(out.cpu().numpy().reshape(-1, 64, 64), exp2, "init = 0 merges, general=%s" % general)


# ------------------------------------------------------------------------------------------------------ (3) LOS
LOS_MAPS = ["3x3", "strip", "c2", "faction", "layer1"]
_los_exp = {}


@pytest.mark.parametrize("variant", [0, 1, 2])
@pytest.mark.parametrize("name", LOS_MAPS)
def test_los_unslotted(torch, maps, stream, name, variant):
    """requests in the caller's order, parents by raw index: equal to the port and to the host call, which packs the
    same batch by depth through a slot table"""
    m = maps(name)
    reqs = m.lr
    d = los_depth(reqs)
    assert (np.diff(d) < 0).any(), "the batch is sorted by depth"
    if name not in _los_exp:
        _los_exp[name] = m.om[m.layer].los_fields_create(reqs)
    exp = _los_exp[name]
    assert (exp.reshape(len(exp), -1) != 0).any(axis=1).sum() > len(exp) // 8
    assert ((exp & LOS_BLOCKED) != 0).reshape(len(exp), -1).any(axis=1).sum() > 0
    if name == "strip":
        assert d.max() == 15
    if name == "c2":
        assert len(reqs) > torch.cuda.get_device_properties(0).multi_processor_count * 2 * LOS_WARPS_PER_CTA * 3
    if name == "faction":
        assert (reqs["faction_id"] == 0).sum() > 0
    if name == "layer1":
        assert (reqs["layer"] == 1).all() and (m.om[0].los_fields_create(reqs) != exp).any()
    m.nav.set_los_variant(variant)
    try:
        _same(los_dev(torch, m.nav, reqs, stream), exp, "los_fields_create_dev variant %d" % variant)
        _same(m.nav.los_fields_create(reqs), exp, "los_fields_create variant %d" % variant)
    finally:
        m.nav.set_los_variant(2)


# ------------------------------------------------------------------------------------------------------ (4) region
@pytest.fixture(scope="module")
def region_nav():
    nav = capi.Nav(0)
    yield nav
    nav.close()


def _region_setup(nav, pforacle, cost, blockers, wars, cw=3, ch=3):
    nav.map_create(cw, ch, 1)
    nav.map_upload_layer(0, cost); nav.map_build_nav(0)
    en = np.zeros(16, np.uint16)
    for a, b in wars:
        en[a] |= 1 << b; en[b] |= 1 << a
    for f in range(15):
        nav.set_enemy_factions(f, int(en[f]))
    for x, z, r, f in blockers:
        nav.blockers_incref(float(x), float(z), float(r), int(f), 0)
    nav.map_commit()
    blk = nav.blockers(0)
    return blk, pforacle.OracleMap(cw, ch, cost, blk, None, factions=nav.faction_counts(0))


def _region_dev(torch, nav, dim, rec, sd, ov, st, inout=None):
    d_req = _dev(torch, rec)
    d_sd = torch.from_numpy(sd).cuda() if len(sd) else None
    d_ov = torch.from_numpy(ov).cuda() if len(ov) else None
    out = (torch.zeros((len(rec), dim * dim // 2), dtype=torch.uint8, device="cuda") if inout is None
           else torch.from_numpy(np.ascontiguousarray(inout).reshape(len(rec), -1)).cuda())
    nav.region_fields_dev(dim, d_req.data_ptr(), len(rec), 0 if d_sd is None else d_sd.data_ptr(),
                          0 if d_ov is None else d_ov.data_ptr(), out.data_ptr(), st.cuda_stream)
    return out.cpu().numpy().reshape(len(rec), dim, dim // 2)


@pytest.mark.parametrize("dim", [96, 128])
def test_region_dev(torch, pforacle, region_nav, stream, dim):
    """CREATE | CELL with and without FIXUP, CREATE with many seeds, and FIXUP alone in place on a caller-held field
    (no seeds and no overlay in that batch: null pointers) == OracleMap.region_field_create / region_field_fixup"""
    nav, seed = region_nav, 0x5EED0D10 + dim
    p, blockers, wars, reqs = cases.region_case(seed, 3, 3, 40, dim)
    cost = synth.cost_from_pathable(p, 3, 3)
    blk, om = _region_setup(nav, pforacle, cost, blockers, wars)
    cases.region_pick_starts(reqs, cost, blk, 3, 3, seed, dim)
    fix = [i for i, q in enumerate(reqs) if q["start"] is not None]
    assert 0 < len(fix) < len(reqs) and sum(q["overlay"] is not None for q in reqs) > 0
    assert sum(q["enemies"] != 0 for q in reqs) > 0
    create = np.stack([om.region_field_create(dim, q["enemies"], 1, [q["target"]], q["center"], q["overlay"]) for q in reqs])
    exp = create.copy()
    for i in fix:
        exp[i] = om.region_field_fixup(dim, reqs[i]["start"], reqs[i]["center"], create[i], reqs[i]["overlay"])
    assert (exp[fix] != create[fix]).any() and (create != 0).reshape(len(reqs), -1).any(axis=1).sum() > len(reqs) // 2
    rec, sd, ov = capi.pack_region_reqs(reqs)
    assert ((rec["flags"] & capi.REGION_FIXUP) != 0).sum() == len(fix) and (rec["flags"] & capi.REGION_CELL).all()
    _same(_region_dev(torch, nav, dim, rec, sd, ov, stream), exp, "region CREATE | CELL [| FIXUP]")
    # FIXUP alone on the create-only fields, no seed and no overlay anywhere in the batch
    fq = [dict(reqs[i], overlay=None, no_create=True, cell=False) for i in fix]
    rec, sd, ov = capi.pack_region_reqs(fq)
    rec["seed_n"] = 0; rec["seed_off"] = 0
    assert (rec["flags"] == capi.REGION_FIXUP).all()
    efix = np.stack([om.region_field_fixup(dim, q["start"], q["center"], create[i]) for q, i in zip(fq, fix)])
    assert (efix != create[fix]).any()
    _same(_region_dev(torch, nav, dim, rec, np.zeros((0, 2), np.int32), np.zeros((0, 2), np.int32), stream,
                      inout=create[fix]), efix, "region FIXUP in place")
    # CREATE with many seeds (tile-space group arrival), no base shift
    rng = np.random.default_rng(seed)
    greqs = [dict(center=q["center"], seeds=np.stack([rng.integers(0, 192, 20), rng.integers(0, 192, 20)], 1),
                  enemies=q["enemies"], overlay=q["overlay"], start=None, cell=False) for q in reqs[:16]]
    rec, sd, ov = capi.pack_region_reqs(greqs)
    assert (rec["flags"] == capi.REGION_CREATE).all()
    eg = np.stack([om.region_field_create(dim, q["enemies"], 0, q["seeds"], q["center"], q["overlay"]) for q in greqs])
    _same(_region_dev(torch, nav, dim, rec, sd, ov, stream), eg, "region CREATE")


# ------------------------------------------------------------------------------------------------------ (5) streams
def _fresh(pforacle, name="3x3"):
    """a context of its own: nothing else has sized its LOS scheduler buffer"""
    return _map_case(name, pforacle, capi.Nav(0))


def test_dev_calls_return_while_stream_busy(torch, pforacle, stream):
    m = _fresh(pforacle)
    try:
        w0 = np.nonzero(m.fw == 0)[0]
        fr = m.fr[w0]
        ef = m.om[0].flow_fields_update(fr)
        el = m.om[0].los_fields_create(m.lr)
        rq = [dict(center=(96, 96), target=(100, 101), enemies=0, overlay=None, start=None)]
        rec, sd, ov = capi.pack_region_reqs(rq)
        er = m.om[0].region_field_create(96, 0, 1, [rq[0]["target"]], rq[0]["center"])
        d_fr, d_lr, d_rq, d_sd = _dev(torch, fr), _dev(torch, m.lr), _dev(torch, rec), torch.from_numpy(sd).cuda()
        f1 = torch.zeros((len(fr), 4096), dtype=torch.uint8, device="cuda")
        f2, lo = torch.zeros_like(f1), torch.zeros((len(m.lr), 4096), dtype=torch.uint8, device="cuda")
        ro = torch.zeros((1, 96 * 48), dtype=torch.uint8, device="cuda")
        st = stream.cuda_stream

        def calls():
            m.nav.flow_fields_update_dev(d_fr.data_ptr(), len(fr), f1.data_ptr(), st)
            m.nav.flow_fields_update_dev(d_fr.data_ptr(), len(fr), f2.data_ptr(), st, general=True)
            m.nav.los_fields_create_dev(d_lr.data_ptr(), len(m.lr), lo.data_ptr(), [0, len(m.lr)], st)
            m.nav.region_fields_dev(96, d_rq.data_ptr(), 1, d_sd.data_ptr(), 0, ro.data_ptr(), st)
        calls()                                                 # sizes the context's buffers
        torch.cuda.synchronize()
        for t in (f1, f2, lo, ro):
            t.zero_()
        torch.cuda._sleep(200_000_000)                          # a bounded spin on the stream, about 0.1 s
        calls()
        busy = not stream.query()
        torch.cuda.synchronize()
        assert busy, "a dev call waited for its stream"
        _same(f1.cpu().numpy().reshape(-1, 64, 64), ef, "flow")
        _same(f2.cpu().numpy().reshape(-1, 64, 64), ef, "general")
        _same(lo.cpu().numpy().reshape(-1, 64, 64), el, "LOS")
        _same(ro.cpu().numpy().reshape(1, 96, 48), er[None], "region")
    finally:
        m.nav.close()


def test_null_stream_is_the_context_stream(torch, pforacle, stream):
    """stream NULL queues on the context's own stream: the synchronous host call that follows on the same context
    returns after the device call's work, so its fields can be read without a synchronise"""
    m = _fresh(pforacle)
    try:
        w0 = np.nonzero(m.fw == 0)[0]
        fr = m.fr[w0]
        d_fr, d_lr = _dev(torch, fr), _dev(torch, m.lr)
        fo = torch.zeros((len(fr), 4096), dtype=torch.uint8, device="cuda")
        lo = torch.zeros((len(m.lr), 4096), dtype=torch.uint8, device="cuda")
        torch.cuda.synchronize()                                # the inputs are on the device before the context's stream reads them
        m.nav.flow_fields_update_dev(d_fr.data_ptr(), len(fr), fo.data_ptr(), 0)
        m.nav.los_fields_create_dev(d_lr.data_ptr(), len(m.lr), lo.data_ptr(), [0, len(m.lr)], 0)
        host = m.nav.los_fields_create(m.lr[:1])
        fo_h, lo_h = fo.cpu().numpy().reshape(-1, 64, 64), lo.cpu().numpy().reshape(-1, 64, 64)
        _same(fo_h, m.om[0].flow_fields_update(fr), "flow on stream NULL")
        el = m.om[0].los_fields_create(m.lr)
        _same(lo_h, el, "LOS on stream NULL")
        _same(host, el[:1], "host call")
    finally:
        m.nav.close()


def test_los_batches_on_two_streams(torch, pforacle, stream):
    """back-to-back LOS batches on two caller streams of one context: the second is larger than any earlier one, so the
    scheduler buffer grows; a third, smaller one follows on the first stream. All equal the port."""
    m = _fresh(pforacle)
    try:
        other = torch.cuda.Stream()
        n = len(m.lr)
        big = m.lr.copy()
        big2 = m.lr.copy()
        big2["prev_index"] = np.where(big2["prev_index"] >= 0, big2["prev_index"] + n, -1)
        big = np.concatenate([big, big2])
        small = m.lr[:n // 2]
        assert (small["prev_index"] < len(small)).all()
        batches = [(m.lr[:n - 1], stream), (big, other), (small, stream)]
        exp = [m.om[0].los_fields_create(b) for b in (m.lr, big)]
        d = [(_dev(torch, b), torch.full((len(b), 4096), 0xA5, dtype=torch.uint8, device="cuda"), s) for b, s in batches]
        torch.cuda.synchronize()
        torch.cuda._sleep(200_000_000)                          # the first stream is still busy when the others queue
        for (dr, out, s), (b, _) in zip(d, batches):
            m.nav.los_fields_create_dev(dr.data_ptr(), len(b), out.data_ptr(), [0, len(b)], s.cuda_stream)
        torch.cuda.synchronize()
        _same(d[0][1].cpu().numpy().reshape(-1, 64, 64), exp[0][:n - 1], "first batch, stream A")
        _same(d[1][1].cpu().numpy().reshape(-1, 64, 64), exp[1], "larger batch, stream B")
        _same(d[2][1].cpu().numpy().reshape(-1, 64, 64), exp[0][:n // 2], "smaller batch, stream A")
    finally:
        m.nav.close()


def test_los_and_flow_on_two_streams(torch, maps, stream):
    m = maps("5x2")
    other = torch.cuda.Stream()
    el = m.om[0].los_fields_create(m.lr)
    w0 = np.nonzero(m.fw == 0)[0]
    ef = m.om[0].flow_fields_update(m.fr[w0])
    d_lr, d_fr = _dev(torch, m.lr), _dev(torch, m.fr[w0])
    lo = torch.zeros((len(m.lr), 4096), dtype=torch.uint8, device="cuda")
    fo = torch.zeros((len(w0), 4096), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    m.nav.los_fields_create_dev(d_lr.data_ptr(), len(m.lr), lo.data_ptr(), [0, len(m.lr)], stream.cuda_stream)
    m.nav.flow_fields_update_dev(d_fr.data_ptr(), len(w0), fo.data_ptr(), other.cuda_stream)
    torch.cuda.synchronize()
    _same(lo.cpu().numpy().reshape(-1, 64, 64), el, "LOS on stream A")
    _same(fo.cpu().numpy().reshape(-1, 64, 64), ef, "flow on stream B")


# ------------------------------------------------------------------------------------------------------ (6) arguments
def _calls(nav, fp, lp, rp, out, n, wo, dim=96, seeds=None, overlay=None):
    """the four dev calls with raw arguments -> their return codes"""
    L, h = nav.L, nav.h
    w = np.ascontiguousarray(wo, np.int32)
    return (L.pfnav_flow_fields_update_dev(h, fp, n, out, None),
            L.pfnav_flow_fields_update_general_dev(h, fp, n, out, None),
            L.pfnav_los_fields_create_dev(h, lp, n, out, len(w) - 1, w.ctypes.data_as(C.c_void_p) if len(w) else None, None),
            L.pfnav_region_fields_dev(h, dim, rp, n, seeds, overlay, out, None))


def test_argument_contract(torch, pforacle, maps):
    m = maps("3x3")
    nav = m.nav
    lr, fr = m.lr[:1], m.fr[:1]
    assert lr["prev_index"][0] == -1 and fr["init"][0] == 1    # a destination-chunk LOS request, a first flow request
    rq, sd, _ = capi.pack_region_reqs([dict(center=(96, 96), target=(100, 101), enemies=0, overlay=None, start=None)])
    d_fr, d_lr, d_rq, d_sd = _dev(torch, fr), _dev(torch, lr), _dev(torch, rq), torch.from_numpy(sd).cuda()
    out = torch.zeros(96 * 48 + 4096, dtype=torch.uint8, device="cuda")
    fp, lp, rp, op, sp = (C.c_void_p(t.data_ptr()) for t in (d_fr, d_lr, d_rq, out, d_sd))
    torch.cuda.synchronize()
    n0 = nav.launch_count()
    assert _calls(nav, fp, lp, rp, op, 1, [0, 1], seeds=sp) == (capi.OK,) * 4 and nav.launch_count() > n0
    torch.cuda.synchronize()
    ERR = capi.ERR_ARG
    cases_ = [
        ("n = 0", (fp, lp, rp, op, 0, [0, 0]), (capi.OK,) * 4),
        ("n = 0, null buffers", (None, None, None, None, 0, []), (capi.OK,) * 4),
        ("null requests", (None, None, None, op, 1, [0, 1]), (ERR,) * 4),
        ("null fields", (fp, lp, rp, None, 1, [0, 1]), (ERR,) * 4),
    ]
    for what, args, want in cases_:
        n0 = nav.launch_count()
        assert _calls(nav, *args, seeds=sp) == want, what
        assert nav.launch_count() == n0, what
    L, h = nav.L, nav.h
    for what, nw, wo in (("n_waves = 0", 0, [0]), ("n_waves < 0", -1, [0, 1]), ("null offsets", 1, None),
                         ("offsets start at 1", 1, [1, 1]), ("offsets end short", 1, [0, 0]), ("offsets end past n", 2, [0, 1, 2]),
                         ("offsets decrease", 3, [0, 1, 0, 1])):
        n0 = nav.launch_count()
        w = None if wo is None else np.ascontiguousarray(wo, np.int32)
        rc = L.pfnav_los_fields_create_dev(h, lp, 1, op, nw, None if w is None else w.ctypes.data_as(C.c_void_p), None)
        assert rc == ERR and nav.launch_count() == n0, what
    n0 = nav.launch_count()
    assert L.pfnav_los_fields_create_dev(h, lp, 1, op, 3, np.array([0, 0, 1, 1], np.int32).ctypes.data_as(C.c_void_p), None) == capi.OK
    assert nav.launch_count() == n0 + 1                        # empty waves are fine
    for dim in (95, 0, 130, -2):
        n0 = nav.launch_count()
        assert L.pfnav_region_fields_dev(h, dim, rp, 1, sp, None, op, None) == ERR, dim
        assert nav.launch_count() == n0
    torch.cuda.synchronize()
    # a host-only context has no compute path: with a map, every call says so; without one, the map is missing
    ho = capi.Nav(hostonly=True)
    try:
        assert _calls(ho, fp, lp, rp, op, 1, [0, 1], seeds=sp) == (ERR,) * 4
        ho.map_create(3, 3, 1)
        want = (capi.ERR_NO_DEVICE,) * 4
        assert _calls(ho, fp, lp, rp, op, 1, [0, 1], seeds=sp) == want
        assert _calls(ho, fp, lp, rp, op, 0, [0, 0], seeds=sp) == want
        assert ho.launch_count() == 0
    finally:
        ho.close()
