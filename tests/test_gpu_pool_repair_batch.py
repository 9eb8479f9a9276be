"""GPU suite: pfnav_pool_repair_batch, the on-miss chain of N_DesiredPointSeekVelocity in device rounds, against the
serial loop pfnav_pool_repair on two contexts built from the same seeds. After every call the counts, every pool entry
(has bits, ff_id, flow and LOS bytes) and the next tick's velocities, desired velocities and LOS flags are equal."""
import ctypes as C
import os

import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
ST_SEEK, ST_SURROUND = 3, 5
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


class Pair:
    """two identically built contexts: [0] runs the serial loop, [1] the batch"""

    def __init__(self, cw, ch, seed, nlayers=1, frac_blocked=0.2, cost=None, blk=None, liid=None, rivers=None):
        self.cw, self.ch = cw, ch
        if cost is None:
            rivers = cw > 1 if rivers is None else rivers
            cost = synth.cost_from_pathable(synth.make_map(cw, ch, seed, frac_blocked=frac_blocked, rivers=rivers), cw, ch)
        self.navs = [capi.Nav(0) for _ in range(2)]
        for nav in self.navs:
            nav.map_create(cw, ch, nlayers)
            for layer in range(nlayers):
                if blk is None:
                    nav.map_upload_layer(layer, cost)
                else:
                    nav.map_upload_layer(layer, cost, blk, liid)
                nav.map_build_nav(layer)
                nav.route_build(layer)
        self.cost = cost

    def each(self, fn):
        return [fn(nav) for nav in self.navs]

    def close(self):
        for nav in self.navs:
            nav.close()

    def pool(self, ndests):
        out = []
        for d in range(ndests):
            for c in range(self.cw * self.ch):
                rows = [nav.pool_get(d, divmod(c, self.cw)) for nav in self.navs]
                out.append(rows)
        return out

    def repair(self, ndests, tick_flags=capi.TICK_VDES_FROM_POOL):
        """tick both, serial on one and batch on the other; -> (nreq, nrep, nrounds); asserts equal pools and ticks"""
        self.each(lambda nav: nav.agents_tick(tick_flags))
        s = self.navs[0].pool_repair()
        b = self.navs[1].pool_repair_batch()
        assert s == b[:2], (s, b)
        self.stats = self.navs[1].pool_repair_batch_stats()
        self.assert_same(ndests)
        return b

    def assert_same(self, ndests):
        for (fa, la, ia), (fb, lb, ib) in self.pool(ndests):
            assert ia == ib
            assert (fa is None) == (fb is None) and (la is None) == (lb is None)
            assert fa is None or (fa == fb).all()
            assert la is None or (la == lb).all()
        self.each(lambda nav: nav.agents_tick(capi.TICK_VDES_FROM_POOL))
        n = self.navs[0].nwork
        a = [nav.agents_read_debug(n) for nav in self.navs]
        v = [nav.agents_read_velocities(n) for nav in self.navs]
        assert (a[0][1] == a[1][1]).all() and (a[0][2] == a[1][2]).all()
        assert (v[0] == v[1]).all()


def _agents(cost, cw, ch, n, seed, flocks, on_blocked=0.5, radius=1.0):
    """n agents, a share of them on blocked tiles, spread over `flocks` flocks"""
    rng = np.random.default_rng(seed)
    img = synth.blocked_to_image(cost, cw, ch)
    free, wall = np.argwhere(img != 255), np.argwhere(img == 255)
    nb = int(n * on_blocked) if len(wall) else 0
    t = np.concatenate([wall[rng.integers(0, len(wall), nb)] if nb else np.zeros((0, 2), np.int64),
                        free[rng.integers(0, len(free), n - nb)]])
    t = t[rng.permutation(n)]
    pos = np.stack([-(t[:, 1] + rng.uniform(0.05, 0.95, n)) * 4.0, (t[:, 0] + rng.uniform(0.05, 0.95, n)) * 4.0], 1).astype(np.float32)
    rec = np.zeros(n, capi.AGENT)
    rec["pos"] = pos; rec["prev_pos"] = pos; rec["radius"] = radius; rec["max_speed"] = 20.0; rec["speed"] = 20.0
    rec["flags"] = capi.FLAG_MOVABLE; rec["flock"] = rng.integers(0, len(flocks), n)
    fl = np.zeros(len(flocks), capi.FLOCK)
    for f, (tile, dest, layer) in enumerate(flocks):
        fl["target"][f] = (-(tile[1] + 0.5) * 4.0, (tile[0] + 0.5) * 4.0)
        fl["dest"][f] = dest; fl["layer"][f] = layer
    return rec, fl


def _wp(r, c):
    """world position of the centre of absolute tile (r, c)"""
    return (-(c + 0.5) * 4.0, (r + 0.5) * 4.0)


def _walled_2x2():
    """a unit-cost 2 x 2 map: chunk (0, 1) cut into an upper and a lower part by a wall row (each part has its own
    portal to chunk (0, 0)); chunk (1, 1) sealed from chunk (1, 0) and cut into a left and a right part, each with its
    own portal up into the lower part of chunk (0, 1)"""
    img = np.ones((128, 128), np.uint8)
    img[30, 64:128] = 255
    img[64:128, 64] = 255
    img[64:128, 96] = 255
    return synth.image_to_blocked(img, 2, 2)


def _place(rec, tiles, prev):
    """agent i stands on tiles[i]; every previous position is `prev` (a tile whose chunk holds its LOS field)"""
    rec["pos"] = np.array([_wp(*t) for t in tiles], np.float32)
    rec["prev_pos"] = np.array(_wp(*prev), np.float32)


def _free_tile(cost, cw, ch, seed):
    img = synth.blocked_to_image(cost, cw, ch)
    free = np.argwhere(img != 255)
    return tuple(int(v) for v in free[np.random.default_rng(seed).integers(0, len(free))])


def _upload(P, rec, fl, ndests, pool_max):
    for nav in P.navs:
        nav.pool_create(ndests, pool_max)
        nav.agents_upload(rec, fl, 20)
        nav.agents_set_work(np.arange(len(rec), dtype=np.uint32))


def _drive(P, ndests, steps=4):
    rounds = []
    for _ in range(steps):
        r = P.repair(ndests)
        rounds.append(r[2])
        if r[0] + r[1] == 0:
            break
    return rounds


def test_golden_repair_pool():
    """repair_pool.npz driven to its golden desired velocities and LOS flags, the batch on one side"""
    g = np.load(os.path.join(GOLDEN, "repair_pool.npz"))
    pos, target = g["pos"], g["target"]
    n = len(pos)
    P = Pair(2, 2, 0, cost=g["cost"], blk=g["blk"], liid=g["liid"])
    try:
        for nav in P.navs:
            nav.pool_create(1, 8)
            nav.pool_request_path(0, (float(pos[0, 0]), float(pos[0, 1])), (float(target[0]), float(target[1])))
        rec = np.zeros(n, capi.AGENT)
        rec["pos"] = pos; rec["prev_pos"] = pos; rec["radius"] = 1.0; rec["max_speed"] = 20.0; rec["speed"] = 20.0
        rec["flags"] = capi.FLAG_MOVABLE; rec["flock"] = 0
        fl = np.zeros(1, capi.FLOCK); fl["target"] = target; fl["dest"] = 0; fl["layer"] = 0
        for nav in P.navs:
            nav.agents_upload(rec, fl, 20)
            nav.agents_set_work(np.arange(n, dtype=np.uint32))
        total = sum(P.repair(1)[:2] != (0, 0) for _ in range(4))
        assert total > 0
        P.navs[1].agents_tick(capi.TICK_VDES_FROM_POOL)
        _, vdes, los = P.navs[1].agents_read_debug(n)
        assert (vdes == g["vdes"]).all() and (los == g["los"]).all()
    finally:
        P.close()


@pytest.mark.parametrize("cw", [1, 2, 4])
def test_maps_and_flocks(cw):
    """1x1, 2x2 and 4x4 maps, several flocks, two of them sharing a destination, half the agents on blocked tiles"""
    P = Pair(cw, cw, 0x5EED0700 + cw)
    try:
        flocks = [(_free_tile(P.cost, cw, cw, k), k % 3, 0) for k in range(4)]
        rec, fl = _agents(P.cost, cw, cw, 1500, cw, flocks)
        _upload(P, rec, fl, 3, 3 * cw * cw)
        assert _drive(P, 3)
    finally:
        P.close()


def test_islands_cut_off_by_blockers_and_churn():
    """islands cut off by blockers (ISLAND_TO_NEAREST) and blockers landing on agents over churn + commit +
    REQUEST_MISSING_ONLY steps"""
    cw = 4
    P = Pair(cw, cw, 0x5EED0720, frac_blocked=0.1)
    try:
        flocks = [(_free_tile(P.cost, cw, cw, k), k, 0) for k in range(2)]
        rec, fl = _agents(P.cost, cw, cw, 3000, 5, flocks, on_blocked=0.1)
        _upload(P, rec, fl, 2, 2 * cw * cw)
        goals = np.array([[t[0] // 64, t[1] // 64, t[0] % 64, t[1] % 64] for t, _, _ in flocks], np.int32)
        rng = np.random.default_rng(3)
        bl = rec["pos"][rng.integers(0, len(rec), 60)].copy()
        for nav in P.navs:
            nav.pool_request_goals(np.arange(2, dtype=np.int32), goals, 0)
        for step in range(4):
            for nav in P.navs:
                for x, z in bl:
                    nav.blockers_incref(float(x), float(z), 10.0, 0)
                nav.map_commit()
                nav.pool_request_goals(np.arange(2, dtype=np.int32), goals, 0, 0, capi.REQUEST_MISSING_ONLY)
            P.repair(2)
            bl += rng.integers(-1, 2, size=bl.shape).astype(np.float32) * 4.0
    finally:
        P.close()


@pytest.mark.parametrize("nlayers,faction,pool_max", [(2, None, 64), (1, 2, 64), (1, None, 10), (2, 2, 10)])
def test_layers_faction_and_eviction(nlayers, faction, pool_max):
    """flocks on two layers, an attacking faction, and a pool small enough to evict"""
    cw = 4
    P = Pair(cw, cw, 0x5EED0730, nlayers=nlayers)
    try:
        if faction is not None:          # attacking requests read the enemy tables (pfnav_set_enemy_factions)
            for nav in P.navs:
                for f in range(15):
                    nav.set_enemy_factions(f, 1 << ((f + 1) % 15))
                nav.request_faction(faction)
        flocks = [(_free_tile(P.cost, cw, cw, 10 + k), k, k % nlayers) for k in range(4)]
        rec, fl = _agents(P.cost, cw, cw, 2500, 7, flocks, on_blocked=0.3)
        _upload(P, rec, fl, 4, pool_max)
        rounds = _drive(P, 4)
        assert max(rounds) >= 1
        if pool_max < 16:
            assert max(rounds) >= 2
    finally:
        P.close()


def test_boundary_rules():
    """rounds end where a request depends on bytes written earlier in the round, writes a slot with a pending repair, or
    evicts: agents on free tiles and walls of every chunk, fields present for some chunks only; with a pool that must
    evict and with one that need not, the batch takes several rounds and still leaves the serial loop's pool"""
    cw = 2
    P = Pair(cw, cw, 0x5EED0740, frac_blocked=0.25)
    try:
        tgt = _free_tile(P.cost, cw, cw, 5)
        rec, fl = _agents(P.cost, cw, cw, 800, 8, [(tgt, 0, 0)], on_blocked=0.5)
        for pool_max in (3, 64):
            _upload(P, rec, fl, 1, pool_max)
            P.each(lambda nav: nav.pool_clear())
            src = rec["pos"][np.nonzero(synth.blocked_to_image(P.cost, cw, cw)[(rec["pos"][:, 1] // 4).astype(int),
                                                                                (-rec["pos"][:, 0] // 4).astype(int)] != 255)[0][0]]
            for nav in P.navs:
                nav.pool_request_path(0, (float(src[0]), float(src[1])), (float(fl["target"][0][0]), float(fl["target"][0][1])))
            rounds = _drive(P, 1, steps=3)
            assert max(rounds) >= 2, rounds
    finally:
        P.close()


def test_enemy_seek_and_surround_fields():
    """TARGET_ENEMIES / TARGET_ENTITY destinations, consumers on blocked and cut-off tiles (kind-2 repairs only)"""
    cw = 4
    P = Pair(cw, cw, 0x5EED0750)
    try:
        ndests = 6
        img = synth.blocked_to_image(P.cost, cw, cw)
        free, wall = np.argwhere(img != 255), np.argwhere(img == 255)
        rng = np.random.default_rng(12)
        fp = capi.Nav.footprints(np.stack([-(free[rng.integers(0, len(free), 40), 1] + 0.5) * 4.0,
                                           (free[rng.integers(0, len(free), 40), 0] + 0.5) * 4.0], 1).astype(np.float32), 2.0)
        allch = np.array([divmod(c, cw) for c in range(cw * cw)], np.int32)
        reqs, chunks = [], []
        for d in range(ndests):
            r = np.zeros(1, capi.ENTITY_FIELD_REQ)
            r["dest"], r["layer"], r["ref_layer"] = d, 0, 0
            r["target_kind"] = capi.TARGET_ENEMIES if d % 2 else capi.TARGET_ENTITY
            r["ent_off"], r["ent_n"], r["chunk_off"], r["chunk_n"] = 5 * d, 5 if d % 2 else 1, len(chunks), len(allch)
            reqs.append(r); chunks.extend(allch.tolist())
        reqs = np.concatenate(reqs)
        n = 2000
        t = np.concatenate([wall[rng.integers(0, len(wall), n // 2)], free[rng.integers(0, len(free), n - n // 2)]])
        pos = np.stack([-(t[:, 1] + 0.5) * 4.0, (t[:, 0] + 0.5) * 4.0], 1).astype(np.float32)
        rec = np.zeros(n, capi.AGENT)
        rec["pos"] = pos; rec["prev_pos"] = pos; rec["radius"] = 1.0; rec["max_speed"] = 20.0; rec["speed"] = 20.0
        rec["flags"] = capi.FLAG_MOVABLE; rec["aux_dest1"] = rng.integers(1, ndests + 1, n)
        rec["state"][: n // 2] = ST_SEEK; rec["flock"][: n // 2] = -1
        rec["state"][n // 2:] = ST_SURROUND; rec["flock"][n // 2:] = 0
        fl = np.zeros(1, capi.FLOCK); fl["target"] = pos[0]; fl["dest"] = -1
        ext = np.zeros(n, capi.MOVESTATE_EXT)
        ext["surround_target_uid"] = capi.NULL_UID
        ext["surround_target_uid"][n // 2:] = 0; ext["using_surround_field"][n // 2:] = 1
        for nav in P.navs:
            nav.pool_create(ndests, ndests * cw * cw)
            nav.pool_request_entity_fields_batch(reqs, fp, np.array(chunks, np.int32))
            nav.agents_upload(rec, fl, 20)
            nav.agents_upload_movestate_ext(ext)
            nav.agents_set_work(np.arange(n, dtype=np.uint32))
        r = P.repair(ndests)
        assert r[1] > 0 and r[2] == 1
        P.repair(ndests)
    finally:
        P.close()


def test_empty_work_clear_and_errors():
    """an empty work list, pool_clear straight before the batch on a caller's stream, a NOMEM stop at the same
    representative as the serial loop's, and the argument errors"""
    cw = 2
    P = Pair(cw, cw, 0x5EED0760)
    try:
        tgt = _free_tile(P.cost, cw, cw, 1)
        rec, fl = _agents(P.cost, cw, cw, 600, 9, [(tgt, 0, 0), (tgt, 1, 0)], on_blocked=0.4)
        _upload(P, rec, fl, 2, 8)
        for nav in P.navs:
            nav.agents_set_work(np.zeros(0, np.uint32))
        assert P.navs[1].pool_repair_batch() == (0, 0, 0)
        for nav in P.navs:
            nav.agents_set_work(np.arange(len(rec), dtype=np.uint32))
        P.repair(2)
        # pfnav_pool_clear straight before the calls (no tick in between), the batch on a stream of the caller's: it
        # must order itself after the clear on that stream
        import torch
        P.each(lambda nav: nav.agents_tick(capi.TICK_VDES_FROM_POOL))
        P.each(lambda nav: nav.pool_clear())
        stream = torch.cuda.Stream()
        s = P.navs[0].pool_repair()
        b = P.navs[1].pool_repair_batch(stream.cuda_stream)
        assert s == b[:2] and s[0] > 0, (s, b)
        P.assert_same(2)
    finally:
        P.close()
    # NOMEM: every path from chunk (1, 1) to the target in chunk (0, 0) needs three chunks, the pool holds one slot
    P = Pair(2, 2, 0, cost=_walled_2x2(), rivers=False)
    try:
        rec, fl = _agents(P.cost, 2, 2, 3, 1, [((10, 10), 0, 0)], on_blocked=0.0)
        _place(rec, [(20, 20), (80, 80), (80, 110)], (20, 20))
        _upload(P, rec, fl, 1, 1)
        for nav in P.navs:
            nav.pool_request_path(0, _wp(20, 20), _wp(10, 10))
        P.each(lambda nav: nav.agents_tick(capi.TICK_VDES_FROM_POOL))
        a, b, r = C.c_int(0), C.c_int(0), C.c_int(0)
        rs = P.navs[0].L.pfnav_pool_repair(P.navs[0].h, C.byref(a), C.byref(b))
        rb = P.navs[1].L.pfnav_pool_repair_batch(P.navs[1].h, None, C.byref(a), C.byref(b), C.byref(r))
        assert rs == rb == capi.ERR_NOMEM, (rs, rb)
        for (fa, la, ia), (fb, lb, ib) in P.pool(1):
            assert ia == ib and (fa is None) == (fb is None) and (la is None) == (lb is None)
            assert fa is None or (fa == fb).all()
            assert la is None or (la == lb).all()
        # no pool / no agents / host-only
        nav = capi.Nav(0)
        try:
            assert nav.L.pfnav_pool_repair_batch(nav.h, None, None, None, None) == capi.ERR_ARG
        finally:
            nav.close()
        ho = capi.Nav(hostonly=True)
        try:
            assert ho.L.pfnav_pool_repair_batch(ho.h, None, None, None, None) == capi.ERR_NO_DEVICE
        finally:
            ho.close()
    finally:
        P.close()


def test_rule_i_own_slot_written_in_the_round():
    """rule (i): two entities in the two parts of chunk (1, 1), neither with a field. The first one's request builds the
    chunk's field toward the left portal; the second one's request merges the right portal into that same slot, so it
    needs the byte the first request wrote and the round ends before it"""
    P = Pair(2, 2, 0, cost=_walled_2x2(), rivers=False)
    try:
        tgt = (10, 10)
        rec, fl = _agents(P.cost, 2, 2, 2, 1, [(tgt, 0, 0)], on_blocked=0.0)
        _place(rec, [(80, 80), (80, 110)], (20, 20))
        _upload(P, rec, fl, 1, 16)
        for nav in P.navs:
            nav.pool_request_path(0, _wp(20, 20), _wp(*tgt))
        r = P.repair(1)
        assert r[0] == 2 and r[2] >= 2, r
        assert P.stats[1][0] >= 1, P.stats
    finally:
        P.close()


def test_rule_ii_emission_writes_a_slot_with_a_pending_repair():
    """rule (ii): an entity under a blocker in the upper part of chunk (0, 1) needs only a repair of that chunk's field
    (its request emits nothing); the next entity, in chunk (1, 1), reaches the target through the lower part of chunk
    (0, 1), so its request merges a second portal into the slot with the pending repair: the round ends before it"""
    P = Pair(2, 2, 0, cost=_walled_2x2(), rivers=False)
    try:
        tgt = (10, 10)
        rec, fl = _agents(P.cost, 2, 2, 2, 1, [(tgt, 0, 0)], on_blocked=0.0)
        _place(rec, [(10, 100), (80, 80)], (20, 20))
        _upload(P, rec, fl, 1, 16)
        for nav in P.navs:
            nav.blockers_incref(*_wp(10, 100), 2.0, 0)
            nav.map_commit()
            nav.pool_request_path(0, _wp(5, 120), _wp(*tgt))
            nav.pool_request_path(0, _wp(20, 20), _wp(*tgt))
        r = P.repair(1)
        assert r[0] >= 1 and r[2] >= 2, r
        assert P.stats[1][1] >= 1, P.stats
    finally:
        P.close()


def test_rule_iii_reservation_that_evicts():
    """rule (iii): two destinations whose paths need one chunk each, a pool of one slot. The second destination's
    request must evict the slot the first one's request filled in the same round: the round ends before it"""
    P = Pair(2, 2, 0, cost=_walled_2x2(), rivers=False)
    try:
        rec, fl = _agents(P.cost, 2, 2, 2, 1, [((10, 10), 0, 0), ((100, 10), 1, 0)], on_blocked=0.0)
        rec["flock"] = [0, 1]
        _place(rec, [(20, 20), (110, 20)], (20, 20))
        rec["prev_pos"] = (8.0, -8.0)      # off the map: no LOS-state miss, both requests come from the velocity phase
        _upload(P, rec, fl, 2, 1)
        r = P.repair(2)
        assert r[2] >= 2, r
        assert P.stats[1][2] >= 1, P.stats
    finally:
        P.close()


def test_crowd_on_one_blob_is_one_round():
    """a crowd under one blocker, the fields of its chunk rebuilt around the blocker: no request, repairs only, one
    round, no boundary"""
    cw = 2
    P = Pair(cw, cw, 0x5EED0710, frac_blocked=0.0, rivers=False)
    try:
        tgt = (100, 70)
        centre = (90, 100)
        rng = np.random.default_rng(1)
        n = 300
        rec, fl = _agents(P.cost, cw, cw, n, 2, [(tgt, 0, 0)], on_blocked=0.0)
        rec["pos"] = (np.array(_wp(*centre), np.float32) + rng.uniform(-6.0, 6.0, (n, 2))).astype(np.float32)
        rec["prev_pos"] = np.array(_wp(*tgt), np.float32)
        _upload(P, rec, fl, 1, 16)
        for nav in P.navs:
            nav.blockers_incref(*_wp(*centre), 14.0, 0)
            nav.map_commit()
            nav.pool_request_path(0, _wp(120, 120), _wp(*tgt))
        r = P.repair(1)
        assert r[0] == 0 and r[1] >= 1 and r[2] == 1, r
        assert P.stats[1] == (0, 0, 0) and P.stats[0][1] > 1, P.stats
    finally:
        P.close()


def test_c5_churn():
    """the C5 map and population of bench.py: obstacles moved onto the herds, commit, REQUEST_MISSING_ONLY goals and a
    tick, then the chain; pools, counts and the next tick equal the serial loop's after every step"""
    import importlib
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    if root not in sys.path:
        sys.path.insert(0, root)
    bench = importlib.import_module("bench")
    bench.set_workload("C5")
    pf = importlib.import_module("permafrost-engine_b200")
    W = bench.build_workload(pf, 1, 0)
    C = bench.CHUNKS
    ngoals = W["g_hi"] - W["g_lo"]
    goals = np.array([[int(v) for v in W["agents"]["flock_target_tile"][f]] for f in range(W["g_lo"], W["g_hi"])], np.int32)
    dests = np.arange(ngoals, dtype=np.int32)
    P = Pair(C, C, 0, cost=W["cost"])
    try:
        churns = []
        for nav in P.navs:
            ch = bench.Churn(W["agents"], bench.WORKLOADS["C5"]["blockers"], C, bench.MAP_SEED + 77)
            ch.place(nav, capi)
            nav.map_commit()
            nav.pool_create(ngoals, ngoals * C * C)
            nav.agents_upload(W["rec"], W["flocks"], bench.HZ)
            nav.agents_set_work(np.arange(W["lo"], W["hi"], dtype=np.uint32))
            nav.pool_request_goals(dests, goals, 0)
            churns.append(ch)
        total, rules = 0, [0, 0, 0]
        for _ in range(2):
            for nav, ch in zip(P.navs, churns):
                ch.move(nav, capi)
                nav.map_commit()
                nav.pool_request_goals(dests, goals, 0, 0, capi.REQUEST_MISSING_ONLY)
            r = P.repair(ngoals)
            total += r[0] + r[1]
            rules = [a + b for a, b in zip(rules, P.stats[1])]
        assert total > 0 and rules[0] + rules[1] > 0, (total, rules)
    finally:
        P.close()
