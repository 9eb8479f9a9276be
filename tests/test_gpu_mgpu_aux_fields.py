"""Zone and entity-field batches of a multi-GPU job (pfnav_group_request_zones, pfnav_group_request_entity_fields_batch):
each (dest, chunk) field is built on one member and copied to every member. Every member is compared with a single
context that gets the same calls, with the solo batch in place of the job's:
- every (dest, chunk) entry: has bits, ff_id, flow bytes;
- the slot choices: a later solo batch that fills the pool evicts by each pool's own slot history, and must leave the
  member equal to its twin;
- entity batches: the footprints each destination remembers, through a pfnav_pool_repair_batch after the group is gone.
The test hook pfnav_mgpu_fields_stats shows every written key built on exactly one member.

Groups of 2 and 3 members on device 0, and on further devices where the box has them. The NCCL transport is checked by
tests/tools/mgpu_nccl_aux_fields_check.py under torchrun."""
import numpy as np
import pytest

import cases
from test_gpu_entity_field_batch import _agents_on, _footprints, _mixed, _req, _tick
from test_gpu_zone_batch import _map, _reach, _reqs, _xz

capi, synth = cases.capi, cases.synth


def _devices(world):
    import torch
    n = torch.cuda.device_count()
    return [i % n for i in range(world)]


def _nav(dev, cost, cw, ndests, max_fields):
    nv = capi.Nav(dev)
    nv.map_create(cw, cw, 1)
    nv.map_upload_layer(0, cost)
    nv.map_build_nav(0)
    nv.route_build(0)
    nv.pool_create(ndests, max_fields)
    return nv


def _pool(nav, ndests):
    """every (dest, chunk) entry: has bits, ffid, flow bytes"""
    out = []
    for d in range(ndests):
        for c in range(nav.cw * nav.ch):
            f, l, ffid = nav.pool_get(d, divmod(c, nav.cw))
            out.append((int(f is not None) | int(l is not None) << 1, ffid, b"" if f is None else f.tobytes()))
    return out


def _zone_keys(reqs, tiles, cw):
    """the (dest, chunk) keys of every zone request, in the order the serial calls write them (tiles[i] None: off the map)"""
    return [[] if t is None else [(int(q["dest"]), cr * cw + cc) for cr, cc in _reach(t, int(q["radius"]), cw, cw)]
            for q, t in zip(reqs, tiles)]


def _entity_keys(reqs, chunks, cw):
    ch = np.asarray(chunks, np.int32).reshape(-1, 2)
    return [[(int(q["dest"]), int(r) * cw + int(c)) for r, c in ch[int(q["chunk_off"]):int(q["chunk_off"]) + int(q["chunk_n"])]]
            for q in reqs]


class Twins:
    """`world` members of an in-process group, and for member r a single context `solo[r]` that gets every call member r
    gets, with the solo batch in place of the job's"""

    def __init__(self, cost, cw, ndests, max_fields, world, small=None):
        self.cw, self.ndests, self.world = cw, ndests, world
        cap = lambda r: small if small is not None and r == world - 1 else max_fields
        self.navs = [_nav(d, cost, cw, ndests, cap(r)) for r, d in enumerate(_devices(world))]
        self.solo = [_nav(0, cost, cw, ndests, cap(r)) for r in range(world)]
        self.grp = capi.Group(self.navs)

    def close(self):
        if self.grp is not None:
            self.grp.close()
        for X in self.navs + self.solo:
            X.close()

    def each(self, fn):
        for X in self.navs + self.solo:
            fn(X)

    def solo_on(self, r, fn):
        """the same solo call on member r and its twin (how members come to hold different fields)"""
        a, b = fn(self.navs[r]), fn(self.solo[r])
        assert np.array_equal(np.asarray(a), np.asarray(b))

    def check_owners(self, m, keys):
        """every key written is built on exactly one member, the owner of the request that writes it last"""
        last = {}
        for i, ks in enumerate(keys):
            for k in ks:
                last[k] = i
        writes = set(last.values())
        stats = [nv.mgpu_fields_stats(m) for nv in self.navs]
        owner = stats[0][2]
        for s in stats:
            assert np.array_equal(s[2], owner), "members disagree on the owners"
            assert s[1] == 0
        for i in range(m):
            assert (owner[i] >= 0) == (i in writes), (i, owner[i])
        for r, (built, _, _) in enumerate(stats):
            assert built == sum(1 for i in last.values() if owner[i] == r), r
        assert sum(s[0] for s in stats) == len(last)
        return owner

    def zones(self, reqs, tiles):
        nf = self.grp.request_zones(reqs)
        for S in self.solo:
            nd, snf = S.pool_request_zones(reqs)
            assert nd == len(reqs) and np.array_equal(snf, nf), "solo counts differ"
        self.compare()
        return self.check_owners(len(reqs), _zone_keys(reqs, tiles, self.cw))

    def entity(self, reqs, fp, chunks):
        self.grp.request_entity_fields_batch(reqs, fp, chunks)
        for S in self.solo:
            assert S.pool_request_entity_fields_batch(reqs, fp, chunks) == len(reqs)
        self.compare()
        return self.check_owners(len(reqs), _entity_keys(reqs, chunks, self.cw))

    def compare(self):
        for r, (nv, S) in enumerate(zip(self.navs, self.solo)):
            a, b = _pool(nv, self.ndests), _pool(S, self.ndests)
            bad = [i for i in range(len(a)) if a[i] != b[i]]
            assert not bad, "member %d: %d entries differ, first (dest, chunk) %s" % (r, len(bad), divmod(bad[0], nv.cw * nv.ch))

    def fill(self, fp, rng):
        """slot choices: solo entity batches naming every (dest, chunk) evict by each pool's own history"""
        nch = self.cw * self.cw
        chunks = np.array([divmod(c, self.cw) for c in range(nch)], np.int32)
        for d in rng.permutation(self.ndests)[:3]:
            req = _req(int(d), capi.TARGET_ENEMIES, (0, len(fp)), (0, nch))
            for r in range(self.world):
                self.solo_on(r, lambda X: X.pool_request_entity_fields_batch(req, fp, chunks))
        self.compare()

    def repair_after_close(self, seed, ndests):
        """the group is gone: agents naming entity destinations 1 .. ndests on every context, a tick,
        pfnav_pool_repair_batch from the remembered footprints"""
        self.grp.close()
        self.grp = None
        rec, fl, ext = _agents_on(self.navs[0], self.cw, self.cw, ndests, 1500, seed)
        for nv, S in zip(self.navs, self.solo):
            out = []
            for X in (nv, S):
                _tick(X, rec, fl, ext)
                out.append(X.pool_repair_batch())
            assert out[0] == out[1]
        self.compare()


def _zone_case(cw, seed, n, radii, rng):
    cost, _ = _map(cw, cw, seed)
    img = synth.blocked_to_image(cost, cw, cw)
    free = np.argwhere(img != 0xFF)
    tiles = [tuple(int(v) for v in free[rng.integers(len(free))]) for _ in range(n)]
    return cost, tiles, [int(rng.choice(radii)) for _ in range(n)]


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_zones_host_flood(pf, world):
    """a few large zones (the owners flood on the host), a zone centred off the map, a repeated dest"""
    rng = np.random.default_rng(1)
    cost, tiles, radii = _zone_case(4, 0x5EED0A01, 4, [40, 60, 90], rng)
    T = Twins(cost, 4, 6, 6 * 16, world)
    try:
        dests = [0, 1, 1, 3, 2]                                 # dest 1 twice; request 3 centred off the map
        tiles = tiles[:3] + [None] + tiles[3:]
        xz = [(1000.0, -1000.0) if t is None else _xz(t) for t in tiles]
        reqs = _reqs([(d, p, r) for d, p, r in zip(dests, xz, radii[:3] + [30] + radii[3:])])
        owner = T.zones(reqs, tiles)
        assert owner[3] == -1
        T.zones(reqs, tiles)                                    # again: every key rebuilt, no new slot
        T.fill(_footprints(4, 4, 40, 3), rng)
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_zones_device_flood(pf, world):
    """80 zones of small radii (the owners flood on the device), spread over every member"""
    rng = np.random.default_rng(2)
    cost, tiles, radii = _zone_case(4, 0x5EED0A02, 80, [3, 6, 10, 16], rng)
    T = Twins(cost, 4, 90, 90 * 16, world)
    try:
        reqs = _reqs([(i, _xz(t), r) for i, (t, r) in enumerate(zip(tiles, radii))])
        owner = T.zones(reqs, tiles)
        assert len(set(owner.tolist())) == world, owner
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_entity_fields(pf, world):
    """TARGET_ENEMIES with shared footprint ranges, TARGET_ENTITY with a building, a repeated (dest, chunk) where the last
    request wins; then the slot choices and the repairs from the remembered footprints"""
    cw = 4
    cost, _ = _map(cw, cw, 0x5EED0A03)
    T = Twins(cost, cw, 41, 41 * 16, world)
    try:
        fp, reqs, chunks = _mixed(cw, cw, 200, 120, 40, 7)
        bld = int(np.nonzero(fp["is_building"])[0][0])
        extra = [_req(3, capi.TARGET_ENTITY, (bld, 1), (len(chunks), 4)),
                 _req(3, capi.TARGET_ENEMIES, (0, 50), (len(chunks) + 2, 2))]      # overwrites two keys of the previous one
        chunks = np.concatenate([chunks, np.array([(0, 0), (1, 1), (1, 1), (2, 2)], np.int32)])
        reqs = np.concatenate([reqs] + extra)
        T.entity(reqs, fp, chunks)
        T.fill(fp, np.random.default_rng(4))
        T.repair_after_close(9, 40)
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_fewer_requests_than_members(pf, world):
    rng = np.random.default_rng(3)
    cost, tiles, radii = _zone_case(3, 0x5EED0A04, 1, [12], rng)
    T = Twins(cost, 3, 2, 2 * 9, world)
    try:
        owner = T.zones(_reqs([(1, _xz(tiles[0]), radii[0])]), tiles)
        assert owner.tolist() == [0]
        fp = _footprints(3, 3, 30, 5)
        owner = T.entity(_req(0, capi.TARGET_ENEMIES, (0, 30), (0, 2)), fp, [(0, 0), (2, 1)])
        assert owner.tolist() == [0]
    finally:
        T.close()


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_diverged_pools(pf, world):
    """members whose pools differ -- earlier solo batches, commits that drop fields, evictions in a small pool -- before
    the job's batches, which evict by each member's own LRU order"""
    cw, nd = 4, 24
    cost, _ = _map(cw, cw, 0x5EED0A05)
    T = Twins(cost, cw, nd, 60, world)
    try:
        rng = np.random.default_rng(6)
        fp, reqs, chunks = _mixed(cw, cw, 150, 60, nd - 4, 11)
        for r in range(world):                   # member r: a different slice of solo entity batches and zones
            t = [tuple(int(v) for v in rng.integers(0, 64 * cw, 2))]
            T.solo_on(r, lambda X: X.pool_request_zones(_reqs([(nd - 1 - r, _xz(t[0]), 8)]))[1])
            part = reqs[r * 7:(r + 1) * 7 + 5 * r]
            T.solo_on(r, lambda X: X.pool_request_entity_fields_batch(part, fp, chunks))
        x, z = float(rng.uniform(-cw * 256 + 40, -40)), float(rng.uniform(40, cw * 256 - 40))
        T.each(lambda X: X.blockers_incref(x, z, 14.0))
        T.each(lambda X: X.map_commit())
        T.compare()
        T.entity(reqs[20:50], fp, chunks)
        T.entity(reqs[:30], fp, chunks)
        T.repair_after_close(13, nd - 4)
    finally:
        T.close()


def _call_zones(g, reqs, nf=None):
    reqs = np.ascontiguousarray(reqs, capi.ZONE_REQ)
    return capi.load().pfnav_group_request_zones(g, capi._p(reqs), len(reqs), None if nf is None else capi._p(nf))


def _call_entity(g, reqs, fp, chunks):
    reqs = np.ascontiguousarray(reqs, capi.ENTITY_FIELD_REQ)
    fp = np.ascontiguousarray(fp, capi.FOOTPRINT)
    ch = np.ascontiguousarray(chunks, np.int32).reshape(-1, 2)
    return capi.load().pfnav_group_request_entity_fields_batch(g, capi._p(reqs), len(reqs), capi._p(fp), len(fp),
                                                               capi._p(ch), len(ch))


@pytest.mark.gpu
def test_errors(pf):
    """a bad argument, and a pool too small on one member: every member refuses and no pool changes (no partial
    batch); a context in no job and the NCCL form on a group member -> PFNAV_ERR_STATE"""
    L = capi.load()
    rng = np.random.default_rng(8)
    cost, tiles, radii = _zone_case(3, 0x5EED0A06, 4, [10, 20], rng)
    T = Twins(cost, 3, 4, 4 * 9, 2, small=8)
    try:
        fp = _footprints(3, 3, 30, 5)
        T.zones(_reqs([(0, _xz(tiles[0]), 4)]), tiles[:1])
        before = [_pool(nv, 4) for nv in T.navs]
        bad = _reqs([(1, _xz(tiles[1]), 10), (4, _xz(tiles[2]), 10)])
        assert _call_zones(T.grp.g, bad) == capi.ERR_ARG
        assert _call_entity(T.grp.g, _req(1, 7, (0, 30), (0, 1)), fp, [(0, 0)]) == capi.ERR_ARG
        # member 1 holds 8 fields: requests of 9 fields fit member 0 only
        allc = [divmod(c, 3) for c in range(9)]
        big = np.concatenate([_req(d, capi.TARGET_ENEMIES, (0, 30), (0, 9)) for d in (1, 2, 3)])
        assert _call_entity(T.grp.g, big, fp, allc) == capi.ERR_NOMEM
        many = _reqs([(d, _xz(t), 200) for d, t in zip((1, 2, 3), tiles[1:])])
        assert _call_zones(T.grp.g, many) == capi.ERR_NOMEM
        assert [_pool(nv, 4) for nv in T.navs] == before
        # a context outside any job; the NCCL form on a group member
        q = np.ascontiguousarray(bad[:1], capi.ZONE_REQ)
        e = np.ascontiguousarray(_req(1, capi.TARGET_ENEMIES, (0, 30), (0, 1)), capi.ENTITY_FIELD_REQ)
        f = np.ascontiguousarray(fp, capi.FOOTPRINT)
        c = np.zeros(2, np.int32)
        for h in (T.solo[0].h, T.navs[0].h):
            assert L.pfnav_mgpu_request_zones(h, capi._p(q), 1, None, None) == capi.ERR_STATE
            assert L.pfnav_mgpu_request_entity_fields_batch(h, capi._p(e), 1, capi._p(f), len(f), capi._p(c), 1, None) == capi.ERR_STATE
        T.compare()
    finally:
        T.close()


@pytest.mark.gpu
def test_unexchanged_blocker_ops(pf):
    """device blocker ops decided on one member and not yet exchanged: PFNAV_ERR_STATE, no pool changed; after the
    exchange and the commit the batches go through"""
    from test_gpu_mgpu_blockers import Job, _case
    cost, a, ms = _case(12, 20)
    J = Job(cost, a, ms, 20, 2)
    try:
        lo0 = J.ranges[0][0]
        J.navs[0].agents_set_blocking(np.arange(lo0, lo0 + 40, dtype=np.uint32), True)
        before = [_pool(nv, J.nflocks) for nv in J.navs]
        zr = _reqs([(0, (-300.0, 300.0), 10)])
        fp = capi.Nav.footprints(np.array([[-100.0, 100.0]], np.float32), 3.0)
        er = _req(1, capi.TARGET_ENEMIES, (0, 1), (0, 1))
        assert _call_zones(J.grp.g, zr) == capi.ERR_STATE
        assert _call_entity(J.grp.g, er, fp, [(0, 0)]) == capi.ERR_STATE
        assert [_pool(nv, J.nflocks) for nv in J.navs] == before
        J.grp.exchange_blocker_ops()
        for nv in J.navs:
            nv.map_commit()
        J.grp.request_zones(zr)
        J.grp.request_entity_fields_batch(er, fp, [(0, 0)])
    finally:
        J.close()


def test_errors_host_only(pf):
    """a host-only context has no device: PFNAV_ERR_NO_DEVICE"""
    L = capi.load()
    nav = capi.Nav(hostonly=True)
    try:
        q = np.zeros(1, capi.ZONE_REQ)
        e = np.zeros(1, capi.ENTITY_FIELD_REQ)
        assert L.pfnav_mgpu_request_zones(nav.h, capi._p(q), 1, None, None) == capi.ERR_NO_DEVICE
        assert L.pfnav_mgpu_request_entity_fields_batch(nav.h, capi._p(e), 1, None, 0, None, 0, None) == capi.ERR_NO_DEVICE
    finally:
        nav.close()
