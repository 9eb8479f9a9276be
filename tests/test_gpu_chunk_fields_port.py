"""GPU suite: the field pool's padded-chunk fields, and the two calls that read or build the same kind of field, against
the plain-C port (oracle/pf_oracle.c) on maps placed where the engine places them.

- (a) TARGET_ZONE fields, pfnav_pool_request_zones (N_RequestAsyncGroupArrivalField, nav.c:3921): world-space centres on
  open, blocked and impassable tiles, on tile and chunk borders and one float32 ulp either side, on the map's corners and
  edges and just outside it; radii 0 .. 90; one batch that floods on the host and one that floods on the device. The
  chunks that get a field == the selection of nav.c:3945-3951 restated here with the map origin, nfields == its size,
  every field == OracleMap.flow_field_zone.
- (b) TARGET_ENTITY / TARGET_ENEMIES fields, pfnav_pool_request_entity_fields_batch: circles across chunk borders and
  map edges on both sides of the device / host rasterisation bound, buildings, four factions at war, reference layers
  0 .. 3. Every field == OracleMap.chunk_field_seeded of the host seeds of a host-only twin. Two properties that do not
  go through pfnav_tile_geom.cuh or enemies_search_rect: at reference layer 0 the seeds are the window's tiles under the
  circles (float64 geometry from the map origin, 1e-3 wu slack), and a TARGET_ENEMIES field is seeded only by enemies
  inside its chunk's search rectangle (field.c:1229-1243), probed just inside and just outside its bounds.
- (c) N_DesiredGroupArrivalVelocity, pfnav_group_arrival_velocity, over the pools (a) built: velocities and flags ==
  OracleMap.group_arrival_velocity bit for bit, at tile centres around every zone, on borders +- 1 ulp, on the map box
  edges and one ulp outside, in chunks without fields, and with a centre off the map.
- (d) N_GroupArrivalFieldCreate with world-space arguments, pfnav_group_arrival_field: dims 64, 96, 128, with and
  without enemies, centres and targets near the map edges and off the map == OracleMap.group_arrival_field.

Maps: 3 x 3 chunks at the origin (the goldens' placement), 5 x 2 centred at the origin as M_CenterAtOrigin does
(map.c:420), 2 x 5 at an offset that is not tile-aligned, 1 x 1 (zone windows of 64), and bench.py's 16 x 16 C2 map
centred, with fewer cases. Blockers of four factions are committed through the device; some close off pockets of
open tiles. Every output is an integer, a direction byte or a float copied from a table: every comparison is exact."""
import numpy as np
import pytest

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
C2_SEED = 0x5EED0001            # bench.py's C2 map
# (chunk_w, chunk_h, (map_x, map_z), seed)
MAPS = {
    "3x3_origin": (3, 3, (0.0, 0.0), 0x5EED0C00),
    "5x2_centred": (5, 2, (5 * 256 / 2.0, -(2 * 256 / 2.0)), 0x5EED0C01),
    "2x5_offset": (2, 5, (601.3, -250.9), 0x5EED0C02),
    "1x1": (1, 1, (0.0, 0.0), 0x5EED0C03),
    "c2_centred": (16, 16, (16 * 256 / 2.0, -(16 * 256 / 2.0)), C2_SEED),
}
RADII = [0, 1, 2, 5, 13, 40, 73, 90]
# circle radii on both sides of the device / host bound: 40 wu with no ring, 28 wu with three (footprint_on_device)
FP_RADII = np.array([0.0, 4.0, 16.0, 27.9, 28.0, 28.5, 36.0, 40.0, 40.5, 60.0], np.float32)
WARS = [(0, 1), (0, 2), (3, 1)]
COMBATABLE = 1 << 4
SLACK = 1e-3
F = np.float32


class Map:
    """one placed map: cost, the committed blockers and faction counts, the port's map and a host-only twin"""

    def __init__(self, name, pforacle):
        cw, ch, (mx, mz), seed = MAPS[name]
        self.name, self.cw, self.ch, self.seed = name, cw, ch, seed
        self.mx, self.mz = F(mx), F(mz)                     # the library keeps the origin in float32
        self.W, self.H = F(cw * 256), F(ch * 256)
        self.dim = 128 if cw > 1 and ch > 1 else 64
        self.cost = synth.cost_from_pathable(synth.make_map(cw, ch, seed, rivers=cw > 1 and ch > 1), cw, ch)
        self.blockers = _blockers(self, np.random.default_rng(seed))
        self.twin = self._ctx(hostonly=True)
        self.blk, self.fac = self.twin.blockers(0), self.twin.faction_counts(0)
        self.om = pforacle.OracleMap(cw, ch, self.cost, self.blk, None, map_x=float(mx), map_z=float(mz), factions=self.fac)
        img_c = synth.blocked_to_image(self.cost, cw, ch)
        img_b = self.blk.reshape(ch, cw, 64, 64).transpose(0, 2, 1, 3).reshape(ch * 64, cw * 64)
        self.passable = (img_c != 0xFF) & (img_b == 0)
        self.impassable, self.blocked = img_c == 0xFF, (img_c != 0xFF) & (img_b > 0)

    def _ctx(self, hostonly=False):
        nav = capi.Nav(hostonly=True) if hostonly else capi.Nav(0)
        nav.map_create(self.cw, self.ch, 1, float(self.mx), float(self.mz))
        nav.map_upload_layer(0, self.cost)
        nav.map_build_nav(0)
        for x, z, r, f in self.blockers:
            nav.blockers_incref(x, z, r, f)
        nav.map_commit()
        return nav

    def device(self):
        """a device context with the same map; its committed blockers are the twin's"""
        nav = self._ctx()
        assert (nav.blockers(0) == self.blk).all() and (nav.faction_counts(0) == self.fac).all()
        return nav

    def close(self):
        self.twin.close()

    def tile_xz(self, r, c):
        """world centre of absolute tile (r, c)"""
        return F(float(self.mx) - (c + 0.5) * 4.0), F(float(self.mz) + (r + 0.5) * 4.0)

    def col_x(self, k):
        """world x of the border left of column k, and one ulp either side"""
        x = self.mx - F(4 * k)
        return [x, np.nextafter(x, F(np.inf)), np.nextafter(x, F(-np.inf))]

    def row_z(self, k):
        z = self.mz + F(4 * k)
        return [z, np.nextafter(z, F(np.inf)), np.nextafter(z, F(-np.inf))]

    def tile_rect(self, r, c):
        """tile rectangles in float64 from the map origin -> (x_lo, x_hi, z_lo, z_hi) arrays"""
        x_hi = float(self.mx) - 4.0 * np.asarray(c, np.float64)
        z_lo = float(self.mz) + 4.0 * np.asarray(r, np.float64)
        return x_hi - 4.0, x_hi, z_lo, z_lo + 4.0


def _blockers(m, rng):
    """(x, z, radius, faction): scattered discs, and rings of discs that close off pockets of open tiles"""
    nch = m.cw * m.ch
    out = []
    for _ in range(min(12 * nch, 300)):
        x = float(m.mx) - rng.uniform(0.02, 0.98) * float(m.W)
        z = float(m.mz) + rng.uniform(0.02, 0.98) * float(m.H)
        out.append((x, z, float(rng.uniform(2, 12)), int(rng.integers(0, 4))))
    for _ in range(min(nch, 24)):
        cx = float(m.mx) - rng.uniform(0.1, 0.9) * float(m.W)
        cz = float(m.mz) + rng.uniform(0.1, 0.9) * float(m.H)
        f = int(rng.integers(0, 4))
        for a in np.linspace(0, 2 * np.pi, 16, endpoint=False):
            out.append((cx + 24 * np.cos(a), cz + 24 * np.sin(a), 6.0, f))
    return [(float(x), float(z), float(r), f) for x, z, r, f in out]


def desc_for_point(m, px, pz):
    """M_Tile_DescForPoint2D (tile.c:547) in float32, as the port's desc_for_point (pf_oracle.c:348) -> absolute
    (r, c), or None off the map"""
    px, pz = F(px), F(pz)
    if px > m.mx or px < m.mx - m.W or pz < m.mz or pz > m.mz + m.H:
        return None
    cr = min(max(int(abs(m.mz - pz) / F(256)), 0), m.ch - 1)
    cc = min(max(int(abs(m.mx - px) / F(256)), 0), m.cw - 1)
    bx, bz = m.mx - F(cc * 256), m.mz + F(cr * 256)
    tr, tc = int(abs(bz - pz) / F(4)), int(abs(bx - px) / F(4))
    return cr * 64 + min(max(tr, 0), 63), cc * 64 + min(max(tc, 0), 63)


def zone_chunks(m, tile, radius):
    """the chunks N_RequestAsyncGroupArrivalField requests (nav.c:3945-3951): rows and columns of the centre tile +- 2
    radius, divided by the chunk size with C's truncation toward zero, clamped to the map"""
    if tile is None:
        return set()
    def span(t, n):
        lo, hi = t - 2 * radius, t + 2 * radius
        cl = lambda v: min(max(int(v / 64), 0), n - 1)
        return range(cl(lo), cl(hi) + 1)
    return {(cr, cc) for cr in span(tile[0], m.ch) for cc in span(tile[1], m.cw)}


def window_base(m, chunk):
    """the first tile of chunk's padded window (field.c:1566-1571)"""
    if m.dim == 64:
        return chunk[0] * 64, chunk[1] * 64
    return tuple(v * 64 - 32 if v > 0 else 0 for v in chunk)


def _pool_fields(nav, m, dest):
    """-> (fields u8[chunks][64][64], has u8[chunks]) of one pool destination"""
    nch = m.cw * m.ch
    fields, has = np.zeros((nch, 64, 64), np.uint8), np.zeros(nch, np.uint8)
    for c in range(nch):
        f, _, _ = nav.pool_get(dest, divmod(c, m.cw))
        if f is not None:
            fields[c], has[c] = f, 1
    return fields, has


# ---------------------------------------------------------------------------------------------------------------------
# (a) zone fields, (c) group-arrival velocities
# ---------------------------------------------------------------------------------------------------------------------
def _zone_centres(m, rng):
    """world-space centres -> list of float32 (x, z)"""
    H, W = m.ch * 64, m.cw * 64
    small = m.cw * m.ch <= 16
    out = []
    for mask, n in ((m.passable, 14 if small else 8), (m.blocked, 3), (m.impassable, 3)):
        t = np.argwhere(mask)
        out += [m.tile_xz(*t[i]) for i in rng.integers(0, len(t), n)] if len(t) else []
    # tile and chunk borders, exactly and one ulp either side (the other coordinate a random tile centre)
    cols = [64 * int(rng.integers(1, m.cw)) for _ in range(2)] if m.cw > 1 else []
    rows = [64 * int(rng.integers(1, m.ch)) for _ in range(2)] if m.ch > 1 else []
    cols += [int(rng.integers(1, W))]; rows += [int(rng.integers(1, H))]
    for k in cols[:3 if small else 2]:
        z = m.tile_xz(int(rng.integers(0, H)), 0)[1]
        out += [(x, z) for x in m.col_x(k)]
    for k in rows[:3 if small else 2]:
        x = m.tile_xz(0, int(rng.integers(0, W)))[0]
        out += [(x, z) for z in m.row_z(k)]
    # the corners and edges of the map box, exactly
    xs, zs = [m.mx, m.mx - m.W], [m.mz, m.mz + m.H]
    out += [(x, z) for x in xs for z in zs]
    out += [(m.mx, m.mz + m.H / F(2)), (m.mx - m.W, m.mz + F(0.3) * m.H), (m.mx - m.W / F(3), m.mz),
            (m.mx - F(0.7) * m.W, m.mz + m.H)]
    # just outside: one ulp past each edge, and further off
    up, dn = F(np.inf), F(-np.inf)
    out += [(np.nextafter(m.mx, up), m.mz + m.H / F(2)), (np.nextafter(m.mx - m.W, dn), m.mz + m.H / F(2)),
            (m.mx - m.W / F(2), np.nextafter(m.mz, dn)), (m.mx - m.W / F(2), np.nextafter(m.mz + m.H, up)),
            (m.mx + F(10), m.mz + F(5)), (m.mx - m.W / F(2), m.mz - F(3))]
    return [(F(x), F(z)) for x, z in out]


def _zone_reqs(rows):
    """rows: (dest, (x, z), radius) -> ZONE_REQ records"""
    out = np.zeros(len(rows), capi.ZONE_REQ)
    for i, (d, xz, rad) in enumerate(rows):
        out[i]["dest"], out[i]["centre_x"], out[i]["centre_z"], out[i]["radius"] = d, xz[0], xz[1], rad
    return out


@pytest.fixture(scope="module", params=list(MAPS))
def placed(request, pforacle):
    m = Map(request.param, pforacle)
    yield m
    m.close()


@pytest.fixture(scope="module")
def zones(placed):
    """(a)'s pools: a batch of two large zones (flooded on the host), then a batch of every other centre (flooded on the
    device); each request its own destination. -> dict(nav, rows, launches, nfields)"""
    m = placed
    rng = np.random.default_rng(m.seed + 1)
    open_ = np.argwhere(m.passable)
    big = [(m.tile_xz(*open_[i]), r) for i, r in zip(rng.integers(0, len(open_), 2), (90, 73))]
    rest = [(xz, RADII[i % len(RADII)]) for i, xz in enumerate(_zone_centres(m, rng))]
    batches = [[(d, xz, r) for d, (xz, r) in enumerate(big)],
               [(len(big) + d, xz, r) for d, (xz, r) in enumerate(rest)]]
    rows = batches[0] + batches[1]
    need = sum(len(zone_chunks(m, desc_for_point(m, *xz), r)) for _, xz, r in rows)
    nav = m.device()
    nav.pool_create(len(rows), 2 * need + 64)           # room for a wrong selection to show in the comparisons
    launches, nfields = [], []
    for b in batches:
        l0 = nav.launch_count()
        nd, nf = nav.pool_request_zones(_zone_reqs(b))
        assert nd == len(b)
        launches.append(nav.launch_count() - l0)
        nfields += [int(v) for v in nf]
    yield dict(nav=nav, rows=rows, launches=launches, nfields=nfields)
    nav.close()


def test_zone_fields_vs_port(placed, zones):
    m, nav, rows = placed, zones["nav"], zones["rows"]
    # a batch whose floods add up to at most PF_ZONE_HOST_POP_RATIO x its largest floods on the host: the pool scatter and
    # the integration; a larger one adds k_zone_seed_bits
    assert zones["launches"] == [2, 3], zones["launches"]
    seen = dict(no_centre=0, cut=0, unreached=0, last_row=0, last_col=0, off_map=0)
    for (dest, xz, rad), nf in zip(rows, zones["nfields"]):
        tile = desc_for_point(m, *xz)
        want = zone_chunks(m, tile, rad)
        seen["off_map"] += tile is None
        assert nf == len(want), (m.name, xz, rad)
        budget = min(int(np.pi * rad * rad + 0.5), m.dim * m.dim)
        for c in range(m.cw * m.ch):
            chunk = divmod(c, m.cw)
            f, _, _ = nav.pool_get(dest, chunk)
            assert (f is not None) == (chunk in want), (m.name, xz, rad, chunk)
            if f is None:
                continue
            exp = m.om.flow_field_zone(chunk, tile, rad)
            assert (f == exp).all(), (m.name, xz, rad, chunk)
            b = window_base(m, chunk)
            seen["no_centre"] += not (0 <= tile[0] - b[0] < m.dim and 0 <= tile[1] - b[1] < m.dim)
            seeds = m.om.zone_seeds(chunk, tile, rad)
            seen["cut"] += 0 < budget == len(seeds)
            r0, c0 = chunk[0] * 64, chunk[1] * 64
            seed_mask = np.zeros((64, 64), bool)
            s = seeds[(seeds[:, 0] >= r0) & (seeds[:, 0] < r0 + 64) & (seeds[:, 1] >= c0) & (seeds[:, 1] < c0 + 64)]
            seed_mask[s[:, 0] - r0, s[:, 1] - c0] = True
            unreached = m.passable[r0:r0 + 64, c0:c0 + 64] & (exp == 0) & ~seed_mask
            seen["unreached"] += bool(unreached.any() and len(seeds))
            seen["last_row"] += chunk[0] == m.ch - 1 and bool(exp.any())
            seen["last_col"] += chunk[1] == m.cw - 1 and bool(exp.any())
    assert seen["off_map"] > 0 and seen["cut"] > 0 and seen["unreached"] > 0, seen
    assert seen["last_row"] > 0 and seen["last_col"] > 0, seen
    if m.dim > 64:                                  # a 1 x 1 map's one window is the whole map
        assert seen["no_centre"] > 0, seen


def _probe_positions(m, rng):
    """positions shared by every destination: borders +- 1 ulp, the map box edges exactly and one ulp outside, and
    random points everywhere (most in chunks without a field)"""
    H, W = m.ch * 64, m.cw * 64
    up, dn = F(np.inf), F(-np.inf)
    out = []
    cols = sorted({64 * k for k in range(1, m.cw)} | {int(v) for v in rng.integers(1, W, 3)})
    rows = sorted({64 * k for k in range(1, m.ch)} | {int(v) for v in rng.integers(1, H, 3)})
    for k in cols[:8]:
        for x in m.col_x(k):
            out += [(x, m.tile_xz(int(r), 0)[1]) for r in rng.integers(0, H, 3)]
    for k in rows[:8]:
        for z in m.row_z(k):
            out += [(m.tile_xz(0, int(c))[0], z) for c in rng.integers(0, W, 3)]
    zs = [m.mz, m.mz + m.H, np.nextafter(m.mz, dn), np.nextafter(m.mz + m.H, up)] + [m.tile_xz(int(r), 0)[1] for r in rng.integers(0, H, 3)]
    xs = [m.mx, m.mx - m.W, np.nextafter(m.mx, up), np.nextafter(m.mx - m.W, dn)] + [m.tile_xz(0, int(c))[0] for c in rng.integers(0, W, 3)]
    out += [(x, z) for x in xs for z in zs]
    out += list(zip(F(float(m.mx) - rng.uniform(0, float(m.W), 200)), F(float(m.mz) + rng.uniform(0, float(m.H), 200))))
    return np.array(out, np.float32)


def _band(m, tile, rad):
    """the tile centres of a band around the zone: every tile within min(radius + 3, 24) of the centre tile, and the
    tiles whose distance from it is within 1.5 of the radius"""
    H, W = m.ch * 64, m.cw * 64
    k = rad + 3
    r = np.arange(max(tile[0] - k, 0), min(tile[0] + k + 1, H))
    c = np.arange(max(tile[1] - k, 0), min(tile[1] + k + 1, W))
    rr, cc = np.meshgrid(r, c, indexing="ij")
    d = np.hypot(rr - tile[0], cc - tile[1])
    sel = (np.maximum(abs(rr - tile[0]), abs(cc - tile[1])) <= min(rad + 3, 24)) | (abs(d - rad) <= 1.5)
    rr, cc = rr[sel], cc[sel]
    return np.stack([float(m.mx) - (cc + 0.5) * 4.0, float(m.mz) + (rr + 0.5) * 4.0], 1).astype(np.float32)


def test_group_arrival_velocity_vs_port(placed, zones):
    m, nav, rows = placed, zones["nav"], zones["rows"]
    rng = np.random.default_rng(m.seed + 2)
    shared = _probe_positions(m, rng)
    off = (m.mx + F(10), m.mz + F(5))
    flags_seen = set()
    zero_dir = dict(inside=0, outside=0)
    picked = rows if m.cw * m.ch <= 16 else rows[:2] + rows[2::3]
    calls = []
    for dest, xz, rad in picked:
        tile = desc_for_point(m, *xz)
        pos = shared if tile is None else np.concatenate([_band(m, tile, rad), shared])
        calls.append((dest, xz, rad, pos))
    calls.append((rows[0][0], off, rows[0][2], shared))            # fields in the pool, centre off the map
    for dest, xz, rad, pos in calls:
        fields, has = _pool_fields(nav, m, dest)
        v, f = nav.group_arrival_velocity(dest, np.array(xz, np.float32), rad, pos)
        ev, ef = m.om.group_arrival_velocity(fields, has, np.array(xz, np.float32), rad, pos)
        bad = np.nonzero((f != ef) | (v.view(np.uint32) != ev.view(np.uint32)).any(axis=1))[0]
        assert not len(bad), (m.name, xz, rad, pos[bad[:5]], v[bad[:5]], ev[bad[:5]], f[bad[:5]], ef[bad[:5]])
        flags_seen |= set(int(x) for x in np.unique(ef))
        zero_dir["inside"] += int((ef == 3).sum())
        zero_dir["outside"] += int(((ef == 1) & (ev == 0).all(axis=1)).sum())
    # the last call: a destination with fields and a centre off the map returns nothing (nav.c:3561)
    assert desc_for_point(m, *off) is None and not f.any() and not v.any()
    assert {0, 1, 3} <= flags_seen, flags_seen
    assert zero_dir["inside"] > 0 and zero_dir["outside"] > 0, zero_dir


# ---------------------------------------------------------------------------------------------------------------------
# (b) TARGET_ENTITY / TARGET_ENEMIES fields
# ---------------------------------------------------------------------------------------------------------------------
def _building(cx, cz, hx, hz, ang):
    c, s = np.cos(ang), np.sin(ang)
    pts = [(-hx, -hz), (hx, -hz), (hx, hz), (-hx, hz)]
    return np.array([(cx + c * a - s * b, cz + s * a + c * b) for a, b in pts], np.float32).reshape(-1)


def search_rect(m, chunk):
    """field_chunk_bounds (field.c:863) widened by half a chunk plus 16 wu on every side (field.c:1229-1243), float64
    -> (x_lo, x_hi, z_lo, z_hi)"""
    cr, cc = chunk
    x_hi = float(m.mx) - 256.0 * cc
    z_lo = float(m.mz) + 256.0 * cr
    return x_hi - 256.0 - 144.0, x_hi + 144.0, z_lo - 144.0, z_lo + 256.0 + 144.0


def _footprints(m, rng):
    """-> (FOOTPRINT records, faction, flags, probes): circles across chunk borders and map edges, interior circles,
    buildings with every corner on the map, and (maps with more than one chunk) circles 0.05 wu inside and outside the
    interior bounds of the TARGET_ENEMIES search rectangles"""
    mx, mz, W, H = float(m.mx), float(m.mz), float(m.W), float(m.H)
    n = 40 if m.cw * m.ch <= 16 else 60
    rad = FP_RADII[rng.integers(0, len(FP_RADII), n)]
    x = mx - rng.uniform(0.05, 0.95, n) * W
    z = mz + rng.uniform(0.05, 0.95, n) * H
    k = n // 5
    if m.cw > 1:
        x[:k] = mx - 256.0 * rng.integers(1, m.cw, k) + rng.uniform(-1, 1, k) * rad[:k]         # across a column border
    if m.ch > 1:
        z[k:2 * k] = mz + 256.0 * rng.integers(1, m.ch, k) + rng.uniform(-1, 1, k) * rad[k:2 * k]
    e = rng.integers(0, 4, k)                                                                    # across a map edge
    d = rng.uniform(0, 1, k) * rad[2 * k:3 * k]
    x[2 * k:3 * k] = np.where(e == 0, mx - d, np.where(e == 1, mx - W + d, x[2 * k:3 * k]))
    z[2 * k:3 * k] = np.where(e == 2, mz + d, np.where(e == 3, mz + H - d, z[2 * k:3 * k]))
    probes = []
    for cr in range(m.ch):
        for cc in range(m.cw):
            xl, xh, zl, zh = search_rect(m, (cr, cc))
            zc, xc = mz + 256.0 * cr + 128.0, mx - 256.0 * cc - 128.0
            for bx, ok in ((xh, cc > 0), (xl, cc < m.cw - 1)):
                if ok:
                    probes += [(bx - 0.05, zc + rng.uniform(-100, 100)), (bx + 0.05, zc + rng.uniform(-100, 100))]
            for bz, ok in ((zl, cr > 0), (zh, cr < m.ch - 1)):
                if ok:
                    probes += [(xc + rng.uniform(-100, 100), bz - 0.05), (xc + rng.uniform(-100, 100), bz + 0.05)]
    if len(probes) > 24:
        probes = [probes[i] for i in rng.choice(len(probes), 24, replace=False)]
    pr = np.array(probes, np.float64).reshape(-1, 2)
    xy = np.concatenate([np.stack([x, z], 1), pr])
    radii = np.concatenate([rad, rng.uniform(30.0, 40.0, len(pr)).astype(np.float32)])
    fp = capi.Nav.footprints(xy.astype(np.float32), radii)
    nb = 4
    for i in range(n - nb, n):
        hx, hz = rng.uniform(2, 10, 2)
        cx, cz = mx - rng.uniform(24, W - 24), mz + rng.uniform(24, H - 24)
        fp["is_building"][i] = 1
        fp["corners_xz"][i] = _building(cx, cz, hx, hz, rng.uniform(0, np.pi))
        fp["x"][i], fp["z"][i] = cx, cz
    faction = rng.integers(0, 4, len(fp)).astype(np.int32)
    flags = np.full(len(fp), capi.FLAG_MOVABLE | COMBATABLE, np.uint32)
    flags[rng.random(len(fp)) < 0.15] &= ~np.uint32(COMBATABLE)
    probe = np.zeros(len(fp), bool)
    probe[n:] = True
    return fp, faction, flags, probe


def _ent_req(dest, kind, ent, chunk, ref_layer):
    r = np.zeros(1, capi.ENTITY_FIELD_REQ)
    r["dest"], r["layer"], r["ref_layer"], r["target_kind"] = dest, 0, ref_layer, kind
    r["ent_off"], r["ent_n"], r["chunk_off"], r["chunk_n"] = ent[0], ent[1], chunk[0], chunk[1]
    return r


def _near_dist(m, fp, r, c):
    """float64 distance from each circle centre to the nearest point of each tile -> [circles][tiles]"""
    xl, xh, zl, zh = m.tile_rect(r, c)
    px = np.asarray(fp["x"], np.float64)[:, None]
    pz = np.asarray(fp["z"], np.float64)[:, None]
    dx = np.maximum(np.maximum(xl[None] - px, px - xh[None]), 0.0)
    dz = np.maximum(np.maximum(zl[None] - pz, pz - zh[None]), 0.0)
    return np.hypot(dx, dz)


def _check_circles(m, chunk, seeds, allowed, must):
    """seeds of one field at reference layer 0 against the circles themselves: every seed within radius + SLACK of an
    allowed circle; every in-map window tile within radius - SLACK of a `must` circle is a seed. -> number of window
    tiles some allowed circle covers"""
    b = window_base(m, chunk)
    H, W = m.ch * 64, m.cw * 64
    r = np.arange(b[0], min(b[0] + m.dim, H)); c = np.arange(b[1], min(b[1] + m.dim, W))
    rr, cc = [a.ravel() for a in np.meshgrid(r, c, indexing="ij")]
    is_seed = np.zeros((H, W), bool)
    if len(seeds):
        is_seed[seeds[:, 0], seeds[:, 1]] = True
    is_seed = is_seed[rr, cc]
    near = np.zeros(len(rr), bool)
    if len(allowed):
        d = _near_dist(m, allowed, rr, cc)
        near = (d <= np.asarray(allowed["sel_radius"], np.float64)[:, None] + SLACK).any(axis=0)
    assert not (is_seed & ~near).any(), (m.name, chunk, np.stack([rr, cc], 1)[is_seed & ~near][:5])
    if len(must):
        d = _near_dist(m, must, rr, cc)
        inside = (d <= np.asarray(must["sel_radius"], np.float64)[:, None] - SLACK).any(axis=0)
        assert not (inside & ~is_seed).any(), (m.name, chunk, np.stack([rr, cc], 1)[inside & ~is_seed][:5])
    return int(near.sum())


def _in_rect(m, fp, chunk, margin):
    xl, xh, zl, zh = search_rect(m, chunk)
    x, z = np.asarray(fp["x"], np.float64), np.asarray(fp["z"], np.float64)
    return (x >= xl + margin) & (x <= xh - margin) & (z >= zl + margin) & (z <= zh - margin)


def _on_map(m, fp):
    return np.array([desc_for_point(m, x, z) is not None for x, z in zip(fp["x"], fp["z"])], bool)


def test_entity_fields_vs_port(placed):
    m = placed
    rng = np.random.default_rng(m.seed + 3)
    fp, faction, flags, probe = _footprints(m, rng)
    nch = m.cw * m.ch
    allc = [divmod(c, m.cw) for c in range(nch)]
    if nch > 16:                # the last row and column, the corners, and random chunks
        pick = {(m.ch - 1, c) for c in range(0, m.cw, 3)} | {(r, m.cw - 1) for r in range(0, m.ch, 3)} | {(0, 0)}
        pick |= {allc[i] for i in rng.choice(nch, 12, replace=False)}
        allc = sorted(pick)
    # footprint arrays: all, the enemies of each faction (cases.enemies_of, as the engine picks them), the probe circles
    circ = (fp["is_building"] == 0) & (fp["sel_radius"] <= 40.0)
    lists = [fp] + [fp[cases.enemies_of(f, WARS, faction, flags)] for f in range(4)]
    lists.append(fp[circ & (probe | (rng.random(len(fp)) < 0.5))])
    off = np.cumsum([0] + [len(a) for a in lists])
    fps = np.concatenate(lists)
    ents = [int(i) for i in np.nonzero(fp["is_building"])[0][:2]] + [int(i) for i in np.argsort(-fp["sel_radius"])[:2]]
    ents += [int(i) for i in rng.choice(len(fp) - int(probe.sum()), 6, replace=False)]
    chunks, reqs, meta = [], [], []
    for L in range(4):
        for k in range(1, len(lists)):
            reqs.append(_ent_req(len(meta), capi.TARGET_ENEMIES, (off[k], off[k + 1] - off[k]), (len(chunks), len(allc)), L))
            chunks += allc
            meta.append((capi.TARGET_ENEMIES, L, off[k], off[k + 1], allc))
        for e in ents:
            t = desc_for_point(m, fp["x"][e], fp["z"][e])
            near = allc if t is None else [c for c in allc if abs(c[0] - t[0] // 64) <= 1 and abs(c[1] - t[1] // 64) <= 1]
            reqs.append(_ent_req(len(meta), capi.TARGET_ENTITY, (e, 1), (len(chunks), len(near)), L))
            chunks += near
            meta.append((capi.TARGET_ENTITY, L, e, e + 1, near))
    nav = m.device()
    try:
        nav.pool_create(len(meta), len(chunks))
        assert nav.pool_request_entity_fields_batch(np.concatenate(reqs), fps, np.array(chunks, np.int32)) == len(meta)
        seen = dict(last_row=0, last_col=0, excluded=0, probe_in=0, probe_out=0, host_raster=0)
        for dest, (kind, L, a, b, chs) in enumerate(meta):
            sub = fps[a:b]
            for chunk in chs:
                f, _, _ = nav.pool_get(dest, chunk)
                seeds = m.twin.entity_seeds(kind, sub, chunk, L)
                exp = m.om.chunk_field_seeded(chunk, seeds)
                assert f is not None and (f == exp).all(), (m.name, kind, L, dest, chunk)
                seen["last_row"] += chunk[0] == m.ch - 1 and bool(len(seeds))
                seen["last_col"] += chunk[1] == m.cw - 1 and bool(len(seeds))
                if L != 0 or not (sub["is_building"] == 0).all():
                    continue
                onm = _on_map(m, sub)
                small = sub["sel_radius"] <= 40.0
                if kind == capi.TARGET_ENTITY:
                    _check_circles(m, chunk, seeds, sub[onm], sub[onm & small])
                    continue
                inside = _in_rect(m, sub, chunk, 0.01)
                maybe = _in_rect(m, sub, chunk, -0.01)
                _check_circles(m, chunk, seeds, sub[maybe & onm], sub[inside & onm & small])
                # enemies outside the rectangle whose circles reach into the window: their tiles must not be seeds
                # unless an enemy inside covers them
                out = ~maybe & onm
                if out.any():
                    seen["excluded"] += _check_circles(m, chunk, np.zeros((0, 2), np.int32), sub[out], sub[:0])
                seen["probe_in"] += int((inside & onm).sum())
            if kind == capi.TARGET_ENEMIES and L == 0:
                seen["host_raster"] += int((~((sub["is_building"] == 0) & (sub["sel_radius"] <= 40.0))).sum())
    finally:
        nav.close()
    # the footprints cross chunk borders and map edges
    x, z, r = [np.asarray(fp[k][~fp["is_building"].astype(bool)], np.float64) for k in ("x", "z", "sel_radius")]
    u, v = (float(m.mx) - x) / 256.0, (z - float(m.mz)) / 256.0
    crosses_chunk = (np.floor(u - r / 256.0) != np.floor(u + r / 256.0)) | (np.floor(v - r / 256.0) != np.floor(v + r / 256.0))
    inner = (u > 0) & (u < m.cw) & (v > 0) & (v < m.ch)
    crosses_edge = inner & ((u - r / 256.0 < 0) | (u + r / 256.0 > m.cw) | (v - r / 256.0 < 0) | (v + r / 256.0 > m.ch))
    assert crosses_edge.any() and (nch == 1 or (crosses_chunk & inner & ~crosses_edge).any())
    assert seen["last_row"] > 0 and seen["last_col"] > 0 and seen["host_raster"] > 0, seen
    if nch > 1:
        assert seen["excluded"] > 0 and seen["probe_in"] > 0, seen


# ---------------------------------------------------------------------------------------------------------------------
# (d) N_GroupArrivalFieldCreate with world-space arguments
# ---------------------------------------------------------------------------------------------------------------------
def test_group_arrival_field_vs_port(placed):
    m = placed
    rng = np.random.default_rng(m.seed + 4)
    open_ = np.argwhere(m.passable)
    up, dn = F(np.inf), F(-np.inf)
    near_edge = [(m.mx - F(3), m.mz + m.H / F(2)), (m.mx - m.W + F(1), m.mz + F(7)), (m.mx - m.W / F(2), m.mz + m.H - F(2)),
                 (m.mx, m.mz), (m.mx - m.W, m.mz + m.H)]
    outside = [(np.nextafter(m.mx, up), m.mz + F(9)), (m.mx - m.W / F(2), np.nextafter(m.mz, dn)), (m.mx + F(40), m.mz - F(40))]
    centres = [m.tile_xz(*open_[i]) for i in rng.integers(0, len(open_), 2)] + near_edge + outside[:1]
    nonempty = empty = 0
    nav = m.device()
    try:
        for i, cxz in enumerate(centres):
            t = desc_for_point(m, *cxz)
            tg = []
            if t is not None:                       # targets around the centre, some of them off the map
                for _ in range(3):
                    tr = min(max(t[0] + int(rng.integers(-40, 41)), 0), m.ch * 64 - 1)
                    tc = min(max(t[1] + int(rng.integers(-40, 41)), 0), m.cw * 64 - 1)
                    tg.append(m.tile_xz(tr, tc))
            tg += [near_edge[i % len(near_edge)], outside[i % len(outside)]]
            targets = np.array(tg, np.float32)
            for dim in (64, 96, 128):
                for enemies in (0, 0b0110):
                    got = nav.group_arrival_field(dim, targets, np.array(cxz, np.float32), enemies)
                    exp = m.om.group_arrival_field(dim, enemies, targets, np.array(cxz, np.float32))
                    assert (got == exp).all(), (m.name, cxz, dim, enemies)
                    nonempty += bool(exp.any()); empty += t is None
    finally:
        nav.close()
    assert nonempty > 0 and empty > 0
