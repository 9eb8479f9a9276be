"""ClearPath case families for tests/test_clearpath_emu.py (device source on CPU threads vs the port) and
tests/test_gpu_clearpath.py (the same families as populations on the device).

A case is one entity and its neighbour lists as find_neighbours (movement.c:2768) hands them to G_ClearPath_NewVelocity:
`self` {px, pz, vx, vz, radius}, `vpref` {vx, vz}, `dyn` / `stat` [32][5] with `ndyn` / `nstat` rows used (static
neighbours have zero velocity, dynamic ones |vel| >= 0.3), `max_len` the truncation length (max_speed / hz). Every family
builds its cases around caller-given centres (float32, map-sized, negative x) and keeps every neighbour within 9.5 wu of
its centre, so that on a map with centres 64 wu apart no two cases meet. Offsets that must stay exact (lattice distances,
mirror images) are small dyadic numbers added to integer centres."""
import numpy as np

EPS = np.float32(1.0 / 1024)
CAP = 32
F = np.float32


class Cases:
    def __init__(self, n):
        self.self5 = np.zeros((n, 5), F)
        self.vpref = np.zeros((n, 2), F)
        self.dyn = np.zeros((n, CAP, 5), F)
        self.stat = np.zeros((n, CAP, 5), F)
        self.ndyn = np.zeros(n, np.int32)
        self.nstat = np.zeros(n, np.int32)
        self.max_len = np.ones(n, F)

    def __len__(self):
        return len(self.self5)

    def case(self, i):
        return (self.self5[i], self.vpref[i], self.dyn[i, :self.ndyn[i]], self.stat[i, :self.nstat[i]], self.max_len[i])

    @staticmethod
    def concat(parts):
        out = Cases(sum(len(p) for p in parts))
        for k in ("self5", "vpref", "dyn", "stat", "ndyn", "nstat", "max_len"):
            setattr(out, k, np.concatenate([getattr(p, k) for p in parts]))
        return out

    def put(self, i, centre, vel, radius, vpref, dyn, stat, max_len=1.0):
        """dyn / stat: lists of (dx, dz, vx, vz, r) relative to the centre (float32 sums)"""
        c = np.asarray(centre, F)
        self.self5[i] = (c[0], c[1], vel[0], vel[1], radius)
        self.vpref[i] = vpref
        self.max_len[i] = max_len
        assert len(dyn) <= CAP and len(stat) <= CAP
        for lst, arr, nattr in ((dyn, self.dyn, self.ndyn), (stat, self.stat, self.nstat)):
            for k, (dx, dz, vx, vz, r) in enumerate(lst):
                arr[i, k] = (c[0] + F(dx), c[1] + F(dz), vx, vz, r)
            nattr[i] = len(lst)


def centres(rng, n, span=4000.0):
    """map-sized centres: x in (-span, -10), z in (10, span)"""
    return np.stack([-rng.uniform(10.0, span, n), rng.uniform(10.0, span, n)], axis=1).astype(F)


def int_centres(rng, n, span=4000):
    return np.stack([-rng.integers(10, span, n), rng.integers(10, span, n)], axis=1).astype(F)


def _disc(rng, rmax=9.5, rmin=0.0):
    a = rng.uniform(0, 2 * np.pi)
    d = np.sqrt(rng.uniform(rmin * rmin, rmax * rmax))
    return d * np.cos(a), d * np.sin(a)


def _vel(rng, lo, hi):
    a = rng.uniform(0, 2 * np.pi)
    s = rng.uniform(lo, hi)
    return s * np.cos(a), s * np.sin(a)


def _dyn(rng, dx, dz, r=None):
    vx, vz = _vel(rng, 0.35, 2.0)
    return (dx, dz, vx, vz, rng.uniform(0.5, 3.0) if r is None else r)


def _stat(rng, dx, dz, r=None):
    return (dx, dz, 0.0, 0.0, rng.uniform(0.5, 3.0) if r is None else r)


COUNTS = (0, 1, 2, 5, 31, 32)


def random_sets(rng, cen, counts=COUNTS):
    """neighbours anywhere within 9.5 wu, radii 0.5-3, every (ndyn, nstat) pair of `counts` in turn"""
    n = len(cen)
    cs = Cases(n)
    pairs = [(a, b) for a in counts for b in counts]
    for i in range(n):
        nd, ns = pairs[i % len(pairs)]
        dyn = [_dyn(rng, *_disc(rng, rmin=0.3)) for _ in range(nd)]
        stat = [_stat(rng, *_disc(rng, rmin=0.3)) for _ in range(ns)]
        cs.put(i, cen[i], _vel(rng, 0.0, 1.5), rng.uniform(0.5, 3.0), _vel(rng, 0.0, 1.5), dyn, stat, rng.uniform(0.3, 2.0))
    return cs


def _ring(rng, k, rad, jitter=0.2):
    a0 = rng.uniform(0, 2 * np.pi)
    return [(rad * np.cos(a0 + 2 * np.pi * j / k) + rng.uniform(-jitter, jitter),
             rad * np.sin(a0 + 2 * np.pi * j / k) + rng.uniform(-jitter, jitter)) for j in range(k)]


def forced_retries(rng, cen):
    """a closed ring of static neighbours plus moving ones inside and outside it, the preferred velocity pointing into
    them: the first solve finds no admissible velocity with both lists non-empty"""
    n = len(cen)
    cs = Cases(n)
    for i in range(n):
        stat = [_stat(rng, dx, dz, rng.uniform(2.0, 3.0)) for dx, dz in _ring(rng, int(rng.integers(6, 13)), rng.uniform(3.0, 5.0))]
        dyn = [_dyn(rng, *_disc(rng, 9.0, 2.0)) for _ in range(int(rng.integers(1, 10)))]
        if rng.random() < 0.5:      # more moving neighbours on a second ring
            dyn += [_dyn(rng, dx, dz) for dx, dz in _ring(rng, int(rng.integers(4, 10)), rng.uniform(6.0, 9.0))]
        tgt = stat[int(rng.integers(len(stat)))]
        vp = np.array(tgt[:2]) / np.hypot(*tgt[:2]) * rng.uniform(0.2, 1.5)
        cs.put(i, cen[i], _vel(rng, 0.0, 1.0), rng.uniform(0.5, 2.0), vp, dyn[:CAP], stat, rng.uniform(0.3, 2.0))
    return cs


LATTICE5 = [(3, 4), (4, 3), (5, 0), (0, 5), (-3, 4), (-4, 3), (-5, 0), (0, -5), (3, -4), (4, -3), (-3, -4), (-4, -3)]
LATTICE_OTHER = [(6, 8), (8, 6), (0, 9), (1, 1), (2, 2), (-2, 2), (6, 0), (0, 6), (-6, 0), (0, -6)]


def equal_distances(rng, cen_int):
    """neighbours on integer lattice offsets with bit-equal float distances (5 = |(3,4)| = |(5,0)| ..., 6, ...), dynamic
    and static ones at the same distance, around a first solve that fails: the literal removal schedule"""
    n = len(cen_int)
    cs = Cases(n)
    for i in range(n):
        offs = list(LATTICE5)
        rng.shuffle(offs)
        k = int(rng.integers(6, len(offs) + 1))
        sel = offs[:k]
        extra = [LATTICE_OTHER[j] for j in rng.choice(len(LATTICE_OTHER), int(rng.integers(0, 5)), replace=False)]
        dyn, stat = [], []
        for j, (dx, dz) in enumerate(sel + extra):
            r = float(rng.choice([1.5, 2.0, 2.5, 3.0]))
            (dyn if (j % 3 == 0) else stat).append(_dyn(rng, dx, dz, r) if j % 3 == 0 else _stat(rng, dx, dz, r))
        vp = np.array(sel[0], float) / 5.0 * rng.uniform(0.3, 1.5)
        cs.put(i, cen_int[i], _vel(rng, 0.0, 0.8), rng.uniform(1.0, 2.5), vp, dyn, stat, rng.uniform(0.3, 2.0))
    return cs


def point_ties(rng, cen_int):
    """configurations mirror-symmetric about the preferred velocity's axis (x): mirrored neighbours (dx, dz) / (dx, -dz)
    with mirrored velocities and an own velocity on the axis, so candidate points come in mirror pairs at the same time and
    distance; offsets are multiples of 1/8 on integer centres, so the mirror is exact in float"""
    n = len(cen_int)
    cs = Cases(n)
    q = lambda v: np.round(v * 8.0) / 8.0
    for i in range(n):
        dyn, stat = [], []
        k = int(rng.integers(3, 7))                    # a closed ring of mirrored static pairs, and both axis points
        rad, r = rng.uniform(3.0, 5.0), q(rng.uniform(2.0, 3.0))
        stat.append((q(rad), 0.0, 0.0, 0.0, r))
        for j in range(1, k):
            t = np.pi * j / k
            dx, dz = q(rad * np.cos(t)), q(rad * np.sin(t))
            stat += [(dx, dz, 0.0, 0.0, r), (dx, -dz, 0.0, 0.0, r)]
        stat.append((q(-rad), 0.0, 0.0, 0.0, r))
        for _ in range(int(rng.integers(1, 4))):       # mirrored moving pairs, heading (roughly) for the entity
            dx, dz = q(rng.uniform(-7.0, 7.0)), q(rng.uniform(1.0, 6.5))
            sp = rng.uniform(0.5, 1.5) / np.hypot(dx, dz)
            vx, vz = q(-dx * sp + rng.uniform(-0.3, 0.3)), q(min(-dz * sp, -0.375))
            rr = q(rng.uniform(0.5, 2.5))
            dyn += [(dx, dz, vx, vz, rr), (dx, -dz, vx, -vz, rr)]
        vx = q(rng.uniform(0.25, 1.5))
        cs.put(i, cen_int[i], (q(rng.uniform(-0.5, 0.5)), 0.0), q(rng.uniform(0.5, 2.0)), (vx, 0.0), dyn, stat,
               q(rng.uniform(0.5, 2.0)))
    return cs


def degenerate_neighbours(rng, cen):
    """a neighbour exactly at the entity's position or closer than EPS (it gets a removal rank but no obstacle), mixed
    into rings that make the first solve fail"""
    n = len(cen)
    cs = Cases(n)
    for i in range(n):
        stat = [_stat(rng, dx, dz, rng.uniform(2.0, 3.0)) for dx, dz in _ring(rng, int(rng.integers(5, 10)), rng.uniform(3.0, 5.0))]
        dyn = [_dyn(rng, *_disc(rng, 9.0, 2.0)) for _ in range(int(rng.integers(1, 6)))]
        for _ in range(int(rng.integers(1, 3))):
            d = [0.0, 0.0] if rng.random() < 0.5 else [rng.uniform(-6e-4, 6e-4), rng.uniform(-6e-4, 6e-4)]
            lst = dyn if rng.random() < 0.5 else stat
            lst.insert(int(rng.integers(0, len(lst) + 1)), (_dyn if lst is dyn else _stat)(rng, d[0], d[1]))
        tgt = stat[0] if abs(stat[0][0]) + abs(stat[0][1]) > 1 else stat[-1]
        vp = np.array(tgt[:2]) / max(np.hypot(*tgt[:2]), 1e-3) * rng.uniform(0.2, 1.5)
        cs.put(i, cen[i], _vel(rng, 0.0, 1.0), rng.uniform(0.5, 2.0), vp, dyn[:CAP], stat[:CAP], rng.uniform(0.3, 2.0))
    return cs


def early_end(rng, cen):
    """the schedule ends early: one list empty (no second solve), or the furthest neighbour alone in its list
    (t_end == 1: the loop ends right after the first removal)"""
    n = len(cen)
    cs = Cases(n)
    for i in range(n):
        ring = [_stat(rng, dx, dz, rng.uniform(2.0, 3.0)) for dx, dz in _ring(rng, int(rng.integers(6, 12)), rng.uniform(3.0, 5.0))]
        kind = i % 3
        if kind == 0:          # only static neighbours
            dyn, stat = [], ring
        elif kind == 1:        # only moving ones
            dyn, stat = [(dx, dz) + _vel(rng, 0.35, 1.5) + (r,) for dx, dz, _, _, r in ring], []
        else:                  # one moving neighbour, furthest of all
            a = rng.uniform(0, 2 * np.pi)
            dyn, stat = [_dyn(rng, 9.3 * np.cos(a), 9.3 * np.sin(a))], ring
        tgt = ring[0]
        vp = np.array(tgt[:2]) / np.hypot(*tgt[:2]) * rng.uniform(0.2, 1.5)
        cs.put(i, cen[i], _vel(rng, 0.0, 1.0), rng.uniform(0.5, 2.0), vp, dyn, stat, rng.uniform(0.3, 2.0))
    return cs


def degenerate_geometry(rng, cen):
    """zero own velocity; HRVO det (centreline x own velocity) within +-EPS; rays with |dir.x| < EPS (NaN slope, incl. the
    preserved l2.point line of C_InfiniteLineIntersection); parallel rays; zero preferred velocity"""
    n = len(cen)
    cs = Cases(n)
    for i in range(n):
        kind = i % 5
        stat = [_stat(rng, dx, dz, rng.uniform(1.5, 3.0)) for dx, dz in _ring(rng, int(rng.integers(3, 9)), rng.uniform(3.0, 6.0), 0.5)]
        dyn = [_dyn(rng, *_disc(rng, 9.0, 2.0)) for _ in range(int(rng.integers(1, 5)))]
        vel = _vel(rng, 0.0, 1.0)
        vp = _vel(rng, 0.1, 1.5)
        if kind == 0:
            vel = (0.0, 0.0)
        elif kind == 1:        # own velocity (nearly) along the centreline of a moving neighbour
            dx, dz, vx, vz, r = dyn[0]
            d = np.hypot(dx, dz)
            s = rng.uniform(0.2, 1.0)
            e = rng.uniform(-1.5, 1.5) * float(EPS)
            vel = (s * dx / d - e * dz / d, s * dz / d + e * dx / d)
        elif kind == 2:        # an edge of a neighbour's cone vertical: D cos(t) - R sin(t) = 0 -> tan(t) = D / R
            own = 0.5
            for lst in (dyn, stat):
                dd, rr = rng.uniform(3.0, 8.0), rng.uniform(0.5, 2.5)
                t = np.arctan2(dd, rr + own) + (np.pi if rng.random() < 0.5 else 0.0)
                item = (dd * np.cos(t), dd * np.sin(t))
                lst.insert(0, _dyn(rng, *item, rr) if lst is dyn else _stat(rng, *item, rr))
            cs.put(i, cen[i], vel, own, vp, dyn, stat, rng.uniform(0.3, 2.0))
            continue
        elif kind == 3:        # parallel rays: a neighbour and its double (twice as far, twice the combined radius)
            own = rng.uniform(0.5, 1.5)
            dx, dz = _disc(rng, 4.5, 2.0)
            r1 = rng.uniform(0.5, 1.5)
            stat.insert(0, _stat(rng, dx, dz, r1))
            stat.append(_stat(rng, 2 * dx, 2 * dz, 2 * (r1 + own) - own))
            cs.put(i, cen[i], vel, own, vp, dyn, stat, rng.uniform(0.3, 2.0))
            continue
        else:
            vp = (0.0, 0.0)
        cs.put(i, cen[i], vel, rng.uniform(0.5, 2.0), vp, dyn, stat, rng.uniform(0.3, 2.0))
    return cs


def overflow(rng, cen):
    """32 + 32 neighbours spread over the disc: phase A finds more than 64 admissible intersections for some"""
    n = len(cen)
    cs = Cases(n)
    for i in range(n):
        dyn = [_dyn(rng, *_disc(rng, 9.5, 3.0), rng.uniform(0.5, 1.2)) for _ in range(CAP)]
        stat = [_stat(rng, *_disc(rng, 9.5, 3.0), rng.uniform(0.5, 1.2)) for _ in range(CAP)]
        cs.put(i, cen[i], _vel(rng, 0.0, 1.0), rng.uniform(0.5, 1.0), _vel(rng, 0.0, 1.5), dyn, stat, rng.uniform(0.3, 2.0))
    return cs


GENERATORS = {"random": random_sets, "forced_retries": forced_retries, "equal_distances": equal_distances,
              "point_ties": point_ties, "degenerate_neighbours": degenerate_neighbours, "early_end": early_end,
              "degenerate_geometry": degenerate_geometry, "overflow": overflow}
INTEGER_CENTRES = ("equal_distances", "point_ties")        # their exact offsets need integer centres
FAMILIES = {name: (lambda g, ic: lambda rng, n: g(rng, int_centres(rng, n) if ic else centres(rng, n)))(g, name in INTEGER_CENTRES)
            for name, g in GENERATORS.items()}


def distances(cs, i):
    """float32 distances of case i's neighbours from the entity, dyn then stat (remove_furthest's v2_len)"""
    p = cs.self5[i, :2]
    nb = np.concatenate([cs.dyn[i, :cs.ndyn[i], :2], cs.stat[i, :cs.nstat[i], :2]])
    d = (p - nb).astype(F)
    return np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]).astype(F)).astype(F)


def has_distance_tie(cs, i):
    d = distances(cs, i)
    return len(np.unique(d)) < len(d)


def same_position(cs, i):
    """a neighbour closer than EPS: no obstacle for it (clearpath.c:123)"""
    return bool((distances(cs, i) < EPS).any())


def ends_after_first_removal(cs, i):
    """t_end <= 1: the first removal (furthest, first in dyn ++ stat order) empties a list, or one list is empty"""
    nd, ns = int(cs.ndyn[i]), int(cs.nstat[i])
    if nd == 0 or ns == 0:
        return True
    d = distances(cs, i)
    k = int(np.argmax(d))          # first maximum, as remove_furthest
    return (k < nd and nd == 1) or (k >= nd and ns == 1)
