"""ctypes binding of oracle/libpforacle.so -- the plain-C CPU restatement (pf_oracle.c).
TEST INFRASTRUCTURE: see the header of pf_oracle.h for who may import this."""
import ctypes as C
import os
import subprocess
import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libpforacle.so")
_lib = None


class _Map(C.Structure):
    _fields_ = [("chunk_w", C.c_int), ("chunk_h", C.c_int), ("map_x", C.c_float), ("map_z", C.c_float),
                ("cost", C.c_void_p), ("blockers", C.c_void_p), ("local_islands", C.c_void_p),
                ("factions", C.c_void_p), ("enemies", C.c_uint16 * 16)]


def build():
    subprocess.run(["make", "-s", "-C", _HERE, "port"], check=True)
    return LIB_PATH


def lib():
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            build()
        L = C.CDLL(LIB_PATH)
        L.pfo_flow_fields_update.argtypes = [C.POINTER(_Map), C.c_void_p, C.c_size_t, C.c_void_p]
        L.pfo_los_fields_create.argtypes = [C.POINTER(_Map), C.c_void_p, C.c_size_t, C.c_void_p]
        L.pfo_world_create.restype = C.c_void_p
        L.pfo_world_create.argtypes = [C.POINTER(_Map), C.c_void_p, C.c_size_t, C.c_void_p, C.c_size_t, C.c_int]
        L.pfo_world_destroy.argtypes = [C.c_void_p]
        L.pfo_ents_in_circle.argtypes = [C.c_void_p, C.c_float, C.c_float, C.c_float, C.c_void_p, C.c_int]
        L.pfo_velocity_work.argtypes = [C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p]
        L.pfo_desired_velocity.argtypes = [C.POINTER(_Map), C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t,
                                           C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
        L.pfo_flow_update_nearest_pathable.argtypes = [C.POINTER(_Map)] + [C.c_int] * 4 + [C.c_void_p]
        L.pfo_flow_update_island_to_nearest.argtypes = [C.POINTER(_Map), C.c_void_p, C.c_void_p, C.c_uint16, C.c_void_p]
        L.pfo_cost_from_tiles.argtypes = [C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.pfo_region_field_create.argtypes = [C.POINTER(_Map), C.c_int, C.c_uint16, C.c_int, C.c_void_p, C.c_int,
                                              C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.pfo_group_arrival_field.argtypes = [C.POINTER(_Map), C.c_int, C.c_uint16, C.c_void_p, C.c_int, C.c_void_p,
                                              C.c_void_p, C.c_int, C.c_void_p]
        L.pfo_world_set_states.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        L.pfo_entity_updates.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p, C.c_void_p,
                                         C.c_void_p]
        L.pfo_entity_apply.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_size_t, C.c_void_p]
        L.pfo_zone_seeds.restype = C.c_int
        L.pfo_zone_seeds.argtypes = [C.POINTER(_Map)] + [C.c_int] * 5 + [C.c_void_p]
        L.pfo_chunk_field_seeded.argtypes = [C.POINTER(_Map), C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_void_p]
        L.pfo_flow_field_zone.argtypes = [C.POINTER(_Map)] + [C.c_int] * 5 + [C.c_void_p]
        L.pfo_group_arrival_velocity.argtypes = [C.POINTER(_Map), C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p,
                                                 C.c_int, C.c_void_p, C.c_void_p]
        L.pfo_region_field_update_to_nearest_pathable.argtypes = [C.POINTER(_Map)] + [C.c_int] * 5 + [C.c_void_p, C.c_int, C.c_void_p]
        L.pfo_clearpath.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_float, C.c_void_p]
        L.pfo_inside_pcr.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_long, C.c_void_p]
        L.pfo_line_isect.argtypes = [C.c_void_p, C.c_long, C.c_void_p]
        _lib = L
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p) if a is not None else None


def cost_from_tiles(chunk_w, chunk_h, tiles, ref_layer):
    """tiles: int32[H32][W32][4] -> cost_base u8[chunks][64][64] (nav.c:267, 431)."""
    tiles = np.ascontiguousarray(tiles, np.int32)
    assert tiles.shape == (chunk_h * 32, chunk_w * 32, 4)
    out = np.zeros((chunk_w * chunk_h, 64, 64), np.uint8)
    lib().pfo_cost_from_tiles(chunk_w, chunk_h, _p(tiles), ref_layer, _p(out))
    return out


class OracleMap:
    def __init__(self, chunk_w, chunk_h, cost, blockers=None, local_islands=None, map_x=0.0, map_z=0.0,
                 factions=None, enemies=None):
        """factions: u8[chunks][15][64][64] per-faction blocker refcounts; enemies[f] = war bit mask of faction f"""
        self.cw, self.ch = chunk_w, chunk_h
        self.cost = np.ascontiguousarray(cost, np.uint8)
        self.blockers = None if blockers is None else np.ascontiguousarray(blockers, np.uint16)
        self.liid = None if local_islands is None else np.ascontiguousarray(local_islands, np.uint16)
        self.factions = None if factions is None else np.ascontiguousarray(factions, np.uint8)
        en = (C.c_uint16 * 16)(*([0] * 16))
        if enemies is not None:
            for f in range(16):
                en[f] = int(enemies[f])
        self.m = _Map(chunk_w, chunk_h, map_x, map_z, _p(self.cost), _p(self.blockers), _p(self.liid), _p(self.factions), en)

    def flow_fields_update(self, reqs, inout=None):
        reqs = np.ascontiguousarray(reqs)
        n = len(reqs)
        buf = np.zeros((n, 64, 64), np.uint8) if inout is None else np.ascontiguousarray(inout, np.uint8).reshape(n, 64, 64).copy()
        lib().pfo_flow_fields_update(C.byref(self.m), _p(reqs), n, _p(buf))
        return buf

    def flow_nearest_pathable(self, chunk, start, inout):
        buf = np.ascontiguousarray(inout, np.uint8).reshape(-1).copy()
        lib().pfo_flow_update_nearest_pathable(C.byref(self.m), chunk[0], chunk[1], start[0], start[1], _p(buf))
        return buf.reshape(64, 64)

    def flow_island_to_nearest(self, gisl, req, local_iid, inout):
        """req: the FIELD_REQ record (1 element) that built the field; gisl: global islands [chunks][64][64]"""
        buf = np.ascontiguousarray(inout, np.uint8).reshape(-1).copy()
        gisl = np.ascontiguousarray(gisl, np.uint16)
        req = np.ascontiguousarray(req)
        lib().pfo_flow_update_island_to_nearest(C.byref(self.m), _p(gisl), _p(req), int(local_iid), _p(buf))
        return buf.reshape(64, 64)

    # ---- region fields (absolute tile coordinates = chunk * 64 + tile) ----
    @staticmethod
    def _pairs(a):
        a = np.ascontiguousarray(a if a is not None else np.zeros((0, 2)), np.int32).reshape(-1, 2)
        return a, len(a)

    def region_field_create(self, dim, enemies, cell_mode, seeds, center, overlay=None):
        """N_CellArrivalFieldCreate (cell_mode=1, seeds = [target]) / tile-space N_GroupArrivalFieldCreate"""
        sd, ns = self._pairs(seeds); ov, no = self._pairs(overlay)
        out = np.zeros((dim, dim // 2), np.uint8)
        lib().pfo_region_field_create(C.byref(self.m), dim, int(enemies), int(cell_mode), _p(sd), ns,
                                      int(center[0]), int(center[1]), _p(ov), no, _p(out))
        return out

    def group_arrival_field(self, dim, enemies, targets_xz, center_xz, overlay=None):
        t = np.ascontiguousarray(targets_xz, np.float32).reshape(-1, 2); ov, no = self._pairs(overlay)
        c = np.ascontiguousarray(center_xz, np.float32)
        out = np.zeros((dim, dim // 2), np.uint8)
        lib().pfo_group_arrival_field(C.byref(self.m), dim, int(enemies), _p(t), len(t), _p(c), _p(ov), no, _p(out))
        return out

    def region_field_fixup(self, dim, start, center, inout, overlay=None):
        """N_CellArrivalFieldUpdateToNearestPathable"""
        ov, no = self._pairs(overlay)
        buf = np.ascontiguousarray(inout, np.uint8).copy()
        lib().pfo_region_field_update_to_nearest_pathable(C.byref(self.m), dim, int(start[0]), int(start[1]),
                                                          int(center[0]), int(center[1]), _p(ov), no, _p(buf))
        return buf

    def zone_seeds(self, chunk, centre, radius):
        out = np.zeros((4 * 4096, 2), np.int32)
        n = lib().pfo_zone_seeds(C.byref(self.m), chunk[0], chunk[1], int(centre[0]), int(centre[1]), int(radius), _p(out))
        return out[:n].copy()

    def chunk_field_seeded(self, chunk, seeds, inout=None):
        """padded-chunk field (zone / entity / enemies targets) from its zero-cost tiles"""
        sd, ns = self._pairs(seeds)
        buf = np.zeros((64, 64), np.uint8) if inout is None else np.ascontiguousarray(inout, np.uint8).reshape(64, 64).copy()
        lib().pfo_chunk_field_seeded(C.byref(self.m), chunk[0], chunk[1], _p(sd), ns, _p(buf))
        return buf

    def flow_field_zone(self, chunk, centre, radius, inout=None):
        """N_FlowFieldInit + N_FlowFieldUpdate(TARGET_ZONE); centre = absolute (r, c)"""
        buf = np.zeros((64, 64), np.uint8) if inout is None else np.ascontiguousarray(inout, np.uint8).reshape(64, 64).copy()
        lib().pfo_flow_field_zone(C.byref(self.m), chunk[0], chunk[1], int(centre[0]), int(centre[1]), int(radius), _p(buf))
        return buf

    def group_arrival_velocity(self, fields, has, centre_xz, radius, pos_xz):
        fields = np.ascontiguousarray(fields, np.uint8); has = np.ascontiguousarray(has, np.uint8)
        pos = np.ascontiguousarray(pos_xz, np.float32).reshape(-1, 2); c = np.ascontiguousarray(centre_xz, np.float32)
        vel = np.zeros((len(pos), 2), np.float32); fl = np.zeros(len(pos), np.uint8)
        lib().pfo_group_arrival_velocity(C.byref(self.m), _p(fields), _p(has), _p(c), int(radius), _p(pos), len(pos), _p(vel), _p(fl))
        return vel, fl

    def los_fields_create(self, reqs):
        reqs = np.ascontiguousarray(reqs)
        out = np.zeros((len(reqs), 64, 64), np.uint8)
        lib().pfo_los_fields_create(C.byref(self.m), _p(reqs), len(reqs), _p(out))
        return out

    def desired_velocity(self, agents, flocks, work, slot, flow, los):
        work = np.ascontiguousarray(work, np.uint32)
        slot = np.ascontiguousarray(slot, np.int32)
        vdes = np.zeros((len(work), 2), np.float32); lo = np.zeros(len(work), np.uint8)
        lib().pfo_desired_velocity(C.byref(self.m), _p(agents), _p(flocks), _p(work), len(work), _p(slot),
                                   _p(flow), _p(los), _p(vdes), _p(lo))
        return vdes, lo


def clearpath(self5, vpref, dyn, stat, max_len=float("inf")):
    """G_ClearPath_NewVelocity then vec2_truncate(max_len); self5 / dyn / stat rows: {px, pz, vx, vz, radius}"""
    self5 = np.ascontiguousarray(self5, np.float32)
    vpref = np.ascontiguousarray(vpref, np.float32)
    dyn = np.ascontiguousarray(dyn, np.float32).reshape(-1, 5)
    stat = np.ascontiguousarray(stat, np.float32).reshape(-1, 5)
    assert len(dyn) <= 32 and len(stat) <= 32
    out = np.zeros(2, np.float32)
    lib().pfo_clearpath(_p(self5), _p(vpref), _p(dyn), len(dyn), _p(stat), len(stat), float(max_len), _p(out))
    return out


def inside_pcr(rays4, pts):
    """inside_pcr over the ray table rays4 [n_rays][4] {px, pz, dx, dz} for every point of pts [n][2] -> bool [n]"""
    rays4 = np.ascontiguousarray(rays4, np.float32).reshape(-1, 4)
    pts = np.ascontiguousarray(pts, np.float32).reshape(-1, 2)
    out = np.zeros(len(pts), np.uint8)
    lib().pfo_inside_pcr(_p(rays4), len(rays4), _p(pts), len(pts), _p(out))
    return out.astype(bool)


def line_isect(lines):
    """C_InfiniteLineIntersection for lines [n][2][4] {px, pz, dx, dz} -> [n][3] {ok, x, z}"""
    lines = np.ascontiguousarray(lines, np.float32).reshape(-1, 8)
    out = np.zeros((len(lines), 3), np.float32)
    lib().pfo_line_isect(_p(lines), len(lines), _p(out))
    return out


def entity_apply(agents, movestate, work, patches, ext=None):
    """entity_apply_update's movestate part -> (agents, movestate) copies after the patches, and the movestate_ext copy
    (64-B records, uid order) when `ext` is given: (agents, movestate, ext)"""
    a = np.ascontiguousarray(agents).copy(); ms = np.ascontiguousarray(movestate).copy()
    ex = None if ext is None else np.ascontiguousarray(ext).copy()
    assert ex is None or ex.dtype.itemsize == 64
    work = np.ascontiguousarray(work, np.uint32); p = np.ascontiguousarray(patches)
    assert p.dtype.itemsize == 160
    lib().pfo_entity_apply(_p(a), _p(ms), _p(ex), _p(work), len(work), _p(p))
    return (a, ms) if ext is None else (a, ms, ex)


class _Arrival(C.Structure):
    _fields_ = [("nearest_ok", C.c_int32), ("nearest", C.c_float * 2), ("mc_n", C.c_int32), ("mc", C.c_void_p)]




class OracleWorld:
    def __init__(self, omap, agents, flocks, hz=20, formation=None, ext=None):
        """formation / ext: per-uid FORMATION_IN / MOVESTATE_EXT records (64 B each) of the states beyond point seeking,
        or None (no formation; NULL_UID targets and zero counters)"""
        self.omap = omap
        self.agents = np.ascontiguousarray(agents)
        self.flocks = np.ascontiguousarray(flocks)
        self.formation = None if formation is None else np.ascontiguousarray(formation)
        self.ext = None if ext is None else np.ascontiguousarray(ext)
        for r in (self.formation, self.ext):
            assert r is None or (r.dtype.itemsize == 64 and len(r) == len(self.agents))
        self.h = lib().pfo_world_create(C.byref(omap.m), _p(self.agents), len(self.agents), _p(self.flocks),
                                        len(self.flocks), hz)
        lib().pfo_world_set_states(self.h, _p(self.formation), _p(self.ext))

    def close(self):
        if self.h:
            lib().pfo_world_destroy(self.h)
            self.h = None

    def ents_in_circle(self, x, z, r, maxout=512):
        out = np.zeros(maxout, np.uint32)
        n = lib().pfo_ents_in_circle(self.h, x, z, r, _p(out), maxout)
        return out[:n].copy()

    @staticmethod
    def _arrivals(arrival):
        """(nearest_ok, nearest[2], mc[n, 2]) tuples (None: no tiles) -> ctypes array, arrays kept alive"""
        keep = [np.zeros((0, 2), np.float32) if a is None else np.ascontiguousarray(a[2], np.float32).reshape(-1, 2) for a in arrival]
        arr = (_Arrival * max(len(arrival), 1))()
        for i, a in enumerate(arrival):
            if a is not None:
                arr[i].nearest_ok = int(a[0]); arr[i].nearest[0], arr[i].nearest[1] = float(a[1][0]), float(a[1][1])
            arr[i].mc_n = len(keep[i]); arr[i].mc = keep[i].ctypes.data
        return arr, keep

    def entity_updates(self, movestate, arrival, work, new_vel, vdes, patch_dtype, target_arrival=None):
        """entity_compute_update per work item. movestate: 176-B records (uid order); arrival: per flock
        (nearest_ok, nearest[2], mc[n, 2]); target_arrival: per work item the same for the target of an
        ENTER_ENTITY_RANGE item (None for the others), or None; -> record array of patch_dtype (160 B)"""
        ms = np.ascontiguousarray(movestate); work = np.ascontiguousarray(work, np.uint32)
        nv = np.ascontiguousarray(new_vel, np.float32); vd = np.ascontiguousarray(vdes, np.float32)
        arr, keep = self._arrivals(arrival)
        tarr, tkeep = (None, None) if target_arrival is None else self._arrivals(target_arrival)
        assert target_arrival is None or len(target_arrival) == len(work)
        out = np.zeros(len(work), patch_dtype)
        assert out.dtype.itemsize == 160 and ms.dtype.itemsize == 176
        lib().pfo_entity_updates(self.h, _p(ms), C.byref(arr), None if tarr is None else C.byref(tarr), _p(work), len(work),
                                 _p(nv), _p(vd), _p(out))
        return out

    def velocity_work(self, work):
        work = np.ascontiguousarray(work, np.uint32)
        vel = np.zeros((len(work), 2), np.float32); vpref = np.zeros((len(work), 2), np.float32)
        lib().pfo_velocity_work(self.h, _p(work), len(work), _p(vel), _p(vpref))
        return vel, vpref
