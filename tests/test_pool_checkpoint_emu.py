"""The pool segment of pfnav_pool_save / pfnav_pool_restore and the map digest on the CPU (csrc/pfnav_pool_host.h through
tests/emu/pool_checkpoint_emu.cpp; the device's touch stamps and field bytes are host arrays there).

- Round trip: pools built with the real slot policies (pf_pool_reserve with evictions, pf_pool_zone_take, pf_pool_drop,
  pf_pool_reset, fields built, aux targets) from seeded op sequences save, load into a fresh pool and save again to the
  same bytes; the loaded pool equals the original member for member.
- Refusals: one segment per validation rule, each refused with its own message, and a refusal changes nothing.
- Digest: the header's function equals a numpy restatement on random images, and summing the tile and block terms in any
  order gives the same value."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
MAGIC = 0x4C504650
HDR = np.dtype([("magic", "<u4"), ("version", "<u4"), ("req_size", "<u2"), ("fp_size", "<u2"), ("chunk_w", "u1"),
                ("chunk_h", "u1"), ("nlayers", "u1"), ("_pad0", "u1"), ("ndests", "<i4"), ("max", "<i4"), ("used", "<i4"),
                ("nzone", "<i4"), ("tick_no", "<u4"), ("nfree", "<u4"), ("naux", "<u4"), ("nfp", "<u4"), ("nstored", "<u4"),
                ("_pad1", "<u4"), ("digest", "<u8")])
assert HDR.itemsize == 64
AUX = np.dtype([("kind", "<i4"), ("layer", "<i4"), ("ref_layer", "<i4"), ("nents", "<u4")])
FP = np.dtype([("x", "<f4"), ("z", "<f4"), ("sel_radius", "<f4"), ("is_building", "<u4"), ("corners", "<f4", 8)])
assert FP.itemsize == 48
REQ = 64                    # sizeof(pfnav_field_req)
CW, CH, NL = 3, 2, 3        # the map geometry the segments of these tests name
DIGEST = 0x0123456789ABCDEF


# ---------------------------------------------------------------------------------------------------------------------
# the map digest, restated
# ---------------------------------------------------------------------------------------------------------------------
U = np.uint64
K_TILE, K_MIX = U(0xD6E8FEB86659FD93), U(0xA0761D6478BD642F)


def splitmix64(x):
    x = np.asarray(x, np.uint64)
    with np.errstate(over="ignore"):
        x = x + U(0x9E3779B97F4A7C15)
        x = (x ^ (x >> U(30))) * U(0xBF58476D1CE4E5B9)
        x = (x ^ (x >> U(27))) * U(0x94D049BB133111EB)
    return x ^ (x >> U(31))


def tile_terms(cost, blk, liid, fmask):
    """[..., 4096] chunk-blocked tiles -> splitmix64(v ^ t * K) per tile"""
    t = np.arange(4096, dtype=np.uint64)
    v = cost.astype(U) | blk.astype(U) << U(8) | liid.astype(U) << U(24) | fmask.astype(U) << U(40)
    with np.errstate(over="ignore"):
        return splitmix64(v ^ (t * K_TILE))


def block_terms(block_hash, nlayers, chunks):
    lay = np.repeat(np.arange(nlayers, dtype=np.uint64), chunks)
    ch = np.tile(np.arange(chunks, dtype=np.uint64), nlayers)
    with np.errstate(over="ignore"):
        return splitmix64(block_hash.reshape(-1) ^ (((lay << U(32)) | ch) * K_MIX))


def fold(total, nlayers, cw, ch, map_x, map_z, enemies):
    h = np.asarray(total, np.uint64)
    bits = np.array([map_x, map_z], np.float32).view(np.uint32)
    for x in [nlayers, cw, ch, int(bits[0]), int(bits[1])] + [int(e) for e in enemies]:
        h = splitmix64(h ^ U(x))
    return int(h)


def map_digest_np(cost, blk, liid, fmask, cw, ch, map_x=0.0, map_z=0.0, enemies=None):
    """images [nlayers][chunks][64][64] (the chunk-blocked layout of map_get_layer / blockers / local_islands); fmask
    may be None (zeros)"""
    cost = np.asarray(cost).reshape(-1, cw * ch, 4096)
    nl = cost.shape[0]
    blk = np.asarray(blk).reshape(nl, -1, 4096); liid = np.asarray(liid).reshape(nl, -1, 4096)
    fmask = np.zeros_like(blk) if fmask is None else np.asarray(fmask).reshape(nl, -1, 4096)
    with np.errstate(over="ignore"):
        bh = tile_terms(cost, blk, liid, fmask).sum(axis=-1, dtype=np.uint64)
        total = block_terms(bh, nl, cw * ch).sum(dtype=np.uint64)
    return fold(total, nl, cw, ch, map_x, map_z, [0] * 16 if enemies is None else enemies)


def fmask_of(faction_counts):
    """[chunks][15][64][64] per-faction blocker counts -> [chunks][64][64] masks, bit f set where faction f counts"""
    fc = np.asarray(faction_counts)
    m = np.zeros((fc.shape[0], 64, 64), np.uint16)
    for f in range(15):
        m |= ((fc[:, f] > 0).astype(np.uint16) << f)
    return m


# ---------------------------------------------------------------------------------------------------------------------
# the emulator
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def emu(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libpool_checkpoint_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-D_GLIBCXX_ASSERTIONS", "-fPIC", "-shared",
                    os.path.join(HERE, "emu", "pool_checkpoint_emu.cpp"), "-o", so], check=True)
    L = C.CDLL(so)
    p, sz, u64 = C.c_void_p, C.c_size_t, C.c_uint64
    L.emu_pc_new.restype = p
    L.emu_pc_new.argtypes = [C.c_int, C.c_int, C.c_int]
    L.emu_pc_clone.restype = p
    L.emu_pc_clone.argtypes = [p]
    L.emu_pc_delete.argtypes = [p]
    L.emu_pc_set_tick.argtypes = [p, C.c_uint32]
    L.emu_pc_reserve.argtypes = [p, p, C.c_int, p]
    L.emu_pc_zone_take.argtypes = [p, u64]
    L.emu_pc_built.argtypes = [p, u64, C.c_int, C.c_int, u64, p]
    L.emu_pc_drop.argtypes = [p, u64]
    L.emu_pc_reset.argtypes = [p]
    L.emu_pc_set_aux.argtypes = [p, C.c_int, C.c_int, C.c_int, C.c_int, p, C.c_int]
    L.emu_pc_size.restype = sz
    L.emu_pc_size.argtypes = [p]
    L.emu_pc_save.restype = sz
    L.emu_pc_save.argtypes = [p, C.c_int, C.c_int, C.c_int, u64, p]
    L.emu_pc_load.argtypes = [p, p, sz, C.c_int, C.c_int, C.c_int, u64, C.c_char_p]
    L.emu_pc_equal.argtypes = [p, p, C.c_int]
    L.emu_pc_counts.argtypes = [p, p]
    L.emu_pc_digest.restype = u64
    L.emu_pc_digest.argtypes = [p, p, p, p, C.c_int, C.c_int, C.c_int, C.c_float, C.c_float, p]
    L.emu_pc_digest_tile.restype = u64
    L.emu_pc_digest_tile.argtypes = [C.c_uint32] * 5
    L.emu_pc_digest_block.restype = u64
    L.emu_pc_digest_block.argtypes = [u64, C.c_int, C.c_int]
    return L


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


def save(L, h, digest=DIGEST):
    out = np.zeros(L.emu_pc_size(h), np.uint8)
    assert L.emu_pc_save(h, CW, CH, NL, digest, _p(out)) == len(out)
    return out.tobytes()


def load(L, h, seg, geom=(CW, CH, NL), digest=DIGEST):
    """-> None or the refusal's message; a refusal must leave the pool as it was"""
    before = L.emu_pc_clone(h)
    try:
        buf = np.frombuffer(seg, np.uint8) if len(seg) else np.zeros(1, np.uint8)
        err = C.create_string_buffer(256)
        rc = L.emu_pc_load(h, _p(buf), len(seg), geom[0], geom[1], geom[2], digest, err)
        if rc:
            assert L.emu_pc_equal(h, before, 1), "a refused load changed the pool"
            return err.value.decode()
        return None
    finally:
        L.emu_pc_delete(before)


def footprints(rng, n):
    f = np.zeros(n, FP)
    f["x"], f["z"] = rng.random(n) * 300, rng.random(n) * 300
    f["sel_radius"] = rng.random(n) * 5
    f["is_building"] = rng.integers(0, 2, n)
    f["corners"] = rng.random((n, 8)) * 300
    return f


def build(L, rng, ndests, mx, nops):
    """a pool driven by the real policies through a seeded op sequence"""
    chunks = CW * CH
    nkeys = ndests * chunks
    h = L.emu_pc_new(ndests, chunks, mx)
    tick = 1
    for _ in range(nops):
        op = rng.random()
        if op < 0.45:
            tick += int(rng.integers(0, 3))
            L.emu_pc_set_tick(h, tick)
            keys = rng.integers(0, nkeys, int(rng.integers(1, min(nkeys, mx) + 1))).astype(np.uint64)
            dev = rng.integers(0, tick + 1, mx).astype(np.uint32)
            L.emu_pc_reserve(h, _p(keys), len(keys), _p(dev))
        elif op < 0.55:
            L.emu_pc_zone_take(h, int(rng.integers(0, nkeys)))
        elif op < 0.80:
            b = rng.integers(0, 256, 8192).astype(np.uint8)
            L.emu_pc_built(h, int(rng.integers(0, nkeys)), int(rng.integers(1, 4)), int(rng.integers(0, NL)),
                           int(rng.integers(1, 1 << 40)), _p(b))
        elif op < 0.88:
            L.emu_pc_drop(h, int(rng.integers(0, nkeys)))
        elif op < 0.90:
            L.emu_pc_reset(h)
        else:
            kind = int(rng.integers(0, 2))
            n = 1 if kind == capi.TARGET_ENTITY else int(rng.integers(0, 5))
            f = footprints(rng, max(n, 1))
            L.emu_pc_set_aux(h, int(rng.integers(0, ndests)), kind, int(rng.integers(0, NL)), int(rng.integers(0, 12)), _p(f), n)
    return h


def counts(L, h):
    c = np.zeros(4, np.int64)
    L.emu_pc_counts(h, _p(c))
    return dict(zip(("used", "nzone", "nfree", "tick"), c.tolist()))


# ---------------------------------------------------------------------------------------------------------------------
# the segment, parsed and composed in Python (the layout of pfnav_pool_host.h, restated)
# ---------------------------------------------------------------------------------------------------------------------
SECTIONS = ("slot", "ffid", "has", "req", "touch", "owner", "free", "aux", "fp", "dtouch", "fields")


def layout(nkeys, mx, nfree, naux, nfp, nstored):
    sizes = dict(slot=nkeys * 4, ffid=nkeys * 8, has=mx, req=mx * REQ, touch=mx * 4, owner=mx * 8, free=nfree * 4,
                 aux=naux * 16, fp=nfp * 48, dtouch=mx * 4, fields=nstored * 8192)
    o, out = 64, {}
    for name in SECTIONS:
        out[name] = o
        o = (o + sizes[name] + 15) & ~15
    out["size"] = o
    return out


def parse(seg):
    h = np.frombuffer(seg[:64], HDR)[0].copy()
    mx, nkeys = int(h["max"]), int(h["ndests"]) * int(h["chunk_w"]) * int(h["chunk_h"])
    L = layout(nkeys, mx, int(h["nfree"]), int(h["naux"]), int(h["nfp"]), int(h["nstored"]))
    assert L["size"] == len(seg)
    b = np.frombuffer(seg, np.uint8)

    def arr(name, dtype, n):
        return b[L[name]:L[name] + n * np.dtype(dtype).itemsize].view(dtype).copy()

    return dict(h=h, slot=arr("slot", "<i4", nkeys), ffid=arr("ffid", "<u8", nkeys), has=arr("has", "u1", mx),
                req=arr("req", "u1", mx * REQ).reshape(mx, REQ), touch=arr("touch", "<u4", mx), owner=arr("owner", "<i8", mx),
                free=arr("free", "<i4", int(h["nfree"])), aux=arr("aux", AUX, int(h["naux"])), fp=arr("fp", FP, int(h["nfp"])),
                dtouch=arr("dtouch", "<u4", mx), fields=arr("fields", "u1", int(h["nstored"]) * 8192).reshape(-1, 8192))


def compose(d, counts_from_arrays=True):
    h = d["h"].copy()
    if counts_from_arrays:
        h["nfree"], h["naux"], h["nfp"], h["nstored"] = len(d["free"]), len(d["aux"]), len(d["fp"]), len(d["fields"])
    mx, nkeys = int(h["max"]), len(d["slot"])
    L = layout(nkeys, mx, int(h["nfree"]), int(h["naux"]), int(h["nfp"]), int(h["nstored"]))
    out = np.zeros(L["size"], np.uint8)
    out[:64] = np.frombuffer(h.tobytes(), np.uint8)
    for name in SECTIONS:
        raw = np.ascontiguousarray(d[name]).view(np.uint8).reshape(-1)
        out[L[name]:L[name] + len(raw)] = raw
    return out.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# tests
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("seed", range(10))
def test_round_trip_of_policy_built_pools(emu, seed):
    rng = np.random.default_rng(0x90C0 + seed)
    ndests = int(rng.integers(1, 5))
    mx = int(rng.integers(1, ndests * CW * CH + 3))
    for step in range(12):
        h = build(emu, np.random.default_rng(seed * 100 + step), ndests, mx, 40 * (step + 1))
        try:
            seg = save(emu, h)
            d = parse(seg)
            c = counts(emu, h)
            assert d["h"]["magic"] == MAGIC and d["h"]["used"] == c["used"] and d["h"]["nzone"] == c["nzone"]
            assert d["h"]["tick_no"] == c["tick"] and d["h"]["digest"] == DIGEST
            assert compose(d) == seg, "the Python layout differs from the header's"
            fresh = emu.emu_pc_new(ndests, CW * CH, mx)
            try:
                assert load(emu, fresh, seg) is None
                assert emu.emu_pc_equal(fresh, h, 1), "the loaded pool differs from the saved one"
                assert save(emu, fresh) == seg, "save -> load -> save changed bytes"
            finally:
                emu.emu_pc_delete(fresh)
            # a load replaces a pool that is already populated, whatever it held
            other = build(emu, np.random.default_rng(seed * 100 + step + 50), ndests, mx, 60)
            try:
                assert load(emu, other, seg) is None
                assert emu.emu_pc_equal(other, h, 1) and save(emu, other) == seg
            finally:
                emu.emu_pc_delete(other)
        finally:
            emu.emu_pc_delete(h)


def test_policies_reach_evictions_zones_and_fields(emu):
    """the op sequences above are not vacuous: full pools with zone-held slots, stored fields and aux targets"""
    seen = dict(full=0, zone=0, stored=0, aux=0)
    for seed in range(10):
        rng = np.random.default_rng(seed)
        h = build(emu, rng, 3, 8, 300)
        d = parse(save(emu, h))
        seen["full"] += int(d["h"]["used"]) == 8
        seen["zone"] += int(d["h"]["nzone"]) > 0
        seen["stored"] += len(d["fields"]) > 0
        seen["aux"] += len(d["fp"]) > 0
        emu.emu_pc_delete(h)
    assert all(v > 0 for v in seen.values()), seen


def test_cleared_pool_saves_empty(emu):
    h = build(emu, np.random.default_rng(3), 2, 9, 200)
    try:
        emu.emu_pc_reset(h)
        d = parse(save(emu, h))
        assert d["h"]["used"] == 0 and d["h"]["nzone"] == 0 and len(d["fields"]) == 0 and len(d["free"]) == 0
        assert (d["slot"] == -1).all() and (d["has"] == 0).all() and (d["dtouch"] == 0).all()
    finally:
        emu.emu_pc_delete(h)


def crafted(emu):
    """a pool with owned, zone-held and free-listed slots, stored fields, aux targets, and room above `used`"""
    rng = np.random.default_rng(77)
    ndests, mx = 3, 12
    chunks = CW * CH
    h = emu.emu_pc_new(ndests, chunks, mx)
    emu.emu_pc_set_tick(h, 5)
    keys = np.arange(6, dtype=np.uint64)
    emu.emu_pc_reserve(h, _p(keys), 6, _p(np.zeros(mx, np.uint32)))                # slots 0..5 owned
    emu.emu_pc_zone_take(h, 12); emu.emu_pc_zone_take(h, 13)                       # slots 6, 7 zone-held
    for k, bits in ((0, 3), (1, 1), (2, 2), (12, 1)):
        b = rng.integers(0, 256, 8192).astype(np.uint8)
        emu.emu_pc_built(h, k, bits, 1, 1000 + k, _p(b))
    f = footprints(rng, 3)
    emu.emu_pc_set_aux(h, 1, capi.TARGET_ENEMIES, 2, 0, _p(f), 3)
    emu.emu_pc_set_aux(h, 2, capi.TARGET_ENTITY, 0, 1, _p(f[1:]), 1)
    d = parse(save(emu, h))
    emu.emu_pc_delete(h)
    # free slots 4 and 5 by hand, as evictions leave them (unmapped, no owner, no fields); the free list is in order
    for s in (4, 5):
        k = int(d["owner"][s])
        d["slot"][k], d["ffid"][k], d["owner"][s] = -1, 0, -1
    d["free"] = np.array([5, 4], np.int32)
    d["h"]["nfree"] = 2
    return d, ndests, mx


def test_layout_and_a_hand_made_free_list(emu):
    d, ndests, mx = crafted(emu)
    h = d["h"]
    assert (h["magic"], h["version"], h["req_size"], h["fp_size"]) == (MAGIC, 1, REQ, 48)
    assert (h["chunk_w"], h["chunk_h"], h["nlayers"], h["ndests"], h["max"]) == (CW, CH, NL, ndests, mx)
    assert (h["used"], h["nzone"], h["tick_no"]) == (8, 2, 5)
    assert list(d["aux"]["kind"]) == [-1, capi.TARGET_ENEMIES, capi.TARGET_ENTITY] and list(d["aux"]["nents"]) == [0, 3, 1]
    assert len(d["fields"]) == 4
    seg = compose(d)
    t = emu.emu_pc_new(ndests, CW * CH, mx)
    try:
        assert load(emu, t, seg) is None
        assert save(emu, t) == seg
        assert counts(emu, t)["nfree"] == 2
    finally:
        emu.emu_pc_delete(t)


def _mut(d, fn):
    e = {k: (v.copy() if hasattr(v, "copy") else v) for k, v in d.items()}
    fn(e)
    return e


def test_each_rule_refuses_with_its_own_message(emu):
    d, ndests, mx = crafted(emu)
    good = compose(d)
    owned = [s for s in range(8) if d["owner"][s] >= 0]
    zone = [s for s in range(8) if d["owner"][s] < 0 and s not in (4, 5)]
    key_of = {int(s): k for k, s in enumerate(d["slot"]) if s >= 0}
    unmapped = [k for k, s in enumerate(d["slot"]) if s < 0]
    flow_built = [s for s in range(mx) if d["has"][s] & 1]
    empty_mapped = [s for s in key_of if d["has"][s] == 0]

    def hdr(field, value):
        return lambda e: e["h"].__setitem__(field, value)

    def setv(name, i, v):
        return lambda e: e[name].__setitem__(i, v)

    def req_layer(e):
        r = e["req"][flow_built[0]].view("<i4")
        r[2] = NL
        e["req"][flow_built[0]] = r.view(np.uint8)

    cases_ = {
        "magic": (hdr("magic", 0x12345678), "magic"),
        "version": (hdr("version", 2), "version"),
        "record size": (hdr("req_size", 60), "record sizes"),
        "header padding": (hdr("_pad1", 1), "padding"),
        "map geometry": (hdr("chunk_w", CW + 1), "map geometry"),
        "layers": (hdr("nlayers", NL + 1), "map geometry"),
        "pool geometry": (hdr("max", mx - 1), "(ndests, max_fields)"),
        "dests": (hdr("ndests", ndests + 1), "(ndests, max_fields)"),
        "counts": (hdr("used", mx + 1), "counts outside"),
        "digest": (hdr("digest", DIGEST ^ 1), "map digest"),
        "slot outside": (setv("slot", unmapped[0], mx), "outside the pool"),
        "mapped above used": (setv("slot", unmapped[0], 9), "at or above used"),
        "slot mapped twice": (setv("slot", unmapped[0], owned[0]), "more than one key"),
        "ff_id unmapped": (setv("ffid", unmapped[0], 7), "ff_id on an unmapped key"),
        "free outside": (lambda e: e.__setitem__("free", np.array([5, 8], np.int32)), "free-list entry outside"),
        "free repeated": (lambda e: e.__setitem__("free", np.array([5, 5, 4], np.int32)), "repeated"),
        "free mapped": (lambda e: e.__setitem__("free", np.array([5, 4, owned[0]], np.int32)), "free-list entry is mapped"),
        "fields above used": (setv("has", 10, 1), "at or above used"),
        "owner above used": (setv("owner", 11, 0), "at or above used"),
        "neither": (lambda e: e.__setitem__("free", np.array([5], np.int32)), "neither free, owned nor zone-held"),
        "wrong owner": (setv("owner", owned[0], key_of[owned[1]]), "not mapped by its owner"),
        "nzone": (hdr("nzone", 1), "nzone"),
        "has bits": (setv("has", flow_built[0], 5), "has byte"),
        "touch": (setv("touch", owned[0], 6), "touch stamp"),
        "device touch": (setv("dtouch", zone[0], 6), "touch stamp"),
        "req layer": (req_layer, "layer that is not created"),
        "aux kind": (lambda e: e["aux"].__setitem__(1, (7, 2, 0, 3)), "bad kind"),
        "entity with two footprints": (lambda e: (e["aux"].__setitem__(2, (capi.TARGET_ENTITY, 0, 1, 2)),
                                                  e["aux"].__setitem__(1, (capi.TARGET_ENEMIES, 2, 0, 2))), "bad kind"),
        "aux layer": (lambda e: e["aux"].__setitem__(1, (capi.TARGET_ENEMIES, NL, 0, 3)), "bad layer"),
        "aux ref layer": (lambda e: e["aux"].__setitem__(1, (capi.TARGET_ENEMIES, 0, 12, 3)), "bad layer"),
        "aux counts": (lambda e: e["aux"].__setitem__(1, (capi.TARGET_ENEMIES, 2, 0, 2)), "do not add up"),
        "aux footprint": (lambda e: e["fp"]["corners"].__setitem__((2, 3), np.nan), "not finite"),
        "more aux than dests": (lambda e: e.__setitem__("aux", np.concatenate([e["aux"], e["aux"][:2]])), "counts outside"),
    }
    if empty_mapped:
        cases_["stored count"] = (setv("has", empty_mapped[0], 2), "stored field count")
    t = emu.emu_pc_new(ndests, CW * CH, mx)
    try:
        assert load(emu, t, good) is None                     # the target holds the crafted pool; refusals keep it
        msgs = {}
        for name, (fn, want) in cases_.items():
            seg = compose(_mut(d, fn), counts_from_arrays=name not in ("counts", "stored count"))
            err = load(emu, t, seg)
            assert err is not None, name
            assert want in err, (name, err)
            msgs[name] = err
        # truncated, padded, shorter than the header
        for seg, want in ((good[:-1], "truncated or padded"), (good + b"\0" * 16, "truncated or padded"),
                          (good[:40], "shorter than its header"), (b"", "shorter than its header")):
            assert want in load(emu, t, seg)
        # the context's own geometry and digest, not only the header's
        assert "map geometry" in load(emu, t, good, geom=(CW, CH, NL + 1))
        assert "map digest" in load(emu, t, good, digest=DIGEST + 1)
        small = emu.emu_pc_new(ndests, CW * CH, mx + 1)
        try:
            assert "(ndests, max_fields)" in load(emu, small, good)
        finally:
            emu.emu_pc_delete(small)
        assert save(emu, t) == good
    finally:
        emu.emu_pc_delete(t)
    # the bookkeeping rules each have their own message
    rules = ["slot outside", "mapped above used", "slot mapped twice", "ff_id unmapped", "free outside", "free repeated",
             "free mapped", "neither", "wrong owner", "nzone", "has bits", "touch", "req layer", "aux kind", "aux layer",
             "aux counts", "aux footprint"]
    assert len({msgs[r] for r in rules}) == len(rules)


def test_digest_matches_restatement(emu):
    rng = np.random.default_rng(11)
    for nl, cw, ch in ((1, 1, 1), (2, 3, 2), (3, 2, 4)):
        n = nl * cw * ch * 4096
        cost = rng.integers(0, 256, n).astype(np.uint8)
        blk = rng.integers(0, 65536, n).astype(np.uint16)
        liid = rng.integers(0, 65536, n).astype(np.uint16)
        fmask = rng.integers(0, 1 << 15, n).astype(np.uint16)
        en = rng.integers(0, 1 << 15, 16).astype(np.uint16)
        mx, mz = float(rng.random() * 100 - 50), float(rng.random() * 100 - 50)
        got = emu.emu_pc_digest(_p(cost), _p(blk), _p(liid), _p(fmask), nl, cw, ch, mx, mz, _p(en))
        assert got == map_digest_np(cost, blk, liid, fmask, cw, ch, np.float32(mx), np.float32(mz), en)
        z = np.zeros(n, np.uint16)
        assert emu.emu_pc_digest(_p(cost), _p(blk), _p(liid), None, nl, cw, ch, mx, mz, _p(en)) == \
            emu.emu_pc_digest(_p(cost), _p(blk), _p(liid), _p(z), nl, cw, ch, mx, mz, _p(en))
        # every input moves it: one tile, the enemy table, the position
        cost2 = cost.copy(); cost2[n // 2] ^= 1
        assert emu.emu_pc_digest(_p(cost2), _p(blk), _p(liid), _p(fmask), nl, cw, ch, mx, mz, _p(en)) != got
        en2 = en.copy(); en2[3] ^= 1
        assert emu.emu_pc_digest(_p(cost), _p(blk), _p(liid), _p(fmask), nl, cw, ch, mx, mz, _p(en2)) != got
        assert emu.emu_pc_digest(_p(cost), _p(blk), _p(liid), _p(fmask), nl, cw, ch, mx + 1, mz, _p(en)) != got


def test_digest_terms_and_order(emu):
    """the per-tile and per-block terms equal the restatement's, and the sums do not depend on their order"""
    rng = np.random.default_rng(5)
    nl, chunks = 2, 6
    cost = rng.integers(0, 256, (nl, chunks, 4096)).astype(np.uint8)
    blk = rng.integers(0, 65536, (nl, chunks, 4096)).astype(np.uint16)
    liid = rng.integers(0, 65536, (nl, chunks, 4096)).astype(np.uint16)
    fm = rng.integers(0, 1 << 15, (nl, chunks, 4096)).astype(np.uint16)
    tt = tile_terms(cost, blk, liid, fm)
    for _ in range(50):
        li, ci, t = int(rng.integers(0, nl)), int(rng.integers(0, chunks)), int(rng.integers(0, 4096))
        assert emu.emu_pc_digest_tile(t, int(cost[li, ci, t]), int(blk[li, ci, t]), int(liid[li, ci, t]), int(fm[li, ci, t])) == \
            int(tt[li, ci, t])
    with np.errstate(over="ignore"):
        bh = tt.sum(axis=-1, dtype=np.uint64)
        bt = block_terms(bh, nl, chunks)
        for li in range(nl):
            for ci in range(chunks):
                assert emu.emu_pc_digest_block(int(bh[li, ci]), li, ci) == int(bt[li * chunks + ci])
        ref = int(bt.sum(dtype=np.uint64))
        for _ in range(5):
            perm = rng.permutation(tt.shape[-1])
            bh2 = np.zeros((nl, chunks), np.uint64)
            for j in np.array_split(perm, 7):                  # tiles in another order, in partial sums
                bh2 += tt[..., j].sum(axis=-1, dtype=np.uint64)
            assert (bh2 == bh).all()
            bt2 = block_terms(bh2, nl, chunks)[rng.permutation(nl * chunks)]
            acc = np.uint64(0)
            for x in bt2:
                acc = acc + x
            assert int(acc) == ref
