"""The state digests of pfnav_state_digest on the CPU (csrc/pfnav_digest_host.h through tests/emu/digest_emu.cpp): the
functions of checkpoint and pool segments that the device's values must equal.

- The header's population, block, flock and record digests of checkpoint segments equal a numpy restatement, for every
  combination of optional tables; so does its pool digest of pool segments built with the real slot policies.
- Segments saved by 1..8 members sum to the one-member population digest, block array and record digest, and carry the
  same flock digest.
- Flipping any single byte of a row changes the population value and exactly one block, the block of that uid; the
  record digest changes exactly when the byte feeds the neighbour record.
- The pool digest ignores the header's map digest word and changes with any byte of the bookkeeping, the device touch
  stamps or the stored fields."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from test_checkpoint_emu import BLK, EXT, FORM, MS, population, ranges
from test_pool_checkpoint_emu import CH, CW, NL, build, layout, parse, splitmix64

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
U = np.uint64
K = U(0xD6E8FEB86659FD93)
MIX = U(0xA0761D6478BD642F)
SEED_ROW, SEED_REC, SEED_FLOCK = U(0x8EBC6AF09C88C6E3), U(0x589965CC75374CC3), U(0x1D8E4E27C47D124F)
SEED_POOL, SEED_FIELD, SEED_TOUCH = U(0xE7037ED1A0B428DB), U(0x2D358DCCAA6C78A5), U(0x8BB84B93962EACC9)
ALL = MS | EXT | FORM | BLK
TABLE_SETS = [0, MS, EXT, FORM, BLK, MS | EXT, MS | BLK, EXT | FORM, MS | EXT | FORM, ALL]
RECORD_BYTES = set(range(0, 8)) | set(range(16, 24)) | set(range(32, 36)) | {44} | set(range(48, 51))   # pos, velocity,
# radius, the state's low byte (state << 24) and the flags' low 24 bits


def _so(tmp_path_factory, src, name):
    so = str(tmp_path_factory.mktemp("emu") / name)
    subprocess.run(["g++", "-std=c++17", "-O2", "-D_GLIBCXX_ASSERTIONS", "-fPIC", "-shared", "-pthread",
                    os.path.join(HERE, "emu", src), "-o", so], check=True)
    return C.CDLL(so)


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    p, sz = C.c_void_p, C.c_size_t
    D = _so(tmp_path_factory, "digest_emu.cpp", "libdigest_emu.so")
    D.emu_dg_nblocks.restype = sz
    D.emu_dg_nblocks.argtypes = [sz, C.c_int]
    D.emu_dg_agents.argtypes = [p, sz, C.c_int, p, p, C.c_char_p]
    D.emu_dg_pool.argtypes = [p, sz, p, C.c_char_p]
    D.emu_dg_splitmix64.restype = C.c_uint64
    D.emu_dg_splitmix64.argtypes = [C.c_uint64]
    K_ = _so(tmp_path_factory, "checkpoint_emu.cpp", "libcheckpoint_emu.so")
    K_.emu_ckpt_size.restype = sz
    K_.emu_ckpt_size.argtypes = [C.c_uint32, sz, sz]
    K_.emu_ckpt_save.restype = sz
    K_.emu_ckpt_save.argtypes = [C.c_uint32, sz, sz, sz, C.c_int, p, sz, p, p, p, p, p, C.c_int, p]
    P = _so(tmp_path_factory, "pool_checkpoint_emu.cpp", "libpool_checkpoint_emu.so")
    P.emu_pc_new.restype = p
    P.emu_pc_new.argtypes = [C.c_int, C.c_int, C.c_int]
    P.emu_pc_delete.argtypes = [p]
    P.emu_pc_set_tick.argtypes = [p, C.c_uint32]
    P.emu_pc_reserve.argtypes = [p, p, C.c_int, p]
    P.emu_pc_zone_take.argtypes = [p, C.c_uint64]
    P.emu_pc_built.argtypes = [p, C.c_uint64, C.c_int, C.c_int, C.c_uint64, p]
    P.emu_pc_drop.argtypes = [p, C.c_uint64]
    P.emu_pc_reset.argtypes = [p]
    P.emu_pc_set_aux.argtypes = [p, C.c_int, C.c_int, C.c_int, C.c_int, p, C.c_int]
    P.emu_pc_size.restype = sz
    P.emu_pc_size.argtypes = [p]
    P.emu_pc_save.restype = sz
    P.emu_pc_save.argtypes = [p, C.c_int, C.c_int, C.c_int, C.c_uint64, p]
    return D, K_, P


def _p(a):
    return None if a is None else a.ctypes.data_as(C.c_void_p)


def ckpt_save(K_, T, tables, lo, hi, hz=20):
    n = len(T["agents"])
    out = np.zeros(K_.emu_ckpt_size(tables, len(T["flocks"]), hi - lo), np.uint8)
    K_.emu_ckpt_save(tables, n, lo, hi, hz, _p(T["flocks"]), len(T["flocks"]), _p(T["agents"]), _p(T.get("ms")),
                     _p(T.get("ext")), _p(T.get("form")), _p(T.get("blk")), 2, _p(out))
    return out.tobytes()


# ---------------------------------------------------------------------------------------------------------------------
# the header's functions, called
# ---------------------------------------------------------------------------------------------------------------------
def agents_digest(D, seg, k, n_total=None):
    """-> (population, flocks, records, blocks or None) of one checkpoint segment"""
    b = np.frombuffer(seg, np.uint8)
    n_total = int(np.frombuffer(seg[32:40], np.uint64)[0]) if n_total is None else n_total
    blocks = np.zeros(max(D.emu_dg_nblocks(n_total, k), 1), np.uint64)
    out = np.zeros(3, np.uint64)
    err = C.create_string_buffer(256)
    rc = D.emu_dg_agents(_p(b), len(b), k, _p(blocks), _p(out), err)
    assert rc == 0, err.value
    return int(out[0]), int(out[1]), int(out[2]), blocks[:D.emu_dg_nblocks(n_total, k)]


def pool_digest(D, seg):
    b = np.frombuffer(seg, np.uint8)
    out = np.zeros(1, np.uint64)
    err = C.create_string_buffer(256)
    rc = D.emu_dg_pool(_p(b), len(b), _p(out), err)
    assert rc == 0, err.value
    return int(out[0])


# ---------------------------------------------------------------------------------------------------------------------
# the definitions, restated in numpy
# ---------------------------------------------------------------------------------------------------------------------
def chain(h, words):
    """h uint64[n], words uint64[n, m]: h = splitmix64(h ^ w) for each column in order"""
    for j in range(words.shape[1]):
        h = splitmix64(h ^ words[:, j])
    return h


def row_words(tables):
    return 4 + (11 if tables & MS else 0) + (4 if tables & EXT else 0) + (4 if tables & FORM else 0) + (2 if tables & BLK else 0)


def agents_np(seg, k):
    h = np.frombuffer(seg[:64], np.uint32)
    tables, nflocks = int(h[7]), int(h[15])
    n_total, lo, hi = (int(v) for v in np.frombuffer(seg[32:56], np.uint64))
    fl = np.frombuffer(seg[64:64 + 16 * nflocks], np.uint64).reshape(1, -1)
    flocks = int(chain(splitmix64(np.array([nflocks], U) ^ SEED_FLOCK), fl)[0])
    W = row_words(tables)
    rows = np.frombuffer(seg[64 + 16 * nflocks:], np.uint64).reshape(hi - lo, 2 * W)
    uids = np.arange(lo, hi, dtype=np.uint64)
    with np.errstate(over="ignore"):
        hr = chain(splitmix64(uids * K ^ U(tables) ^ SEED_ROW), rows)
        a = np.frombuffer(seg[64 + 16 * nflocks:], np.uint8).reshape(hi - lo, 16 * W)[:, :64].copy().view(np.uint32)
        sf = ((a[:, 11] << np.uint32(24)) | (a[:, 12] & np.uint32(0xFFFFFF))).astype(np.uint64)
        w = np.stack([rows[:, 0], rows[:, 2], a[:, 8].astype(np.uint64) | sf << U(32)], axis=1)
        hrec = chain(splitmix64(uids * K ^ SEED_REC), w)
        blocks = np.zeros((n_total + (1 << k) - 1) >> k, np.uint64)
        for b in np.unique(uids >> U(k)):
            blocks[int(b)] = hr[(uids >> U(k)) == b].sum(dtype=np.uint64)
        return int(hr.sum(dtype=np.uint64)), flocks, int(hrec.sum(dtype=np.uint64)), blocks


def pool_np(seg):
    d = parse(seg)
    h = d["h"]
    mx, nkeys = int(h["max"]), len(d["slot"])
    L = layout(nkeys, mx, int(h["nfree"]), int(h["naux"]), int(h["nfp"]), int(h["nstored"]))
    head = np.frombuffer(seg[:L["dtouch"]], np.uint64).copy()
    head[7] = 0                                                     # the map digest word
    hc = splitmix64(np.array([L["dtouch"]], U) ^ SEED_POOL)
    hc = chain(hc, head.reshape(1, -1))
    s = np.arange(mx, dtype=np.uint64)
    with np.errstate(over="ignore"):
        dev = splitmix64((s << U(32) | d["dtouch"].astype(U)) ^ SEED_TOUCH).sum(dtype=np.uint64)
        stored = np.nonzero(d["has"])[0].astype(np.uint64)
        if len(stored):
            f = d["fields"].view(np.uint64).reshape(len(stored), 512, 2)
            wk = splitmix64(np.arange(512, dtype=np.uint64) * K ^ SEED_FIELD)
            t = splitmix64(splitmix64(wk[None, :] ^ f[:, :, 0]) ^ f[:, :, 1]).sum(axis=1, dtype=np.uint64)
            dev += splitmix64(t ^ stored * MIX ^ SEED_POOL).sum(dtype=np.uint64)
        return int(splitmix64(hc ^ dev)[0])


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tables", TABLE_SETS)
def test_agents_digest_restated(libs, tables):
    D, K_, _ = libs
    assert [D.emu_dg_splitmix64(x) for x in (0, 1, 2 ** 63)] == [int(v) for v in splitmix64(np.array([0, 1, 2 ** 63], U))]
    rng = np.random.default_rng(tables + 11)
    for n in (0, 1, 5, 257):
        T = population(rng, n, 3, tables)
        for lo, hi in ((0, n), (n // 3, n)):
            seg = ckpt_save(K_, T, tables, lo, hi)
            for k in (6, 8):
                got = agents_digest(D, seg, k)
                want = agents_np(seg, k)
                assert got[:3] == want[:3], (n, lo, hi, k)
                assert (got[3] == want[3]).all()


@pytest.mark.parametrize("tables", [0, MS | BLK, ALL])
def test_members_sum_to_one_context(libs, tables):
    D, K_, _ = libs
    rng = np.random.default_rng(tables + 3)
    for n in (0, 3, 200, 1000):
        T = population(rng, n, 5, tables)
        one = agents_digest(D, ckpt_save(K_, T, tables, 0, n), 6)
        for world in range(1, 9):
            lo = ranges(n, world)
            parts = [agents_digest(D, ckpt_save(K_, T, tables, lo[r], lo[r + 1]), 6, n) for r in range(world)]
            with np.errstate(over="ignore"):
                assert sum(p[0] for p in parts) % 2 ** 64 == one[0], (n, world)
                assert sum(p[2] for p in parts) % 2 ** 64 == one[2], (n, world)
                assert (np.sum([p[3] for p in parts], axis=0, dtype=np.uint64) == one[3]).all(), (n, world)
            assert all(p[1] == one[1] for p in parts)
            for r, p in enumerate(parts):                             # zero outside the member's range
                nz = np.nonzero(p[3])[0]
                assert all((lo[r] >> 6) <= b <= ((lo[r + 1] - 1) >> 6) for b in nz)


def test_single_byte_flips(libs):
    D, K_, _ = libs
    rng = np.random.default_rng(77)
    n, k = 300, 6
    T = population(rng, n, 4, ALL)
    seg = ckpt_save(K_, T, ALL, 0, n)
    pop, flocks, records, blocks = agents_digest(D, seg, k)
    row = 16 * row_words(ALL)
    start = 64 + 16 * 4
    uids = [0, 63, 64, 150, n - 1] + list(rng.integers(0, n, 5))
    for u in uids:
        offs = range(row) if u in (0, 64, n - 1) else rng.integers(0, row, 60)
        for o in offs:
            b = bytearray(seg)
            b[start + u * row + int(o)] ^= 1 << int(rng.integers(0, 8))
            p2, f2, r2, bl2 = agents_digest(D, bytes(b), k)
            assert p2 != pop, (u, o)
            assert list(np.nonzero(bl2 != blocks)[0]) == [u >> k], (u, o)
            assert f2 == flocks
            assert (r2 != records) == (int(o) in RECORD_BYTES), (u, o)
    b = bytearray(seg)
    b[64 + 5] ^= 0x10                                                 # a flock's target
    p2, f2, r2, bl2 = agents_digest(D, bytes(b), k)
    assert f2 != flocks and p2 == pop and r2 == records


def test_refused_segments(libs):
    D, K_, _ = libs
    T = population(np.random.default_rng(1), 10, 2, MS)
    seg = ckpt_save(K_, T, MS, 0, 10)
    err = C.create_string_buffer(256)
    out = np.zeros(3, np.uint64)
    for bad, k in ((seg[:-1], 6), (seg + b"\0" * 16, 6), (b"\1" + seg[1:], 6), (seg[:40], 6), (seg, 5), (seg, 21)):
        buf = np.frombuffer(bad, np.uint8)
        assert D.emu_dg_agents(_p(buf), len(buf), k, None, _p(out), err) == 1 and err.value
        assert not out.any()


@pytest.mark.parametrize("seed", range(6))
def test_pool_digest_restated(libs, seed):
    D, _, P = libs
    rng = np.random.default_rng(seed)
    h = build(P, rng, int(rng.integers(2, 6)), int(rng.integers(4, 24)), 60)
    try:
        out = np.zeros(P.emu_pc_size(h), np.uint8)
        P.emu_pc_save(h, CW, CH, NL, 0x0123456789ABCDEF, _p(out))
        seg = out.tobytes()
    finally:
        P.emu_pc_delete(h)
    got = pool_digest(D, seg)
    assert got == pool_np(seg)
    d = parse(seg)
    L = layout(len(d["slot"]), int(d["h"]["max"]), len(d["free"]), len(d["aux"]), len(d["fp"]), len(d["fields"]))
    b = bytearray(seg); b[56:64] = bytes(8)                           # the map digest word is not hashed
    assert pool_digest(D, bytes(b)) == got
    held = np.nonzero(d["has"])[0]
    for o in [24, 32, L["slot"], L["req"] + 3] + ([L["has"] + int(held[0])] if len(held) else []) + [
            L["touch"], L["owner"], L["dtouch"], L["dtouch"] + 4 * (int(d["h"]["max"]) - 1)] + \
            ([L["fields"], L["fields"] + 4096, len(seg) - 1] if len(d["fields"]) else []):
        b = bytearray(seg); b[o] ^= 0x20
        assert pool_digest(D, bytes(b)) != got, o
