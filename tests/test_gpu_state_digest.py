"""pfnav_state_digest / pfnav_state_digest_read / pfnav_group_state_digest: the device-resident game state digested on the
device, checked against the host functions of csrc/pfnav_digest_host.h (tests/emu/digest_emu.cpp) applied to the segments
pfnav_agents_save and pfnav_pool_save write at the same point.

- Equality with the oracle: every combination of optional tables, a population of over 1 M rows (several passes of the
  grid-stride kernels), a cold pool, a pool after ticks of misses with zone and entity fields present, and every tick of
  the headless loop of test_gpu_checkpoint.py.
- Sensitivity: one input delta or command record changes the population value and only its uid's block; a committed
  blocker op changes the map value; one pool request changes the pool value.
- Stream order: a digest queued before an apply on the same stream reads the state before the apply.
- Determinism: twin contexts fed the same inputs, and a game restored from agents + pool segments, give the digests of the
  saved game's own continuation, tick by tick.
- Jobs: groups of 2 and 3 members give the single context's population, block array, flocks, records and map, with empty
  masks; a member whose record column differs shows in the records mask.
- Refusals change nothing."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import cases
from test_gpu_checkpoint import map_ready, population, start_group, start_solo
from test_gpu_mgpu_commands import _devices
from test_gpu_pool_checkpoint import aux_fields, ndests, resumed, with_seekers

capi = cases.capi
HERE = os.path.dirname(os.path.abspath(__file__))
ALL = capi.DIGEST_ALL
AGENT_TABLES = capi.DIGEST_POPULATION | capi.DIGEST_FLOCKS | capi.DIGEST_RECORDS
K = 6


@pytest.fixture(scope="module")
def oracle(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("emu") / "libdigest_emu.so")
    subprocess.run(["g++", "-std=c++17", "-O2", "-fPIC", "-shared", os.path.join(HERE, "emu", "digest_emu.cpp"), "-o", so],
                   check=True)
    D = C.CDLL(so)
    D.emu_dg_nblocks.restype = C.c_size_t
    D.emu_dg_nblocks.argtypes = [C.c_size_t, C.c_int]
    D.emu_dg_agents.argtypes = [C.c_void_p, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, C.c_char_p]
    D.emu_dg_pool.argtypes = [C.c_void_p, C.c_size_t, C.c_void_p, C.c_char_p]
    return D


def agents_oracle(D, segs, k=K):
    """the host functions over the segments of one save -> dict population, flocks, records, blocks"""
    n_total = int(np.frombuffer(segs[0][32:40], np.uint64)[0])
    blocks = np.zeros(max(D.emu_dg_nblocks(n_total, k), 1), np.uint64)
    pop = rec = 0
    flocks = set()
    for s in segs:
        b = np.frombuffer(s, np.uint8)
        out = np.zeros(3, np.uint64)
        err = C.create_string_buffer(256)
        assert D.emu_dg_agents(b.ctypes.data, len(b), k, blocks.ctypes.data, out.ctypes.data, err) == 0, err.value
        pop, rec = (pop + int(out[0])) % 2 ** 64, (rec + int(out[2])) % 2 ** 64
        flocks.add(int(out[1]))
    assert len(flocks) == 1
    return dict(population=pop, flocks=flocks.pop(), records=rec, blocks=blocks[:D.emu_dg_nblocks(n_total, k)])


def pool_oracle(D, seg):
    b = np.frombuffer(seg, np.uint8)
    out = np.zeros(1, np.uint64)
    err = C.create_string_buffer(256)
    assert D.emu_dg_pool(b.ctypes.data, len(b), out.ctypes.data, err) == 0, err.value
    return int(out[0]), int(np.frombuffer(seg[56:64], np.uint64)[0])          # the pool digest, the header's map digest


def digest(nv, what=ALL, k=K):
    nv.state_digest(what, k)
    return nv.state_digest_read()


def check_solo(D, nv, what=ALL):
    """the device's digest against the oracle of the segments saved at the same point"""
    d, blocks = digest(nv, what)
    if what & AGENT_TABLES:
        o = agents_oracle(D, [nv.agents_save()])
        assert int(d["population"]) == o["population"] and int(d["flocks"]) == o["flocks"]
        assert int(d["records"]) == o["records"]
        assert (blocks == o["blocks"]).all() and len(blocks) == int(d["nblocks"])
        with np.errstate(over="ignore"):
            assert int(blocks.sum(dtype=np.uint64)) == int(d["population"])
    if what & (capi.DIGEST_POOL | capi.DIGEST_MAP):
        pool, mp = pool_oracle(D, nv.pool_save())
        if what & capi.DIGEST_POOL:
            assert int(d["pool"]) == pool
        if what & capi.DIGEST_MAP:
            assert int(d["map"]) == mp
    return d, blocks


def values(d, blocks, keys=("population", "flocks", "records", "map", "pool")):
    return tuple(int(d[k]) for k in keys) + (blocks.tobytes(),)


@pytest.mark.gpu
def test_symbols(pf):
    assert {"pfnav_state_digest", "pfnav_state_digest_read", "pfnav_group_state_digest",
            "pfnav_mgpu_state_digest"} <= set(capi.SYMBOLS)


@pytest.mark.gpu
def test_every_table_combination(pf, oracle):
    P = population()
    n = len(P["rec"])
    for tables in range(16):
        X = capi.Nav(0)
        try:
            map_ready(X, P)
            X.agents_upload(P["rec"], P["fl"], 20)
            if tables & 1:
                X.agents_upload_movestate(P["ms"])
            if tables & 2:
                X.agents_upload_movestate_ext(P["ext"])
            if tables & 4:
                X.agents_upload_formation(P["form"])
            if tables & 8:
                X.agents_upload_blocking(P["blk"])
            X.map_commit()
            d, _ = check_solo(oracle, X)                    # the cold pool too
            assert int(d["tables"]) == tables and int(d["n_total"]) == n and (int(d["lo"]), int(d["hi"])) == (0, n)
            assert int(d["nblocks"]) == (n + 63) // 64 and int(d["hz"]) == 20
        finally:
            X.close()


@pytest.mark.gpu
def test_over_a_million_rows(pf, oracle):
    P = population()
    N = 1_100_003
    reps = -(-N // len(P["rec"]))
    X = capi.Nav(0)
    try:
        map_ready(X, P, route=False, buildings=False)
        X.agents_upload(np.tile(P["rec"], reps)[:N], P["fl"], 20)
        X.agents_upload_movestate(np.tile(P["ms"], reps)[:N])
        ext = np.tile(P["ext"], reps)[:N]
        X.agents_upload_movestate_ext(ext)
        X.agents_upload_formation(np.tile(P["form"], reps)[:N])
        X.agents_upload_blocking(np.tile(P["blk"], reps)[:N])
        for k in (6, 20):
            d, blocks = digest(X, AGENT_TABLES, k)
            o = agents_oracle(oracle, [X.agents_save()], k)
            assert (int(d["population"]), int(d["flocks"]), int(d["records"])) == (o["population"], o["flocks"], o["records"])
            assert (blocks == o["blocks"]).all()
    finally:
        X.close()


@pytest.mark.gpu
def test_loop_ticks_equal_the_oracle(pf, oracle):
    P = with_seekers()
    R = start_solo(P)
    X = R.navs[0]
    try:
        check_solo(oracle, X)
        aux_fields(X, P)
        d0, _ = check_solo(oracle, X)
        for t in range(3):
            R.tick()
            d, _ = check_solo(oracle, X)
            assert int(d["pool"]) != int(d0["pool"])
        seg = X.pool_save()
        assert int(np.frombuffer(seg[48:52], np.uint32)[0]) > 0, "no stored field"
        assert int(np.frombuffer(seg[44:48], np.uint32)[0]) > 0, "no entity-field footprints"
    finally:
        R.close()


def delta_of(P, uid):
    d = np.zeros(1, capi.INPUT_DELTA)
    d["uid"] = uid
    d["mask"] = capi.INPUT_ROT
    d["rot"] = [0.0, 0.6, 0.0, 0.8]
    return d


@pytest.mark.gpu
def test_sensitivity(pf, oracle):
    P = population()
    R = start_solo(P)
    X = R.navs[0]
    nd = ndests(P)
    try:
        d0, b0 = digest(X)
        for uid in (0, 77, len(P["rec"]) - 1):
            X.agents_input_deltas(delta_of(P, uid))
            d1, b1 = digest(X)
            assert int(d1["population"]) != int(d0["population"])
            assert list(np.nonzero(b1 != b0)[0]) == [uid >> K]
            assert (int(d1["records"]), int(d1["map"]), int(d1["pool"])) == (int(d0["records"]), int(d0["map"]), int(d0["pool"]))
            check_solo(oracle, X)
            d0, b0 = d1, b1
        c = np.zeros(1, capi.AGENT_DELTA)
        c["uid"] = 5
        c["mask"] = 1 << 4                                   # PFNAV_DELTA_SPEEDS
        c["max_speed"] = P["rec"]["max_speed"][5]
        c["speed"] = float(P["rec"]["speed"][5]) + 1.0
        X.agents_commands(c)
        d1, b1 = digest(X)
        assert int(d1["population"]) != int(d0["population"]) and list(np.nonzero(b1 != b0)[0]) == [0]
        check_solo(oracle, X)
        d0, b0 = d1, b1
        X.blockers_incref(-300.0, 300.0, 5.0, 2)
        d1, _ = digest(X, capi.DIGEST_MAP)
        assert int(d1["map"]) == int(d0["map"]), "a queued op is not committed: the map is unchanged"
        X.map_commit()
        d1, b1 = digest(X)
        assert int(d1["map"]) != int(d0["map"]) and int(d1["population"]) == int(d0["population"])
        check_solo(oracle, X)
        d0 = d1
        X.pool_request_zone(nd - 2, P["rec"]["pos"][0], 5)
        d1, _ = check_solo(oracle, X)
        assert int(d1["pool"]) != int(d0["pool"]) and int(d1["population"]) == int(d0["population"])
    finally:
        R.close()


@pytest.mark.gpu
def test_stream_order(pf):
    """queue, apply on the same stream, read: the state before the apply"""
    P = population()
    R = start_solo(P)
    X = R.navs[0]
    try:
        for _ in range(2):
            nw = len(X.agents_read_work())
            X.agents_tick(capi.TICK_VDES_FROM_POOL); X.pool_repair(); X.agents_tick(capi.TICK_VDES_FROM_POOL)
            X.agents_compute_updates()
            before = values(*digest(X, ALL))
            X.state_digest(ALL, K)
            X.agents_apply_updates_ex(capi.APPLY_BLOCKERS)
            assert values(*X.state_digest_read()) == before
            after = values(*digest(X, ALL))
            assert after[0] != before[0] and nw > 0
            R.commit(); R.settle()
    finally:
        R.close()


def digests_of_ticks(R, n, what=ALL):
    out = []
    for _ in range(n):
        R.tick()
        out.append([values(*digest(nv, what)) for nv in R.navs])
    return out


@pytest.mark.gpu
def test_twins_and_restore(pf):
    P = population()
    A, B = start_solo(P), start_solo(P)
    try:
        a, b = digests_of_ticks(A, 8), digests_of_ticks(B, 8)
        assert a == b
        asegs, psegs = A.save(), [A.navs[0].pool_save()]
        ref = digests_of_ticks(A, 3)
    finally:
        A.close(); B.close()
    C_ = resumed(P, asegs, psegs, 1)
    try:
        assert digests_of_ticks(C_, 3) == ref
    finally:
        C_.close()


def job_values(out, blocks):
    d = out[0]
    return (int(d["population"]), int(d["flocks"]), int(d["records"]), int(d["map"]), blocks.tobytes())


def command_batch(rng, P, m=40):
    """movement commands for m random entities: new velocities and speeds"""
    n = len(P["rec"])
    c = np.zeros(m, capi.AGENT_DELTA)
    c["uid"] = rng.choice(n, m, replace=False)
    c["mask"] = (1 << 4) | (1 << 6)                          # PFNAV_DELTA_SPEEDS | PFNAV_DELTA_VELOCITY
    c["velocity"] = rng.standard_normal((m, 2)).astype(np.float32)
    c["max_speed"] = P["rec"]["max_speed"][c["uid"]]
    c["speed"] = rng.random(m).astype(np.float32) * c["max_speed"]
    return c


@pytest.mark.gpu
@pytest.mark.parametrize("world", [2, 3])
def test_groups_give_the_single_context(pf, oracle, world):
    """8 steps of the same command batches on one context and on a group: the group's job digest is the single
    context's, with empty masks. Then 3 ticks of the headless loop, whose misses each member serves from its own pool:
    the job digest is the oracle's of the members' own segments."""
    P = population()
    what = AGENT_TABLES | capi.DIGEST_MAP
    S = start_solo(P)
    G = start_group(P, world)
    rng = np.random.default_rng(world)
    try:
        for t in range(8):
            d, b = digest(S.navs[0], what)
            out, blocks = G.grp.state_digest(ALL, K)
            assert job_values(out, blocks) == (int(d["population"]), int(d["flocks"]), int(d["records"]), int(d["map"]),
                                               b.tobytes()), ("step", t)
            assert int(out[0]["differ_flocks"]) == int(out[0]["differ_records"]) == int(out[0]["differ_map"]) == 0
            for r, (lo, hi) in enumerate(G.ranges()):
                m = out[1 + r]
                assert (int(m["lo"]), int(m["hi"])) == (lo, hi) and int(m["pool"]) != 0
            c = command_batch(rng, P)
            S.navs[0].agents_commands(c); S.navs[0].agents_rebuild_index()
            G.grp.commands(c); G.grp.gather()
        for t in range(3):
            G.tick()
            out, blocks = G.grp.state_digest(ALL, K)
            o = agents_oracle(oracle, G.save())
            assert (int(out[0]["population"]), int(out[0]["flocks"]), int(out[0]["records"])) == \
                (o["population"], o["flocks"], o["records"]), ("tick", t)
            assert (blocks == o["blocks"]).all()
            assert int(out[0]["differ_flocks"]) == int(out[0]["differ_records"]) == int(out[0]["differ_map"]) == 0
            for r, nv in enumerate(G.navs):
                assert int(out[1 + r]["pool"]) == pool_oracle(oracle, nv.pool_save())[0]
    finally:
        S.close(); G.close()


@pytest.mark.gpu
def test_group_masks_and_empty_members(pf):
    P = population()
    n = len(P["rec"])
    G = start_group(P, 3)
    try:
        out, _ = G.grp.state_digest(ALL, K)
        assert int(out[0]["differ_records"]) == 0
        lo, hi = G.ranges()[1]
        rec = P["rec"][lo:hi].copy()
        rec["pos"][0] += 1.0
        G.navs[1].agents_upload_shard(rec, lo, hi, n, P["fl"], 20)     # no gather: member 1's column differs
        out, _ = G.grp.state_digest(capi.DIGEST_RECORDS, K)
        assert int(out[0]["differ_records"]) == 0b010
    finally:
        G.close()
    # a population smaller than the group: member 2's range is empty, its population and blocks are zero
    small = P["rec"][:2].copy()
    navs = [capi.Nav(d) for d in _devices(3)]
    S = capi.Nav(0)
    try:
        for nv in navs + [S]:
            map_ready(nv, P, buildings=False)
        grp = capi.Group(navs)
        for r, nv in enumerate(navs):
            lo, hi = capi.mgpu_shard_range(2, r, 3)
            nv.agents_upload_shard(small[lo:hi], lo, hi, 2, P["fl"], 20)
        grp.gather()
        S.agents_upload(small, P["fl"], 20)
        out, blocks = grp.state_digest(AGENT_TABLES, K)
        d, b = digest(S, AGENT_TABLES)
        assert int(out[3]["population"]) == 0 and (int(out[3]["lo"]), int(out[3]["hi"])) == (2, 2)
        assert (int(out[0]["population"]), int(out[0]["records"]), blocks.tobytes()) == \
            (int(d["population"]), int(d["records"]), b.tobytes())
        grp.close()
    finally:
        for nv in navs + [S]:
            nv.close()


@pytest.mark.gpu
def test_refusals_change_nothing(pf):
    P = population()
    R = start_solo(P)
    X = R.navs[0]
    L = capi.load()
    try:
        with pytest.raises(capi.PfnavError, match="error -4"):
            X.state_digest_read()                            # nothing queued yet
        before = values(*digest(X))
        for what, k in ((1 << 5, K), (0, K), (capi.DIGEST_POPULATION, 5), (capi.DIGEST_POPULATION, 21)):
            with pytest.raises(capi.PfnavError, match="error -1"):
                X.state_digest(what, k)
        assert values(*X.state_digest_read()) == before      # the previous digest is still the one read
        d = np.zeros(1, capi.DIGEST)
        n = C.c_size_t(0)
        small = np.zeros(1, np.uint64)
        assert L.pfnav_state_digest_read(X.h, d.ctypes.data, small.ctypes.data, 1, C.byref(n)) == capi.ERR_NOMEM
        assert n.value == (len(P["rec"]) + 63) // 64 and d.tobytes() == bytes(capi.DIGEST.itemsize)
        assert values(*digest(X)) == before
    finally:
        R.close()
    Y = capi.Nav(0)
    try:
        Y.map_create(3, 3, 1)
        Y.map_upload_layer(0, P["cost"]); Y.map_build_nav(0)
        for what in (capi.DIGEST_POOL, capi.DIGEST_RECORDS, capi.DIGEST_POPULATION, capi.DIGEST_FLOCKS):
            with pytest.raises(capi.PfnavError, match="error -1"):
                Y.state_digest(what, K)
        Y.state_digest(capi.DIGEST_MAP, K)
        assert int(Y.state_digest_read()[0]["map"]) != 0
    finally:
        Y.close()
    H = capi.Nav(0, hostonly=True)
    try:
        with pytest.raises(capi.PfnavError, match="error -3"):
            H.state_digest(capi.DIGEST_MAP, K)
        with pytest.raises(capi.PfnavError, match="error -3"):
            H.state_digest_read()
    finally:
        H.close()
