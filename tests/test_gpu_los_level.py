"""The level-parallel LOS kernel (k_los_level, LOS variant 2, the default) against the byte-state replay (k_los_b,
variant 1) on the device: byte for byte on the golden LOS batches and on the C2 cold goal batch read back through
pfnav_pool_get; the C2 cold batch digest with variant 2; and the replayed-field count of the trace against the CPU run of
the same kernel source (tests/emu/los_emu.cpp) on the same batch."""
import hashlib
import importlib
import os
import sys

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import cases  # noqa: E402
import test_gpu_cold_request as cold  # noqa: E402
import test_los_level_emu as lemu  # noqa: E402

pytestmark = pytest.mark.gpu
capi = cases.capi
GOLD = os.path.join(ROOT, "tests", "golden")


def _both_variants(nav, run):
    out = {}
    for v in (1, 2):
        nav.set_los_variant(v)
        out[v] = run()
    nav.set_los_variant(2)
    return out[1], out[2]


def test_level_vs_replay_golden_batches(pf):
    g = np.load(os.path.join(GOLD, "portal_los.npz"))
    nav = pf.capi.Nav(0)
    try:
        nav.map_create(3, 3, 1); nav.map_upload_layer(0, g["cost"])
        reqs = g["los_reqs"].view(capi.LOS_REQ)
        a, b = _both_variants(nav, lambda: nav.los_fields_create(reqs))
        assert (a == b).all() and (b == g["los_exp"]).all()
    finally:
        nav.close()
    g = np.load(os.path.join(GOLD, "faction.npz"))
    nav = pf.capi.Nav(0)
    try:
        nav.map_create(2, 2, 1)
        for f in range(15):
            nav.set_enemy_factions(f, int(g["enemies"][f]))
        nav.map_upload_layer(0, g["cost"], g["blk"], g["liid"])
        nav.map_upload_factions(0, g["factions"])
        reqs = g["lreq"].view(capi.LOS_REQ)
        a, b = _both_variants(nav, lambda: nav.los_fields_create(reqs))
        assert (a == b).all() and (b == g["lexp"]).all()
    finally:
        nav.close()


def test_level_vs_replay_c2_cold_pool():
    pf = importlib.import_module("permafrost-engine_b200")
    nav, W, dests, targets = cold._setup(pf, agents=False)
    try:
        def run():
            nav.pool_clear()
            counts = nav.pool_request_goals(dests, targets, 0)
            return counts, cold._pool_bytes(nav, len(dests), nav.cw * nav.cw)
        a, b = _both_variants(nav, run)
        assert a[0] == b[0]
        assert a[1] == b[1]
        assert sum(1 for e in b[1] if e[0] & 2) > 0
    finally:
        nav.close()


def test_c2_cold_batch_digest_with_level_kernel():
    pf = importlib.import_module("permafrost-engine_b200")
    nav, W, dests, targets = cold._setup(pf, agents=False)
    try:
        nav.set_los_variant(2)
        nav.pool_clear()
        nf, nl = nav.pool_request_goals(dests, targets, 0)
        h = hashlib.sha256(np.array([nf, nl], np.int64).tobytes())
        for has, ffid, f, l in cold._pool_bytes(nav, len(dests), nav.cw * nav.cw):
            h.update(np.array([has, ffid], np.uint64).tobytes()); h.update(f); h.update(l)
    finally:
        nav.close()
    with open(cold.GOLDEN) as fh:
        assert h.hexdigest() == fh.read().split()[0]


def test_replayed_count_matches_emu(pf, tmp_path):
    cw, cost, reqs = lemu.c2_batch()
    L = lemu._build(tmp_path, "level")
    want, etrace = lemu.run_emu(L, cw, cw, cost, reqs)
    nav = pf.capi.Nav(0)
    try:
        nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost)
        nav.los_trace(True)
        got = nav.los_fields_create(reqs)
        tr = nav.los_trace(False, read_cap=len(reqs))
    finally:
        nav.close()
    assert (got == want).all()
    assert len(tr) == len(reqs)
    n_emu = int(lemu.replayed(etrace).sum())
    assert n_emu > 0 and int(lemu.replayed(tr).sum()) == n_emu
