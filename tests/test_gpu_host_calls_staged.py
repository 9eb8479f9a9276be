"""GPU suite: the host-array calls (flow and LOS fields, region and group-arrival fields, zone and entity fields, the
group-arrival velocities, the neighbour query and the serial pool repair) pass their inputs and outputs through the
context's request staging, the buffers the goal batch's plan lives in. One context makes every call right after a goal
batch, while its LOS work is still forked, first at a small size, then at one that grows the staging buffers, then small
again; a twin context makes the same calls with the forked work joined and the device synchronised before each. The
outputs, the pool after pfnav_fields_join, and the tick and pool repair that follow are equal bit for bit."""
import numpy as np
import pytest
import torch

import cases

pytestmark = pytest.mark.gpu
capi, synth = cases.capi, cases.synth
CW = 8                       # 8 x 8 chunks
NGOALS = 8


def _world(nav, cost, rec, fl):
    nav.map_create(CW, CW, 1)
    nav.map_upload_layer(0, cost)
    nav.map_build_nav(0)
    nav.route_build(0)
    nav.pool_create(NGOALS, NGOALS * CW * CW)
    nav.agents_upload(rec, fl, 20)
    nav.agents_set_work(np.arange(len(rec), dtype=np.uint32))
    nav.agents_tick(0)                                  # builds the position index the neighbour query reads


def _calls(nav, n, goal, plan, pos):
    """every host-array call at size n -> list of output arrays"""
    fr, lr = plan
    rng = np.random.default_rng(n)
    out = []
    flow = nav.flow_fields_update(fr[np.arange(n) % len(fr)])
    upd = fr[np.arange(n) % len(fr)].copy()
    upd["init"] = 0                                     # in place on the fields just built
    out += [flow, nav.flow_fields_update(upd, inout=flow)]
    reps = -(-n // len(lr))
    big = np.concatenate([lr] * reps)
    for k in range(1, reps):                            # each copy of the chain names its own parents
        sl = big[k * len(lr):(k + 1) * len(lr)]
        sl["prev_index"] = np.where(sl["prev_index"] >= 0, sl["prev_index"] + k * len(lr), sl["prev_index"])
    los = nav.los_fields_create(big[:max(n, len(lr))])
    out.append(los)
    child = np.flatnonzero(lr["prev_index"] >= 0)
    if len(child):                                      # a caller-held previous field
        q = lr[child[:1]].copy()
        prev = los[int(q["prev_index"][0])]
        q["prev_index"] = capi.LOS_PREV_INPLACE
        out.append(nav.los_fields_create(np.concatenate([lr, q]), prev_fields={len(lr): prev}))
    H = CW * 64
    centres = rng.integers(48, H - 48, (n, 2))
    reqs = [dict(center=tuple(c), target=tuple(c + rng.integers(-20, 20, 2)), enemies=0) for c in centres]
    created = nav.region_fields(96, reqs)
    out.append(created)
    fix = [dict(q, no_create=True, start=q["center"]) for q in reqs]
    out.append(nav.region_fields(96, fix, inout=created))
    out.append(nav.group_arrival_field(64, pos[:n], pos[0]))
    chunks = np.stack([np.arange(n) // CW % CW, np.arange(n) % CW], 1).astype(np.int32)
    out.append(nav.zone_fields(goal[:2] * 64 + goal[2:], 12, chunks))
    fp = capi.Nav.footprints(pos[:n], 1.5)
    out.append(nav.entity_fields(capi.TARGET_ENEMIES, fp, chunks))
    out.append(nav.entity_fields(capi.TARGET_ENTITY, fp[:1], chunks))
    out += list(nav.group_arrival_velocity(0, pos[0], 8, pos[np.arange(n) % len(pos)]))
    out.append(nav.ents_in_circle(float(pos[0, 0]), float(pos[0, 1]), 40.0, max(n, 16)))
    return out


def test_host_calls_share_the_staging_with_the_goal_batch():
    cost = synth.cost_from_pathable(synth.make_map(CW, CW, 0x5EED0900, rivers=True), CW, CW)
    img = synth.blocked_to_image(cost, CW, CW)
    free = np.argwhere(img != 255)
    rng = np.random.default_rng(0x900)
    tiles = free[rng.integers(0, len(free), NGOALS)]
    goals = np.array([[r // 64, c // 64, r % 64, c % 64] for r, c in tiles], np.int32)
    a = synth.make_agents(cost, CW, CW, 4096, NGOALS, 0x5EED0901, radius=1.5, spacing=2.2)
    a["vdes"] = np.zeros((len(a["radius"]), 2), np.float32)
    rec, fl = capi.pack_agents(a)
    fl["dest"] = np.arange(len(fl)) % NGOALS
    fl["target"] = [(-(c + 0.5) * 4.0, (r + 0.5) * 4.0) for r, c in tiles[np.arange(len(fl)) % NGOALS]]
    pos = rec["pos"].copy()
    navs = [capi.Nav(0), capi.Nav(0)]                  # [0] overlaps the forked LOS work, [1] synchronised steps
    try:
        for nav in navs:
            _world(nav, cost, rec, fl)
        fr, _, fw, lr, _ = navs[0].plan_goal(tuple(goals[0]))
        plan = (fr[fw == 0], lr)
        assert len(lr) > 1
        got = [[], []]
        for n in (1, 1024, 3):
            for k, nav in enumerate(navs):
                nav.pool_request_goals(np.arange(NGOALS, dtype=np.int32), goals)
                if k:
                    nav.fields_join()
                    torch.cuda.synchronize()
                got[k] += _calls(nav, n, goals[0], plan, pos)
        assert len(got[0]) == len(got[1])
        for x, y in zip(*got):
            assert x.dtype == y.dtype and x.shape == y.shape and (x == y).all()
        for nav in navs:
            nav.fields_join()
        pool = [cases.pool_fields(nav, NGOALS, CW * CW) for nav in navs]
        _same_pool(*pool)
        res = []
        for nav in navs:
            nav.agents_tick(capi.TICK_VDES_FROM_POOL)
            res.append(nav.pool_repair())
        assert res[0] == res[1]
        _same_pool(*[cases.pool_fields(nav, NGOALS, CW * CW) for nav in navs])
        for nav in navs:
            nav.agents_tick(capi.TICK_VDES_FROM_POOL)
        n = len(rec)
        assert (navs[0].agents_read_velocities(n) == navs[1].agents_read_velocities(n)).all()
        d = [nav.agents_read_debug(n) for nav in navs]
        assert all((x == y).all() for x, y in zip(*d))
    finally:
        for nav in navs:
            nav.close()


def _same_pool(p, q):
    assert len(p) == len(q)
    for x, y in zip(p, q):
        if isinstance(x, np.ndarray):
            assert (x == y).all()
        else:
            assert x == y
