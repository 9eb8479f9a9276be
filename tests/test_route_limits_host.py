"""The host planner on the longest routes a 32 x 32-chunk map can force (cases.serpentine_cost: one gap per chunk-row
boundary, at alternating ends). Every chunk sequence there is forced, so the map is a reference of its own for the host
routine that the device route tests compare with at these lengths (tests/test_gpu_route_limits.py): the portal-graph
search between the map's ends visits the chunks in boustrophedon order with the hop count that order implies, and a
goal plans one flow and one LOS request per chunk, its LOS requests one chain through the whole map. Host-only context:
no GPU."""
import numpy as np
import pytest

import cases

capi = cases.capi
CW = CH = 32


@pytest.fixture(scope="module")
def serpentine():
    cost = cases.serpentine_cost(CW, CH)
    nav = capi.Nav(hostonly=True)
    nav.map_create(CW, CH, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0); nav.route_build(0)
    yield nav, cost
    nav.close()


def _dedup(seq):
    return [int(seq[0])] + [int(b) for a, b in zip(seq, seq[1:]) if b != a]


def test_serpentine_search_is_boustrophedon(serpentine):
    """AStar_PortalGraphPath from the top-left chunk to the bottom-right one: rows 0..30 end to end, then the one chunk
    below the last gap; two hops (exit and entry portal) per chunk crossing"""
    nav, _ = serpentine
    order = cases.serpentine_order(CW, CH)
    last = (CH - 1) * CW + CW - 1
    route = order[:order.index(last) + 1]
    ports = nav.portals(0)
    fin = np.nonzero(ports[:, 0] * CW + ports[:, 1] == last)[0]
    req = np.array([[0, 10, 10, last, 50, 50, last, int(ports[k, 2])] for k in fin], np.int32)
    st, cost, hops = nav.route_graph_paths(req, 4096, on_device=False)
    assert (st == 1).all(), st
    best = int(np.argmin(cost))
    assert _dedup(hops[best][:, 0]) == route
    assert len(hops[best]) == 2 * (len(route) - 1) == 1984
    # consecutive hops alternate: a crossing (the portal's connected portal) and a move inside the chunk
    for k in range(0, len(hops[best]) - 1, 2):
        (c0, p0, _), (c1, p1, _) = hops[best][k], hops[best][k + 1]
        row = ports[(ports[:, 0] * CW + ports[:, 1] == c0) & (ports[:, 2] == p0)][0]
        assert (int(row[7]), int(row[8])) == (int(c1), int(p1)), k


def test_serpentine_request_path_corner_to_corner(serpentine):
    """N_RequestPath across the map: one flow and one LOS request per chunk of the forced route, the LOS requests one
    chain from the target's chunk back to the source's"""
    nav, _ = serpentine
    order = cases.serpentine_order(CW, CH)
    last = (CH - 1) * CW + CW - 1
    route = order[:order.index(last) + 1]
    ok, _, fr, _, fc, lr, lc = nav.route_request_path((-42.0, 42.0), (-(31 * 256 + 202.0), 31 * 256 + 202.0))
    assert ok
    assert sorted(fc.tolist()) == sorted(route) and sorted(lc.tolist()) == sorted(route)
    assert lc.tolist() == route[::-1]
    assert cases.los_depths(lr).max() == len(route) == 993


def test_serpentine_goal_plans_every_chunk(serpentine):
    """N_RequestGoal's plan for a target in the top-left chunk: every chunk one flow and one LOS request, and the LOS
    requests one chain of depth 1024 in the order of the forced route"""
    nav, cost = serpentine
    fr, fc, fw, lr, lc = nav.plan_goal((0, 0, 10, 10))
    assert sorted(fc.tolist()) == list(range(CW * CH)) and sorted(lc.tolist()) == list(range(CW * CH))
    depth = cases.los_depths(lr)
    assert depth.max() == CW * CH
    # walk the chain back from its deepest request: the forced route, reversed
    chain, i = [], int(np.argmax(depth))
    while i >= 0:
        chain.append(int(lc[i])); i = int(lr[i]["prev_index"])
    assert chain[::-1] == cases.serpentine_order(CW, CH)
