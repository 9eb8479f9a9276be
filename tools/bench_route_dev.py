#!/usr/bin/env python
"""AStar_PortalGraphPath throughput on the C2 map (16 x 16 chunks): the device batch (k_portal_graph_path_warp, one warp
per search) against the host planner's routine on host threads, at each given number of searches. Each timing is the
median of 5 calls after one warm-up call; every call ends with its results back on the host.
python tools/bench_route_dev.py [nsearches ...]"""
import importlib
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402


def main():
    sizes = [int(a) for a in sys.argv[1:]] or [64, 1024, 4096]
    pf = importlib.import_module("permafrost-engine_b200")
    capi, synth = pf.capi, pf.synth
    bench.set_workload("C2")
    cw = bench.CHUNKS
    cost = synth.cost_from_pathable(synth.make_map(cw, cw, bench.MAP_SEED), cw, cw)
    nav = capi.Nav(0)
    nav.map_create(cw, cw, 1); nav.map_upload_layer(0, cost); nav.map_build_nav(0)
    t0 = time.perf_counter(); nav.route_build(0); t_build = time.perf_counter() - t0
    ports = nav.portals(0)
    nports = np.bincount(ports[:, 0] * cw + ports[:, 1], minlength=cw * cw)
    rng = np.random.default_rng(7)
    n = max(sizes)
    req = np.zeros((n, 8), np.int32)
    k = 0
    while k < n:
        ec = int(rng.integers(0, cw * cw))
        if nports[ec] == 0:
            continue
        req[k] = [int(rng.integers(0, cw * cw)), int(rng.integers(0, 64)), int(rng.integers(0, 64)), ec,
                  int(rng.integers(0, 64)), int(rng.integers(0, 64)), ec, int(rng.integers(0, nports[ec]))]
        k += 1

    def timed(r, on_device):
        out = nav.route_graph_paths(r, 512, on_device)
        ts = []
        for _ in range(5):
            t0 = time.perf_counter(); out = nav.route_graph_paths(r, 512, on_device); ts.append(time.perf_counter() - t0)
        return statistics.median(ts), out

    print("C2 map %dx%d chunks, %d portals, route_build %.2f s, %d host threads" % (cw, cw, len(ports), t_build, os.cpu_count()))
    for m in sizes:
        r = req[:m]
        t_dev, (st_d, c_d, h_d) = timed(r, True)
        t_host, (st_h, c_h, h_h) = timed(r, False)
        same = bool((st_d == st_h).all() and (c_d.view(np.uint32) == c_h.view(np.uint32)).all() and
                    all(np.array_equal(a, b) for a, b in zip(h_d, h_h)))
        print("%5d searches (%d with a path, longest %d hops): device %.2f ms = %.0f searches/s, host threads %.2f ms = "
              "%.0f searches/s, identical = %s" % (m, int((st_h == 1).sum()), max(len(h) for h in h_h), t_dev * 1e3, m / t_dev,
                                                  t_host * 1e3, m / t_host, same))


if __name__ == "__main__":
    main()
