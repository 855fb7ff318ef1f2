#!/usr/bin/env python
"""tools/bench_nearest.py -- nearest-first iteration on the device (ufo_b200_nearest) on the config #2
map after three scans; one JSON line per case.

    python tools/bench_nearest.py [--steps K] [--warmup W]

* queries: from the first scan's sensor origin, beginNNLeaves(p, occupied only): the first element
           (want = 1: the planner's nearest-obstacle question) and a 10 000-node sequence (want = 10000).
* cases:   "after scan" -- the first query after a scan, which rebuilds the kept tree shape (the scan is
           not timed); "unchanged" -- repeated queries on the same map; "iterate+sort" -- the baseline a
           caller has without this call: ufo_b200_iterate of the same filter plus a host sort by distance.
* steps:   --steps / --warmup for the unchanged map; 5 timed queries after a scan, one untimed before them.
* times:   wall_ms on the host clock around the call (it ends with the results on the host);
           device_ms = CUDA-event time of the brick kernels and the sort (ufo_b200_last_nearest_stats),
           rebuild_ms = host time of the shape rebuild; medians over the steps.  The card's name and
           power limit are part of each line.
"""
import argparse
import ctypes as C
import json
import math
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import CONFIGS, make_scans  # noqa: E402
from bench_writes import card_info  # noqa: E402

CAP = 1 << 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from ufomap_b200 import capi
    cfg = CONFIGS[2]
    after = 5  # timed first-after-scan queries per want, each after a scan of its own (one untimed before them)
    origins, _, _, xyzs, _ = make_scans(cfg, 3 + 2 * (after + 1), 0)
    m = capi.Map(cfg["resolution"], initial_bricks=cfg["bricks"])
    for k in range(3):
        m.insert(origins[k], xyzs[k], max_range=cfg["max_range"])
    m.wait()
    n_bricks = int(m.stats()["bricks_in_map"])
    name, limit = card_info()
    p = np.ascontiguousarray(origins[0], np.float64)
    codes, depths = np.empty(CAP, np.uint64), np.empty(CAP, np.uint8)
    occ, flags, d2 = np.empty(CAP, np.float32), np.empty(CAP, np.uint8), np.empty(CAP, np.float64)
    n, nxt = C.c_size_t(), C.c_double()
    st = capi.NearestStats()

    def query(want):
        t0 = time.perf_counter()
        m._check(m.lib.ufo_b200_nearest(m.h, p.ctypes.data, None, 0, 1, 1, 0, 0, 0, 0, 0.0, want, codes.ctypes.data,
                                        depths.ctypes.data, occ.ctypes.data, flags.ctypes.data, None, d2.ctypes.data, CAP,
                                        C.byref(n), C.byref(nxt)))
        wall = 1e3 * (time.perf_counter() - t0)
        assert n.value <= CAP
        m._check(m.lib.ufo_b200_last_nearest_stats(m.h, C.byref(st)))
        return wall, st.as_dict(), n.value

    def baseline():
        t0 = time.perf_counter()
        c, d, o, f, _ = m.iterate(leaves=True, occupied=True, free=False)
        hs = np.ldexp(cfg["resolution"], d.astype(np.int64)) / 2.0
        cen = np.zeros((len(c), 3))
        for D in range(16, 0, -1):
            idx = ((c >> np.uint64(3 * (D - 1))) & np.uint64(7)).astype(np.int64)
            step = np.where(((idx[:, None] >> np.arange(3)[None, :]) & 1) == 1, math.ldexp(cfg["resolution"], D - 1) / 2.0,
                            -math.ldexp(cfg["resolution"], D - 1) / 2.0)
            cen = np.where((D > d)[:, None], cen + step, cen)
        s = p[None, :] - np.minimum(np.maximum(p[None, :], cen - hs[:, None]), cen + hs[:, None])
        order = np.argsort((s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2], kind="stable")
        return 1e3 * (time.perf_counter() - t0), len(order)

    med = lambda v: float(np.median(v)) if v else None  # noqa: E731
    common = dict(bricks=n_bricks, steps=args.steps, warmup=args.warmup, gpu=name, power_limit=limit,
                  map="%s; 3 scans inserted" % cfg["workload"])
    scan = 3
    for want in (1, 10000):
        # the first query after a scan: the shape is rebuilt
        walls, dev, reb, nodes, bv = [], [], [], 0, []
        for k in range(after + 1):
            m.insert(origins[scan], xyzs[scan], max_range=cfg["max_range"])
            scan += 1
            m.wait()
            w, s, nodes = query(want)
            assert s["rebuilt"] == 1
            if k >= 1:
                walls.append(w)
                dev.append(s["ms_device"])
                reb.append(s["ms_rebuild"])
                bv.append(s["bricks_visited"])
        print(json.dumps({"tool": "bench_nearest", "case": "after scan", "want": want, "nodes": nodes, "wall_ms": med(walls),
                          "device_ms": med(dev), "rebuild_ms": med(reb), "bricks_visited": med(bv), **common}), flush=True)
        walls, dev, bv, shells = [], [], [], []
        for k in range(args.warmup + args.steps):
            w, s, nodes = query(want)
            assert s["rebuilt"] == 0
            if k >= args.warmup:
                walls.append(w)
                dev.append(s["ms_device"])
                bv.append(s["bricks_visited"])
                shells.append(s["shells"])
        print(json.dumps({"tool": "bench_nearest", "case": "unchanged", "want": want, "nodes": nodes, "wall_ms": med(walls),
                          "device_ms": med(dev), "bricks_visited": med(bv), "shells": med(shells), **common}), flush=True)
    walls = []
    for k in range(args.warmup + min(args.steps, 5)):
        w, cnt = baseline()
        if k >= args.warmup:
            walls.append(w)
    print(json.dumps({"tool": "bench_nearest", "case": "iterate+sort", "nodes": cnt, "wall_ms": med(walls), **common}),
          flush=True)
    m.close()


if __name__ == "__main__":
    main()
