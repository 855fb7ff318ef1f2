#!/usr/bin/env python
"""tools/bench_clone.py -- device copies (ufo_b200_clone) and the tree counters / known box
(ufo_b200_tree_info) on the config #2 map after three scans; one JSON line per case.

    python tools/bench_clone.py [--steps K] [--warmup W]

* clone:      Map.clone() against what the reference's copy constructor does, write() of the file
              image plus read() of it into a new map (map creation not timed).
* tree_info:  Map.tree_info() against iterate() of every occupied and free leaf, which is how the
              reference gets its known box (occupancy_map_base.h:828-852).
* times:      wall_ms on the host clock (every call returns with its work finished); device_ms the sum
              of the call's CUDA kernel, memcpy and memset activity from torch.profiler, a profile of its
              own per step, and cuda_records the number of activity records it saw; k_brick_info_ms the
              CUDA-event time ufo_b200_tree_info reports for its brick pass.  Medians over the steps.
              The card's name and power limit are on every line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import CONFIGS, make_scans  # noqa: E402
from bench_writes import card_info  # noqa: E402


def timed(call, steps, warmup, after=None):
    """Medians of (wall ms, device ms) of call(); after(result) runs outside the timed window."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    for _ in range(warmup):
        r = call()
        if after:
            after(r)
    walls, devs, seen = [], [], []
    for _ in range(steps):
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            t0 = time.perf_counter()
            r = call()
            walls.append(1e3 * (time.perf_counter() - t0))
            torch.cuda.synchronize()
        cuda = [e for e in prof.events() if e.device_type.name == "CUDA"]
        devs.append(sum(e.time_range.elapsed_us() for e in cuda) / 1e3)
        seen.append(len(cuda))
        if after:
            after(r)
    return dict(wall_ms=float(np.median(walls)), device_ms=float(np.median(devs)), cuda_records=int(np.median(seen)))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=7)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    from ufomap_b200 import capi
    cfg = CONFIGS[2]
    n_scans = 3
    origins, _, _, xyzs, _ = make_scans(cfg, n_scans, 0)
    m = capi.Map(cfg["resolution"], initial_bricks=cfg["bricks"], device=0)
    for k in range(n_scans):
        m.insert(origins[k], xyzs[k], max_range=cfg["max_range"])
    m.wait()
    pools = m.pool_stats()
    name, limit = card_info()
    common = {"tool": "bench_clone", "config": 2, "bricks": int(pools["bricks"]), "device_bytes": int(pools["device_bytes"]),
              "steps": args.steps, "warmup": args.warmup, "gpu": name, "power_limit": limit,
              "map": "%s; %d scans inserted" % (cfg["workload"], n_scans)}

    t = timed(m.clone, args.steps, args.warmup, after=lambda c: c.close())
    print(json.dumps({**common, "case": "clone", **t}), flush=True)

    twins = []

    def write_read():
        t = twins.pop()
        t.read(m.write())
        return t

    def fresh():
        twins.append(capi.Map(cfg["resolution"], initial_bricks=cfg["bricks"], device=0))

    fresh()
    t = timed(write_read, args.steps, args.warmup, after=lambda t: (t.close(), fresh()))
    print(json.dumps({**common, "case": "write + read", "image_bytes": len(m.write()), **t}), flush=True)

    info = m.tree_info()
    t = timed(m.tree_info, args.steps, args.warmup)
    kernel = float(np.median([m.tree_info()["ms_device"] for _ in range(args.steps)]))
    print(json.dumps({**common, "case": "tree_info", "k_brick_info_ms": kernel, **t,
                      "num_leaf_nodes": info["num_leaf_nodes"], "num_inner_nodes": info["num_inner_nodes"]}), flush=True)
    n_leaves = len(m.iterate(occupied=True, free=True, unknown=False)[0])
    t = timed(lambda: m.iterate(occupied=True, free=True, unknown=False), args.steps, args.warmup)
    print(json.dumps({**common, "case": "iterate(leaves, occupied, free)", "records": n_leaves, **t}), flush=True)
    m.close()


if __name__ == "__main__":
    main()
