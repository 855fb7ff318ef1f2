#!/usr/bin/env python
"""tools/bench_iterate.py -- beginLeaves on the device (ufo_b200_iterate) on a BASELINE config map; one
JSON line per case.

    python tools/bench_iterate.py [--config 2|4] [--steps K] [--warmup W]

* map:    config #2 holds one full scan, config #4 two (bench.py's scan streams).
* cases:  beginLeaves() over the whole map at min_depth 0 (occupied + free), and the RViz plugin's
          call -- beginLeaves(AABB, occupied, free, unknown = false, contains = false, min_depth) -- over
          a 20 m box around the sensor at min_depth 0, 1, 2 and 4 (depth 1 values are the max of the
          octet's leaf sector, depth 2 values the max of the block's pair maxima).
* times:  device time of the size pass and of the emit pass (the two k_brick_iter launches of a call)
          and of the call's device-to-host copies, from torch.profiler's CUDA activity records; medians
          over the steps.  wall_ms: the whole call on the host clock.
* bytes:  written = 16 B per brick (size-pass info) + 16 B per record of a reached brick (emit pass);
          read_min = what the size pass cannot avoid reading: every brick's key (8 B) and 64 meta
          words (256 B).  The card's name and power limit are part of each line.
"""
import argparse
import ctypes as C
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


def run_case(m, volume, min_depth, steps, warmup):
    """(records, per-step dicts) for one beginLeaves call shape."""
    import torch
    from torch.profiler import ProfilerActivity, profile

    bv, bp, nb = m._bv(volume)
    args = (1, 1, 1, 0, 0, int(min_depth), bp, nb)
    n = C.c_size_t()
    m._check(m.lib.ufo_b200_iterate(m.h, *args, None, None, None, None, None, 0, C.byref(n)))
    cnt = n.value
    codes = np.empty(max(cnt, 1), np.uint64)
    depths = np.empty(max(cnt, 1), np.uint8)
    occ = np.empty(max(cnt, 1), np.float32)
    flags = np.empty(max(cnt, 1), np.uint8)

    def call():
        m._check(m.lib.ufo_b200_iterate(m.h, *args, codes.ctypes.data, depths.ctypes.data, occ.ctypes.data,
                                        flags.ctypes.data, None, cnt, C.byref(n)))
        assert n.value == cnt

    for _ in range(warmup):
        call()
    walls = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(steps):
            t0 = time.perf_counter()
            call()
            walls.append(1e3 * (time.perf_counter() - t0))
        torch.cuda.synchronize()
    events = sorted((e for e in prof.events() if e.device_type.name == "CUDA"), key=lambda e: e.time_range.start)
    size, emit, d2h = [], [], []
    per_call_d2h = 0.0
    expect_emit = False
    for e in events:
        if "k_brick_iter" in e.name:
            if expect_emit:
                emit.append(e.time_range.elapsed_us() / 1e3)
                expect_emit = False
            else:
                if size:
                    d2h.append(per_call_d2h)
                per_call_d2h = 0.0
                size.append(e.time_range.elapsed_us() / 1e3)
                expect_emit = True
        elif "DtoH" in e.name or "Device -> Host" in e.name:
            per_call_d2h += e.time_range.elapsed_us() / 1e3
    d2h.append(per_call_d2h)
    med = lambda v: float(np.median(v)) if v else None  # noqa: E731
    return cnt, dict(size_ms=med(size), emit_ms=med(emit), d2h_ms=med(d2h), wall_ms=med(walls),
                     launches_seen=len(size))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, default=2, choices=[2, 4])
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    from ufomap_b200 import capi
    cfg = CONFIGS[args.config]
    n_scans = 1 if args.config == 2 else 2
    origins, _, _, xyzs, _ = make_scans(cfg, n_scans, 0)
    m = capi.Map(cfg["resolution"], initial_bricks=cfg["bricks"])
    for k in range(n_scans):
        m.insert(origins[k], xyzs[k], max_range=cfg["max_range"])
    m.wait()
    n_bricks = int(m.stats()["bricks_in_map"])
    name, limit = card_info()
    o = np.asarray(origins[0], np.float64)
    box = [capi.aabb(o - 10.0, o + 10.0)]
    for label, vol, md in (("whole map", [], 0), ("RViz box 20 m", box, 0), ("RViz box 20 m", box, 1),
                          ("RViz box 20 m", box, 2), ("RViz box 20 m", box, 4)):
        cnt, t = run_case(m, vol, md, args.steps, args.warmup)
        line = {"tool": "bench_iterate", "config": args.config, "case": "beginLeaves(%s, occupied, free, min_depth=%d)" % (label, md),
                "records": cnt, "bricks": n_bricks, **t,
                "bytes_written": 16 * n_bricks + 16 * cnt, "record_bytes": 16 * cnt,
                "bytes_read_min": 264 * n_bricks,
                "steps": args.steps, "warmup": args.warmup, "gpu": name, "power_limit": limit,
                "map": "%s; %d scan(s) inserted" % (cfg["workload"], n_scans)}
        print(json.dumps(line), flush=True)
    m.close()


if __name__ == "__main__":
    main()
