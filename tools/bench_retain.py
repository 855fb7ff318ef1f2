#!/usr/bin/env python
"""tools/bench_retain.py -- page_out, retain and page_in on the BASELINE config #2 map; one JSON line.

    python tools/bench_retain.py [--scans S] [--keep F]

* map:    config #2 (OccupancyMap 2 cm, max_range 30 m) after S scans along bench.py's sensor path.
* volume: a box around the last sensor position whose half width along x is chosen by bisection on
          the brick centres so that it keeps about the fraction F of the bricks.
* times:  wall_ms is the host clock around each call (every call ends with the stream idle);
          ms_classify / ms_compact / ms_upper are the CUDA-event times of ufo_b200_retain_stats.
* bytes:  the compaction gather reads and writes the surviving bricks' arrays once: 2 x kept bricks x
          bytes per brick of the compacted arrays (leaves, masks, meta, pair maxima, keys, stamps,
          depth-3 / 4 aggregates), over ms_compact -- which also holds the allocation and release of
          each array, so it is a rate of the whole step, not of the kernel alone.  The card's name and
          power limit are part of the line.

Needs a GPU: it fails without one.
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

# bytes per brick the compaction moves on a mono map without change detection / alias arrays: leaf,
# miss + hit masks, meta, pair maxima, key, two stamps, depth-3 and depth-4 aggregates
MOVED_PER_BRICK = 64 * 64 * 4 + 2 * 64 * 8 + 64 * 4 + 64 * 16 + 8 + 4 + 4 + 8 * 8 + 8


def timed(call):
    t0 = time.perf_counter()
    out = call()
    return out, (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scans", type=int, default=3)
    ap.add_argument("--keep", type=float, default=0.5)
    args = ap.parse_args()
    from ufomap_b200 import capi
    from ufomap_b200.capi import Map

    cfg = CONFIGS[2]
    origins, packed, layout, _, _ = make_scans(cfg, args.scans, 0)
    m = Map(cfg["resolution"], initial_bricks=cfg["bricks"])
    for k in range(args.scans):
        m.insert_packed(origins[k], packed[k].ctypes.data, len(packed[k]), layout, max_range=cfg["max_range"])
    m.wait()
    pools = m.pool_stats()

    # brick centres from a page of the whole map (a volume that keeps nothing), then the box
    everything = m.page_out([capi.sphere([1e6, 1e6, 1e6], 1.0)])
    bx = capi.page_keys(everything)[:, 0].astype(np.float64)
    del everything
    centre_x = (bx - (1 << 11) + 0.5) * 16 * cfg["resolution"]
    o = origins[-1]
    half_x = float(np.quantile(np.abs(centre_x - o[0]), args.keep))
    box = (o - np.array([half_x, 1e3, 1e3]), o + np.array([half_x, 1e3, 1e3]))

    blob, ms_out = timed(lambda: m.page_out(box=box))
    st, ms_retain = timed(lambda: m.retain(box=box))
    after = m.pool_stats()
    back, ms_in = timed(lambda: m.page_in(blob))
    name, limit = card_info()
    moved = 2 * st["bricks_kept"] * MOVED_PER_BRICK
    print(json.dumps({
        "tool": "bench_retain", "gpu": name, "power_limit": limit, "workload": cfg["workload"], "scans": args.scans,
        "bricks": pools["bricks"], "brick_cap": pools["brick_cap"], "device_bytes": pools["device_bytes"],
        "kept": st["bricks_kept"], "removed": st["bricks_removed"], "brick_cap_after": after["brick_cap"],
        "device_bytes_after": after["device_bytes"], "blob_bytes": int(len(blob)),
        "page_out_wall_ms": round(ms_out, 2), "page_out_GBps": round(len(blob) / ms_out / 1e6, 2),
        "retain_wall_ms": round(ms_retain, 2), "retain_ms_classify": round(st["ms_classify"], 3),
        "retain_ms_compact": round(st["ms_compact"], 3), "retain_ms_upper": round(st["ms_upper"], 3),
        "compact_moved_bytes": moved, "compact_GBps": round(moved / max(st["ms_compact"], 1e-6) / 1e6, 2),
        "page_in_wall_ms": round(ms_in, 2), "page_in_GBps": round(len(blob) / ms_in / 1e6, 2),
        "page_in_ms_create": round(back["ms_classify"], 3), "page_in_ms_scatter": round(back["ms_compact"], 3),
        "page_in_ms_derive": round(back["ms_upper"], 3), "bricks_after_page_in": back["bricks_kept"],
    }))
    assert back["bricks_kept"] == st["bricks_kept"] + capi.page_info(blob)["n_bricks"]
    m.close()


if __name__ == "__main__":
    main()
