#!/usr/bin/env python
"""tools/bench_route_read.py -- readData into the ranks of a routed map: the config #2 map (2 cm,
three 131 072-point scans of up to 30 m) is written by one map, and its node stream is read into
1 (a plain map: the single map's readData), 2 and 4 routed ranks on ONE device; one JSON line per
stream and number of ranks, printed as soon as it is measured.

    python tools/bench_route_read.py [--reps R] [--streams box20m,whole]

* wall_ms: host wall time of each rank's ufo_b200_read_data call (it parses the stream on the host,
  runs the import on the map's stream and ends in a stream synchronisation), into empty ranks,
  median over R repetitions after one warm-up.  Every rank parses the whole stream.
* device_ms: per rank, the device time of one more such call: the summed durations of its kernels
  and copies, traced with torch.profiler in a separate pass (the host parse, which precedes all
  device work, is not in it).
* Both for the whole map and for a 20 m box around the last sensor pose (the mapping server's
  change box).  After the timed reads the ranks' parts are assembled and checked against the
  single map's image.  The card's name, power limit and maximum SM clock are part of the line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CONFIGS, make_scans  # noqa: E402


def card_info():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    return [x.strip() for x in out.strip().split(",")[:3]]


def stats(ms):
    return {"median": float(np.median(ms)), "min": float(np.min(ms)), "max": float(np.max(ms))}


def make_group(capi, cfg, world, bricks):
    maps = [capi.Map(cfg["resolution"], initial_bricks=bricks) for _ in range(world)]
    if world > 1:
        ptrs = [m.route_setup(r, world) for r, m in enumerate(maps)]
        for m in maps:
            m.route_connect(ptrs)
    return maps


def device_ms(torch, call):
    """Summed duration of the device work (kernels, copies, memsets) of one call."""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        call()
        torch.cuda.synchronize()
    us = sum(e.time_range.elapsed_us() for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA)
    return us / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--streams", default="box20m,whole")
    args = ap.parse_args()
    import torch
    from ufomap_b200 import capi
    cfg = CONFIGS[2]
    torch.cuda.init()
    name, limit, clock = card_info()
    origins, packed, layout, _, _ = make_scans(cfg, 3, 0)
    bricks = 1 << 19
    src = capi.Map(cfg["resolution"], initial_bricks=bricks)
    for k in range(3):
        buf = packed[k]
        src.insert_packed(origins[k], buf.ctypes.data, len(buf), layout, max_range=cfg["max_range"])
    src.wait()
    o = origins[-1]
    boxes = {"whole": None, "box20m": (o - 10.0, o + 10.0)}
    streams = [(n, src.write_data(boxes[n]), boxes[n]) for n in args.streams.split(",")]
    src_bricks = src.pool_stats()["bricks"]
    src.close()
    head = {"tool": "bench_route_read", "gpu": name, "power_limit": limit, "max_sm_clock": clock, "reps": args.reps,
            "workload": cfg["workload"], "scans": 3, "source_bricks": src_bricks,
            "box20m": "AABB of half size 10 m around the last sensor pose"}
    for sname, data, box in streams:
        for world in (1, 2, 4):
            # per rank: enough bricks for its share of the map, so that no pool grows in a timed call
            per_rank = max(1 << 14, int(1.25 * src_bricks / world))
            wall = [[] for _ in range(world)]
            for rep in range(args.reps + 1):  # the first repetition warms up
                maps = make_group(capi, cfg, world, per_rank)
                for r, m in enumerate(maps):
                    t0 = time.perf_counter()
                    m.read_data(data, box=box)
                    t = 1e3 * (time.perf_counter() - t0)
                    if rep:
                        wall[r].append(t)
                if rep < args.reps:
                    for m in maps:
                        m.close()
            image = capi.assemble_image([m.image_part() for m in maps])
            if world == 1:
                single_image = image
            assert image == single_image, "%s: the union of %d ranks differs from the single map" % (sname, world)
            bricks_held = [m.pool_stats()["bricks"] for m in maps]
            for m in maps:
                m.close()
            maps = make_group(capi, cfg, world, per_rank)
            dev = [device_ms(torch, lambda: m.read_data(data, box=box)) for m in maps]
            for m in maps:
                m.close()
            print(json.dumps(dict(head, stream=sname, stream_bytes=len(data), ranks=world,
                                  wall_ms=[stats(w) for w in wall], device_ms=dev, bricks=bricks_held)), flush=True)


if __name__ == "__main__":
    main()
