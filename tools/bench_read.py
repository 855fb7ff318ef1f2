#!/usr/bin/env python
"""tools/bench_read.py -- what opening a saved map costs: the config #2 map (2 cm, three 131 072-point
scans of up to 30 m) is written once, then read into empty maps; one JSON line per input.

    python tools/bench_read.py [--reps R] [--root DIR]

Inputs: the whole map's node stream and the 20 m change box's (around the last sensor pose) through
read_data (Octree::readData), and the whole map's file image through read (Octree::read) where the
library has it.  Per input, medians over R calls into fresh maps after one warm-up:

* wall_ms: host wall time of the call (it ends in a stream synchronisation);
* host_ms: from the call's start to the start of its first device activity -- the host walk of the
  stream, everything the host builds from it and the allocations before the first copy;
* h2d_ms: summed durations of the host-to-device copies;
* device_ms: summed durations of the kernels, memsets and other copies.

The split comes from a torch.profiler trace of each call (CPU and CUDA activities on one clock),
taken in passes separate from the wall-time passes.  --root DIR imports ufomap_b200 from DIR, so
that two builds can be measured in one session.  The card's name, power limit and maximum SM clock
are part of every line.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def card_info():
    out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                          "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
    return [x.strip() for x in out.strip().split(",")[:4]]


def split_ms(torch, call):
    """(host_ms, h2d_ms, device_ms) of one call, from a profiler trace."""
    from torch.profiler import ProfilerActivity, profile, record_function
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        with record_function("read_call"):
            call()
        torch.cuda.synchronize()
    events = prof.events()
    start = min(e.time_range.start for e in events if e.name == "read_call")
    dev = [e for e in events if e.device_type == torch.autograd.DeviceType.CUDA]
    if not dev:
        raise RuntimeError("no device activity in the trace")
    first = min(e.time_range.start for e in dev)
    h2d = sum(e.time_range.elapsed_us() for e in dev if "HtoD" in e.name)
    other = sum(e.time_range.elapsed_us() for e in dev if "HtoD" not in e.name)
    return (first - start) / 1e3, h2d / 1e3, other / 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--root", default=ROOT, help="import ufomap_b200 from this tree")
    args = ap.parse_args()
    sys.path.insert(0, ROOT)
    from bench import CONFIGS, make_scans  # noqa: E402
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    from ufomap_b200 import capi
    assert os.path.dirname(capi.__file__).startswith(os.path.abspath(args.root)), capi.__file__
    cfg = CONFIGS[2]
    torch.cuda.init()
    name, limit, max_clock, clock = card_info()
    origins, packed, layout, _, _ = make_scans(cfg, 3, 0)
    bricks = 1 << 19
    src = capi.Map(cfg["resolution"], initial_bricks=bricks)
    for k in range(3):
        buf = packed[k]
        src.insert_packed(origins[k], buf.ctypes.data, len(buf), layout, max_range=cfg["max_range"])
    src.wait()
    o = origins[-1]
    box = (o - 10.0, o + 10.0)
    whole, box_data = src.write_data(), src.write_data(box)
    inputs = [("whole", "read_data", whole, lambda m: m.read_data(whole)),
              ("box20m", "read_data", box_data, lambda m: m.read_data(box_data, box=box))]
    if hasattr(capi.Map, "read"):
        image = src.write()
        inputs.append(("whole", "read", image, lambda m: m.read(image)))
    src_bricks = src.pool_stats()["bricks"]
    src.close()
    head = {"tool": "bench_read", "root": os.path.abspath(args.root), "gpu": name, "power_limit": limit,
            "max_sm_clock": max_clock, "sm_clock_at_start": clock, "reps": args.reps, "workload": cfg["workload"],
            "scans": 3, "source_bricks": src_bricks}
    fresh = lambda: capi.Map(cfg["resolution"], initial_bricks=int(1.25 * src_bricks))  # noqa: E731
    for sname, how, data, call in inputs:
        wall, splits = [], []
        check = None
        for rep in range(args.reps + 1):  # the first repetition warms up
            m = fresh()
            t0 = time.perf_counter()
            call(m)
            t = 1e3 * (time.perf_counter() - t0)
            if rep:
                wall.append(t)
            elif sname == "whole":
                check = m.write() if how == "read" else m.write_data()
            m.close()
        # (a box's stream need not come back byte for byte: the read map lacks what lies outside)
        assert sname != "whole" or check == data, "%s via %s: the map does not write the input back" % (sname, how)
        for rep in range(args.reps):
            m = fresh()
            splits.append(split_ms(torch, lambda: call(m)))
            m.close()
        s = np.array(splits)
        print(json.dumps(dict(head, stream=sname, call=how, input_bytes=len(data),
                              wall_ms=float(np.median(wall)), host_ms=float(np.median(s[:, 0])),
                              h2d_ms=float(np.median(s[:, 1])), device_ms=float(np.median(s[:, 2])),
                              wall_all_ms=[round(w, 2) for w in wall])), flush=True)


if __name__ == "__main__":
    main()
