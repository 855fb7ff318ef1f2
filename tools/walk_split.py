#!/usr/bin/env python
"""Device time of the two ray-walk kernels, k_split and k_walk_mark, on the bench configurations.

    python tools/walk_split.py [--config 2 3 4] [--scans 12] [--out DIR]

One map per configuration, fed the bench's seeded scans (host buffers, synchronous inserts);
the first three scans are warm-up.  The timed scans run under torch.profiler with CUDA activities,
which gives the device time of every kernel launch by name; ms_rays (CUDA events around the
walk, profiling level 1) is printed next to it.  UFOMAP_B200_LIB selects another build of the
library, so a variant is timed by the same script.  One JSON line per configuration; with --out,
the profiler's key averages are written there as well.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

CONFIGS = {
    2: dict(res=0.02, max_range=30.0, kind="velodyne", bricks=1 << 19),
    3: dict(res=0.002, max_range=5.0, kind="rgbd", bricks=1 << 20),
    4: dict(res=0.05, max_range=100.0, kind="velodyne", bricks=1 << 18),
}
KERNELS = ("k_split", "k_walk_mark", "k_gather_scan", "k_gather", "k_update_brick")


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0] if out else None
    except Exception:
        return None


def kernel_base(name):
    """'void ufo_b200::k_walk_mark<0, false, false, true>(...)' -> 'k_walk_mark'"""
    s = name.split("(")[0].split("<")[0]
    return s.split("::")[-1].split(" ")[-1]


def run(config, n_scans, out_dir):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from ufomap_b200 import capi, scans

    cfg = CONFIGS[config]
    rgbd = cfg["kind"] == "rgbd"
    m = capi.Map(cfg["res"], color=rgbd, initial_bricks=cfg["bricks"])
    m.set_profiling(1)

    def feed(k):
        if rgbd:
            o, p, c = scans.rgbd(k=k)
            m.insert(o, p, rgb=c, max_range=cfg["max_range"], dtype=np.float32, discrete=True)
        else:
            o, p = scans.velodyne64(k=k)
            m.insert(o, p, max_range=cfg["max_range"], dtype=np.float32)
        return m.stats()

    warm = 3
    for k in range(warm):
        feed(k)
    torch.cuda.synchronize()
    rows = []
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for k in range(warm, n_scans):
            rows.append(feed(k))
        torch.cuda.synchronize()
    m.close()
    timed = n_scans - warm
    per_kernel = {}
    for ev in prof.key_averages():
        base = kernel_base(ev.key)
        if base not in KERNELS:
            continue
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        d = per_kernel.setdefault(base, {"ms_per_scan": 0.0, "launches": 0})
        d["ms_per_scan"] += t * 1e-3 / timed
        d["launches"] += ev.count
    if out_dir:
        os.makedirs(out_dir, exist_ok=True)
        with open(os.path.join(out_dir, "walk_split_config%d.txt" % config), "w") as f:
            f.write(prof.key_averages().table(sort_by="cuda_time_total", row_limit=30))
    return {
        "config": config, "lib": os.environ.get("UFOMAP_B200_LIB", "default"), "card": card(),
        "scans_timed": timed, "kernels": per_kernel,
        "ms_rays_events": float(np.median([r["ms_rays"] for r in rows])),
        "ms_total_events": float(np.median([r["ms_total"] for r in rows])),
        "note": "kernel times from torch.profiler (profiled run); ms_*_events: CUDA events, median over the profiled scans",
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, nargs="+", default=[2, 3, 4], choices=sorted(CONFIGS))
    ap.add_argument("--scans", type=int, default=12)
    ap.add_argument("--out", default=None, help="directory for the profiler tables")
    args = ap.parse_args()
    if args.scans < 4:
        ap.error("--scans must be >= 4 (three warm-up scans)")
    import torch
    if not torch.cuda.is_available():
        sys.exit("walk_split.py needs a CUDA device")
    for c in args.config:
        print(json.dumps(run(c, args.scans, args.out)), flush=True)


if __name__ == "__main__":
    main()
