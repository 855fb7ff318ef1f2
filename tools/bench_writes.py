#!/usr/bin/env python
"""tools/bench_writes.py -- ordered per-node writes (ufo_b200_update_nodes) and insertRay batches
(ufo_b200_insert_rays) on a map that holds two scans of a BASELINE config; one JSON line.

    python tools/bench_writes.py --workload writes|rays [--steps K] [--warmup W] [--config 2|4]
                                 [--impl reference]

* writes: per step 1 M depth-0 entries (90 % ADD of a hit / miss / larger log-odds, 10 % SET) at
  uniform voxels of a 30 m cube around the sensor.
* rays:   per step insertRay of every point of one config scan (config #2: 131 072 rays of up to 30 m).
* value:  updates (entries or rays) per second of device time (CUDA events around the whole batch);
  ms_per_batch_wall adds the host side of the call (validation, copies).  The card's name and power
  limit are part of the line.
* --impl reference: the compiled reference on every 16th entry / ray, one host thread (ADD entries
  only: setNodeValue does not compile in the reference).
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

from bench import CONFIGS, make_scans  # noqa: E402


def card_info(index=0):
    """(name, power limit) of the GPU a number was measured on, as nvidia-smi reports them."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        name, limit = [x.strip() for x in out.strip().split(",")[:2]]
        return name, limit
    except Exception:
        return None, None


def write_batches(cfg, total, seed=7, n=1 << 20, half_m=15.0):
    """Per step n depth-0 entries (90 % ADD, 10 % SET) at uniform voxels of a cube of half edge
    half_m around the map centre: (codes, ops, values)."""
    rng = np.random.default_rng(seed)
    half = int(half_m / cfg["resolution"])
    out = []
    for _ in range(total):
        k = (32768 + rng.integers(-half, half, size=(n, 3))).astype(np.uint64)
        codes = np.zeros(n, np.uint64)
        for b in range(16):
            for a in range(3):
                codes |= ((k[:, a] >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b + a)
        ops = (rng.random(n) < 0.1).astype(np.uint8)
        vals = np.float32([0.8473, -0.4055, 2.0, -2.0])[rng.integers(0, 4, n)]
        out.append((codes, ops, vals))
    return out


def run_writes(args, cfg):
    """One JSON line for --workload writes | rays (module docstring)."""
    total = args.steps + args.warmup
    origins, _, _, xyzs, _ = make_scans(cfg, total + 2, 0)
    batches = write_batches(cfg, total) if args.workload == "writes" else None
    if args.impl == "reference":
        import writes_lib
        writes_lib.build()
        kind, cls = ("reference", writes_lib.WritesRefMap) if writes_lib.have_ref() else ("port", writes_lib.WritesOracleMap)
        stride = 16
        m = cls(cfg["resolution"])
        times, n_up = [], []
        for k in range(total):
            t0 = time.perf_counter()
            if batches:
                codes, ops, vals = batches[k]
                m.update_nodes(codes[::stride], 0, 0, vals[::stride])  # the reference has no SET
                n = len(codes[::stride])
            else:
                ends = xyzs[k][::stride]
                m.insert_rays(origins[k], ends, max_range=cfg["max_range"], hit_end=True)
                n = len(ends)
            if k >= args.warmup:
                times.append(time.perf_counter() - t0)
                n_up.append(n)
        line = {"impl": "reference", "kind": kind, "workload": args.workload, "metric": "updates_per_s",
                "value": float(np.sum(n_up) / np.sum(times)), "unit": "updates/s",
                "ms_per_batch": 1e3 * float(np.median(times)), "batch": int(np.median(n_up)),
                "sample": "every %d-th entry / ray of each batch, one host thread" % stride,
                "steps": args.steps, "warmup": args.warmup, "higher_is_better": True}
        print(json.dumps(line), flush=True)
        return
    from ufomap_b200 import capi
    name, limit = card_info()
    m = capi.Map(cfg["resolution"], initial_bricks=cfg["bricks"])
    for k in range(2):
        m.insert(origins[total + k], xyzs[total + k], max_range=cfg["max_range"])
    ms, wall, n_up, bricks = [], [], [], []
    for k in range(total):
        t0 = time.perf_counter()
        if batches:
            codes, ops, vals = batches[k]
            m.update_nodes(codes, 0, ops, vals)
            n = len(codes)
        else:
            m.insert_rays(origins[k], xyzs[k], max_range=cfg["max_range"], hit_end=True)
            n = len(xyzs[k])
        t1 = time.perf_counter()
        st = m.stats()
        if k >= args.warmup:
            ms.append(st["ms_total"])
            wall.append(1e3 * (t1 - t0))
            n_up.append(n)
            bricks.append(st["touched_bricks"])
    m.close()
    line = {"impl": args.impl, "workload": args.workload, "metric": "updates_per_s",
            "value": float(np.sum(n_up) / (1e-3 * np.sum(ms))), "unit": "updates/s",
            "ms_per_batch": float(np.median(ms)), "ms_per_batch_wall": float(np.median(wall)),
            "batch": int(np.median(n_up)), "touched_bricks": int(np.median(bricks)),
            "steps": args.steps, "warmup": args.warmup, "higher_is_better": True,
            "gpu": name, "power_limit": limit,
            "config": {"workload": cfg["workload"],
                       "batch": ("1 M depth-0 updateValue / setNodeValue entries over a 30 m cube" if batches
                                 else "insertRay of every point of a scan, max_range %g m" % cfg["max_range"]),
                       "map": "two config scans inserted first"}}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", required=True, choices=["writes", "rays"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--impl", default="b200", choices=["b200", "reference"])
    ap.add_argument("--config", type=int, default=2, choices=[2, 4])
    args = ap.parse_args()
    run_writes(args, CONFIGS[args.config])


if __name__ == "__main__":
    main()
