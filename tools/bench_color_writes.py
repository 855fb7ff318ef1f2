#!/usr/bin/env python
"""tools/bench_color_writes.py -- op-0 (ADD) batches through ufo_b200_update_nodes and through
ufo_b200_update_nodes_color, on a mono and on a colour map, plus a batch of colour ops; one JSON line
per case.

    python tools/bench_color_writes.py [--steps K] [--warmup W] [--config 2|4]

* maps: two scans of the BASELINE config inserted first (the colour map with per-point colours).
* batches: per step 1 M depth-0 entries at uniform voxels of a 30 m cube around the sensor
  (tools/bench_writes.py's batches with every op set to ADD); the "colour ops" case makes 40 % of
  them ADD_COLOR and 20 % SET_COLOR.
* The cases run interleaved, one step of each in turn, so that drift of the card affects them alike.
* value: entries per second of device time (CUDA events around the whole batch, ms_total of the
  call's stats); ms_per_batch_wall adds the host side (validation, copies).  The card's name and
  power limit are part of every line.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from bench import CONFIGS, make_scans  # noqa: E402
from bench_writes import card_info, write_batches  # noqa: E402

CASES = [("mono", "update_nodes"), ("mono", "update_nodes_color"), ("colour", "update_nodes"),
         ("colour", "update_nodes_color"), ("colour", "colour_ops")]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--config", type=int, default=2, choices=[2, 4])
    args = ap.parse_args()
    cfg = CONFIGS[args.config]
    total = args.steps + args.warmup
    origins, _, _, xyzs, _ = make_scans(cfg, 2, 0)
    batches = write_batches(cfg, total)
    rng = np.random.default_rng(11)
    from ufomap_b200 import capi
    name, limit = card_info()
    maps = {}
    for kind in ("mono", "colour"):
        m = capi.Map(cfg["resolution"], color=kind == "colour", initial_bricks=cfg["bricks"])
        for k in range(2):
            rgb = rng.integers(1, 256, size=(len(xyzs[k]), 3)).astype(np.uint8) if kind == "colour" else None
            m.insert(origins[k], xyzs[k], rgb=rgb, max_range=cfg["max_range"])
        maps[kind] = m
    n = len(batches[0][0])
    colour_ops = rng.choice(np.uint8([0, 2, 3]), size=n, p=[0.4, 0.4, 0.2])
    colours = rng.integers(0, 256, size=(n, 3)).astype(np.uint8)
    res = {c: ([], [], []) for c in CASES}
    for k in range(total):
        codes, _, vals = batches[k]
        for case in CASES:
            kind, call = case
            m = maps[kind]
            t0 = time.perf_counter()
            if call == "update_nodes":
                m.update_nodes(codes, 0, 0, vals)
            elif call == "update_nodes_color":
                m.update_nodes_color(codes, 0, 0, vals, None)
            else:
                m.update_nodes_color(codes, 0, colour_ops, vals, colours)
            t1 = time.perf_counter()
            st = m.stats()
            if k >= args.warmup:
                res[case][0].append(st["ms_total"])
                res[case][1].append(1e3 * (t1 - t0))
                res[case][2].append(st["touched_bricks"])
    for m in maps.values():
        m.close()
    for case in CASES:
        ms, wall, bricks = res[case]
        line = {"map": case[0], "call": case[1] if case[1] != "colour_ops" else "update_nodes_color",
                "ops": "40 % ADD, 40 % ADD_COLOR, 20 % SET_COLOR" if case[1] == "colour_ops" else "ADD",
                "metric": "entries_per_s", "value": float(n * len(ms) / (1e-3 * np.sum(ms))), "unit": "entries/s",
                "ms_per_batch": float(np.median(ms)), "ms_per_batch_min": float(np.min(ms)),
                "ms_per_batch_max": float(np.max(ms)), "ms_per_batch_wall": float(np.median(wall)),
                "batch": n, "touched_bricks": int(np.median(bricks)), "steps": args.steps, "warmup": args.warmup,
                "gpu": name, "power_limit": limit, "config": cfg["workload"]}
        print(json.dumps(line), flush=True)


if __name__ == "__main__":
    main()
