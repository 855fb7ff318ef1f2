#!/usr/bin/env python
"""tools/bench_route_grow.py -- what pool growth during routed passes costs.  One JSON line per part.

    python tools/bench_route_grow.py [--parent-lib PATH] [--steps K] [--warmup W] [--rounds R]

* wait:   route_mark now waits for its marking kernels (to grow a full pool before anything is
          published).  tools/bench_route.py --case 2disc and --case 3d0 (2 ranks on one device, one
          process each) are run with this build and, given --parent-lib, with a library built from
          the parent commit, alternating R rounds; the line gives every run's mark-phase ms per rank.
* stream: a routed stream of config #2 scans (2 cm Velodyne-64, discrete, 2 ranks on one device) on
          ranks started from a small pool (initial_bricks 1024) and on ranks sized for the run:
          host ms per pass (mark, barrier, apply, wait), regrows and the final brick capacities.
These are overhead figures of ranks that share one GPU, not multi-GPU scaling figures.  The card's
name and power limit are part of each line.
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
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import CONFIGS, make_scans  # noqa: E402
from bench_route import capacities, rank_parts  # noqa: E402
from bench_writes import card_info  # noqa: E402


def bench_route(case, lib, steps, warmup):
    env = dict(os.environ)
    if lib:
        env["UFOMAP_B200_LIB"] = os.path.abspath(lib)
    cmd = [sys.executable, os.path.join(ROOT, "tools", "bench_route.py"), "--case", case, "--ranks", "2",
           "--steps", str(steps), "--warmup", str(warmup), "--no-single"]
    out = subprocess.run(cmd, env=env, check=True, capture_output=True, text=True).stdout
    line = json.loads([x for x in out.splitlines() if x.startswith("{")][-1])
    return [round(p["mark_ms"], 3) for p in line["per_rank"]], [round(p["apply_ms"], 3) for p in line["per_rank"]]


def part_wait(args):
    libs = [("this", None)] + ([("parent", args.parent_lib)] if args.parent_lib else [])
    runs = {c: {name: [] for name, _ in libs} for c in ("2disc", "3d0")}
    for _ in range(args.rounds):
        for case in runs:
            for name, lib in libs:
                mark, apply_ = bench_route(case, lib, args.steps, args.warmup)
                runs[case][name].append({"mark_ms_per_rank": mark, "apply_ms_per_rank": apply_})
    name, limit = card_info(0)
    print(json.dumps({"tool": "bench_route_grow", "part": "wait", "ranks": 2, "shared_device": True,
                      "steps": args.steps, "warmup": args.warmup, "runs": runs, "gpu": name,
                      "power_limit": limit}), flush=True)


def part_stream(args):
    import torch
    from ufomap_b200 import capi

    cfg = CONFIGS[2]
    world, passes = 2, args.passes
    origins, packed, layout, _, _ = make_scans(cfg, passes, 0)
    parts = rank_parts(cfg, packed, world)
    case = dict(depth=0, discrete=True)
    bricks, cap_b, cap_h = capacities(cfg, case, world, len(packed[0]))
    dev = torch.device("cuda", 0)
    d_parts = [[torch.from_numpy(p[0]).to(dev) for p in parts[r]] for r in range(world)]
    out = {}
    for label, initial in (("presized", bricks), ("small", 1024), ("presized_again", bricks)):
        maps = [capi.Map(cfg["resolution"], initial_bricks=initial) for _ in range(world)]
        ptrs = [m.route_setup(r, world, cap_bricks=cap_b, cap_hits=cap_h) for r, m in enumerate(maps)]
        for m in maps:
            m.route_connect(ptrs)
        torch.cuda.synchronize(dev)
        ms, regrows = [], []
        for k in range(passes):
            t0 = time.perf_counter()
            for r, m in enumerate(maps):
                t = d_parts[r][k]
                m.route_mark_ex(origins[k], t.data_ptr(), t.shape[0], layout, on_device=True,
                                max_range=cfg["max_range"], discrete=True)
            for m in maps:
                m.wait()
            for m in maps:
                m.route_apply(0, world, True)
            for m in maps:
                m.wait()
            ms.append((time.perf_counter() - t0) * 1e3)
            regrows.append([m.stats()["regrows"] for m in maps])
        out[label] = {"initial_bricks": initial, "ms_per_pass": [round(x, 2) for x in ms],
                      "ms_total": round(sum(ms), 2), "regrows_per_pass": regrows,
                      "brick_cap": [m.pool_stats()["brick_cap"] for m in maps],
                      "bricks": [m.pool_stats()["bricks"] for m in maps]}
        for m in maps:
            m.close()
        torch.cuda.empty_cache()
    name, limit = card_info(0)
    print(json.dumps({"tool": "bench_route_grow", "part": "stream", "workload": cfg["workload"], "ranks": world,
                      "shared_device": True, "passes": passes, "results": out, "gpu": name, "power_limit": limit}),
          flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--parent-lib", default=None, help="a library built from the parent commit (A/B of the wait)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--passes", type=int, default=8)
    ap.add_argument("--part", choices=["wait", "stream", "all"], default="all")
    args = ap.parse_args()
    if args.part in ("wait", "all"):
        part_wait(args)
    if args.part in ("stream", "all"):
        part_stream(args)


if __name__ == "__main__":
    main()
