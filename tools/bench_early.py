#!/usr/bin/env python
"""Device time of insertPointCloud with early stopping (ufo_early.cuh) on the bench configurations.

    python tools/bench_early.py [--config 2 3 4] [--stop 0 1 3 10] [--scans 6] [--warmup 2]

One map per (configuration, E), fed the bench's seeded scans (host buffers, synchronous inserts,
the scans of a moving sensor as bench.py feeds them).  E = 0 is the unchanged path, measured in the
same call.  Per timed scan: ms_total (CUDA events around the insert's device work), the E1 / E2 / E3
split (walks and node ids / prefix rounds / marking, CUDA events at profiling level 1), the round
count, visits, distinct nodes, free-set nodes and the bytes of the node table and id buffers.  One
JSON line per (configuration, E), with the card's name, power limit and maximum SM clock read in the
same call.  A workload whose buffers do not fit the card is reported with its error.
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


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return out.strip().splitlines()[0] if out.strip() else None
    except Exception:
        return None


def run(config, stop, n_scans, warm):
    from ufomap_b200 import capi, scans

    cfg = CONFIGS[config]
    rgbd = cfg["kind"] == "rgbd"
    m = capi.Map(cfg["res"], color=rgbd, initial_bricks=cfg["bricks"])
    m.set_profiling(1)
    m.set_early_stopping(True)
    rows = []
    try:
        for k in range(n_scans):
            if rgbd:
                o, p, c = scans.rgbd(k=k)
                m.insert(o, p, rgb=c, max_range=cfg["max_range"], dtype=np.float32, discrete=True,
                         early_stopping=stop)
            else:
                o, p = scans.velodyne64(k=k)
                m.insert(o, p, max_range=cfg["max_range"], dtype=np.float32, early_stopping=stop)
            if k >= warm:
                rows.append(dict(m.stats(), **{"early_" + n: v for n, v in m.early_stats().items()}))
    except capi.UfoError as e:
        return {"config": config, "stop": stop, "error": str(e)}
    finally:
        m.close()

    def med(key):
        return float(np.median([r[key] for r in rows]))
    return {
        "config": config, "stop": stop, "scans_timed": len(rows), "points": int(rows[-1]["points"]),
        "ms_total": med("ms_total"), "ms_rays": med("ms_rays"), "ms_update": med("ms_update"),
        "ms_e1_walk": med("early_ms_walk"), "ms_e2_rounds": med("early_ms_rounds"), "ms_e3_mark": med("early_ms_mark"),
        "rounds": [int(r["early_rounds"]) for r in rows], "visits": int(rows[-1]["early_visits"]),
        "nodes": int(rows[-1]["early_nodes"]), "free_nodes": int(rows[-1]["early_free_nodes"]),
        "table_bytes": int(rows[-1]["early_table_bytes"]), "id_bytes": int(rows[-1]["early_id_bytes"]),
        "device_bytes": int(rows[-1]["device_bytes"]),
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", type=int, nargs="+", default=[2, 3, 4], choices=sorted(CONFIGS))
    ap.add_argument("--stop", type=int, nargs="+", default=[0, 1, 3, 10])
    ap.add_argument("--scans", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    if args.scans <= args.warmup:
        ap.error("--scans must exceed --warmup")
    import torch
    if not torch.cuda.is_available():
        sys.exit("bench_early.py needs a CUDA device")
    print(json.dumps({"card": card()}), flush=True)
    for c in args.config:
        for e in args.stop:
            print(json.dumps(run(c, e, args.scans, args.warmup)), flush=True)
            torch.cuda.empty_cache()
    print(json.dumps({"card": card()}), flush=True)


if __name__ == "__main__":
    main()
