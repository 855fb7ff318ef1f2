#!/usr/bin/env python
"""tools/bench_route.py -- the routed multi-GPU mode (ufo_b200_route_mark_ex) on the mapping server's
own call: discrete insertion, colour maps, insert depth 0..6.  One JSON line per run.

    python tools/bench_route.py --case 3d0|3d6|2disc [--ranks N] [--steps K] [--warmup W]
    torchrun --nproc-per-node N tools/bench_route.py --case ...     (one process per GPU)

* 3d0:   config #3 (2 mm colour RGB-D, 307 200 points, max_range 5 m), insertPointCloudDiscrete, depth 0
* 3d6:   the same at insert depth 6 (the mapping server's 2 mm setting is depth 4-6)
* 2disc: config #2 (2 cm Velodyne-64, 131 072 points, max_range 30 m) with discrete=1

A scan is split over the ranks as one stream (route_apply(0, N, 1)): config #3 by contiguous image
rows (global index offset, stride 1), config #2 by azimuth sector (bench.route_slice).

Without torchrun (one process), N maps on ONE device play the ranks: every rank's mark pass and
then every rank's apply pass run one after the other, each timed with CUDA events on the map's
stream.  These are OVERHEAD figures of the routed mode -- device time each rank spends and the
records it forwards -- not scaling figures: the ranks share one GPU.  The same call on one map
(single_ms) is measured after the routed maps are freed.  Under torchrun every process drives its
own GPU; the inboxes are mapped over cudaIpc and a 4-byte NCCL all-reduce on the map's stream is
the barrier, as in bench.py --mode route.  The card's name and power limit are part of the line.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from bench import CONFIGS, make_scans, route_slice  # noqa: E402
from bench_writes import card_info  # noqa: E402

CASES = {
    "3d0": dict(config=3, depth=0, discrete=True),
    "3d6": dict(config=3, depth=6, discrete=True),
    "2disc": dict(config=2, depth=0, discrete=True),
}


def rank_parts(cfg, packed, world):
    """Per rank: (point buffer, index_base, index_stride) of every scan."""
    out = []
    for r in range(world):
        scans_r = []
        for buf in packed:
            n = len(buf)
            if cfg["kind"] == "rgbd":
                lo, hi = r * n // world, (r + 1) * n // world  # contiguous image rows
                scans_r.append((np.ascontiguousarray(buf[lo:hi]), lo, 1))
            else:
                scans_r.append((np.ascontiguousarray(buf[route_slice(n, r, world)]), 0, 1))  # mono: index unused
        out.append(scans_r)
    return out


def capacities(cfg, case, world, n_pts):
    """Per-rank brick pool and inbox capacities (pools do not grow during a routed pass)."""
    # a rank keeps the bricks its own rays cross (fused walk, depth <= 2) and the ones it owns; colour
    # ranks at 2 mm also hold a 16 GB scan volume each (depth 0), so their pools are kept smaller
    bricks = cfg["bricks"] if not cfg["color"] else max(1 << 16, int(cfg["bricks"] * 0.8) // world)
    cap_hits = 1 << 19 if case["depth"] >= 5 or cfg["color"] else 1 << 18
    cap_bricks = max(1 << 16, 400000 // world)
    return bricks, cap_bricks, max(cap_hits, n_pts // world + 1)


def run(args):
    import torch
    from ufomap_b200 import capi

    case = CASES[args.case]
    cfg = CONFIGS[case["config"]]
    total = args.steps + args.warmup
    world_env = int(os.environ.get("WORLD_SIZE", "1"))
    distributed = world_env > 1
    rank = int(os.environ.get("RANK", "0")) if distributed else 0
    local = int(os.environ.get("LOCAL_RANK", "0")) if distributed else 0
    world = world_env if distributed else args.ranks
    torch.cuda.set_device(local)
    dev = torch.device("cuda", local)
    if distributed:
        import torch.distributed as dist
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        dist.init_process_group("nccl", device_id=dev)
    origins, packed, layout, _, _ = make_scans(cfg, total, 0)
    n_pts = len(packed[0])
    parts = rank_parts(cfg, packed, world)
    bricks, cap_b, cap_h = capacities(cfg, case, world, n_pts)
    opts = dict(max_range=cfg["max_range"], depth=case["depth"], discrete=case["discrete"])
    mine = [rank] if distributed else list(range(world))
    streams = {r: torch.cuda.Stream(dev) for r in mine}
    maps = {}
    for r in mine:
        m = capi.Map(cfg["resolution"], color=cfg["color"], device=local, initial_bricks=bricks)
        m.set_stream(streams[r].cuda_stream)
        maps[r] = m
    ptrs = {r: maps[r].route_setup(r, world, cap_bricks=cap_b, cap_hits=cap_h) for r in mine}
    opened = []
    if distributed:
        handles = [None] * world
        dist.all_gather_object(handles, capi.ipc_export(ptrs[rank]))
        peers = [ptrs[rank] if r == rank else capi.ipc_open(handles[r]) for r in range(world)]
        opened = [p for r, p in enumerate(peers) if r != rank]
        dist.barrier()
    else:
        peers = [ptrs[r] for r in range(world)]
    for m in maps.values():
        m.route_connect(peers)
    token = torch.zeros(1, device=dev)
    d_parts = {r: [torch.from_numpy(p[0]).to(dev) for p in parts[r]] for r in mine}
    torch.cuda.synchronize(dev)

    def timed(r, fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(streams[r])
        fn()
        e1.record(streams[r])
        e1.synchronize()
        return e0.elapsed_time(e1)

    mark_ms = {r: [] for r in mine}
    apply_ms = {r: [] for r in mine}
    sent = {r: [] for r in mine}
    for k in range(total):
        for r in mine:
            _, base, stride = parts[r][k]
            t = d_parts[r][k]
            ms = timed(r, lambda: maps[r].route_mark_ex(origins[k], t.data_ptr(), t.shape[0], layout, on_device=True,
                                                         index_base=base, index_stride=stride, **opts))
            if k >= args.warmup:
                mark_ms[r].append(ms)
                sent[r].append(maps[r].route_sent())
        if distributed:
            with torch.cuda.stream(streams[rank]):
                dist.all_reduce(token)  # the barrier between forwarding and applying
        for r in mine:
            ms = timed(r, lambda: maps[r].route_apply(0, world, True))
            if k >= args.warmup:
                apply_ms[r].append(ms)
        for m in maps.values():
            m.wait()
    bricks_in_map = {r: maps[r].stats()["bricks_in_map"] for r in mine}
    for m in maps.values():
        m.wait()
    if distributed:
        dist.barrier()
        for p in opened:
            capi.ipc_close(p)
        dist.barrier()
    for m in maps.values():
        m.close()
    del d_parts
    torch.cuda.empty_cache()

    single_ms = None
    if not distributed and not args.no_single:
        m = capi.Map(cfg["resolution"], color=cfg["color"], device=local, initial_bricks=cfg["bricks"])
        times = []
        for k in range(total):
            t = torch.from_numpy(packed[k]).to(dev)
            m.insert_packed(origins[k], t.data_ptr(), n_pts, layout, on_device=True, **opts)
            if k >= args.warmup:
                times.append(m.stats()["ms_total"])
        m.close()
        single_ms = float(np.median(times))

    inbox = capi.route_inbox_bytes(world, cap_b, cap_h, color=cfg["color"])
    per_rank = []
    for r in mine:
        s = sent[r]
        bricks_rec = [x["brick_records"] for x in s]
        full_rec = [x["full_brick_records"] for x in s]
        hit_rec = [x["hit_records"] for x in s]
        hit_b = 16 if cfg["color"] else 8
        per_rank.append({
            "rank": r, "points": int(len(parts[r][0][0])),
            "mark_ms": float(np.median(mark_ms[r])), "apply_ms": float(np.median(apply_ms[r])),
            "brick_records": int(np.median(bricks_rec)), "full_brick_records": int(np.median(full_rec)),
            "hit_records": int(np.median(hit_rec)),
            "inbox_bytes_per_scan": int(np.median([8 * 65 * b + 8 * f + hit_b * h
                                                   for b, f, h in zip(bricks_rec, full_rec, hit_rec)])),
            "bricks_in_map": int(bricks_in_map[r])})
    if distributed:
        gathered = [None] * world
        dist.all_gather_object(gathered, per_rank)
        per_rank = [x for g in gathered for x in g]
        dist.destroy_process_group()
        if rank != 0:
            return
    name, limit = card_info(local)
    line = {"tool": "bench_route", "case": args.case, "workload": cfg["workload"],
            "insert": "route_mark_ex(discrete=%d, depth=%d), scan split over %d ranks, route_apply(0, %d, 1)"
                      % (case["discrete"], case["depth"], world, world),
            "ranks": world, "gpus": world if distributed else 1,
            "shared_device": not distributed,
            "note": ("overhead figures: %d ranks share one GPU and run one after the other; not a scaling figure"
                     % world) if not distributed else "one process per GPU",
            "steps": args.steps, "warmup": args.warmup,
            "mark_ms_sum": float(sum(p["mark_ms"] for p in per_rank)),
            "apply_ms_sum": float(sum(p["apply_ms"] for p in per_rank)),
            "single_ms": single_ms, "inbox_allocated_bytes_per_rank": int(inbox),
            "per_rank": per_rank, "gpu": name, "power_limit": limit}
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", required=True, choices=sorted(CASES))
    ap.add_argument("--ranks", type=int, default=2, help="maps on one device (without torchrun)")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--no-single", action="store_true", help="skip the single-map comparison")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
