#!/usr/bin/env python
"""tools/bench_route_image.py -- one file image from the ranks of a routed map: ufo_b200_image_part_bv
per rank and ufo_b200_image_assemble, on the config #2 map (2 cm, three 131 072-point scans of up to
30 m) split over two routed ranks on ONE device; one JSON line.

    python tools/bench_route_image.py [--reps R] [--before LIB]

* part_ms / assemble_ms: host wall time of each call (both end in a stream synchronisation or run
  on the host), median over R repetitions, for the whole map and for a 20 m change box around the
  last sensor pose (what the mapping server publishes after each scan).  The assembled image is
  checked against the single map's write_data of the same volume.
* write_data_ms: the single-map ufo_b200_write_data of the same map (whole map and the box), which
  is now its own part assembled alone.  --before LIB times the same call of another build of the
  library (e.g. the previous commit's) on an identical map, alternated with this one call by call,
  and checks that both write the same bytes.
* Moving the parts between GPUs (an all-gather over NCCL or gloo) is not measured: on one device
  the parts are host byte strings already.  The card's name and power limit are part of the line.
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


class RawMap:
    """A map of another build of the library, through the few calls this script makes."""

    def __init__(self, path, cfg, bricks):
        from ufomap_b200 import capi
        self.lib = lib = C.CDLL(path)
        vp, sz = C.c_void_p, C.c_size_t
        lib.ufo_b200_default_params.argtypes = [C.POINTER(capi.Params)]
        lib.ufo_b200_create.argtypes = [C.POINTER(capi.Params), C.POINTER(vp)]
        lib.ufo_b200_insert_pointcloud.argtypes = [vp, vp, vp, sz, C.c_int, C.c_double, C.c_uint32, C.c_int,
                                                   C.c_uint32, C.c_int, C.c_int]
        lib.ufo_b200_write_data.argtypes = [vp, vp, C.c_uint32, vp, sz, C.POINTER(sz)]
        lib.ufo_b200_destroy.argtypes = [vp]
        p = capi.Params()
        lib.ufo_b200_default_params(C.byref(p))
        p.resolution = cfg["resolution"]
        p.initial_bricks = bricks
        self.h = vp()
        assert lib.ufo_b200_create(C.byref(p), C.byref(self.h)) == 0

    def insert(self, origin, buf, layout, max_range):
        o = np.ascontiguousarray(origin, np.float64)
        assert self.lib.ufo_b200_insert_pointcloud(self.h, o.ctypes.data, buf.ctypes.data, len(buf), layout, max_range,
                                                   0, 0, 0, 0, 0) == 0

    def write_data(self, box6):
        bp = None if box6 is None else box6.ctypes.data
        n = C.c_size_t()
        assert self.lib.ufo_b200_write_data(self.h, bp, 0, None, 0, C.byref(n)) == 0
        out = np.empty(max(n.value, 1), np.uint8)
        assert self.lib.ufo_b200_write_data(self.h, bp, 0, out.ctypes.data, n.value, C.byref(n)) == 0
        return out[:n.value].tobytes()


def timed(f):
    t0 = time.perf_counter()
    out = f()
    return 1e3 * (time.perf_counter() - t0), out


def stats(ms):
    return {"median": float(np.median(ms)), "min": float(np.min(ms)), "max": float(np.max(ms))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=9)
    ap.add_argument("--before", default=None, help="another build of libufomap_b200.so to time write_data against")
    args = ap.parse_args()
    from ufomap_b200 import capi
    cfg = CONFIGS[2]
    name, limit = card_info()
    origins, packed, layout, _, _ = make_scans(cfg, 3, 0)
    world, bricks = 2, 1 << 18
    single = capi.Map(cfg["resolution"], initial_bricks=bricks)
    ranks = [capi.Map(cfg["resolution"], initial_bricks=bricks) for _ in range(world)]
    ptrs = [m.route_setup(r, world, cap_bricks=max(1 << 16, 400000 // world), cap_hits=1 << 18)
            for r, m in enumerate(ranks)]  # the inbox sizes bench.py uses for config #2
    for m in ranks:
        m.route_connect(ptrs)
    before = RawMap(args.before, cfg, bricks) if args.before else None
    for k in range(3):
        buf = packed[k]
        single.insert_packed(origins[k], buf.ctypes.data, len(buf), layout, max_range=cfg["max_range"])
        if before is not None:
            before.insert(origins[k], buf, layout, cfg["max_range"])
        keep = [np.ascontiguousarray(buf[r::world]) for r in range(world)]
        for m, part in zip(ranks, keep):
            m.route_mark(origins[k], part.ctypes.data, len(part), layout, max_range=cfg["max_range"])
        for m in ranks:
            m.wait()
        for m in ranks:
            m.route_apply(0, world, True)
        for m in ranks:
            m.wait()
    single.wait()
    o = origins[-1]
    box = (o - 10.0, o + 10.0)
    box6 = capi.Map._box6(box)
    volumes = {"whole": (None, None), "box20m": (capi.aabb(*box), box6)}
    out = {"tool": "bench_route_image", "gpu": name, "power_limit": limit, "reps": args.reps,
           "config": {"workload": cfg["workload"], "scans": 3, "ranks": "%d routed ranks on one device" % world,
                      "box20m": "AABB of half size 10 m around the last sensor pose",
                      "transport": "not measured"}}
    for vname, (vol, b6) in volumes.items():
        part_ms, asm_ms, new_ms, old_ms = [[] for _ in range(world)], [], [], []
        sizes = None
        for rep in range(args.reps + 1):  # the first repetition warms up
            parts = []
            for r, m in enumerate(ranks):
                t, p = timed(lambda: m.image_part(volume=vol))
                parts.append(p)
                if rep:
                    part_ms[r].append(t)
            t, image = timed(lambda: capi.assemble_image(parts, with_header=False))
            if rep:
                asm_ms.append(t)
            t, ref = timed(lambda: single.write_data(None if vol is None else box))
            if rep:
                new_ms.append(t)
            assert image == ref, "assembled image differs from the single map's (%s)" % vname
            if before is not None:
                t, old = timed(lambda: before.write_data(b6))
                if rep:
                    old_ms.append(t)
                assert old == ref, "the two builds write different bytes (%s)" % vname
            sizes = {"part_bytes": [len(p) for p in parts], "image_bytes": len(image)}
        out[vname] = dict(sizes, part_ms=[stats(x) for x in part_ms], assemble_ms=stats(asm_ms),
                          write_data_ms=stats(new_ms), write_data_before_ms=stats(old_ms) if old_ms else None)
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
