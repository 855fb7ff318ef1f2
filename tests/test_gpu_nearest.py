"""Nearest-first iteration on the device (ufo_b200_nearest, beginNNTree / beginNNLeaves) against the CPU
checker built from the reference's unmodified sources: the reference's beginTree / beginLeaves,
stable-sorted by its own squared distance.  Element for element over the whole sequence -- code, depth,
log-odds bits, colour, flags, centre and d2 bits -- for every filter, contains, min_depth 0/1/4/5/7,
tree and leaves, and a set of volumes and query points (free space, inside an occupied voxel, on voxel
faces and corners, far outside the known box, outside the map).  Plus: shells of any size concatenate to
the same sequence, an unchanged map is answered from the kept tree shape and only near bricks, every
kind of map write invalidates that shape, and the facade's loops give the same nodes."""
import itertools
import math
import subprocess

import numpy as np
import pytest

import nearest_lib
import writes_lib
from test_facade_nearest import build_facade_nearest
from test_gpu_iterate import L, _velodyne_inserts, _volumes
from ufomap_b200 import capi, scans
from ufomap_b200.capi import Map

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not nearest_lib.have_ref(), reason="reference nearest checker not built")]

ALL = 1 << 40  # a want larger than any sequence: one shell holds everything


def _history(name):
    """(device map, checker map, colour, resolution) after the named history (test_gpu_iterate's)."""
    if name == "velodyne":
        kw, ins, color = dict(resolution=0.1), _velodyne_inserts(), False
    elif name == "rgbd_color_discrete":
        kw, color = dict(resolution=0.04), True
        ins = []
        for k in range(2):
            o, p, c = scans.rgbd(k=k, width=48, height=36)
            ins.append(dict(origin=o, xyz=p, rgb=c, max_range=3.0, discrete=True))
    elif name == "thresholds":
        kw, ins, color = dict(resolution=0.1, occupied_thres=0.6, free_thres=0.3), _velodyne_inserts(2), False
    else:  # setValueVolume and node writes, read back through the file image
        kw, ins, color = dict(resolution=0.1), _velodyne_inserts(2), False
    gpu = Map(color=color, initial_blocks=1 << 12, **kw)
    ref = nearest_lib.NearestRefMap(color=color, **kw)
    for i in ins:
        gpu.insert(**i)
    if name != "writes":
        for i in ins:
            ref.insert(**i)
        return gpu, ref, color, kw["resolution"]
    wref = writes_lib.WritesRefMap(**kw)
    for i in ins:
        wref.insert(**i)
    box = (np.array([-1.0, -2.0, -0.5]), np.array([2.0, 1.5, 0.7]))
    gpu.set_value_volume(box, 0.2, 0)
    wref.set_value_volume(box, 0.2, 0)
    rng = np.random.default_rng(5)
    pts = rng.uniform(-4, 4, size=(300, 3))
    depths = rng.integers(0, 4, size=300).astype(np.uint32)
    codes = np.array([gpu.to_code(p, int(d)) for p, d in zip(pts, depths)], np.uint64)
    vals = rng.choice([0.85, -0.4, 1.3, -2.0], size=300).astype(np.float32)
    gpu.update_nodes(codes, depths, 0, vals)
    wref.update_nodes(codes, depths, 0, vals)
    assert ref.read(wref.write())
    return gpu, ref, color, kw["resolution"]


def _points(gpu, res):
    """Query points: free space, inside an occupied voxel, on a voxel face, on a voxel corner, far
    outside the known box, outside the map's cube."""
    codes, depths, *_ = gpu.iterate(leaves=True, occupied=True, free=False)
    occ_centre = _centres(codes[len(codes) // 2:len(codes) // 2 + 1], depths[len(codes) // 2:len(codes) // 2 + 1], res)[0]
    mn, mx = gpu.change_bbox()
    half = math.ldexp(res, L) / 2.0
    return {"free": np.array([0.31, -0.17, 0.23]), "occupied": occ_centre + 0.23 * res,
            "face": np.array([7 * res, 0.37 * res - 2 * res, 0.61 * res]), "corner": np.array([3 * res, -5 * res, 2 * res]),
            "far": mx + np.array([40.0, -25.0, 30.0]), "outside": np.array([half * 1.5, -half * 2.0, 0.5])}


def _centres(codes, depths, resolution):
    """getChildCenter accumulated from the root (octree.h:625-633), vectorised."""
    codes = np.asarray(codes, np.uint64)
    depths = np.asarray(depths).astype(np.int64)
    c = np.zeros((len(codes), 3))
    for D in range(L, 0, -1):
        idx = ((codes >> np.uint64(3 * (D - 1))) & np.uint64(7)).astype(np.int64)
        hs = math.ldexp(resolution, D - 1) / 2.0
        on = (D > depths)[:, None]
        step = np.where(((idx[:, None] >> np.arange(3)[None, :]) & 1) == 1, hs, -hs)
        c = np.where(on, c + step, c)
    return c


def _d2(point, centres, depths, res):
    """The reference's squaredDistance in numpy: clamp, subtract, (x*x + y*y) + z*z."""
    hs = np.ldexp(res, depths.astype(np.int64)) / 2.0
    lo, hi = centres - hs[:, None], centres + hs[:, None]
    s = point[None, :] - np.minimum(np.maximum(point[None, :], lo), hi)
    return (s[:, 0] * s[:, 0] + s[:, 1] * s[:, 1]) + s[:, 2] * s[:, 2]


def _compare(got, want, res, what):
    gc, gd, go, gf, gr, gd2 = got
    wc, wd, wo, wf, wr, wcen, wd2 = want
    assert len(gc) == len(wc), (what, len(gc), len(wc))
    assert np.array_equal(gc, wc), what
    assert np.array_equal(gd, wd), what
    assert np.array_equal(go.view(np.uint32), wo.view(np.uint32)), what
    assert np.array_equal(gf, wf & 7), what
    assert np.array_equal(gr, wr), what
    assert np.array_equal(gd2.view(np.uint64), wd2.view(np.uint64)), what
    if len(gc):
        assert np.array_equal(_centres(gc, gd, res).view(np.uint64), wcen.view(np.uint64)), what


def _all(gpu, point, vol=None, **kw):
    *rec, nxt = gpu.nearest(point, vol, want=ALL, **kw)
    assert nxt == math.inf
    return tuple(rec)


def _shells(gpu, point, want, vol=None, **kw):
    parts = list(gpu.nearest_shells(point, vol, want=want, **kw))
    for p in parts[:-1]:
        assert len(p[0]) >= want
    return tuple(np.concatenate([p[i] for p in parts]) for i in range(6))


@pytest.mark.parametrize("name", ["velodyne", "rgbd_color_discrete", "writes", "thresholds"])
def test_nearest_matches_the_reference(name):
    gpu, ref, color, res = _history(name)
    assert gpu.write() == ref.write(), "file images differ: the trees are not the same shape"
    vols = _volumes(gpu)
    pts = _points(gpu, res)
    filters = list(itertools.product((0, 1), repeat=3))
    checked, k = 0, 0
    for (pname, p), (vname, vol), leaves, contains, md in itertools.product(
            pts.items(), vols.items(), (True, False), (False, True), (0, 1, 4, 5, 7)):
        flt = filters[k % len(filters)]
        k += 1
        kw = dict(leaves=leaves, occupied=flt[0], free=flt[1], unknown=flt[2], contains=contains, min_depth=md)
        got = _all(gpu, p, vol, **kw)
        want = ref.nearest(p, vol, **kw)
        _compare(got, want, res, (name, pname, vname, kw))
        checked += len(got[0])
    assert checked > 0
    gpu.close()


def test_every_filter_from_one_point():
    gpu, ref, color, res = _history("velodyne")
    p = _points(gpu, res)["face"]
    for flt, leaves, contains in itertools.product(itertools.product((0, 1), repeat=3), (True, False), (False, True)):
        kw = dict(leaves=leaves, occupied=flt[0], free=flt[1], unknown=flt[2], contains=contains)
        _compare(_all(gpu, p, **kw), ref.nearest(p, **kw), res, kw)
    gpu.close()


def test_shell_boundaries():
    gpu, ref, color, res = _history("velodyne")
    pts = _points(gpu, res)
    for pname in ("free", "corner", "far"):
        for kw in (dict(leaves=True, occupied=1, free=0, unknown=0), dict(leaves=False, occupied=1, free=1, unknown=1),
                   dict(leaves=True, occupied=0, free=1, unknown=0, min_depth=1)):
            whole = _all(gpu, pts[pname], **kw)
            assert np.all(np.diff(whole[5]) >= 0)
            for want in (1, 7, 1000):
                if want == 1 and len(whole[0]) > 3000:
                    continue  # one node per call: covered by the smaller sequences
                parts = _shells(gpu, pts[pname], want, **kw)
                for a, b in zip(parts, whole):
                    assert np.array_equal(a, b), (pname, kw, want)
    gpu.close()


def test_repeated_queries_stay_local():
    gpu, ref, color, res = _history("velodyne")
    p = _points(gpu, res)["free"]
    gpu.nearest(p, want=1, occupied=True, free=False)
    first = gpu.last_nearest_stats()
    assert first["rebuilt"] == 1
    codes, depths, occ, flags, rgb, d2, hi = gpu.nearest(p, want=50, occupied=True, free=False)
    st = gpu.last_nearest_stats()
    assert st["rebuilt"] == 0 and st["revision"] == first["revision"] and len(codes) >= 50
    # the live bricks: those holding a non-default voxel; a brick of cube distance d2 >= hi is never read
    leaf_codes, _, _ = gpu.value_field()
    bricks = np.unique(leaf_codes.astype(np.uint64) >> np.uint64(12)) << np.uint64(12)
    bd = _d2(p, _centres(bricks, np.full(len(bricks), 4, np.uint8), res), np.full(len(bricks), 4), res)
    near = int(np.count_nonzero(bd < hi * (1 + 1e-6)))
    assert 0 < st["bricks_visited"] <= near * st["shells"], (st, near, len(bricks))
    assert st["bricks_visited"] < len(bricks)
    gpu.close()


def _sorted_by_distance(gpu, p, res, **kw):
    """The fresh checker of a changed map: the device's beginTree / beginLeaves order (checked against
    the reference in test_gpu_iterate.py), stable-sorted by the reference's distance."""
    codes, depths, occ, flags, rgb = gpu.iterate(**kw)
    d2 = _d2(p, _centres(codes, depths, res), depths, res)
    o = np.argsort(d2, kind="stable")
    return codes[o], depths[o], occ[o], flags[o], rgb[o], d2[o]


def test_every_write_invalidates_the_shape(tmp_path):
    gpu, _, _, res = _history("velodyne")
    p = np.array([0.45, -0.35, 0.15])
    kw = dict(leaves=True, occupied=True, free=True, unknown=False)
    box = (np.array([-0.6, -0.6, -0.6]), np.array([0.9, 0.7, 0.8]))
    img = gpu.write()
    data = gpu.write_data()
    o, pts = scans.velodyne64(k=5, rings=8, azimuths=128)
    cases = [
        ("scan", lambda m: m.insert(o, pts, max_range=20.0)),
        ("update_nodes", lambda m: m.update_nodes(np.array([m.to_code(p + 0.2, 0)], np.uint64), np.zeros(1, np.uint32), 1,
                                                  np.array([2.5], np.float32))),
        ("insert_rays", lambda m: m.insert_rays(np.array([[0.0, 0.0, 0.0]]), np.array([[0.8, -0.5, 0.3]]))),
        ("set_value_volume", lambda m: m.set_value_volume(box, 0.9, 0)),
        ("set_value_volume_bv", lambda m: m.set_value_volume_bv(capi.sphere(p, 0.4), 0.1, 0)),
        ("read_data", lambda m: m.read_data(data)),
        ("read", lambda m: m.read(img)),
        ("sensor_model", lambda m: m.set_sensor_model_field(0, 0.55)),
        ("retain", lambda m: m.retain(box=box)),
        ("page_in", lambda m: (lambda blob: (m.retain(capi.sphere([50.0, 50.0, 50.0], 1.0)), m.page_in(blob)))(
            m.page_out(box=box))),
        ("clear", lambda m: m.clear()),
        ("clear_resize", lambda m: (m.clear_resize(res, L), m.read(img))),
    ]
    gpu.nearest(p, want=ALL, **kw)
    for what, change in cases:
        rev = gpu.last_nearest_stats()["revision"]
        change(gpu)
        got = _all(gpu, p, **kw)
        st = gpu.last_nearest_stats()
        assert st["rebuilt"] == 1 and st["revision"] != rev, what
        want = _sorted_by_distance(gpu, p, res, **kw)
        for a, b in zip(got, want):
            assert np.array_equal(np.asarray(a).view(np.uint8), np.asarray(b).view(np.uint8)), what
    # a clone answers like its source
    gpu.read(img)
    twin = gpu.clone()
    a, b = _all(gpu, p, **kw), _all(twin, p, **kw)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    twin.close()
    gpu.close()


def test_nearest_arguments():
    m = Map(0.1, depth_levels=4)
    with pytest.raises(capi.UfoError) as e:
        m.nearest([0, 0, 0])
    assert e.value.status == capi.E_UNSUPPORTED
    m.close()
    m = Map(0.1)
    for bad in ([math.nan, 0, 0], [0, math.inf, 0]):
        with pytest.raises(capi.UfoError) as e:
            m.nearest(bad)
        assert e.value.status == capi.E_INVALID
    # an empty map: the root, a default leaf, at distance 0 from a point inside the map
    codes, depths, occ, flags, rgb, d2, nxt = m.nearest([0.3, 0.2, 0.1], unknown=True, want=5)
    assert codes.tolist() == [0] and depths.tolist() == [L] and d2.tolist() == [0.0] and nxt == math.inf
    assert len(m.nearest([0, 0, 0], min_depth=L + 1)[0]) == 0
    assert len(m.nearest([0, 0, 0], capi.sphere([1e9, 0, 0], 1.0), unknown=True)[0]) == 0
    m.close()


@pytest.mark.parametrize("name", ["velodyne", "rgbd_color_discrete"])
def test_facade_loops(name, tmp_path):
    gpu, ref, color, res = _history(name)
    data = gpu.write_data()
    path = tmp_path / "map.data"
    path.write_bytes(data)
    p = _points(gpu, res)["free"]
    exe = build_facade_nearest(tmp_path)
    out = subprocess.run([exe, str(path), repr(res), str(L), str(int(color))] + [repr(float(v)) for v in p],
                         capture_output=True, text=True)
    assert out.returncode == 0 and "facade nearest ok" in out.stdout, (out.returncode, out.stdout[-800:], out.stderr)
    assert "FAILED" not in out.stdout
    lines = out.stdout.splitlines()

    def expect(tag, vol=None, **kw):
        codes, depths, occ, flags, rgb, d2 = _all(gpu, p, vol, **kw)
        hs = np.ldexp(res, depths.astype(np.int64)) / 2.0
        c = _centres(codes, depths, res)
        mn, mx = c - hs[:, None], c + hs[:, None]
        return ["%s %d %d %08x %d %d %d %d %016x %016x %016x %016x %016x %016x %016x" % (
            tag, codes[i], depths[i], occ[i:i + 1].view(np.uint32)[0], rgb[i][0], rgb[i][1], rgb[i][2], flags[i] & 7,
            d2[i:i + 1].view(np.uint64)[0], *mn[i].view(np.uint64), *mx[i].view(np.uint64)) for i in range(len(codes))]

    sphere = capi.sphere(p, 1.5)
    box = capi.aabb(p + np.array([-0.7, -0.4, -0.3]), p + np.array([0.6, 0.9, 0.5]))
    want = {
        "tree": expect("tree", leaves=False, occupied=1, free=0, unknown=0, min_depth=1),
        "tree_var": expect("tree_var", [sphere], leaves=False, occupied=1, free=1, unknown=0, contains=True),
        "tree_volume": expect("tree_volume", [box, sphere], leaves=False),
        "leaves": expect("leaves", leaves=True, occupied=1, free=0, unknown=0),
        "leaves_var": expect("leaves_var", [box], leaves=True, occupied=0, free=1, unknown=0, min_depth=2),
        "leaves_volume": expect("leaves_volume", [box, sphere], leaves=True, occupied=1, free=1, unknown=1),
    }
    for tag, rows in want.items():
        assert [ln for ln in lines if ln.split(" ", 1)[0] == tag] == rows, tag
    assert sum(len(r) for r in want.values()) > 0
    d = math.sqrt(_all(gpu, p, leaves=True, occupied=1, free=0, unknown=0)[5][0])
    assert "planner %016x" % np.array([d]).view(np.uint64)[0] in lines
    changed = [ln for ln in lines if ln.startswith("changed")][0].split()
    assert int(changed[2]) == capi.E_INVALID and int(changed[1]) < 100000
    gpu.close()
