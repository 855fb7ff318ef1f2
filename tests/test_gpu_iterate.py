"""beginTree / beginLeaves on the device (ufo_b200_iterate) against the reference's own iterators,
compiled from its unmodified sources: element for element, in order -- code, depth, log-odds bits,
colour bytes, isLeaf and the contains flags -- for every filter, contains, min_depth and a set of
bounding volumes, on histories whose file image is first checked byte-identical (that fixes the tree
shape both sides iterate).  Plus: every record agrees with ufo_b200_query, and the RViz plugin's loop
through the C++ facade prints what the same loop over the reference gives."""
import itertools
import math
import struct
import subprocess

import numpy as np
import pytest

import iterate_lib
import volumes_lib
import writes_lib
from test_facade_iterate import build_facade_iterate
from ufomap_b200 import capi, scans
from ufomap_b200.capi import E_UNSUPPORTED, Map, UfoError

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not iterate_lib.have_ref(), reason="reference iteration checker not built")]

L = 16


def _velodyne_inserts(k_max=3):
    ins = []
    for k in range(k_max):
        o, p = scans.velodyne64(k=k, rings=8, azimuths=128)
        ins.append(dict(origin=o, xyz=p, max_range=20.0))
    return ins


def _history(name):
    """(device map, reference map, colour) after the named history."""
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
    else:  # setValueVolume and node writes
        kw, ins, color = dict(resolution=0.1), _velodyne_inserts(2), False
    gpu = Map(color=color, initial_blocks=1 << 12, **kw)
    ref = iterate_lib.IterateRefMap(color=color, **kw)
    for i in ins:
        gpu.insert(**i)
    if name != "writes":
        for i in ins:
            ref.insert(**i)
        return gpu, ref, color
    # the reference's node writes live in another checker: the history runs there and its file image
    # is read into the iteration checker (the image is the whole tree: shape and leaf values)
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
    return gpu, ref, color


def _volumes(gpu):
    mn, mx = gpu.change_bbox()
    mid, span = (mn + mx) / 2, float(np.min(mx - mn))
    s = 0.3 * span
    box = capi.aabb(mid - 0.4 * s, mid + np.array([0.3, 0.5, 0.2]) * s)
    sph = capi.sphere(mid + 0.2 * s, 0.45 * s)
    fru = capi.frustum(volumes_lib.ref_frustum7(mid - np.array([s, 0, 0]), mid, [0, 0, 1], math.pi / 4, math.pi / 3,
                                                0.1 * s, 2.0 * s))
    return {"none": [], "aabb": [box], "sphere": [sph], "frustum": [fru], "union": [box, sph, fru],
            "miss": [capi.sphere([1e4, 1e4, 1e4], 1.0)]}


def _compare(got, want, what):
    gc, gd, go, gf, gr = got
    wc, wd, wo, wf, wr = want[:5]
    assert len(gc) == len(wc), (what, len(gc), len(wc))
    assert np.array_equal(gc, wc), what
    assert np.array_equal(gd, wd), what
    assert np.array_equal(go.view(np.uint32), wo.view(np.uint32)), what
    assert np.array_equal(gf, wf & 7), what
    assert np.array_equal(gr, wr), what


def _centres(codes, depths, resolution):
    """getChildCenter accumulated from the root (octree.h:625-633)."""
    out = np.zeros((len(codes), 3))
    for i, (code, d) in enumerate(zip(codes.tolist(), depths.tolist())):
        c = [0.0, 0.0, 0.0]
        for D in range(L, d, -1):
            idx = (code >> (3 * (D - 1))) & 7
            hs = math.ldexp(resolution, D - 1) / 2.0
            for k in range(3):
                c[k] += hs if (idx >> k) & 1 else -hs
        out[i] = c
    return out


@pytest.mark.parametrize("name", ["velodyne", "rgbd_color_discrete", "writes", "thresholds"])
def test_iteration_matches_the_reference(name):
    gpu, ref, color = _history(name)
    assert gpu.write() == ref.write(), "file images differ: the trees are not the same shape"
    vols = _volumes(gpu)
    res = 0.04 if color else 0.1
    checked = 0
    for (vname, vol), leaves, flt, contains, md in itertools.product(
            vols.items(), (True, False), itertools.product((0, 1), repeat=3), (False, True),
            (0, 1, 2, 3, 4, 5, 6, L, L + 1)):
        kw = dict(leaves=leaves, occupied=flt[0], free=flt[1], unknown=flt[2], contains=contains, min_depth=md)
        got = gpu.iterate(vol, **kw)
        want = ref.iterate(vol, **kw)
        _compare(got, want, (name, vname, kw))
        checked += len(got[0])
        if vname in ("aabb", "union") and flt == (1, 1, 0) and len(got[0]):
            # the consistency check: each record is what ufo_b200_query reports for its node
            occ, fl, rgb = gpu.query(got[0], got[1].astype(np.uint32))
            assert np.array_equal(occ.view(np.uint32), got[2].view(np.uint32)), (name, kw)
            assert np.array_equal(fl & 3, got[3] & 3), (name, kw)
            if color:
                assert np.array_equal(rgb, got[4]), (name, kw)
            if md <= 2:
                assert np.array_equal(_centres(got[0], got[1], res).view(np.uint64), want[5].view(np.uint64)), (name, kw)
    assert checked > 0
    gpu.close()


def test_centres_are_the_references():
    gpu, ref, _ = _history("velodyne")
    vols = _volumes(gpu)
    for md in (0, 3):
        got = gpu.iterate(vols["sphere"], leaves=False, min_depth=md, unknown=True)
        want = ref.iterate(vols["sphere"], leaves=False, min_depth=md, unknown=True)
        assert len(got[0]) and np.array_equal(got[0], want[0])
        assert np.array_equal(_centres(got[0], got[1], 0.1).view(np.uint64), want[5].view(np.uint64))
    gpu.close()


def test_iterate_arguments():
    m = Map(0.1, depth_levels=4)
    with pytest.raises(UfoError) as e:
        m.iterate()
    assert e.value.status == E_UNSUPPORTED
    m.close()
    m = Map(0.1)
    codes, depths, occ, flags, _ = m.iterate(leaves=True, unknown=True)
    # an empty map: the root, a default leaf
    assert codes.tolist() == [0] and depths.tolist() == [L] and occ.tolist() == [0.0] and flags[0] & 4
    assert len(m.iterate(min_depth=L + 1)[0]) == 0
    bad = np.zeros(1, capi.VOLUME_DTYPE)
    bad["type"] = 99
    with pytest.raises(UfoError) as e:
        m.iterate(bad)
    assert e.value.status == capi.E_INVALID
    m.close()


def _hex_doubles(values):
    return ["%016x" % struct.unpack("<Q", struct.pack("<d", float(v)))[0] for v in values]


@pytest.mark.parametrize("name,min_depth,unknown", [("velodyne", 0, 0), ("velodyne", 4, 1), ("rgbd_color_discrete", 0, 0)])
def test_rviz_loop_through_the_facade(name, min_depth, unknown, tmp_path):
    gpu, ref, color = _history(name)
    data = gpu.write_data()
    path = tmp_path / "map.data"
    path.write_bytes(data)
    res = 0.04 if color else 0.1
    mn, mx = gpu.change_bbox()
    lo, hi = mn + 0.25 * (mx - mn), mn + 0.75 * (mx - mn)
    exe = build_facade_iterate(tmp_path)
    args = [exe, str(path), repr(res), str(L), str(int(color)), str(min_depth), "1", "1", str(unknown)] + [repr(float(v)) for v in
                                                                                                 (*lo, *hi)]
    out = subprocess.run(args, capture_output=True, text=True)
    assert out.returncode == 0 and "facade iterate ok" in out.stdout, (out.returncode, out.stdout[-500:], out.stderr)
    lines = [ln for ln in out.stdout.splitlines() if ln.startswith(("node", "extent"))]
    # the same loop over the reference: the box as the plugin builds it (clamped to the map)
    half = math.ldexp(res, L) / 2.0
    lo_c = np.maximum(np.array([float(v) for v in args[9:12]]), -half)
    hi_c = np.minimum(np.array([float(v) for v in args[12:15]]), half)
    want = ref.iterate([capi.aabb(lo_c, hi_c)], leaves=True, occupied=True, free=True, unknown=bool(unknown),
                       min_depth=min_depth)
    codes, depths, occ, flags, rgb, centres, probs = want
    expect, ext = [], {}
    for i in range(len(codes)):
        t = 0 if flags[i] & 8 else (1 if flags[i] & 16 else 2)
        hs = math.ldexp(res, int(depths[i])) / 2.0
        bmin, bmax = centres[i] - hs, centres[i] + hs
        point = [rgb[i][0] / 255.0, rgb[i][1] / 255.0, rgb[i][2] / 255.0, probs[i]] if color else [0.0] * 4
        expect.append("node %d %d %d " % (t, min_depth, depths[i]) + " ".join(_hex_doubles([probs[i], *bmin, *bmax, *point])))
        if t in ext:
            ext[t] = (np.minimum(ext[t][0], bmin), np.maximum(ext[t][1], bmax))
        else:
            ext[t] = (bmin, bmax)
    for t in sorted(ext):
        expect.append("extent %d " % t + " ".join(_hex_doubles([*ext[t][0], *ext[t][1]])))
    assert len(codes) > 0
    assert lines == expect
    gpu.close()
