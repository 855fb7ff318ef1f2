"""Bounding volumes on the device against the reference compiled from its unmodified sources:
writeData / write / compressed write, readData, setValueVolume and leaf iteration with any union
of AABBs, frustums, line segments, OBBs, planes, points, rays and spheres -- streams byte for
byte, value fields bit for bit."""
import math

import numpy as np
import pytest

import volumes_lib
from helpers import assert_value_fields_equal, check_inner_against_field
from ufomap_b200 import capi, scans
from ufomap_b200.capi import E_UNSUPPORTED, Map, UfoError

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not volumes_lib.have_ref(), reason="reference volume checker not built")]


def _scenario(name):
    if name == "velodyne":
        ins = []
        for k in range(3):
            o, p = scans.velodyne64(k=k, rings=8, azimuths=128)
            ins.append(dict(origin=o, xyz=p, max_range=25.0))
        return dict(resolution=0.2), ins, False
    ins = []
    for k in range(2):
        o, p, c = scans.rgbd(k=k, width=48, height=36)
        ins.append(dict(origin=o, xyz=p, rgb=c, max_range=3.0, discrete=True))
    return dict(resolution=0.04), ins, True


def _maps(name, **extra):
    kw, inserts, color = _scenario(name)
    kw.update(extra)
    gpu = Map(color=color, initial_blocks=1 << 12, **kw)
    ref = volumes_lib.VolumesRefMap(color=color, **kw)
    for ins in inserts:
        gpu.insert(**ins)
        ref.insert(**ins)
    return gpu, ref, inserts, color


def _shapes(centre, size, rng):
    """One shape of every type around centre, of extent ~size."""
    c = np.asarray(centre, np.float64)
    s = float(size)
    q = rng.normal(size=4)
    n = rng.normal(size=3)
    n /= np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])
    return [
        capi.aabb(c - 0.4 * s, c + np.array([0.3, 0.5, 0.2]) * s),
        capi.frustum(volumes_lib.ref_frustum7(c - np.array([s, 0, 0]), c, [0, 0, 1], math.pi / 4, math.pi / 3,
                                              0.1 * s, 2.0 * s)),
        capi.line_segment(c - np.array([s, 0.3 * s, 0.1 * s]), c + np.array([0.8 * s, 0.2 * s, 0.4 * s])),
        capi.obb(c, np.array([0.5, 0.2, 0.3]) * s, q / np.linalg.norm(q)),
        capi.plane(n, (n[0] * c[0] + n[1] * c[1]) + n[2] * c[2]),
        capi.point(c + 0.1 * s),
        capi.volume_record(capi.RAY, volumes_lib.ref_ray(c, [1.0, 0.5, -0.2])),
        capi.sphere(c + 0.2 * s, 0.45 * s),
    ]


def _volumes(gpu, ref, rng):
    mn, mx = ref.change_bbox()
    mid, span = (mn + mx) / 2, float(np.min(mx - mn))
    shapes = _shapes(mid, 0.4 * span, rng)
    vols = [[s] for s in shapes]
    for k in (2, 3, 4):
        pick = rng.choice(len(shapes), k, replace=False)
        vols.append([shapes[i] for i in pick])
    vols.append([])  # the whole map
    vols.append([capi.sphere([1e4, 1e4, 1e4], 1.0), capi.aabb([2e4, 2e4, 2e4], [3e4, 3e4, 3e4])])  # misses the map
    return vols


@pytest.mark.parametrize("name", ["velodyne", "rgbd_color_discrete"])
def test_streams_are_byte_identical(name):
    gpu, ref, _, _ = _maps(name)
    rng = np.random.default_rng(31)
    for i, vol in enumerate(_volumes(gpu, ref, rng)):
        for md in range(5):
            got = gpu.write_data_bv(vol, md)
            assert got == ref.write_data_bv(vol, md), (i, md, len(got))
        for md in (0, 3):
            assert gpu.write_bv(vol, md) == ref.write_bv(vol, md), (i, md)
        if i in (1, 3, 9):
            image, _ = gpu.write_compressed_bv(vol, 0, acceleration=1, level=0)
            assert image == ref.write_bv(vol, 0, compress=True, acceleration=1, level=0), i
    gpu.close()


@pytest.mark.parametrize("name", ["velodyne", "rgbd_color_discrete"])
def test_aabb_volume_equals_the_box_calls(name):
    gpu, ref, inserts, color = _maps(name)
    mn, mx = ref.change_bbox()
    box = (mn + 0.2 * (mx - mn), mn + 0.7 * (mx - mn))
    vol = capi.aabb(*box)
    for md in range(5):
        assert gpu.write_data_bv(vol, md) == gpu.write_data(box, md)
    assert gpu.write_bv(vol, 2) == gpu.write(box=box, min_depth=2)
    c1, o1, _ = gpu.export_nodes(depth=0, box=box)
    c2, o2, _ = gpu.export_nodes_bv(vol, depth=0)
    assert len(c2) and np.array_equal(c1, c2) and np.array_equal(o1.view(np.uint32), o2.view(np.uint32))
    kw, _, _ = _scenario(name)
    twin = Map(color=color, initial_blocks=1 << 12, **kw)
    for ins in inserts:
        twin.insert(**ins)
    gpu.set_value_volume(box, 0.3, 0)
    twin.set_value_volume_bv(vol, 0.3, 0)
    assert_value_fields_equal(gpu.value_field(), twin.value_field())
    gpu.close()
    twin.close()


@pytest.mark.parametrize("name", ["velodyne", "rgbd_color_discrete"])
def test_read_data_with_a_volume(name):
    src, ref_src, inserts, color = _maps(name)
    rng = np.random.default_rng(5)
    vols = _volumes(src, ref_src, rng)
    kw, _, _ = _scenario(name)
    for i in (0, 1, 3, 4, 6, 7, 9, 11):
        vol = vols[i]
        # a stream is read with the volume it was written with (the reader skips what the writer skipped)
        data = src.write_data_bv(vol, i % 3)
        gpu = Map(color=color, initial_blocks=1 << 12, **kw)
        ref = volumes_lib.VolumesRefMap(color=color, **kw)
        other = dict(inserts[-1])
        other["origin"] = np.array(other["origin"]) + np.array([0.37, -0.21, 0.05])
        gpu.insert(**other)
        ref.insert(**other)
        gpu.read_data_bv(data, vol)
        assert ref.read_data_bv(data, vol)
        field = gpu.value_field()
        assert_value_fields_equal(field, ref.value_field(), what="volume %d" % i)
        check_inner_against_field(gpu, field, ref.sensor_model(), levels=(1, 2, 3, 4, 5, 7))
        gpu.close()
    src.close()


@pytest.mark.parametrize("color", [False, True])
def test_set_value_volume_every_shape(color):
    kw = dict(resolution=0.05)
    gpu = Map(color=color, initial_blocks=1 << 12, **kw)
    ref = volumes_lib.VolumesRefMap(color=color, **kw)
    rng = np.random.default_rng(41)
    values = [0.1192, 0.7, 0.5, 0.99, 0.3]
    i = 0
    for k in range(3):
        o, p, c = scans.rgbd(k=k, width=56, height=42)
        ins = dict(origin=o, xyz=p, rgb=c if color else None, max_range=3.0, discrete=True)
        gpu.insert(**ins)
        ref.insert(**ins)
        # centres straddle brick borders (16 voxels = 0.8 m)
        shapes = _shapes(np.array([0.8, 0.0, 0.0]) + rng.uniform(-0.3, 0.3, 3), 0.6, rng)
        for kind, shape in enumerate(shapes):
            if kind in (capi.PLANE, capi.RAY):
                continue  # a 0.05 m map of 16 levels is too large for these (below)
            md = 0 if color else (i % 5)
            val = values[i % len(values)]
            gpu.set_value_volume_bv(shape, val, md)
            ref.set_value_volume_bv(shape, val, md)
            field = gpu.value_field()
            assert_value_fields_equal(field, ref.value_field(), color_tol=0,
                                      what="shape %d, scan %d, depth %d" % (kind, k, md))
            i += 1
    check_inner_against_field(gpu, ref.value_field(), ref.sensor_model(), levels=(1, 2, 3, 4, 5, 6, 9, 16))
    gpu.close()


@pytest.mark.parametrize("depth_levels", [10, 11, 12])
def test_set_value_volume_planes_and_rays_on_small_maps(depth_levels):
    kw = dict(resolution=0.1, depth_levels=depth_levels)
    gpu = Map(initial_blocks=1 << 12, **kw)
    ref = volumes_lib.VolumesRefMap(**kw)
    o, p = scans.random_shell(n=1500)
    gpu.insert(o, p, max_range=5.0)
    ref.insert(o, p, max_range=5.0)
    # the reference's tree of a plane holds (2^L)^2 voxels: planes on the two smaller maps only
    planes = [capi.plane([0, 0, 1], 0.3), capi.plane([0.6, 0.0, 0.8], -1.0)] if depth_levels < 12 else []
    edge = 0.1 * 2 ** (depth_levels - 1)  # the map spans [-edge, edge] on every axis
    q = np.array([0.9, 0.1, 0.3, 0.2]) / np.linalg.norm([0.9, 0.1, 0.3, 0.2])
    shapes = planes + [capi.sphere([edge - 0.2, 0.3, 0.2], 0.8), capi.obb([-edge + 0.1, -edge, 0.0], [0.6, 0.6, 0.6], q),
              capi.aabb([edge - 1.0, -0.5, -0.5], [edge + 3.0, 0.5, 0.5]),
              
              capi.volume_record(capi.RAY, volumes_lib.ref_ray([0.1, 0.2, 0.3], [1, 0, 0])),
              capi.volume_record(capi.RAY, volumes_lib.ref_ray([-2.0, 1.0, 0.5], [0.3, -0.4, 0.5]))]
    for j, shape in enumerate(shapes):
        md = j % 3
        gpu.set_value_volume_bv(shape, 0.2 if j % 2 else 0.8, md)
        ref.set_value_volume_bv(shape, 0.2 if j % 2 else 0.8, md)
        assert_value_fields_equal(gpu.value_field(), ref.value_field(), what="shape %d" % j)
        gpu.insert(o, p, max_range=5.0)
        ref.insert(o, p, max_range=5.0)
    field = gpu.value_field()
    assert_value_fields_equal(field, ref.value_field(), what="after the last scan")
    check_inner_against_field(gpu, field, ref.sensor_model(), levels=(1, 2, 3, 4, 5, 6, 9))
    gpu.close()


def test_set_value_volume_over_the_brick_limit_is_rejected():
    gpu = Map(0.05, initial_blocks=1 << 12)
    o, p = scans.velodyne64(k=0, rings=8, azimuths=128)
    gpu.insert(o, p, max_range=10.0)
    before = gpu.value_field()
    with pytest.raises(UfoError) as e:
        gpu.set_value_volume_bv(capi.plane([0, 0, 1], 0.0), 0.9, 0)  # ~ (3277 m / 0.8 m)^2 bricks
    assert e.value.status == E_UNSUPPORTED
    assert_value_fields_equal(gpu.value_field(), before, what="after the rejected call")
    with pytest.raises(UfoError) as e:
        gpu.set_value_volume_bv(capi.sphere([0, 0, 0], 1.0), 0.9, 5)
    assert e.value.status == E_UNSUPPORTED
    gpu.close()


def _centres_of(codes, d, levels, resolution):
    """Per level l = levels-1 .. d: the centre of the depth-l ancestor of each depth-d cell,
    accumulated from the root like getChildCenter."""
    half = [resolution / 2.0, resolution]
    while len(half) <= levels:
        half.append(half[-1] * 2.0)
    c = np.zeros((len(codes), 3))
    out = []
    for lvl in range(levels - 1, d - 1, -1):
        idx = ((codes >> np.uint64(3 * lvl)) & np.uint64(7)).astype(np.int64)
        c = c + np.stack([np.where(idx & 1, half[lvl], -half[lvl]), np.where(idx & 2, half[lvl], -half[lvl]),
                          np.where(idx & 4, half[lvl], -half[lvl])], 1)
        out.append((lvl, c.copy(), half[lvl]))
    return out


@pytest.mark.parametrize("name", ["velodyne", "rgbd_color_discrete"])
def test_leaf_iteration_matches_the_reference(name):
    """export_nodes_bv == beginLeaves(volume, ...) at depths 0..6.  A leaf the reference returns
    collapsed above the depth is expanded into its cells; of those, the cells whose path below the
    reference's node leaves the volume are not part of the device's answer."""
    gpu, ref, _, _ = _maps(name)
    kw, _, _ = _scenario(name)
    rng = np.random.default_rng(9)
    vols = _volumes(gpu, ref, rng)
    for i in (0, 1, 2, 3, 4, 6, 7, 8, 10, 11, 12):
        vol = vols[i]
        for d in (0, 1, 2, 3, 4, 6):
            for flt in (dict(), dict(free=False), dict(occupied=False)):
                rc, rd, rv = ref.leaves_bv(vol, min_depth=d, **flt)
                cells, cv, cdep = [], [], []
                for D in np.unique(rd):
                    sel = rd == D
                    base = (rc[sel] >> np.uint64(3 * D)) << np.uint64(3 * D)
                    reps = 1 << (3 * (int(D) - d))
                    offs = np.arange(reps, dtype=np.uint64) << np.uint64(3 * d)
                    cells.append((base[:, None] + offs[None, :]).reshape(-1))
                    cv.append(np.repeat(rv[sel], reps))
                    cdep.append(np.full(sel.sum() * reps, D))
                want_c = np.concatenate(cells) if cells else np.empty(0, np.uint64)
                want_v = np.concatenate(cv) if cv else np.empty(0, np.float32)
                want_d = np.concatenate(cdep) if cdep else np.empty(0, np.int64)
                keep = np.ones(len(want_c), bool)
                if len(vol) and len(want_c):
                    for lvl, cen, hs in _centres_of(want_c, d, gpu.depth_levels, kw["resolution"]):
                        below = want_d > lvl
                        if below.any():
                            keep[below] &= capi.volume_intersects(vol, cen[below], hs)
                order = np.argsort(want_c[keep], kind="stable")
                want_c, want_v = want_c[keep][order], want_v[keep][order]
                gc, gv, _ = gpu.export_nodes_bv(vol, depth=d, **flt)
                gc = (gc >> np.uint64(3 * d)) << np.uint64(3 * d)
                assert np.array_equal(gc, want_c), (i, d, flt, len(gc), len(want_c))
                assert np.array_equal(gv.view(np.uint32), want_v.view(np.uint32)), (i, d, flt)
    gpu.close()


def test_rejections():
    gpu = Map(0.1, initial_blocks=1 << 10)
    bad = capi.volume_record(9, [0, 0, 0])
    for call in (lambda: gpu.write_data_bv(bad), lambda: gpu.export_nodes_bv(bad), lambda: gpu.set_value_volume_bv(bad, 0.5),
                 lambda: gpu.read_data_bv(b"\x00" + b"\x00" * 4, bad)):
        with pytest.raises(UfoError) as e:
            call()
        assert e.value.status == capi.E_INVALID
    with pytest.raises(UfoError) as e:
        gpu.write_data_bv(capi.sphere([0, 0, 0], 1.0), 5)
    assert e.value.status == E_UNSUPPORTED
    gpu.close()
    col = Map(0.1, color=True, initial_blocks=1 << 10)
    with pytest.raises(UfoError) as e:
        col.set_value_volume_bv(capi.sphere([0, 0, 0], 1.0), 0.5, 1)
    assert e.value.status == E_UNSUPPORTED
    col.close()
