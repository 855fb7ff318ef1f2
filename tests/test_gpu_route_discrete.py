"""Routed multi-GPU mode with every option of the single-GPU insert except early_stopping
(ufo_b200_route_mark_ex): discrete insertion, colour maps, insert depths 1-6, simple ray casting.
As in test_gpu_route.py, several maps on ONE device play the ranks and a stream synchronisation
stands in for the barrier.

  * one scan split by rays (interleaved and contiguous sectors, world 2 and 4): union of the
    ranks' value fields == single-GPU map fed the whole scan with the same call, colour included
  * colour winner: the lowest GLOBAL cloud index of a hit voxel blends, wherever it sits
  * colour sensors merged in sensor order == single map inserting them one after the other ==
    the reference's insertPointCloudDiscrete on OccupancyMapColor
  * insert depth 5/6 sends whole bricks: no rank allocates a brick it does not own
  * rejected calls apply nothing
"""
import numpy as np
import pytest

from helpers import assert_value_fields_equal
from oracle_lib import RefMap, have_ref
from ufomap_b200 import capi, scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu

_M64 = np.uint64(0xFFFFFFFFFFFFFFFF)


def _ranks(world, resolution, bricks=1 << 15, color=False, **kw):
    maps = [Map(resolution, color=color, initial_bricks=bricks) for _ in range(world)]
    ptrs = [m.route_setup(r, world, **kw) for r, m in enumerate(maps)]
    for m in maps:
        m.route_connect(ptrs)
    return maps


def _union(maps):
    parts = [m.value_field() for m in maps]
    codes = np.concatenate([p[0] for p in parts])
    assert len(np.unique(codes)) == len(codes), "ranks own disjoint bricks"
    order = np.argsort(codes, kind="stable")
    return codes[order], np.concatenate([p[1] for p in parts])[order], np.concatenate([p[2] for p in parts])[order]


def _barrier(maps):
    for m in maps:
        m.wait()


def _compact(c):
    """Every third bit of a Morton code -> one key axis."""
    c = c & np.uint64(0x1249249249249249)
    c = (c ^ (c >> np.uint64(2))) & np.uint64(0x10C30C30C30C30C3)
    c = (c ^ (c >> np.uint64(4))) & np.uint64(0x100F00F00F00F00F)
    c = (c ^ (c >> np.uint64(8))) & np.uint64(0x1F0000FF0000FF)
    c = (c ^ (c >> np.uint64(16))) & np.uint64(0x1F00000000FFFF)
    c = (c ^ (c >> np.uint64(32))) & np.uint64(0x1FFFFF)
    return c


def _brick_owner(codes, world):
    """Owner rank of the bricks of depth-0 voxel codes (brick_owner of ufo_device.cuh)."""
    codes = np.asarray(codes, np.uint64)
    bx, by, bz = (_compact(codes >> np.uint64(a)) >> np.uint64(4) for a in range(3))
    k = bx | (by << np.uint64(21)) | (bz << np.uint64(42))
    k = k ^ np.uint64(0x9E3779B97F4A7C15)
    with np.errstate(over="ignore"):
        k ^= k >> np.uint64(33)
        k = (k * np.uint64(0xFF51AFD7ED558CCD)) & _M64
        k ^= k >> np.uint64(33)
        k = (k * np.uint64(0xC4CEB9FE1A85EC53)) & _M64
        k ^= k >> np.uint64(33)
    h = k & np.uint64(0xFFFFFFFF)
    return ((h >> np.uint64(7)) % np.uint64(world)).astype(np.int64)


def _split(buf, world, how):
    """(part, index_base, index_stride) of every rank."""
    if how == "interleaved":
        return [(np.ascontiguousarray(buf[r::world]), r, world) for r in range(world)]
    cut = np.linspace(0, len(buf), world + 1).astype(np.int64)
    return [(np.ascontiguousarray(buf[cut[r]:cut[r + 1]]), int(cut[r]), 1) for r in range(world)]


# (name, colour, depth, discrete, simple)
CASES = [
    ("mono-discrete-d0", False, 0, True, False),
    ("mono-discrete-d2", False, 2, True, False),
    ("mono-discrete-d3", False, 3, True, False),
    ("mono-discrete-d6", False, 6, True, False),
    ("mono-simple-d0", False, 0, False, True),
    ("mono-simple-d3", False, 3, False, True),
    ("color-plain-d0", True, 0, False, False),
    ("color-plain-d6", True, 6, False, False),
    ("color-discrete-d0", True, 0, True, False),
    ("color-discrete-d6", True, 6, True, False),
]


def _scan(color, k):
    if color:
        o, p, rgb = scans.rgbd(k=k, width=160, height=120)
        return o, p, rgb, 0.02, 5.0
    o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
    return o, p, None, 0.05, 10.0


@pytest.mark.parametrize("how", ["interleaved", "sectors"])
@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_one_scan_split_by_rays(case, world, how):
    _, color, depth, discrete, simple = case
    res = _scan(color, 0)[3]
    maps = _ranks(world, res, color=color)
    single = Map(res, color=color, initial_bricks=1 << 15)
    opts = dict(depth=depth, discrete=discrete, simple=simple)
    for k in range(2):
        o, p, rgb, _, rng_max = _scan(color, k)
        buf, layout = capi.pack_points(p, rgb, np.float32)
        single.insert(o, p, rgb=rgb, max_range=rng_max, dtype=np.float32, **opts)
        parts = _split(buf, world, how)
        for m, (part, base, stride) in zip(maps, parts):
            m.route_mark_ex(o, part.ctypes.data, len(part), layout, max_range=rng_max, index_base=base,
                            index_stride=stride, **opts)
        _barrier(maps)
        for m in maps:
            m.route_apply(0, world, True)
        _barrier(maps)
    ref = single.value_field()
    assert len(ref[0]) > 0
    assert_value_fields_equal(_union(maps), ref, what="routed union vs single GPU")
    st = [m.stats() for m in maps]
    assert sum(s["touched_voxels"] for s in st) == single.stats()["touched_voxels"]


@pytest.mark.parametrize("discrete", [False, True])
def test_colour_winner_is_lowest_global_index(discrete):
    """Two points of one scan hit one voxel with different colours; the lower global index sits on
    the rank that does NOT own the voxel.  Its colour wins, blended as the single map blends it
    (second pass: onto the colour the first pass left)."""
    res, world = 0.05, 2
    maps = _ranks(world, res, bricks=1 << 12, color=True)
    single = Map(res, color=True, initial_bricks=1 << 12)
    swapped = Map(res, color=True, initial_bricks=1 << 12)
    origin = np.array([0.013, 0.021, 0.007])
    # a voxel centre owned by rank 1; rank 0 holds the winning point
    target = None
    for i in range(4096):
        c = np.array([2.0 + 0.8 * (i % 16), 0.8 * ((i // 16) % 16) - 6.0, 0.8 * (i // 256) - 6.0])
        key = np.floor(c / res)
        c = (key + 0.5) * res
        code = single.to_code(c)
        if _brick_owner(np.array([code], np.uint64), world)[0] == 1:
            target = c
            break
    assert target is not None
    a_pt = target + np.array([-0.01, 0.005, 0.0])
    b_pt = target + np.array([0.01, -0.005, 0.01])
    colours = [((200, 10, 30), (20, 220, 40)), ((5, 100, 250), (250, 250, 5))]
    for ca, cb in colours:
        single.insert(origin, [a_pt, b_pt], rgb=[ca, cb], discrete=discrete, dtype=np.float32)
        swapped.insert(origin, [b_pt, a_pt], rgb=[cb, ca], discrete=discrete, dtype=np.float32)
        bufa, layout = capi.pack_points([a_pt], [ca], np.float32)
        bufb, _ = capi.pack_points([b_pt], [cb], np.float32)
        maps[0].route_mark_ex(origin, bufa.ctypes.data, 1, layout, discrete=discrete, index_base=0, index_stride=1)
        maps[1].route_mark_ex(origin, bufb.ctypes.data, 1, layout, discrete=discrete, index_base=1, index_stride=1)
        _barrier(maps)
        for m in maps:
            m.route_apply(0, world, True)
        _barrier(maps)
        field = _union(maps)
        ref = single.value_field()
        assert_value_fields_equal(field, ref, what="routed colour winner vs single GPU")
        i = np.searchsorted(ref[0], np.uint64(single.to_code(target)))
        assert ref[0][i] == single.to_code(target)
        other = swapped.value_field()
        j = np.searchsorted(other[0], ref[0][i])
        if (ca, cb) == colours[0]:
            assert tuple(field[2][i]) == ca  # empty leaf: the winner's colour as it is
        assert tuple(field[2][i]) != tuple(other[2][j]), "the winner decides the colour"


def test_colour_sensors_merged_in_sensor_order():
    """Two overlapping RGB-D views at 8 mm, one per rank, discrete insertion; every owner applies
    sensor 0's marks and colours, then sensor 1's."""
    res, world = 0.008, 2
    maps = _ranks(world, res, bricks=1 << 16, color=True)
    single = Map(res, color=True, initial_bricks=1 << 16)
    ref = RefMap(res, color=True) if have_ref() else None
    for k in range(2):
        keep = []
        for s, m in enumerate(maps):
            origin = np.array([0.0013 + 0.02 * k + 0.3 * s, 0.0021 + 0.01 * k - 0.25 * s, 0.0007])
            o, p, rgb = scans.rgbd(k=k, width=160, height=120, origin=origin)
            single.insert(o, p, rgb=rgb, max_range=6.0, discrete=True, dtype=np.float32)
            if ref is not None:
                ref.insert(o, p, rgb=rgb, max_range=6.0, discrete=True)
            buf, layout = capi.pack_points(p, rgb, np.float32)
            keep.append(buf)
            m.route_mark_ex(o, buf.ctypes.data, len(buf), layout, max_range=6.0, discrete=True, self_too=True)
        _barrier(maps)
        for s in range(world):
            for m in maps:
                m.route_apply(s, 1, s == world - 1)
        _barrier(maps)
    field = _union(maps)
    assert_value_fields_equal(field, single.value_field(), what="merged colour sensors vs single GPU")
    if ref is not None:
        assert_value_fields_equal(field, ref.value_field(), color_tol=0, what="merged colour sensors vs reference")


@pytest.mark.parametrize("color", [False, True])
@pytest.mark.parametrize("depth", [5, 6])
def test_deep_insert_allocates_no_foreign_bricks(depth, color):
    world = 2
    res = 0.02 if color else 0.05
    maps = _ranks(world, res, color=color)
    single = Map(res, color=color, initial_bricks=1 << 15)
    for k in range(2):
        o, p, rgb, _, rng_max = _scan(color, k)
        buf, layout = capi.pack_points(p, rgb, np.float32)
        single.insert(o, p, rgb=rgb, max_range=rng_max, depth=depth, discrete=color, dtype=np.float32)
        for m, (part, base, stride) in zip(maps, _split(buf, world, "interleaved")):
            m.route_mark_ex(o, part.ctypes.data, len(part), layout, max_range=rng_max, depth=depth,
                            discrete=color, index_base=base, index_stride=stride)
        _barrier(maps)
        sent = [m.route_sent() for m in maps]
        assert all(s["full_brick_records"] > 0 for s in sent)
        for m in maps:
            m.route_apply(0, world, True)
        _barrier(maps)
    assert_value_fields_equal(_union(maps), single.value_field(), what="depth %d routed vs single GPU" % depth)
    for r, m in enumerate(maps):
        codes = m.value_field()[0]
        bricks = np.unique(codes >> np.uint64(12))
        assert m.stats()["bricks_in_map"] == len(bricks), "rank %d holds bricks without values" % r
        assert (_brick_owner(bricks << np.uint64(12), world) == r).all(), "rank %d holds a foreign brick" % r


def test_rejected_calls_apply_nothing():
    res, world = 0.05, 2
    maps = _ranks(world, res)
    cmaps = _ranks(world, res, bricks=1 << 12, color=True)
    o, p = scans.velodyne64(k=0, rings=8, azimuths=256)
    buf, layout = capi.pack_points(p, None, np.float32)
    for m in maps:
        m.route_mark_ex(o, buf.ctypes.data, len(buf), layout, max_range=10.0, discrete=True, index_base=0,
                        index_stride=1, self_too=True)
    _barrier(maps)
    for s in range(world):
        for m in maps:
            m.route_apply(s, 1, s == world - 1)
    _barrier(maps)
    before = [m.value_field() for m in maps]
    bad = [(dict(early_stopping=1), capi.E_UNSUPPORTED), (dict(depth=7), capi.E_UNSUPPORTED),
           (dict(index_stride=0), capi.E_INVALID)]
    for kw, status in bad:
        for m in maps:
            with pytest.raises(capi.UfoError) as e:
                m.route_mark_ex(o, buf.ctypes.data, len(buf), layout, max_range=10.0, **kw)
            assert e.value.status == status, kw
    _, pc, rgb = scans.rgbd(width=32, height=24)
    cbuf, clayout = capi.pack_points(pc, rgb, np.float32)
    for m in cmaps:
        with pytest.raises(capi.UfoError) as e:
            m.route_mark(o, cbuf.ctypes.data, len(cbuf), clayout)
        assert e.value.status == capi.E_UNSUPPORTED
        assert m.stats()["bricks_in_map"] == 0
    _barrier(maps)
    for m, b in zip(maps, before):
        assert_value_fields_equal(m.value_field(), b, what="after rejected calls")
    # the ranks still take a pass after the rejections
    for m in maps:
        m.route_mark_ex(o, buf.ctypes.data, len(buf), layout, max_range=10.0, depth=3)
    _barrier(maps)
    for m in maps:
        m.route_apply(0, world, True)
    _barrier(maps)
