"""Writers on routed maps: setValueVolume (both forms), write batches (update_nodes,
update_nodes_color, insert_rays) and the mapping server's loop.  Every rank takes the same call and
applies it to the bricks it owns, so the union of the ranks equals the single map.  As in
test_gpu_route.py, several maps on ONE device play the ranks and a stream synchronisation stands in
for the barrier.

  * setValueVolume, AABB and sphere / frustum, min_depth 0 and 3, colour at 0: union value field
    and depth 1-4 aggregates == single map (== the C restatement for the AABB form); no rank holds
    a brick it does not own
  * update_nodes (ADD / SET at depths 0/3/6), update_nodes_color, insert_rays with hit_end: same
  * a call between route_mark and the last route_apply is refused and changes nothing
  * a rank whose pools grow during a write batch takes further routed scans
  * the server loop -- routed insert, clearing of the robot's box, change-box publish -- gives the
    bytes a single map gives
"""
import numpy as np
import pytest

from color_writes_lib import codes_of, mixed_color_batch
from helpers import assert_value_fields_equal
from oracle_lib import OracleMap
from test_gpu_route_discrete import _barrier, _brick_owner, _ranks, _union
from ufomap_b200 import capi, scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu

CLAMP_MIN = 0.1192


def _routed_scan(maps, k, depth=0, discrete=True, color=False):
    """One velodyne scan (rgbd for colour) split over the ranks; returns what a single map inserts."""
    world = len(maps)
    if color:
        o, p, rgb = scans.rgbd(k=k, width=96, height=72)
        rng_max = 5.0
    else:
        o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
        rgb, rng_max = None, 10.0
    buf, layout = capi.pack_points(p, rgb, np.float32)
    keep = []
    for r, m in enumerate(maps):
        part = np.ascontiguousarray(buf[r::world])
        keep.append(part)
        m.route_mark_ex(o, part.ctypes.data, len(part), layout, max_range=rng_max, depth=depth, discrete=discrete,
                        index_base=r, index_stride=world)
    _barrier(maps)
    for m in maps:
        m.route_apply(0, world, True)
    _barrier(maps)
    return dict(origin=o, xyz=p, rgb=rgb, max_range=rng_max, depth=depth, discrete=discrete, dtype=np.float32)


def _assert_union_equals(maps, single, what):
    assert_value_fields_equal(_union(maps), single.value_field(), what=what)
    for d in (1, 2, 3, 4):
        parts = [m.export_nodes(depth=d) for m in maps]
        codes = np.concatenate([p[0] for p in parts])
        order = np.argsort(codes, kind="stable")
        got = (codes[order], np.concatenate([p[1] for p in parts])[order], np.concatenate([p[2] for p in parts])[order])
        assert_value_fields_equal(got, single.export_nodes(depth=d), what="%s, depth-%d aggregates" % (what, d))


def _assert_owned(maps, single):
    """Every brick of every rank is its own: the ranks' brick counts add up to the single map's,
    and every brick holding a value belongs to the rank that holds it."""
    world = len(maps)
    assert sum(m.pool_stats()["bricks"] for m in maps) == single.pool_stats()["bricks"]
    for r, m in enumerate(maps):
        bricks = np.unique(m.value_field()[0] >> np.uint64(12))
        assert (_brick_owner(bricks << np.uint64(12), world) == r).all(), "rank %d holds a foreign brick" % r


def _frustum():
    return capi.frustum7([-4.0, -1.0, 0.5], [3.0, 1.0, 0.0], [0, 0, 1], 0.6, 0.9, 0.5, 9.0)


# (name, colour, min_depth, shape): shape None is the AABB form
VOLUME_CASES = [
    ("aabb-d0", False, 0, None),
    ("aabb-d3", False, 3, None),
    ("sphere-d0", False, 0, "sphere"),
    ("frustum-d3", False, 3, "frustum"),
    ("color-aabb-d0", True, 0, None),
    ("color-sphere-d0", True, 0, "sphere"),
]


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("case", VOLUME_CASES, ids=[c[0] for c in VOLUME_CASES])
def test_set_value_volume(case, world):
    _, color, min_depth, shape = case
    res = 0.02 if color else 0.05
    maps = _ranks(world, res, color=color)
    single = Map(res, color=color, initial_bricks=1 << 15)
    oracle = OracleMap(res) if not color else None
    box = (np.array([-2.13, -1.07, -0.61]), np.array([1.91, 2.23, 0.87]))
    for k in range(2):
        ins = _routed_scan(maps, k, color=color)
        single.insert(**ins)
        if oracle is not None:
            oracle.insert(ins["origin"], ins["xyz"], max_range=ins["max_range"], discrete=True)
    for occupancy in (CLAMP_MIN, 0.83):
        for m in maps + [single]:
            if shape is None:
                m.set_value_volume(box, occupancy, min_depth)
            elif shape == "sphere":
                m.set_value_volume_bv(capi.sphere([0.37, -0.41, 0.22], 1.7), occupancy, min_depth)
            else:
                m.set_value_volume_bv(_frustum(), occupancy, min_depth)
        if oracle is not None and shape is None:
            oracle.set_value_volume(box, occupancy, min_depth)
    _assert_union_equals(maps, single, "setValueVolume %s" % case[0])
    if oracle is not None and shape is None:
        assert_value_fields_equal(single.value_field(), oracle.value_field(), what="single map vs oracle")


@pytest.mark.parametrize("shape", [None, "sphere", "frustum"])
def test_set_value_volume_creates_only_owned_bricks(shape):
    world, res = 4, 0.05
    maps = _ranks(world, res)
    single = Map(res, initial_bricks=1 << 15)
    for m in maps + [single]:
        if shape is None:
            m.set_value_volume(([-1.5, -2.0, -0.5], [2.5, 1.0, 1.0]), 0.8, 0)
        elif shape == "sphere":
            m.set_value_volume_bv(capi.sphere([0.3, 0.2, -0.1], 1.6), 0.8, 0)
        else:
            m.set_value_volume_bv(_frustum(), 0.8, 0)
    assert single.pool_stats()["bricks"] > 0
    _assert_owned(maps, single)
    _assert_union_equals(maps, single, "setValueVolume into empty ranks")


def _node_batch(rng, n, depths):
    keys = rng.integers(32768 - 300, 32768 + 300, size=(n, 3))
    d = rng.choice(np.asarray(depths, np.uint32), size=n).astype(np.uint32)
    ops = rng.integers(0, 2, size=n).astype(np.uint8)
    vals = rng.choice(np.float32([0.85, -0.41, 2.3, -1.7, 0.0]), size=n).astype(np.float32)
    return codes_of(keys, d), d, ops, vals


@pytest.mark.parametrize("world", [2, 4])
def test_write_batches(world):
    res = 0.05
    maps = _ranks(world, res)
    single = Map(res, initial_bricks=1 << 15)
    rng = np.random.default_rng(7)
    ins = _routed_scan(maps, 0)
    single.insert(**ins)
    # ADD and SET at depths 0 / 3 / 6, every code several times, in one ordered batch
    codes, depths, ops, vals = _node_batch(rng, 3000, [0, 3, 6])
    codes, depths, ops, vals = (np.concatenate([a, a[::-1]]) for a in (codes, depths, ops, vals))
    for m in maps + [single]:
        m.update_nodes(codes, depths, ops, vals)
    _assert_union_equals(maps, single, "update_nodes")
    # rays with the hit on the given end point, at depths 0 and 3
    o, p = scans.velodyne64(k=1, rings=8, azimuths=256)
    for depth in (0, 3):
        for m in maps + [single]:
            m.insert_rays(o, p, max_range=8.0, depth=depth, hit_end=True)
    _assert_union_equals(maps, single, "insert_rays")
    # and the ranks still take routed scans
    single.insert(**_routed_scan(maps, 2))
    _assert_union_equals(maps, single, "routed scan after writes")


@pytest.mark.parametrize("world", [2, 4])
def test_color_write_batches(world):
    res = 0.02
    maps = _ranks(world, res, color=True)
    single = Map(res, color=True, initial_bricks=1 << 15)
    single.insert(**_routed_scan(maps, 0, color=True))
    codes, depths, ops, vals, rgb = mixed_color_batch(4000, seed=11, half=120, set_ops=True)
    for m in maps + [single]:
        m.update_nodes_color(codes, depths, ops, vals, rgb)
    _assert_union_equals(maps, single, "update_nodes_color")


def test_calls_between_mark_and_apply_are_refused():
    world, res = 2, 0.05
    maps = _ranks(world, res)
    _routed_scan(maps, 0)
    o, p = scans.velodyne64(k=1, rings=8, azimuths=256)
    buf, layout = capi.pack_points(p, None, np.float32)
    for m in maps:
        m.route_mark(o, buf.ctypes.data, len(buf), layout, max_range=10.0)
    _barrier(maps)
    code = maps[0].to_code([0.3, 0.2, 0.1])
    calls = [
        lambda m: m.set_value_volume(([-1, -1, -1], [1, 1, 1]), 0.9),
        lambda m: m.set_value_volume_bv(capi.sphere([0, 0, 0], 1.0), 0.9),
        lambda m: m.update_nodes([code], 0, Map.ADD, 1.0),
        lambda m: m.insert_rays([0.0, 0.0, 0.0], [[2.0, 1.0, 0.5]], hit_end=True),
        lambda m: m.image_part(),
    ]
    for call in calls:
        for m in maps:
            with pytest.raises(capi.UfoError) as e:
                call(m)
            assert e.value.status == capi.E_INVALID
    # the pass completes, then the refused calls had left nothing behind
    for m in maps:
        m.route_apply(0, world, True)
    _barrier(maps)
    ref = [Map(res, initial_bricks=1 << 15) for _ in range(world)]
    ptrs = [m.route_setup(r, world) for r, m in enumerate(ref)]
    for m in ref:
        m.route_connect(ptrs)
    _routed_scan(ref, 0)
    for m in ref:
        m.route_mark(o, buf.ctypes.data, len(buf), layout, max_range=10.0)
    _barrier(ref)
    for m in ref:
        m.route_apply(0, world, True)
    _barrier(ref)
    for m, r in zip(maps, ref):
        assert_value_fields_equal(m.value_field(), r.value_field(), what="after refused calls")


def test_pool_growth_during_a_write_batch():
    """Ranks created with a small pool grow inside a write batch (outside any routed pass), then
    take further routed scans.  The batch covers the space the scans reach with depth-6 nodes, so
    the grown pools hold the scans (pools do not grow during a routed pass)."""
    world, res = 2, 0.05
    maps = _ranks(world, res, bricks=1 << 8)
    single = Map(res, initial_bricks=1 << 8)
    cap0 = [m.pool_stats()["brick_cap"] for m in maps]
    lo, hi = np.array([-11.0, -11.0, -2.5]), np.array([11.0, 11.0, 1.5])
    axes = [np.arange(lo[a], hi[a], 64 * res) for a in range(3)]
    centres = np.stack(np.meshgrid(*axes, indexing="ij"), axis=-1).reshape(-1, 3)
    keys = np.floor(centres / res).astype(np.int64) + 32768
    rng = np.random.default_rng(3)
    codes, depths, ops, vals = _node_batch(rng, 3000, [0, 3, 6])
    codes = np.concatenate([codes_of(keys, np.full(len(keys), 6, np.uint32)), codes])
    depths = np.concatenate([np.full(len(keys), 6, np.uint32), depths])
    ops = np.concatenate([np.zeros(len(keys), np.uint8), ops])
    vals = np.concatenate([np.full(len(keys), -0.2, np.float32), vals])
    for m in maps + [single]:
        m.update_nodes(codes, depths, ops, vals)
    assert all(m.pool_stats()["brick_cap"] > c for m, c in zip(maps, cap0)), "the pools grew"
    _assert_union_equals(maps, single, "after growth")
    for k in range(2):
        single.insert(**_routed_scan(maps, k))
    _assert_union_equals(maps, single, "routed scans after growth")


def _box_of(bbs):
    mn = np.min([b[0] for b in bbs], axis=0)
    mx = np.max([b[1] for b in bbs], axis=0)
    return mn, mx


@pytest.mark.parametrize("world", [2, 4])
def test_server_loop(world):
    """Per step: routed discrete insert, clear the robot's box at the clamp minimum, publish the
    change box (the min / max of the ranks' boxes) at depths 0 and 2 -- the bytes a single map
    writes for that box -- and reset the change boxes."""
    res = 0.05
    maps = _ranks(world, res)
    single = Map(res, initial_bricks=1 << 15)
    for k in range(3):
        ins = _routed_scan(maps, k, depth=0, discrete=True)
        single.insert(**ins)
        o = ins["origin"]
        robot = (o - np.array([0.6, 0.4, 0.9]), o + np.array([0.6, 0.4, 0.3]))
        for m in maps + [single]:
            m.set_value_volume(robot, CLAMP_MIN, 0)
        vol = capi.aabb(*_box_of([m.change_bbox() for m in maps]))
        for depth in (0, 2):
            parts = [m.image_part(volume=vol, min_depth=depth) for m in maps]
            got = capi.assemble_image(parts, with_header=False)
            assert got == single.write_data_bv(vol, min_depth=depth), "step %d depth %d" % (k, depth)
        for m in maps + [single]:
            m.reset_change_bbox()
    parts = [m.image_part() for m in maps]
    assert capi.assemble_image(parts) == single.write_bv()
    _assert_union_equals(maps, single, "server loop")
