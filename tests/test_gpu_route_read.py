"""readData on routed maps (ufo_b200_read_data[_bv] after ufo_b200_route_setup): every rank takes the
same stream and applies the part that falls in the bricks it owns, so the union of the ranks equals
one map that read the stream.  As in test_gpu_route.py, several maps on ONE device play the ranks
and a stream synchronisation stands in for the barrier.

  * streams of a scanned map (min_depth 0 / 2 / 4, LZ4, AABB / sphere / frustum + OBB volumes) and a
    stream with non-default collapsed nodes above the brick level, read into empty ranks: union
    value field and image == the single map's (2 and 4 ranks, mono and colour)
  * merged into ranks that hold routed scans -- default-payload nodes above the brick level delete
    subtrees -- and followed by more routed scans: == the single map after every step
  * an image of N ranks read into M ranks re-assembles to the same bytes (== the compiled
    reference's readData + write where it is built)
  * no rank holds a non-empty brick it does not own, and a read creates no foreign brick
  * rejections: the same status on every rank and nothing changed
  * ranks with small pools grow during the read and then take routed scans
"""
import numpy as np
import pytest

from helpers import assert_value_fields_equal
from oracle_lib import RefMap, have_ref
from test_gpu_route_discrete import _barrier, _brick_owner, _ranks, _union
from test_gpu_route_writes import _routed_scan
from ufomap_b200 import capi, scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu


def _res(color):
    return 0.02 if color else 0.05


def _scan(color, k):
    """What a single map inserts for scan k (the one _routed_scan splits over the ranks)."""
    if color:
        o, p, rgb = scans.rgbd(k=k, width=96, height=72)
        return dict(origin=o, xyz=p, rgb=rgb, max_range=5.0, discrete=True, dtype=np.float32)
    o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
    return dict(origin=o, xyz=p, max_range=10.0, discrete=True, dtype=np.float32)


def _source(color, ks):
    m = Map(_res(color), color=color, initial_bricks=1 << 15)
    for k in ks:
        m.insert(**_scan(color, k))
    return m


def _collapsed(color):
    """A map whose stream holds non-default collapsed nodes of depth 7 and 5: setValueVolume over one
    whole depth-7 node and one whole depth-5 node, and over a box that ends inside its nodes."""
    res = _res(color)
    m = Map(res, color=color, initial_bricks=1 << 14)
    e = 0.25 * res
    m.set_value_volume(([e, e, e], [128 * res - e] * 3), 0.9, 0)
    m.set_value_volume(([-32 * res + e, e, -32 * res + e], [-e, 32 * res - e, -e]), 0.3, 0)
    m.set_value_volume(([-40 * res + e, -21 * res, e], [-3 * res, -e, 50 * res]), 0.7, 0)
    return m


def _volumes(color):
    s = 0.4 if color else 1.0
    return {
        "aabb": capi.aabb(np.array([-2.1, -1.3, -0.9]) * s, np.array([1.7, 2.9, 0.6]) * s),
        "sphere": capi.sphere(np.array([1.1, -0.7, 0.1]) * s, 1.9 * s),
        "frustum+obb": [capi.frustum7(np.array([-5.0, 0.5, 0.4]) * s, [0.0, 0.0, 0.0], [0, 0, 1], 0.5, 0.8, 0.3 * s,
                                      6.0 * s),
                        capi.obb(np.array([0.8, 1.9, -0.2]) * s, np.array([1.2, 0.6, 0.4]) * s,
                                 [0.9238795, 0.0, 0.0, 0.3826834])],
    }


def _bricks(maps):
    return [m.pool_stats()["bricks"] for m in maps]


def _check(maps, single, what, before=None):
    """The ranks' union equals `single`: value field and file image.  No rank holds a non-empty
    brick it does not own; with `before` (brick counts of maps + [single] before the last read) the
    read created as many bricks over the ranks as on the single map, so none of them foreign."""
    assert_value_fields_equal(_union(maps), single.value_field(), what=what)
    assert capi.assemble_image([m.image_part() for m in maps]) == single.write(), "%s: image" % what
    for r, m in enumerate(maps):
        bricks = np.unique(m.value_field()[0] >> np.uint64(12))
        assert (_brick_owner(bricks << np.uint64(12), len(maps)) == r).all(), "%s: rank %d holds a foreign brick" % (
            what, r)
    if before is not None:
        after = _bricks(maps + [single])
        grown = [a - b for a, b in zip(after, before)]
        assert sum(grown[:-1]) == grown[-1], "%s: bricks created %r" % (what, grown)


def _read(maps, data, **kw):
    for m in maps:
        m.read_data_bv(data, **kw)
    _barrier(maps)


def _close(maps):
    for m in maps:
        m.close()


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("color", [False, True], ids=["mono", "color"])
def test_union_equals_single_map(color, world):
    src = _source(color, (0, 1))
    streams = [("min_depth %d" % d, src.write_data(min_depth=d), {}) for d in (0, 2, 4)]
    packed, usize = src.write_compressed(data_only=True)
    streams.append(("lz4", packed, dict(compressed=True, uncompressed_size=usize)))
    # a stream is read with the volume it was written with
    streams += [(name, src.write_data_bv(vol), dict(volume=vol)) for name, vol in _volumes(color).items()]
    col = _collapsed(color)
    data = col.write_data()
    assert len(data) < 1 << 16, "the whole depth-7 node is one collapsed node"
    streams.append(("collapsed", data, {}))
    for name, data, kw in streams:
        maps = _ranks(world, _res(color), bricks=1 << 14, color=color)
        single = Map(_res(color), color=color, initial_bricks=1 << 14)
        before = _bricks(maps + [single])
        _read(maps + [single], data, **kw)
        assert single.pool_stats()["bricks"] > 0, name
        _check(maps, single, name, before)
        _close(maps + [single])
    for m in (src, col):
        m.close()


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("color", [False, True], ids=["mono", "color"])
def test_merge_into_routed_scans(color, world):
    """Routed scans, then streams of other maps (their default-payload nodes above the brick level
    delete what the scans left there), then more routed scans."""
    res = _res(color)
    maps = _ranks(world, res, color=color)
    single = Map(res, color=color, initial_bricks=1 << 15)
    single.insert(**_routed_scan(maps, 0, color=color))
    _check(maps, single, "routed scan")
    other = _source(color, (3,))
    col = _collapsed(color)
    vol = _volumes(color)["sphere"]
    steps = [("whole stream", other.write_data(), {}),
             ("min_depth 2 in a sphere", other.write_data_bv(vol, 2), dict(volume=vol)),
             ("collapsed nodes", col.write_data(), {})]
    for name, data, kw in steps:
        before = _bricks(maps + [single])
        _read(maps + [single], data, **kw)
        _check(maps, single, name, before)
    for k in (1, 2):
        single.insert(**_routed_scan(maps, k, color=color))
        _check(maps, single, "routed scan %d after the reads" % k)
    _close(maps + [single, other, col])


def _group(world, res, bricks=1 << 15):
    return _ranks(world, res, bricks=bricks) if world > 1 else [Map(res, initial_bricks=bricks)]


@pytest.mark.parametrize("n,m", [(1, 2), (2, 4), (4, 2), (2, 1)])
def test_load_onto_a_different_number_of_gpus(n, m):
    res = 0.05
    src = _group(n, res)
    for k in range(3):
        if n > 1:
            _routed_scan(src, k)
        else:
            src[0].insert(**_scan(False, k))
    parts = [s.image_part() for s in src]
    image = capi.assemble_image(parts)
    stream = capi.assemble_image(parts, with_header=False)
    dst = _group(m, res)
    single = Map(res, initial_bricks=1 << 15)
    before = _bricks(dst + [single])
    _read(dst + [single], stream)
    assert capi.assemble_image([d.image_part() for d in dst]) == image
    _check(dst, single, "%d -> %d ranks" % (n, m), before)
    if have_ref():
        ref = RefMap(res)
        assert ref.read_data(stream)
        assert ref.write() == image
    # and the loaded ranks take the next scan like one map
    if m > 1:
        single.insert(**_routed_scan(dst, 3))
    else:
        for d in dst + [single]:
            d.insert(**_scan(False, 3))
    _check(dst, single, "scan after the load")
    _close(src + dst + [single])


def _state(m):
    return m.write(), m.pool_stats()


def test_rejections_are_the_same_on_every_rank():
    world, res = 2, 0.05
    maps = _ranks(world, res)
    _routed_scan(maps, 0)
    src = _source(False, (1,))
    data = src.write_data()
    packed, usize = src.write_compressed(data_only=True)
    huge = b"\x00" + np.float32(0.5).tobytes()  # the root as one non-default leaf: 2^36 bricks
    bad = [
        ("truncated", lambda m: m.read_data(data[:-1]), capi.E_INVALID),
        ("truncated lz4 input", lambda m: m.read_data(packed[:len(packed) // 2], compressed=True,
                                                      uncompressed_size=usize), capi.E_INVALID),
        ("lz4 size", lambda m: m.read_data(packed, compressed=True, uncompressed_size=usize - 1), capi.E_INVALID),
        ("volume", lambda m: m.read_data_bv(data, capi.volume_record(9, [0, 0, 0])), capi.E_INVALID),
        ("budget", lambda m: m.read_data(huge), capi.E_UNSUPPORTED),
    ]
    for name, call, status in bad:
        before = [_state(m) for m in maps]
        for m in maps:
            with pytest.raises(capi.UfoError) as e:
                call(m)
            assert e.value.status == status, name
        assert [_state(m) for m in maps] == before, name
    # between route_mark and the last route_apply of a pass
    o, p = scans.velodyne64(k=1, rings=8, azimuths=256)
    buf, layout = capi.pack_points(p, None, np.float32)
    for m in maps:
        m.route_mark(o, buf.ctypes.data, len(buf), layout, max_range=10.0)
    _barrier(maps)
    for m in maps:
        with pytest.raises(capi.UfoError) as e:
            m.read_data(data)
        assert e.value.status == capi.E_INVALID
    for m in maps:
        m.route_apply(0, world, True)
    _barrier(maps)
    ref = _ranks(world, res)
    _routed_scan(ref, 0)
    for m in ref:
        m.route_mark(o, buf.ctypes.data, len(buf), layout, max_range=10.0)
    _barrier(ref)
    for m in ref:
        m.route_apply(0, world, True)
    _barrier(ref)
    for m, r in zip(maps, ref):
        assert _state(m) == _state(r), "the refused read left nothing behind"
    _close(maps + ref + [src])


def test_shallow_ranks_refuse_a_read():
    world = 2
    maps = [Map(0.25, depth_levels=4, initial_bricks=1 << 10) for _ in range(world)]
    ptrs = [m.route_setup(r, world) for r, m in enumerate(maps)]
    for m in maps:
        m.route_connect(ptrs)
    def state(m):  # no file image below depth_levels 5
        return [a.tobytes() for a in m.value_field()] + [m.pool_stats()]

    before = [state(m) for m in maps]
    for m in maps:
        with pytest.raises(capi.UfoError) as e:
            m.read_data(b"\x00" + np.float32(0.5).tobytes())
        assert e.value.status == capi.E_UNSUPPORTED
    assert [state(m) for m in maps] == before
    _close(maps)


def test_pool_growth_during_a_read():
    """Ranks created with a small pool grow inside the read, then take routed scans.  The stream
    covers the space the scans reach, so the grown pools hold the scans (pools do not grow during a
    routed pass)."""
    world, res = 2, 0.05
    maps = _ranks(world, res, bricks=1 << 8)
    single = Map(res, initial_bricks=1 << 8)
    cap0 = [m.pool_stats()["brick_cap"] for m in maps]
    src = Map(res, initial_bricks=1 << 15)
    src.set_value_volume(([-11.0, -11.0, -2.5], [11.0, 11.0, 1.5]), 0.45, 0)
    src.insert(**_scan(False, 4))
    before = _bricks(maps + [single])
    _read(maps + [single], src.write_data())
    assert all(m.pool_stats()["brick_cap"] > c for m, c in zip(maps, cap0)), "the pools grew"
    _check(maps, single, "after growth", before)
    for k in range(2):
        single.insert(**_routed_scan(maps, k))
        _check(maps, single, "routed scan %d after growth" % k)
    _close(maps + [single, src])
