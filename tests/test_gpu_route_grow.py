"""Routed passes grow their pools instead of failing.  Ranks created with tiny pools (16-64 bricks)
run every kind of routed pass; a full pool grows while marking (route_mark waits for its marking
kernels, grows and marks again before anything is published) or while applying (the apply calls from
the one that backed off are replayed at the next synchronising call).  As in test_gpu_route.py,
several maps on ONE device play the ranks and a stream synchronisation stands in for the barrier.

  * one scan split by rays (mono plain, colour discrete, insert depth 3 / 5 / 6, simple ray
    casting, the record path): every rank equals a pre-sized rank leaf for leaf and node for node at
    depths 1-6 and 9, the union equals the single map, the inner aggregates follow from the leaves
  * config #5 shape, mono and colour: one sensor per rank, merged in sensor order with self_too
  * growth only while marking, only while applying (a later apply call of the pass backs off too),
    and an apply left unsynchronised until the next pass's route_mark
  * a grown routed map takes setValueVolume, a write batch and image assembly like a pre-sized one
  * an inbox region that is too small is still refused with UFO_B200_E_NOMEM
"""
import numpy as np
import pytest

from helpers import assert_value_fields_equal, check_inner_against_field
from oracle_lib import OracleMap, RefMap, have_ref
from test_gpu_route_discrete import _barrier, _split, _union
from test_gpu_route_writes import _node_batch
from ufomap_b200 import capi, scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu

TINY = 16
BIG = 1 << 16
LEVELS = (1, 2, 3, 4, 5, 6, 9)


def _ranks(world, res, sizes, color=False, **kw):
    maps = [Map(res, color=color, initial_bricks=b) for b in sizes]
    ptrs = [m.route_setup(r, world, **kw) for r, m in enumerate(maps)]
    for m in maps:
        m.route_connect(ptrs)
    return maps


def _caps(maps):
    return [m.pool_stats()["brick_cap"] for m in maps]


def _same_rank(grown, sized, what):
    """One rank of a grown map holds what the same rank of a pre-sized map holds: leaves, colours and
    the aggregates of every inner level, bit for bit."""
    field = sized.value_field()
    assert_value_fields_equal(grown.value_field(), field, what=what)
    for lvl in LEVELS:
        q = np.unique(field[0] >> np.uint64(3 * lvl)) << np.uint64(3 * lvl)
        a, b = grown.query(q, lvl), sized.query(q, lvl)
        assert np.array_equal(a[0].view(np.uint32), b[0].view(np.uint32)), "%s: level %d max" % (what, lvl)
        assert np.array_equal(a[1], b[1]), "%s: level %d flags" % (what, lvl)
        if grown.color:
            assert np.array_equal(a[2], b[2]), "%s: level %d colours" % (what, lvl)


def _check(grown, sized, single, model, what):
    for r, (g, s) in enumerate(zip(grown, sized)):
        _same_rank(g, s, "%s, rank %d" % (what, r))
        check_inner_against_field(g, g.value_field(), model, levels=LEVELS)
    assert_value_fields_equal(_union(grown), single.value_field(), what="%s: union vs single GPU" % what)


def _scan(color, k):
    if color:
        o, p, rgb = scans.rgbd(k=k, width=160, height=120)
        return o, p, rgb, 0.02, 5.0
    o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
    return o, p, None, 0.05, 10.0


# (name, colour, depth, discrete, simple, UFO_B200_MARK)
CASES = [
    ("mono-plain", False, 0, False, False, None),
    ("mono-records", False, 0, False, False, "records"),
    ("mono-d3", False, 3, False, False, None),
    ("mono-d5", False, 5, False, False, None),
    ("mono-simple", False, 0, False, True, None),
    ("color-discrete", True, 0, True, False, None),
    ("color-discrete-d6", True, 6, True, False, None),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_one_scan_split_by_rays(case, monkeypatch):
    name, color, depth, discrete, simple, mark = case
    if mark:
        monkeypatch.setenv("UFO_B200_MARK", mark)  # read when a map is created
    world = 2
    res = _scan(color, 0)[3]
    grown = _ranks(world, res, [TINY] * world, color=color)
    sized = _ranks(world, res, [BIG] * world, color=color)
    single = Map(res, color=color, initial_bricks=BIG)
    oracle = OracleMap(res) if not color and depth == 0 and not simple else None
    opts = dict(depth=depth, discrete=discrete, simple=simple)
    regrows = [0] * world
    for k in range(2):
        o, p, rgb, _, rng_max = _scan(color, k)
        buf, layout = capi.pack_points(p, rgb, np.float32)
        single.insert(o, p, rgb=rgb, max_range=rng_max, dtype=np.float32, **opts)
        if oracle is not None:
            oracle.insert(o, p, max_range=rng_max)
        parts = _split(buf, world, "interleaved")
        for maps in (grown, sized):
            for m, (part, base, stride) in zip(maps, parts):
                if name == "mono-plain":
                    m.route_mark(o, part.ctypes.data, len(part), layout, max_range=rng_max)
                else:
                    m.route_mark_ex(o, part.ctypes.data, len(part), layout, max_range=rng_max, index_base=base,
                                    index_stride=stride, **opts)
            _barrier(maps)
            for m in maps:
                m.route_apply(0, world, True)
            _barrier(maps)
        regrows = [n + m.stats()["regrows"] for n, m in zip(regrows, grown)]
        assert all(m.stats()["regrows"] == 0 for m in sized)
    assert all(n > 0 for n in regrows), "every rank grew: %r" % regrows
    assert all(c > TINY for c in _caps(grown))
    model = OracleMap(res).sensor_model()
    _check(grown, sized, single, model, name)
    if oracle is not None:
        assert_value_fields_equal(single.value_field(), oracle.value_field(), what="single GPU vs oracle")


@pytest.mark.parametrize("color", [False, True], ids=["mono", "color"])
def test_sensors_merged_in_sensor_order(color):
    """Config #5 shape: one sensor per rank, every owner applies the sensors one after the other."""
    world = 2
    res = 0.008 if color else 0.04
    grown = _ranks(world, res, [TINY, 64], color=color)
    sized = _ranks(world, res, [BIG] * world, color=color)
    single = Map(res, color=color, initial_bricks=BIG)
    cpus = [RefMap(res, color=color)] if have_ref() else []
    if not color:
        cpus.append(OracleMap(res))
    for k in range(2):
        keep = []
        for s in range(world):
            if color:
                origin = np.array([0.0013 + 0.02 * k + 0.3 * s, 0.0021 + 0.01 * k - 0.25 * s, 0.0007])
                o, p, rgb = scans.rgbd(k=k, width=160, height=120, origin=origin)
                opts = dict(max_range=6.0, discrete=True)
            else:
                base = scans.sensor_ring(s, 8) + np.array([0.25 * k, 0.10 * k, 0.0])
                o, p = scans.velodyne64(k=k, rings=16, azimuths=512, origin=base, seed=88172645463325252 + 7919 * s)
                rgb, opts = None, dict(max_range=30.0)
            single.insert(o, p, rgb=rgb, dtype=np.float32, **opts)
            for c in cpus:
                c.insert(o, p, rgb=rgb, **opts)
            buf, layout = capi.pack_points(p, rgb, np.float32)
            keep.append(buf)
            for maps in (grown, sized):
                maps[s].route_mark_ex(o, buf.ctypes.data, len(buf), layout, self_too=True, **opts)
        for maps in (grown, sized):
            _barrier(maps)
            for s in range(world):
                for m in maps:
                    m.route_apply(s, 1, s == world - 1)
            _barrier(maps)
    assert all(c > s for c, s in zip(_caps(grown), [TINY, 64]))
    model = OracleMap(res).sensor_model()
    _check(grown, sized, single, model, "merged sensors")
    for c in cpus:
        assert_value_fields_equal(_union(grown), c.value_field(), what="merged sensors vs %s" % type(c).__name__)


@pytest.mark.parametrize("phase", ["mark", "apply", "apply-async"])
def test_growth_in_one_phase(phase):
    """mark: rank 0 walks every ray into a tiny pool, the other ranks walk none and own large pools;
    rank 0's own marks stay local, so it grows while marking and never while applying.
    apply: rank 0 walks no ray but owns a third of the bricks, ranks 1 and 2 walk one half of the
    scan each, and the owners merge the sensors one after the other (self_too).  Rank 0's pool runs
    full in its second apply call (sensor 1), and its third call (sensor 2) backs off with it: both
    are replayed.  apply-async: the same without a wait after the apply calls, so that the next
    pass's route_mark replays them."""
    world, res = 3, 0.05
    grown = _ranks(world, res, [TINY, BIG, BIG])
    sized = _ranks(world, res, [BIG] * world)
    single = Map(res, initial_bricks=BIG)
    oracle = OracleMap(res)
    for k in range(3):
        o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
        half = len(p) // 2
        clouds = [p] if phase == "mark" else [p[:half], p[half:]]
        for c in clouds:
            single.insert(o, c, max_range=10.0, dtype=np.float32)
            oracle.insert(o, c, max_range=10.0)
        bufs = [capi.pack_points(c, None, np.float32)[0] for c in clouds]
        layout = capi.pack_points(p[:1], None, np.float32)[1]
        empty = bufs[0][:0]
        parts = [bufs[0], empty, empty] if phase == "mark" else [empty] + bufs
        cap0 = _caps(grown) if phase != "apply-async" else None  # (a synchronising call: no replay here)
        for maps in (grown, sized):
            for m, q in zip(maps, parts):
                m.route_mark(o, q.ctypes.data, len(q), layout, max_range=10.0, self_too=phase != "mark")
            _barrier(maps)
        cap_marked = _caps(grown)
        if k == 0:
            assert (cap_marked[0] > TINY) == (phase == "mark"), "growth while marking: %r" % cap_marked
        for maps in (grown, sized):
            if phase == "mark":
                for m in maps:
                    m.route_apply(0, world, True)
            else:
                for s in range(world):
                    for m in maps:
                        m.route_apply(s, 1, s == world - 1)
            if phase != "apply-async" or maps is sized or k == 2:
                _barrier(maps)
        if phase == "mark":
            assert _caps(grown) == cap_marked, "no growth while applying"
        elif phase == "apply" and k == 0:
            assert cap_marked == cap0 and _caps(grown)[0] > TINY, "growth while applying"
            assert grown[0].stats()["regrows"] > 0
    assert _caps(grown)[0] > TINY
    model = OracleMap(res).sensor_model()
    _check(grown, sized, single, model, phase)
    assert_value_fields_equal(single.value_field(), oracle.value_field(), what="single GPU vs oracle")


def test_apply_replayed_inside_the_next_mark():
    """The replay of an unsynchronised apply happens in the next route_mark: rank 0's pool grows
    there, before its own (empty) marking."""
    world, res = 2, 0.05
    grown = _ranks(world, res, [TINY, BIG])
    o, p = scans.velodyne64(k=0, rings=16, azimuths=512)
    buf, layout = capi.pack_points(p, None, np.float32)
    empty = buf[:0]
    grown[0].route_mark(o, empty.ctypes.data, 0, layout, max_range=10.0, self_too=True)
    grown[1].route_mark(o, buf.ctypes.data, len(buf), layout, max_range=10.0, self_too=True)
    _barrier(grown)
    cap = _caps(grown)[0]
    for m in grown:
        m.route_apply(0, world, True)
    grown[1].wait()
    grown[0].route_mark(o, empty.ctypes.data, 0, layout, max_range=10.0, self_too=True)
    assert grown[0].pool_stats()["brick_cap"] > cap
    grown[1].route_mark(o, empty.ctypes.data, 0, layout, max_range=10.0, self_too=True)
    _barrier(grown)
    for m in grown:
        m.route_apply(0, world, True)
    _barrier(grown)
    single = Map(res, initial_bricks=BIG)
    single.insert(o, p, max_range=10.0, dtype=np.float32)
    assert_value_fields_equal(_union(grown), single.value_field(), what="replayed in the next mark")


def _routed_scan(maps, k):
    world = len(maps)
    o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
    buf, layout = capi.pack_points(p, None, np.float32)
    parts = [np.ascontiguousarray(buf[r::world]) for r in range(world)]
    for m, part in zip(maps, parts):
        m.route_mark_ex(o, part.ctypes.data, len(part), layout, max_range=10.0, discrete=True, index_base=0,
                        index_stride=1)
    _barrier(maps)
    for m in maps:
        m.route_apply(0, world, True)
    _barrier(maps)
    return dict(origin=o, xyz=p, max_range=10.0, discrete=True, dtype=np.float32)


def test_grown_map_takes_writers_and_image_assembly():
    world, res = 2, 0.05
    grown = _ranks(world, res, [TINY] * world)
    sized = _ranks(world, res, [BIG] * world)
    single = Map(res, initial_bricks=BIG)
    for k in range(2):
        ins = _routed_scan(grown, k)
        _routed_scan(sized, k)
        single.insert(**ins)
    assert all(c > TINY for c in _caps(grown))
    codes, depths, ops, vals = _node_batch(np.random.default_rng(5), 3000, [0, 3])
    for m in grown + sized + [single]:
        m.set_value_volume(([-1.5, -2.0, -0.5], [2.5, 1.0, 1.0]), 0.8, 0)
        m.update_nodes(codes, depths, ops, vals)
    model = OracleMap(res).sensor_model()
    _check(grown, sized, single, model, "after writers")
    got = capi.assemble_image([m.image_part() for m in grown])
    assert got == capi.assemble_image([m.image_part() for m in sized])
    assert got == single.write_bv()


def test_undersized_inbox_is_still_refused():
    world, res = 2, 0.05
    maps = _ranks(world, res, [TINY] * world, cap_bricks=4, cap_hits=4)
    o, p = scans.velodyne64(k=0, rings=16, azimuths=512)
    buf, layout = capi.pack_points(p, None, np.float32)
    parts = [np.ascontiguousarray(buf[r::world]) for r in range(world)]
    for m, part in zip(maps, parts):
        m.route_mark(o, part.ctypes.data, len(part), layout, max_range=10.0)
    status = []
    for m in maps:
        try:
            m.wait()
            status.append(capi.OK)
        except capi.UfoError as e:
            status.append(e.status)
    assert capi.E_NOMEM in status
