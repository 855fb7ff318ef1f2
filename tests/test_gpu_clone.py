"""Device copies of maps (ufo_b200_clone, Map.clone): the copy holds the source's value field, file
image, iteration and query results, as does a map that read the source's image; the same later calls
(scans, write batches, colour batches, setValueVolume) keep all three equal, and nothing done to the
copy reaches the source.  Change detection and the change box start empty; the copy's pools grow
under later scans.  Routed and sharded maps are refused with nothing changed.  Against the compiled
reference: its copy constructor and the facade's copy (clone, then the sensor model through the
probability getters) store bitwise-equal log-odds and give equal value fields after further scans."""
import ctypes as C

import numpy as np
import pytest

import info_lib
from color_writes_lib import mixed_color_batch
from ufomap_b200 import scans
from ufomap_b200.capi import E_UNSUPPORTED, Map, UfoError

pytestmark = pytest.mark.gpu


def _scan(color, k):
    if color:
        o, p, c = scans.rgbd(k=k, width=64, height=48)
        return dict(origin=o, xyz=p, rgb=c, max_range=3.0, discrete=True)
    o, p = scans.velodyne64(k=k, rings=16, azimuths=256)
    return dict(origin=o, xyz=p, max_range=15.0)


def _source(color, k_max=2, **kw):
    m = Map(0.04 if color else 0.1, 16, color=color, device=0, **kw)
    for k in range(k_max):
        m.insert(**_scan(color, k))
    return m


def _same(a, b, what):
    ca, va, ra = a.value_field()
    cb, vb, rb = b.value_field()
    assert np.array_equal(ca, cb), what
    assert np.array_equal(va.view(np.uint32), vb.view(np.uint32)), what
    assert np.array_equal(ra, rb), what
    assert a.write() == b.write(), what
    ia, ib = a.iterate(), b.iterate()
    for x, y in zip(ia, ib):
        assert np.array_equal(x, y), what
    if len(ca):
        idx = np.linspace(0, len(ca) - 1, 500).astype(np.int64)
        depths = (np.arange(len(idx)) % 7).astype(np.uint32)
        codes = ca[idx] & ~((np.uint64(1) << (np.uint64(3) * depths.astype(np.uint64))) - np.uint64(1))
        qa, qb = a.query(codes, depths), b.query(codes, depths)
        for x, y in zip(qa, qb):
            assert np.array_equal(np.asarray(x).view(np.uint8), np.asarray(y).view(np.uint8)), what


def _twin(src):
    t = Map(src.resolution, src.depth_levels, color=src.color, device=0)
    t.read(src.write())
    return t


@pytest.mark.parametrize("color", [False, True])
def test_clone_equals_source_and_image_twin(color):
    src = _source(color)
    image = src.write()
    c = src.clone()
    assert src.write() == image
    assert np.array_equal(c.sensor_model().view(np.uint64), src.sensor_model().view(np.uint64))
    twin = _twin(src)
    _same(c, src, "clone")
    _same(c, twin, "twin")
    # a change to the copy does not reach the source
    c.insert(**_scan(color, 5))
    assert src.write() == image
    c.close()
    assert src.write() == image


@pytest.mark.parametrize("color", [False, True])
def test_later_calls_keep_source_clone_and_twin_equal(color):
    src = _source(color)
    c = src.clone()
    twin = _twin(src)
    maps = (src, c, twin)
    for k in (2, 3):
        for m in maps:
            m.insert(**_scan(color, k))
    _same(c, src, "scans")
    _same(c, twin, "scans, twin")
    rng = np.random.default_rng(7)
    pts = rng.uniform(-3, 3, size=(400, 3))
    depths = rng.integers(0, 4, size=400).astype(np.uint32)
    codes = np.array([src.to_code(p, int(d)) for p, d in zip(pts, depths)], np.uint64)
    vals = rng.choice([0.85, -0.4, 1.3, -2.0], size=400).astype(np.float32)
    for m in maps:
        m.update_nodes(codes, depths, 0, vals)
    _same(c, src, "write batch")
    if color:
        batch = mixed_color_batch(3000, seed=11)
        for m in maps:
            m.update_nodes_color(*batch)
        _same(c, src, "colour batch")
    box = (np.array([-1.0, -1.5, -0.5]), np.array([1.5, 1.0, 0.6]))
    for m in maps:
        m.set_value_volume(box, 0.3, 0)
    _same(c, src, "setValueVolume")
    _same(c, twin, "setValueVolume, twin")


def test_changes_and_change_box_are_not_carried_over():
    src = Map(0.1, 16, device=0)
    src.enable_change_detection(True)
    src.insert(**_scan(False, 0))
    assert len(src.changed_codes()) > 0
    mn, mx = src.change_bbox()
    assert np.all(mn <= mx)
    c = src.clone()
    assert len(c.changed_codes()) == 0
    cmn, cmx = c.change_bbox()
    assert np.all(cmn > cmx)  # reset: nothing changed yet
    c.insert(**_scan(False, 1))
    assert len(c.changed_codes()) == 0  # detection is off on the copy
    assert len(src.changed_codes()) > 0


def test_pools_and_growth():
    src = _source(False, initial_bricks=64)
    ps = src.pool_stats()
    c = src.clone()
    pc = c.pool_stats()
    assert pc["bricks"] == ps["bricks"]
    assert pc["brick_cap"] == max(64, 2 * ps["bricks"])
    assert pc["up_cap"] >= pc["brick_cap"] // 2
    twin = _twin(src)
    for k in range(2, 8):
        s = _scan(False, k)
        s["origin"] = np.asarray(s["origin"]) + np.array([6.0 * k, 0.0, 0.0])
        s["xyz"] = np.asarray(s["xyz"]) + np.array([6.0 * k, 0.0, 0.0])
        c.insert(**s)
        twin.insert(**s)
    assert c.pool_stats()["brick_cap"] > pc["brick_cap"]
    _same(c, twin, "grown")


def test_refusals_change_nothing():
    routed = Map(0.1, 16, device=0)
    routed.route_setup(0, 2, cap_bricks=1 << 8, cap_hits=1 << 10)
    sharded = Map(0.1, 16, device=0)
    sharded.set_shard(0, 2)
    sharded.insert(**_scan(False, 0))
    for m in (routed, sharded):
        before, field = m.pool_stats(), m.value_field()
        with pytest.raises(UfoError) as e:
            m.clone()
        assert e.value.status == E_UNSUPPORTED
        assert m.pool_stats() == before
        for x, y in zip(m.value_field(), field):
            assert np.array_equal(x, y)


def _expf():
    f = C.CDLL("libm.so.6").expf
    f.restype = C.c_float
    f.argtypes = [C.c_float]
    return f


@pytest.mark.skipif(not info_lib.have_ref(), reason="reference info checker not built")
@pytest.mark.parametrize("color", [False, True])
def test_copy_constructor_matches_the_reference(color):
    model = dict(occupied_thres=0.61, free_thres=0.37, prob_hit=0.7123456789, prob_miss=0.3987654321,
                 clamping_thres_min=0.1234567, clamping_thres_max=0.9712345)
    res = 0.04 if color else 0.1
    src = Map(res, 16, color=color, device=0, **model)
    ref = info_lib.InfoRefMap(res, 16, color=color, **model)
    for k in range(2):
        src.insert(**_scan(color, k))
        ref.insert(**_scan(color, k))
    # the facade's copy: clone, then the reference constructor's toLogit of the probability getters,
    # which evaluate toProb on the float log-odds with the float exponential
    expf = _expf()
    probs = [1.0 / (1.0 + float(expf(-float(np.float32(x))))) for x in src.sensor_model()]
    c = src.clone()
    c.set_sensor_model(*probs)
    rc = ref.copy()
    assert np.array_equal(c.sensor_model().view(np.uint64), rc.sensor_model().view(np.uint64))
    for k in (2, 3):
        c.insert(**_scan(color, k))
        rc.insert(**_scan(color, k))
    gc, gv, gr = c.value_field()
    wc, wv, wr = rc.value_field()
    assert np.array_equal(gc, wc)
    assert np.array_equal(gv.view(np.uint32), wv.view(np.uint32))
    if color:
        assert np.array_equal(gr, wr)
