"""The dense ray walk merges duplicate marks before they reach memory (ufo_walk.cuh, drain_marks):
records of a 32-record drain that mark the same 64-bit word of the scan volume become one global
reduction.  The value field must not change -- it is checked against the generic record path
(UFO_B200_MARK=records, one mark per record, no merging) and against the plain-C oracle -- and the
walk counters (profiling level 2) must show the merge."""
import ctypes as C

import numpy as np
import pytest

from ufomap_b200 import capi, scans


def test_walk_stats_binding():
    assert "ufo_b200_last_walk_stats" in capi.SYMBOLS
    assert [n for n, _ in capi.WalkStats._fields_] == ["records", "mask_reductions", "words_marked",
                                                       "dirty_reductions"]
    assert C.sizeof(capi.WalkStats) == 32
    lib = capi.load()
    st = capi.WalkStats()
    assert lib.ufo_b200_last_walk_stats(None, C.byref(st)) == capi.E_INVALID
    m = capi.Map(0.1, device=-2)  # geometry-only handle: no device needed
    assert lib.ufo_b200_last_walk_stats(m.h, None) == capi.E_INVALID
    m.close()


def _converging(w=160, h=120, seed=3):
    """A depth image: w x h rays in pixel order (neighbouring rays cross the same blocks) from a
    0.8..3 m surface onto one sensor voxel, 60 degree horizontal field of view."""
    rng = np.random.default_rng(seed)
    f = (w / 2) / np.tan(np.radians(30.0))
    u, v = np.meshgrid(np.arange(w) - (w - 1) / 2, np.arange(h) - (h - 1) / 2)
    d = np.stack([np.full(u.size, f), u.ravel(), v.ravel()], axis=1)
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    r = 1.9 + 0.6 * np.sin(u.ravel() / 17.0) * np.cos(v.ravel() / 11.0) + rng.uniform(-0.3, 0.3, u.size)
    origin = np.array([0.013, -0.007, 0.021])
    return origin, origin + d * r[:, None]


def _gpu_map(res, origin, pts, max_range, records, monkeypatch):
    if records:
        monkeypatch.setenv("UFO_B200_MARK", "records")
    else:
        monkeypatch.delenv("UFO_B200_MARK", raising=False)
    m = capi.Map(res, initial_bricks=1 << 19)
    monkeypatch.delenv("UFO_B200_MARK", raising=False)
    m.set_profiling(2)
    m.insert(origin, pts, max_range=max_range)
    return m


def _check(res, origin, pts, max_range, monkeypatch, oracle_stride=1):
    from helpers import assert_value_fields_equal
    from oracle_lib import OracleMap

    dense = _gpu_map(res, origin, pts, max_range, False, monkeypatch)
    ws = dense.walk_stats()
    field = dense.value_field()
    dense.close()
    rec = _gpu_map(res, origin, pts, max_range, True, monkeypatch)
    assert rec.walk_stats()["records"] == 0  # the record path does not use the dense walk
    assert_value_fields_equal(field, rec.value_field(), what="records path")
    rec.close()
    if oracle_stride > 1:
        # the oracle on a subsample of the rays, against the dense walk on the same subsample
        pts = pts[::oracle_stride]
        sub = _gpu_map(res, origin, pts, max_range, False, monkeypatch)
        field = sub.value_field()
        sub.close()
    cpu = OracleMap(res)
    cpu.insert(origin, pts, max_range=max_range)
    assert_value_fields_equal(field, cpu.value_field(), what="oracle")
    cpu.close()
    assert 0 < ws["words_marked"] <= ws["mask_reductions"] <= ws["records"], ws
    assert 0 < ws["dirty_reductions"] <= ws["mask_reductions"], ws
    return ws


@pytest.mark.gpu
def test_converging_scan_merges(monkeypatch):
    origin, pts = _converging()
    ws = _check(0.01, origin, pts, 5.0, monkeypatch)
    # every ray crosses the few blocks around the sensor: most records merge
    assert ws["mask_reductions"] * 2 < ws["records"], ws


@pytest.mark.gpu
def test_velodyne_scan_merges(monkeypatch):
    """Config #2 shape: 2 cm, 131 072-ray Velodyne-64 scan, 30 m."""
    origin, pts = scans.velodyne64(k=0)
    ws = _check(0.02, origin, pts, 30.0, monkeypatch, oracle_stride=8)
    # one reduction per record before merging; about 1.95 records per reduction on the H100
    assert ws["mask_reductions"] * 3 < ws["records"] * 2, ws


@pytest.mark.gpu
def test_counters_off_without_profiling(monkeypatch):
    origin, pts = _converging(w=40, h=30)
    monkeypatch.delenv("UFO_B200_MARK", raising=False)
    m = capi.Map(0.01)
    m.set_profiling(1)
    m.insert(origin, pts, max_range=5.0)
    assert m.walk_stats() == {"records": 0, "mask_reductions": 0, "words_marked": 0, "dirty_reductions": 0}
    m.set_profiling(2)
    m.insert(origin, pts, max_range=5.0)
    assert m.walk_stats()["records"] > 0
    m.close()
