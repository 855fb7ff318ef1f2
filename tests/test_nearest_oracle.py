"""The two CPU checkers of the nearest-first iteration agree (TEST INFRASTRUCTURE, no GPU): the
reference's beginTree / beginLeaves stable-sorted by its own squared distance, and the reference's
best-first search restated with the popped-node test fixed.  Per distance both hold the same nodes
(as a multiset: the queue orders ties its own way), and the sorted sequence is non-decreasing.  The
best-first order itself may step back by an ulp or two: centres accumulate rounding, so a child's cube
can stick out of its parent's by that much."""
import itertools

import numpy as np
import pytest

import nearest_lib
from ufomap_b200 import capi, scans

pytestmark = pytest.mark.skipif(not nearest_lib.have_ref(), reason="reference nearest checker not built")


def _map(color):
    if color:
        m = nearest_lib.NearestRefMap(0.04, color=True)
        for k in range(2):
            o, p, c = scans.rgbd(k=k, width=24, height=18)
            m.insert(o, p, rgb=c, max_range=3.0, discrete=True)
        return m
    m = nearest_lib.NearestRefMap(0.1)
    for k in range(2):
        o, p = scans.velodyne64(k=k, rings=6, azimuths=64)
        m.insert(o, p, max_range=12.0)
    return m


def _groups(res):
    """{d2 bits: sorted list of (code, depth, occ bits, flags, rgb, centre bits)}"""
    codes, depths, occ, flags, rgb, centres, d2 = res
    out = {}
    for i in range(len(codes)):
        key = int(d2[i:i + 1].view(np.uint64)[0])
        out.setdefault(key, []).append((int(codes[i]), int(depths[i]), int(occ[i:i + 1].view(np.uint32)[0]), int(flags[i]),
                                        bytes(rgb[i]), centres[i].tobytes()))
    return {k: sorted(v) for k, v in out.items()}


@pytest.mark.parametrize("color", [False, True])
def test_checkers_agree(color):
    m = _map(color)
    res = 0.04 if color else 0.1
    points = [np.array([0.33, -0.71, 0.12]), np.array([2 * res, -3 * res, res]), np.array([500.0, -20.0, 3.0])]
    vols = {"none": None, "sphere": [capi.sphere([0.2, 0.1, 0.0], 1.5)]}
    total = 0
    for p, (vname, vol), leaves, flt, contains, md in itertools.product(
            points, vols.items(), (True, False), ((1, 0, 0), (1, 1, 0), (0, 1, 1)), (False, True), (0, 5)):
        kw = dict(leaves=leaves, occupied=flt[0], free=flt[1], unknown=flt[2], contains=contains, min_depth=md)
        a = m.nearest(p, vol, kind="sorted", **kw)
        b = m.nearest(p, vol, kind="bestfirst", **kw)
        assert np.all(np.diff(a[6]) >= 0), kw
        assert np.array_equal(a[6].view(np.uint64), np.sort(b[6]).view(np.uint64)), (vname, kw)
        assert _groups(a) == _groups(b), (vname, kw)
        total += len(a[0])
    assert total > 0
    m.close()
