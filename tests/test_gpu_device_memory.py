"""Device memory a map owns: every pool array follows the pool's capacity in every state (the change
masks while detection is switched off included), and ufo_b200_pool_stats' device_bytes is the sum of
the allocations the map holds, whatever order its buffers were sized in."""
import numpy as np
import pytest

from ufomap_b200 import scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu

BIG = 1 << 15  # bricks: no scan below outgrows this pool


def _scan(k, rings, azimuths):
    o, p = scans.velodyne64(k=k, rings=rings, azimuths=azimuths)
    return dict(origin=o, xyz=p)


def test_change_masks_follow_the_pool_while_paused():
    """Two maps take the same calls; one of them grows its brick pool while change detection is
    switched off.  Capacity must not change what is recorded."""
    small = _scan(0, 8, 64)
    wide = [_scan(k, 16, 512) for k in range(1, 4)]
    maps = {"fixed": Map(0.2, initial_bricks=BIG), "growing": Map(0.2, initial_bricks=16)}
    caps, changed = {}, {}
    for name, m in maps.items():
        m.enable_change_detection()
        m.insert(**small, max_range=5.0)
        m.enable_change_detection(False)
        cap_paused = m.pool_stats()["brick_cap"]
        for s in wide:
            m.insert(**s, max_range=40.0)
        caps[name] = (cap_paused, m.pool_stats()["brick_cap"])
        m.reset_change_detection()
        m.enable_change_detection()
        m.insert(**wide[0], max_range=20.0)
        after_enable = (m.changed_codes(0), m.changed_codes(1))
        m.retain(box=(np.array([-12.0, -10.0, -3.0]), np.array([14.0, 9.0, 6.0])))
        m.insert(**small, max_range=30.0)
        changed[name] = after_enable + (m.changed_codes(0), m.changed_codes(1))
        caps[name] += (m.pool_stats()["brick_cap"],)
    assert caps["fixed"] == (BIG, BIG, BIG)
    assert caps["growing"][1] > caps["growing"][0]
    assert len(changed["fixed"][0]) > 0 and len(changed["fixed"][2]) > 0
    for a, b in zip(changed["fixed"], changed["growing"]):
        np.testing.assert_array_equal(a, b)
    for m in maps.values():
        m.close()


def test_device_bytes_after_a_volume_regrow():
    """The dense scan volume is sized by max_range: a map that regrows it holds the same memory as one
    that sized it for the longer range at once."""
    s = _scan(0, 16, 256)
    a = Map(0.2, initial_bricks=BIG)
    b = Map(0.2, initial_bricks=BIG)
    a.insert(**s, max_range=30.0)
    a.insert(**s, max_range=30.0)
    b.insert(**s, max_range=10.0)
    b.insert(**s, max_range=30.0)
    pa, pb = a.pool_stats(), b.pool_stats()
    assert pa["brick_cap"] == pb["brick_cap"] == BIG and pa["up_cap"] == pb["up_cap"]
    assert pa["device_bytes"] == pb["device_bytes"]
    a.close()
    b.close()
