"""GPU: the leaf update (k_update_brick) claims its bricks through a work cursor and stages a
brick's hit masks only when the brick received a hit this scan.  These cases check the paths
that scheduling and the hit flag depend on against the CPU oracle (and the compiled reference
where it travelled): a scan repeated after the brick pool grew in the middle of it, hits in
bricks that no ray crosses, out-of-tree (aliased) + face hits, and setValueVolume (SET mode)
straight after an asynchronous scan."""
import numpy as np
import pytest

import color_lib as cl
from helpers import assert_value_fields_equal, check_inner_against_field
from oracle_lib import OracleMap, RefMap, have_ref
from ufomap_b200 import scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu


def _cpus(**kw):
    return [OracleMap(**kw)] + ([RefMap(**kw)] if have_ref() else [])


def _check(gpu, cpus, levels=(1, 2, 3, 4, 5, 6)):
    field = gpu.value_field()
    for c in cpus:
        assert_value_fields_equal(field, c.value_field(), what=type(c).__name__)
    check_inner_against_field(gpu, field, cpus[0].sensor_model(), levels=levels)
    return field


def test_scan_repeated_after_pool_growth_matches_a_presized_map():
    """A map created with a handful of bricks overflows its pool in the middle of every early scan;
    the scan is repeated with a new scan id and a fresh cursor and must leave the same value field
    as a map that never grew."""
    small = Map(0.05, initial_blocks=16, initial_bricks=4)
    big = Map(0.05, initial_blocks=1 << 16)
    cpus = _cpus(resolution=0.05)
    regrows = 0
    for k in range(3):
        o, p = scans.velodyne64(k=k, rings=32, azimuths=1024)
        for m in [small, big] + cpus:
            m.insert(o, p, max_range=20.0)
        regrows += small.stats()["regrows"]
    assert regrows > 0, "the small map's pool never grew"
    field = _check(small, cpus)
    assert_value_fields_equal(field, big.value_field(), what="pre-sized map")
    assert len(field[0]) > 0
    small.close()
    big.close()


@pytest.mark.parametrize("max_range", [-1.0, 10.0])
def test_hits_in_bricks_no_ray_crosses(max_range):
    """Every end point is the first voxel of its brick on an axis-aligned ray: the brick holding
    the hit gets no free-space mark of its own, so only the hit flag brings its hit masks in."""
    res = 0.02
    brick = 16 * res
    o = np.array([0.5, 0.5, 0.5]) * res  # voxel centre next to the map's origin
    ends = []
    for axis in range(3):
        for sign in (1.0, -1.0):
            for k in range(1, 9):
                e = o.copy()
                # + side: first voxel of brick k; - side: last voxel of brick -k, entered first
                e[axis] = sign * k * brick + (0.5 * res if sign > 0 else -0.5 * res)
                ends.append(e)
    p = np.array(ends)
    gpu = Map(res, initial_blocks=1 << 12)
    cpus = _cpus(resolution=res)
    for m in [gpu] + cpus:
        m.insert(o, p, max_range=max_range)
        m.insert(o + [0.0, 0.0, 3 * res], p + [0.0, 0.0, 3 * res], max_range=max_range)
    field = _check(gpu, cpus)
    assert (field[1] > 0).sum() >= len(p), "every end point is occupied"
    gpu.close()


@pytest.mark.parametrize("color", [False, True])
def test_aliased_and_face_hits(color):
    """Hits on the + faces of a small map land on wrapped (aliased) voxels as well as in-tree ones;
    the scans after the first one take the alias path, the first one the dense path."""
    kw = dict(resolution=cl.FACE_RES, depth_levels=cl.FACE_LEVELS)
    gpu = Map(color=color, initial_blocks=16, **kw)
    cpus = [OracleMap(color=color, **kw)] + ([RefMap(color=color, **kw)] if have_ref() else [])
    for s in cl.face_scans():
        ins = dict(origin=s["origin"], xyz=s["xyz"], rgb=s["rgb"] if color else None, max_range=40.0,
                   discrete=s["discrete"])
        for m in [gpu] + cpus:
            m.insert(**ins)
    _check(gpu, cpus)
    gpu.close()


def test_set_value_volume_straight_after_an_async_scan():
    """SET mode launches the same kernel with a cursor of its own; the asynchronous scan before it
    must not leave the cursor behind."""
    gpu = Map(0.05, initial_blocks=1 << 14)
    cpus = _cpus(resolution=0.05)
    for k in range(2):
        o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
        gpu.insert(o, p, max_range=15.0, async_=True)
        for c in cpus:
            c.insert(o, p, max_range=15.0)
        lo = np.array([-3.0, -2.0, -1.0]) + 0.7 * k
        for m in [gpu] + cpus:
            m.set_value_volume((lo, lo + [4.1, 3.3, 1.7]), 0.8 if k == 0 else 0.25)
    gpu.wait()
    _check(gpu, cpus)
    gpu.close()
