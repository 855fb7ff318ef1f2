"""GPU: the depth-1 / depth-2 values derived from per-block line maxima (max of octets 4h..4h+3,
one 128 B leaf line, an uninitialised octet counting as 0.0) and the leaves, on the paths that read
or rebuild them: scans that touch one octet of a line whose other octets hold larger values, lines
mixing initialised and uninitialised octets, lines with one saturated pair next to one that is not,
maps after readData, setValueVolume and a threshold change, colour maps and out-of-tree (alias)
marks.  Each case checks the value field against the C restatement (and the compiled reference
where it travelled) and the depth 1-5 node answers against the pure function of the field."""
import numpy as np
import pytest

from helpers import assert_value_fields_equal, check_inner_against_field
import writes_lib
from writes_lib import WritesOracleMap as OracleMap, WritesRefMap as RefMap, have_ref
from ufomap_b200 import scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu
writes_lib.build()

LEVELS = (1, 2, 3, 4, 5)


def _maps(color=False, with_ref=True, resolution=0.05, **kw):
    gpu = Map(resolution, color=color, initial_blocks=1 << 12, **kw)
    gpu.set_profiling(2)
    cpus = [OracleMap(resolution=resolution, color=color, **kw)]
    if with_ref and have_ref():
        cpus.append(RefMap(resolution=resolution, color=color, **kw))
    return gpu, cpus


def _check(gpu, cpus, levels=LEVELS):
    field = gpu.value_field()
    for c in cpus:
        assert_value_fields_equal(field, c.value_field(), color_tol=0, what=type(c).__name__)
    check_inner_against_field(gpu, field, gpu.sensor_model(), levels=levels)


def _insert(maps, ins):
    for m in maps:
        m.insert(**ins)


def _velodyne(k, max_range=12.0):
    o, p = scans.velodyne64(k=k, rings=16, azimuths=256)
    return dict(origin=o, xyz=p, max_range=max_range)


def _spread(v):
    v = v.astype(np.uint64) & np.uint64(0x1fffff)
    out = np.zeros_like(v)
    for b in range(21):
        out |= ((v >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b)
    return out


def _batch(n, seed, value, depths, op, spread):
    """n writes (op 0 ADD, 1 SET) of `value` at keys 2^15 +- spread, at `depths`."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(32768 - spread, 32768 + spread, size=(n, 3)).astype(np.uint64)
    d = np.broadcast_to(np.asarray(depths, np.uint32), (n,)).copy()
    du = d.astype(np.uint64)[:, None]
    centre = np.where(du > 0, np.uint64(1) << (np.maximum(du, np.uint64(1)) - np.uint64(1)), np.uint64(0))
    k = ((keys >> du) << du) | centre
    codes = _spread(k[:, 0]) | (_spread(k[:, 1]) << np.uint64(1)) | (_spread(k[:, 2]) << np.uint64(2))
    return codes, d, np.full(n, op, np.uint8), np.full(n, value, np.float32)


def test_one_octet_of_a_line_with_larger_mates():
    """SET writes put the clamp maximum into whole blocks and octets; the next scans touch single
    octets of those lines and must keep the other octets' values in the depth-1 / depth-2 answers."""
    gpu, cpus = _maps()
    _insert([gpu] + cpus, _velodyne(0))
    cpus = cpus[:1]  # the reference has no SET
    for depth, n in ((2, 3000), (1, 8000)):
        batch = _batch(n, seed=depth, value=3.0, depths=depth, op=1, spread=120)
        for m in [gpu] + cpus:
            m.update_nodes(*batch)
    _check(gpu, cpus)
    for k in (1, 2):
        _insert([gpu] + cpus, _velodyne(k))
        _check(gpu, cpus)
    gpu.close()


def test_lines_mixing_initialised_and_uninitialised_octets():
    """Isolated depth-0 writes initialise single octets of new blocks; the scans then touch lines
    whose other octets are partly initialised, partly not (0.0)."""
    gpu, cpus = _maps()
    _insert([gpu] + cpus, _velodyne(0, max_range=6.0))
    batch = _batch(4000, seed=5, value=-0.7, depths=0, op=0, spread=300)
    for m in [gpu] + cpus:
        m.update_nodes(*batch)
    _check(gpu, cpus)
    for k in (1, 2):
        _insert([gpu] + cpus, _velodyne(k, max_range=15.0))
        _check(gpu, cpus)
    gpu.close()


def test_line_with_one_saturated_pair():
    """Scans saturate the free space around the sensor; single voxels written above the clamp then
    leave lines whose one pair is still saturated and whose other is not.  Such a line is read
    whole, and its saturated octets keep their bits."""
    gpu, cpus = _maps(resolution=0.1)
    sat = []
    for k in range(8):
        _insert([gpu] + cpus, _velodyne(k, max_range=8.0))
        sat.append(gpu.update_stats()["saturated_octets"])
    assert sat[-1] > 0, sat
    cpus = cpus[:1]  # the reference has no SET
    batch = _batch(3000, seed=9, value=-0.2, depths=0, op=1, spread=60)
    for m in [gpu] + cpus:
        m.update_nodes(*batch)
    _check(gpu, cpus)
    for k in (8, 9):
        _insert([gpu] + cpus, _velodyne(k, max_range=8.0))
        _check(gpu, cpus)
    gpu.close()


def test_after_read_data_set_value_volume_and_threshold_change():
    rng = np.random.default_rng(11)
    n = 5000
    depths = rng.choice(5, size=n, p=[0.5, 0.2, 0.15, 0.1, 0.05]).astype(np.uint32)
    codes, depths, ops, _ = _batch(n, seed=11, value=0.0, depths=depths, op=1, spread=200)
    vals = rng.choice(np.float32([-2.0, -0.4, 0.3, 0.85, 3.0]), size=n).astype(np.float32)
    src = Map(0.05, initial_blocks=1 << 12)
    src.update_nodes(codes, depths, ops, vals)
    data = src.write_data()
    src.close()
    gpu, cpus = _maps(with_ref=False)
    _insert([gpu] + cpus, _velodyne(1))
    gpu.read_data(data)
    for c in cpus:
        assert c.read_data(data)
    _check(gpu, cpus)
    _insert([gpu] + cpus, _velodyne(0))
    _check(gpu, cpus)
    for m in [gpu] + cpus:
        m.set_value_volume((np.array([0.3, -0.6, -0.5]), np.array([1.1, 0.2, 0.4])), 0.8, 0)
    _check(gpu, cpus)
    gpu.set_sensor_model(occupied_thres=0.6, free_thres=0.45)
    _check(gpu, cpus)
    _insert([gpu] + cpus, _velodyne(2))
    _check(gpu, cpus)
    gpu.close()


def test_colour_map():
    """Colour maps read the untouched octets of a touched line for their maxima only."""
    gpu, cpus = _maps(color=True, resolution=0.04)
    for k in range(2):
        o, p, c = scans.rgbd(k=k, width=96, height=72)
        _insert([gpu] + cpus, dict(origin=o, xyz=p, rgb=c, max_range=3.0, discrete=True))
        _check(gpu, cpus)
        batch = _batch(4000, seed=20 + k, value=0.9, depths=0, op=0, spread=60)
        for m in [gpu] + cpus:
            m.update_nodes(*batch)
        _check(gpu, cpus)
    gpu.close()


def test_alias_path():
    """Rays leaving through the + faces: the wrapped blocks' line maxima are rebuilt from their leaves."""
    rng = np.random.default_rng(13)
    p = rng.uniform(-40, 40.0, size=(4000, 3))
    o = np.array([0.3, -0.2, 0.1])
    special = np.array([[15.99, 15.99, 15.99], [-16.0, -16.0, -16.0], [-100, 0.1, 0.1], [1.0, 1.0, 1.0]])
    p = np.concatenate([special, p]).astype(np.float32).astype(np.float64)
    gpu, cpus = _maps(resolution=0.5, depth_levels=6)
    for _ in range(2):
        _insert([gpu] + cpus, dict(origin=o, xyz=p, max_range=-1.0))
        _check(gpu, cpus, levels=(1, 2, 3, 4, 5, 6))
    gpu.close()
