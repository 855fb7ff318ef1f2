"""GPU: the depth-1 / depth-2 values derived from per-block pair maxima (max of octets 2k and
2k+1) and the leaves, on every path that writes them: scans over values a write batch left in
the untouched partner octet, uninitialised partners, maps read from a file, setValueVolume,
threshold changes, colour maps and out-of-tree (alias) marks.  Each case checks the value field
against the C restatement (and the compiled reference where it travelled), the depth 1-4 node
answers against the pure function of the field; the file image of these values is compared
byte for byte against the reference by tests/test_gpu_export.py."""
import numpy as np
import pytest

from helpers import assert_value_fields_equal, check_inner_against_field
import writes_lib
from writes_lib import WritesOracleMap as OracleMap, WritesRefMap as RefMap, have_ref
from ufomap_b200 import scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu
writes_lib.build()

RES = 0.05
LEVELS = (1, 2, 3, 4, 5)


def _maps(color=False, with_ref=True, **kw):
    kw.setdefault("resolution", RES)
    gpu = Map(color=color, initial_blocks=1 << 12, **kw)
    cpus = [OracleMap(color=color, **kw)]
    if with_ref and have_ref():
        cpus.append(RefMap(color=color, **kw))
    return gpu, cpus


def _each(maps, fn):
    for m in maps:
        fn(m)


def _check(gpu, cpus, levels=LEVELS):
    field = gpu.value_field()
    for c in cpus:
        assert_value_fields_equal(field, c.value_field(), color_tol=0, what=type(c).__name__)
    check_inner_against_field(gpu, field, gpu.sensor_model(), levels=levels)
    return field


def _velodyne(k, max_range=12.0):
    o, p = scans.velodyne64(k=k, rings=16, azimuths=256)
    return dict(origin=o, xyz=p, max_range=max_range)


def _spread(v):
    v = v.astype(np.uint64) & np.uint64(0x1fffff)
    out = np.zeros_like(v)
    for b in range(21):
        out |= ((v >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b)
    return out


def _codes_of(keys, depths):
    """Code of the depth-d node holding each key, with the centre bits a depth-d Key carries."""
    keys = np.asarray(keys, np.uint64)
    d = np.asarray(depths, np.uint64)[:, None]
    centre = np.where(d > 0, np.uint64(1) << (np.maximum(d, np.uint64(1)) - np.uint64(1)), np.uint64(0))
    k = ((keys >> d) << d) | centre
    return _spread(k[:, 0]) | (_spread(k[:, 1]) << np.uint64(1)) | (_spread(k[:, 2]) << np.uint64(2))


def _batch(n, seed, value, depths=1, spread=120):
    """n SET writes (op 1) of `value` around the sensor (keys 2^15 +- spread) at `depths`."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(32768 - spread, 32768 + spread, size=(n, 3))
    depths = np.broadcast_to(np.asarray(depths, np.uint32), (n,)).copy()
    return _codes_of(keys, depths), depths, np.ones(n, np.uint8), np.broadcast_to(np.float32(value), (n,)).copy()


def test_scan_over_a_larger_partner_written_by_a_batch():
    """SET writes put the clamp maximum into whole octets; the next scans touch one octet of many
    such pairs and must keep the partner's value in the depth-1 / depth-2 answers."""
    gpu, cpus = _maps()
    ins = _velodyne(0)
    gpu.insert(**ins)
    _each(cpus, lambda m: m.insert(**ins))
    codes, depths, ops, vals = _batch(20000, seed=1, value=3.0)
    gpu.update_nodes(codes, depths, ops, vals)
    cpus[0].update_nodes(codes, depths, ops, vals)  # the reference has no SET
    cpus = cpus[:1]
    _check(gpu, cpus)
    for k in (1, 2):
        ins = _velodyne(k)
        gpu.insert(**ins)
        _each(cpus, lambda m: m.insert(**ins))
        _check(gpu, cpus)
    gpu.close()


def test_uninitialised_partners():
    """A fresh map: every touched octet's partner starts uninitialised (0.0); isolated depth-0
    writes initialise single octets of new blocks before the next scan."""
    gpu, cpus = _maps()
    ins = _velodyne(0, max_range=8.0)
    gpu.insert(**ins)
    _each(cpus, lambda m: m.insert(**ins))
    _check(gpu, cpus)
    codes, depths, ops, vals = _batch(3000, seed=2, value=-1.5, depths=0, spread=400)
    ops[:] = 0
    for m in [gpu] + cpus:
        m.update_nodes(codes, depths, ops, vals)
    _check(gpu, cpus)
    ins = _velodyne(1, max_range=16.0)
    gpu.insert(**ins)
    _each(cpus, lambda m: m.insert(**ins))
    _check(gpu, cpus)
    gpu.close()


def test_after_reading_a_file_with_arbitrary_values():
    """readData of a node stream with values written at depths 0..6 into a map holding a scan,
    then a scan on top."""
    rng = np.random.default_rng(3)
    n = 6000
    depths = rng.choice(7, size=n, p=[0.5, 0.2, 0.1, 0.08, 0.06, 0.04, 0.02]).astype(np.uint32)
    vals = rng.choice(np.float32([-2.0, -0.4, 0.3, 0.85, 3.0]), size=n).astype(np.float32)
    codes, depths, ops, _ = _batch(n, seed=3, value=0.0, depths=depths, spread=200)
    src = Map(RES, initial_blocks=1 << 12)
    src.update_nodes(codes, depths, ops, vals)
    data = src.write_data()
    src.close()
    gpu, cpus = _maps()
    ins = _velodyne(1)
    gpu.insert(**ins)
    _each(cpus, lambda m: m.insert(**ins))
    gpu.read_data(data)
    for c in cpus:
        assert c.read_data(data)
    _check(gpu, cpus)
    ins = _velodyne(0)
    gpu.insert(**ins)
    _each(cpus, lambda m: m.insert(**ins))
    _check(gpu, cpus)
    gpu.close()


@pytest.mark.parametrize("color", [False, True])
def test_after_set_value_volume(color):
    gpu, cpus = _maps(color=color)
    o, p, c = scans.rgbd(k=0, width=56, height=42)
    ins = dict(origin=o, xyz=p, rgb=c if color else None, max_range=3.0, discrete=True)
    gpu.insert(**ins)
    _each(cpus, lambda m: m.insert(**ins))
    # a colour map supports min_depth 0 only
    for i, (md, val) in enumerate([(0, 0.9), (0, 0.2), (0, 0.7)] if color else [(0, 0.9), (1, 0.2), (2, 0.7)]):
        lo = np.array([0.4, -0.5, -0.4]) + 0.13 * i
        hi = lo + np.array([0.37, 0.41, 0.29])
        _each([gpu] + cpus, lambda m: m.set_value_volume((lo, hi), val, md))
        _check(gpu, cpus)
    o, p, c = scans.rgbd(k=1, width=56, height=42)
    ins = dict(origin=o, xyz=p, rgb=c if color else None, max_range=3.0, discrete=True)
    gpu.insert(**ins)
    _each(cpus, lambda m: m.insert(**ins))
    _check(gpu, cpus)
    gpu.close()


def test_after_a_threshold_change():
    """The depth-2 flags follow the octet flags that the threshold change recomputes."""
    gpu, cpus = _maps(with_ref=False)
    for k in range(2):
        ins = _velodyne(k)
        gpu.insert(**ins)
        _each(cpus, lambda m: m.insert(**ins))
    _check(gpu, cpus)
    gpu.set_sensor_model(occupied_thres=0.6, free_thres=0.45)
    _check(gpu, cpus)
    ins = _velodyne(2)
    gpu.insert(**ins)
    _each(cpus, lambda m: m.insert(**ins))
    _check(gpu, cpus)
    gpu.set_sensor_model()
    _check(gpu, cpus)
    gpu.close()


def test_colour_map():
    gpu, cpus = _maps(color=True, resolution=0.04)
    for k in range(2):
        o, p, c = scans.rgbd(k=k, width=96, height=72)
        ins = dict(origin=o, xyz=p, rgb=c, max_range=3.0, discrete=True)
        gpu.insert(**ins)
        _each(cpus, lambda m: m.insert(**ins))
        _check(gpu, cpus)
        codes, depths, ops, vals = _batch(4000, seed=10 + k, value=0.6, depths=0, spread=60)
        ops[:] = 0
        _each([gpu] + cpus, lambda m: m.update_nodes(codes, depths, ops, vals))
        _check(gpu, cpus)
    gpu.close()


def test_alias_path():
    """Rays leaving through the + faces: the wrapped blocks are refreshed from their leaves."""
    rng = np.random.default_rng(7)
    p = rng.uniform(-40, 40.0, size=(4000, 3))
    o = np.array([0.3, -0.2, 0.1])
    special = np.array([o, o + [0.5, 0, 0], o + [0, 0, 3.0], [1.0, 1.0, 1.0], [0.5, 0.5, 0.5],
                        [-16.0, 0, 0], [-16.0, -16.0, -16.0], [15.99, 15.99, 15.99], [-100, 0.1, 0.1]])
    p = np.concatenate([special, p]).astype(np.float32).astype(np.float64)
    gpu, cpus = _maps(resolution=0.5, depth_levels=6)
    for _ in range(2):
        gpu.insert(origin=o, xyz=p, max_range=-1.0)
        _each(cpus, lambda m: m.insert(origin=o, xyz=p, max_range=-1.0))
        _check(gpu, cpus, levels=(1, 2, 3, 4, 5, 6))
    gpu.close()
