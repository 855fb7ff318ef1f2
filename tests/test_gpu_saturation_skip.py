"""GPU: on mono maps the leaf update leaves saturated pairs alone (two initialised octets, no hit,
every voxel at clamping_thres_min: a miss cannot change them) and writes back only the leaf sectors
that changed; colour maps read and write every touched pair.  Every case runs at profiling level 2,
checks what was skipped (update_stats) and compares the value field against the C restatement and,
where it travelled, the compiled reference, the depth 1-5 answers against the pure function of the
field, and colours / change sets where the case has them."""
import numpy as np
import pytest

from helpers import assert_value_fields_equal, check_inner_against_field
import writes_lib
from writes_lib import WritesOracleMap as OracleMap, WritesRefMap as RefMap, have_ref
from ufomap_b200 import scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu
writes_lib.build()

RES = 0.1
LEVELS = (1, 2, 3, 4, 5)


def _maps(color=False, with_ref=True, initial_blocks=1 << 12, **kw):
    kw.setdefault("resolution", RES)
    gpu = Map(color=color, initial_blocks=initial_blocks, **kw)
    gpu.set_profiling(2)
    cpus = [OracleMap(color=color, **kw)]
    if with_ref and have_ref():
        cpus.append(RefMap(color=color, **kw))
    return gpu, cpus


def _check(gpu, cpus, levels=LEVELS):
    field = gpu.value_field()
    for c in cpus:
        assert_value_fields_equal(field, c.value_field(), color_tol=0, what=type(c).__name__)
    check_inner_against_field(gpu, field, gpu.sensor_model(), levels=levels)
    return field


def _scan(k, color=False, max_range=8.0):
    if color:
        o, p, c = scans.rgbd(k=k, width=64, height=48)
        return dict(origin=o, xyz=p, rgb=c, max_range=3.0, discrete=True)
    o, p = scans.velodyne64(k=k, rings=16, azimuths=256)
    return dict(origin=o, xyz=p, max_range=max_range)


def _insert(gpu, cpus, ins):
    """One scan into every map; returns the GPU's update_stats of it."""
    gpu.insert(**ins)
    for c in cpus:
        c.insert(**ins)
    return gpu.update_stats()


def _saturate(gpu, cpus, n=8, color=False, max_range=8.0):
    """n scans from nearby poses; returns the saturated octets of each."""
    return [_insert(gpu, cpus, _scan(k, color, max_range))["saturated_octets"] for k in range(n)]


@pytest.mark.parametrize("color", [False, True])
def test_saturating_stream(color):
    """Repeated free-space observation drives voxels to the clamp; on a mono map the later scans
    skip their pairs and leave unchanged sectors unwritten, a colour map updates them all, and every
    result stays the reference's."""
    gpu, cpus = _maps(color=color, resolution=0.04 if color else RES)
    sat, clean = [], []
    for k in range(10):
        st = _insert(gpu, cpus, _scan(k, color))
        sat.append(st["saturated_octets"])
        clean.append(st["clean_sectors"])
        if k in (0, 5, 9):
            _check(gpu, cpus)
    if color:
        assert sum(sat) == 0 and sum(clean) == 0, (sat, clean)
    else:
        assert sat[0] == 0
        assert sat[-1] > 0, sat
        assert sum(clean) > 0, clean
    # the skipped octets are still touched octets: part of the scan's counters
    assert gpu.stats()["touched_octets"] >= sat[-1]
    gpu.close()


def test_hit_in_a_saturated_pair():
    """Points in the middle of rays already saturated as free space: their pairs carry a hit bit
    and are updated, the rest of the scan is skipped."""
    gpu, cpus = _maps()
    _saturate(gpu, cpus)
    o, p = scans.velodyne64(k=7, rings=16, azimuths=256)
    mid = o + 0.5 * (p[::7] - o)
    ins = dict(origin=o, xyz=np.concatenate([p, mid]), max_range=8.0)
    st = _insert(gpu, cpus, ins)
    assert st["saturated_octets"] > 0
    assert gpu.stats()["hit_voxels"] > 0
    _check(gpu, cpus)
    gpu.close()


def test_positive_clamp_skips_nothing():
    """clamping_thres_min above 0.5: the clamp is positive, so the maximum of a pair can equal it
    while the pair holds an uninitialised octet (counted as 0.0) or initialised voxels no update has
    reached (0.0): a miss would raise those to the clamp.  Such a map never skips."""
    model = dict(clamping_thres_min=0.6, clamping_thres_max=0.97)
    gpu, cpus = _maps(**model)
    sat = _saturate(gpu, cpus, n=6)
    assert sum(sat) == 0, sat
    _check(gpu, cpus)
    gpu.close()


def test_stream_reaching_new_space_next_to_saturated_space():
    """Scans from nearby poses saturate a region, then scans from poses further away mark both
    saturated pairs and octets no scan has marked yet (fresh octets and partners).  With a negative
    clamp a pair holding an uninitialised octet has a maximum >= 0.0 and so never equals the clamp:
    the kernel's "both octets initialised" condition is a guard that the pair-maximum test already
    implies here (test_positive_clamp_skips_nothing covers the clamp where it would not)."""
    gpu, cpus = _maps()
    sat = []
    for k in range(12):
        sat.append(_insert(gpu, cpus, _scan(k % 6 if k < 8 else 2 * k))["saturated_octets"])
        if k in (7, 11):
            _check(gpu, cpus)
    assert sat[7] > 0 and sum(sat[8:]) > 0, sat
    gpu.close()


def test_pair_with_one_voxel_above_the_clamp():
    """A saturated region, then one voxel of many pairs raised by a node update: those pairs are
    updated, the others skipped."""
    gpu, cpus = _maps()
    _saturate(gpu, cpus)
    codes, occ, _ = gpu.value_field()
    cmin = np.float32(gpu.sensor_model()[4])
    at_clamp = codes[occ == cmin]
    assert len(at_clamp) > 1000
    pick = at_clamp[::97]
    for m in [gpu] + cpus:
        m.update_nodes(pick, np.zeros(len(pick), np.uint32), np.zeros(len(pick), np.uint8),
                       np.full(len(pick), 0.3, np.float32))
    _check(gpu, cpus)
    st = _insert(gpu, cpus, _scan(8))
    assert st["saturated_octets"] > 0
    _check(gpu, cpus)
    gpu.close()


def _restart_cpu(gpu, cpus, **model):
    """The CPU maps have a fixed sensor model: a new one with `model`, holding the GPU map's state."""
    data = gpu.write_data()
    for c in cpus:
        c.close()
    out = []
    for cls in (OracleMap, RefMap) if have_ref() else (OracleMap,):
        c = cls(resolution=RES, **model)
        assert c.read_data(data)
        out.append(c)
    return out


def test_sensor_model_changes():
    """clamping_thres_min raised (values below the new clamp remain: no skipping from then on),
    lowered (skipping resumes once voxels reach the new clamp), and prob_miss > 0.5 (a miss raises
    the value: no skipping)."""
    gpu, cpus = _maps()
    assert _saturate(gpu, cpus)[-1] > 0
    raised = dict(clamping_thres_min=0.2)
    gpu.set_sensor_model(**raised)
    cpus = _restart_cpu(gpu, cpus, **raised)
    for k in range(8, 11):
        assert _insert(gpu, cpus, _scan(k))["saturated_octets"] == 0
    _check(gpu, cpus)
    lowered = dict(clamping_thres_min=0.05)
    gpu.set_sensor_model(**lowered)
    cpus = _restart_cpu(gpu, cpus, **lowered)
    sat = [_insert(gpu, cpus, _scan(k % 6))["saturated_octets"] for k in range(12)]
    assert sat[-1] > 0, sat
    _check(gpu, cpus)
    positive_miss = dict(clamping_thres_min=0.05, prob_miss=0.6)
    gpu.set_sensor_model(**positive_miss)
    cpus = _restart_cpu(gpu, cpus, **positive_miss)
    assert _insert(gpu, cpus, _scan(3))["saturated_octets"] == 0
    _check(gpu, cpus)
    gpu.close()


def test_change_detection():
    """The change set of a scan over saturated space is the reference's: skipped voxels are not
    changes."""
    if not have_ref():
        pytest.skip("the compiled reference did not travel")
    gpu = Map(RES, initial_blocks=1 << 12)
    gpu.set_profiling(2)
    ref = RefMap(resolution=RES)
    for m in (gpu, ref):
        m.enable_change_detection(True)
    sat = []
    for k in range(9):
        for m in (gpu, ref):
            m.reset_change_detection()
        sat.append(_insert(gpu, [ref], _scan(k))["saturated_octets"])
        assert np.array_equal(gpu.changed_codes(0), np.unique(ref.changed_codes()[0])), k
    assert sat[-1] > 0, sat
    _check(gpu, [ref])
    gpu.close()


def test_scan_repeated_after_pool_growth():
    """A small pool saturated by short scans, then a long scan that overflows it: the scan is
    repeated on the grown pools, and its saturated pairs are skipped exactly once."""
    gpu, cpus = _maps(initial_blocks=64)
    _saturate(gpu, cpus, max_range=4.0)
    st = _insert(gpu, cpus, _scan(7, max_range=14.0))
    assert gpu.stats()["regrows"] > 0
    assert st["saturated_octets"] > 0
    _check(gpu, cpus)
    gpu.close()


def test_out_of_tree_keys_turn_the_skip_off():
    """Once a map has met out-of-tree keys, its scans fold nothing and skip nothing."""
    rng = np.random.default_rng(7)
    o = np.array([0.3, -0.2, 0.1])
    inside = rng.uniform(-12.0, 12.0, size=(3000, 3)).astype(np.float32).astype(np.float64)
    # rays that leave through the + faces of a 32 m map (as in test_gpu_pair_maxima's alias case)
    special = np.array([o, o + [0.5, 0, 0], o + [0, 0, 3.0], [1.0, 1.0, 1.0], [0.5, 0.5, 0.5], [-16.0, 0, 0],
                        [-16.0, -16.0, -16.0], [15.99, 15.99, 15.99], [-100, 0.1, 0.1]])
    outside = np.concatenate([inside, special, rng.uniform(-40, 40.0, size=(4000, 3))])
    outside = outside.astype(np.float32).astype(np.float64)
    gpu, cpus = _maps(resolution=0.5, depth_levels=6)
    ins = dict(origin=o, xyz=inside, max_range=-1.0)
    sat = [_insert(gpu, cpus, ins)["saturated_octets"] for _ in range(7)]
    assert sat[-1] > 0, sat
    _check(gpu, cpus, levels=(1, 2, 3, 4, 5, 6))
    for xyz in (outside, inside, inside):
        assert _insert(gpu, cpus, dict(origin=o, xyz=xyz, max_range=-1.0))["saturated_octets"] == 0
        _check(gpu, cpus, levels=(1, 2, 3, 4, 5, 6))
    gpu.close()


def test_async_inserts():
    gpu, cpus = _maps()
    for k in range(10):
        ins = _scan(k)
        gpu.insert(async_=True, **ins)
        for c in cpus:
            c.insert(**ins)
    gpu.wait()
    assert gpu.update_stats()["saturated_octets"] > 0
    _check(gpu, cpus)
    gpu.close()
