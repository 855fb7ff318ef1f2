"""GPU: per-node writes (ufo_b200_update_nodes) and ray insertion (ufo_b200_insert_rays) against
the C restatement and, where the prebuilt harness travelled, the compiled reference.  Value
fields are compared bit for bit, inner aggregates against the pure function of the field."""
import concurrent.futures as cf

import numpy as np
import pytest

from helpers import assert_value_fields_equal, check_inner_against_field, check_inner_sampled, sorted_field_large
import writes_lib
from writes_lib import WritesOracleMap as OracleMap, WritesRefMap as RefMap, have_ref
from ufomap_b200 import scans
from ufomap_b200.capi import Map, UfoError, E_INVALID, E_UNSUPPORTED

pytestmark = pytest.mark.gpu
writes_lib.build()

RES = 0.05
LEVELS = (1, 2, 3, 4, 5, 6, 9, 16)
VALUES = np.float32([0.8473, -0.4055, 1.5, -2.5, 0.3, 3.0, -0.05])


def _spread(v):
    v = v.astype(np.uint64) & np.uint64(0x1fffff)
    out = np.zeros_like(v)
    for b in range(21):
        out |= ((v >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b)
    return out


def codes_of(keys, depths):
    """Code of the depth-d node holding each key, with the centre bits a depth-d Key carries."""
    keys = np.asarray(keys, np.uint64)
    d = np.asarray(depths, np.uint64)[:, None]
    centre = np.where(d > 0, np.uint64(1) << (np.maximum(d, np.uint64(1)) - np.uint64(1)), np.uint64(0))
    k = ((keys >> d) << d) | centre
    return _spread(k[:, 0]) | (_spread(k[:, 1]) << np.uint64(1)) | (_spread(k[:, 2]) << np.uint64(2))


def mixed_batch(n, seed, half=40, ops=True, depth_p=(0.6, 0.15, 0.1, 0.08, 0.06, 0.008, 0.002)):
    """n entries around the map centre (keys 2^15 +- half), depths 0..6, repeated codes."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(32768 - half, 32768 + half, size=(n // 4, 3))
    keys = keys[rng.integers(0, len(keys), n)]  # every code about four times
    p = np.asarray(depth_p, float)
    depths = rng.choice(7, size=n, p=p / p.sum()).astype(np.uint32)
    codes = codes_of(keys, depths)
    op = (rng.random(n) < 0.1).astype(np.uint8) if ops else np.zeros(n, np.uint8)
    vals = VALUES[rng.integers(0, len(VALUES), n)]
    return codes, depths, op, vals


def prefilled(map_cls, **kw):
    m = map_cls(RES, **kw)
    for k in range(2):
        o, p = scans.velodyne64(k=k, rings=16, azimuths=256)
        m.insert(o, p, max_range=20.0)
    return m


def checkers(with_ref=True, color=False):
    cpus = [prefilled(OracleMap, color=color)]
    if with_ref and have_ref():
        cpus.append(prefilled(RefMap, color=color))
    return cpus


def compare(gpu, cpus, color_tol=0):
    field = gpu.value_field()
    for c in cpus:
        assert_value_fields_equal(field, c.value_field(), color_tol=color_tol, what=type(c).__name__)
    check_inner_against_field(gpu, cpus[0].value_field(), cpus[0].sensor_model(), levels=LEVELS)
    return field


def rays(n, seed, r=6.0):
    rng = np.random.default_rng(seed)
    o = np.array([0.013, 0.021, 0.007]) + rng.uniform(-0.3, 0.3, size=(n, 3))
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    return o, o + d * rng.uniform(0.05, r, size=(n, 1))


def test_known_answers():
    """integrateHit then integrateMiss on one voxel; repeated hits stop at the clamp; one insertRay
    marks the computeRay codes free and its end occupied."""
    m = Map(0.02)
    hit, miss = np.float32(np.log(0.7 / 0.3)), np.float32(np.log(0.4 / 0.6))
    c = m.to_code([0.5, 0.5, 0.5])
    m.update_nodes([c, c], 0, 0, [hit, miss])
    _, occ, _ = m.value_field()
    assert occ.view(np.uint32).tolist() == [0x3EE237E7]
    m.update_nodes([c] * 20, 0, 0, hit)
    _, occ, _ = m.value_field()
    assert occ.view(np.uint32).tolist() == [0x4060B4BA]
    m.clear()
    m.insert_rays([0, 0, 0], [[1.0, 0, 0]], hit_end=True)
    codes, occ, _ = m.value_field()
    free = m.compute_ray([0, 0, 0], [1.0, 0, 0])
    end = m.to_code([1.0, 0, 0])
    assert np.array_equal(np.sort(codes), np.sort(np.append(free, end)))
    assert (occ[codes != end].view(np.uint32) == 0xBECF991F).all()
    assert occ[codes == end].tolist() == [hit]
    m.close()


def test_mixed_batch_on_scanned_map():
    """~200 k entries, every op and depth 0..6, on a map holding two 5 cm Velodyne scans."""
    codes, depths, ops, vals = mixed_batch(200_000, seed=1)
    gpu = prefilled(Map)
    gpu.update_nodes(codes, depths, ops, vals)
    st = gpu.stats()
    assert st["points"] == len(codes) and st["touched_bricks"] > 0 and st["ms_total"] > 0
    cpu = checkers(with_ref=False)
    cpu[0].update_nodes(codes, depths, ops, vals)
    compare(gpu, cpu)
    if have_ref():
        # the reference has no SET: the ADD-only batch against it
        codes, depths, ops, vals = mixed_batch(200_000, seed=2, ops=False)
        gpu = prefilled(Map)
        gpu.update_nodes(codes, depths, ops, vals)
        ref = prefilled(RefMap)
        ref.update_nodes(codes, depths, ops, vals)
        assert_value_fields_equal(gpu.value_field(), ref.value_field(), what="RefMap")


@pytest.mark.parametrize("depth,hit_end,max_range", [(0, True, -1.0), (0, False, 3.0), (3, True, 3.0),
                                                       (3, False, -1.0)])
def test_ray_batches(depth, hit_end, max_range):
    o, e = rays(32768, seed=depth + 2 * hit_end)
    gpu = prefilled(Map)
    gpu.insert_rays(o, e, max_range=max_range, depth=depth, hit_end=hit_end)
    assert gpu.stats()["points"] == len(o)
    cpus = checkers()
    for c in cpus:
        c.insert_rays(o, e, max_range=max_range, depth=depth, hit_end=hit_end)
    compare(gpu, cpus)


def test_colour_map():
    """Leaf colours stay as they are; log-odds and inner aggregates as on a mono map."""
    o, p, rgb = scans.rgbd(k=0, width=160, height=120)
    gpu = Map(RES, color=True)
    cpu = OracleMap(RES, color=True)
    for m in (gpu, cpu):
        m.insert(o, p, rgb=rgb, max_range=5.0, discrete=True)
    before = gpu.value_field()
    codes, depths, ops, vals = mixed_batch(50_000, seed=3)
    ops[depths > 0] = 0
    for m in (gpu, cpu):
        m.update_nodes(codes, depths, ops, vals)
    field = gpu.value_field()
    assert_value_fields_equal(field, cpu.value_field(), color_tol=0, what="OracleMap")
    check_inner_against_field(gpu, cpu.value_field(), cpu.sensor_model(), levels=LEVELS)
    keep = np.isin(field[0], before[0])
    assert np.array_equal(field[2][keep], before[2][np.isin(before[0], field[0])])


def test_pool_growth_applies_every_update_once():
    """A map created with 16 bricks has to grow while expanding the batch; the result still equals
    the checker, so no update was applied twice."""
    codes, depths, ops, vals = mixed_batch(100_000, seed=4, half=200)
    gpu = Map(RES, initial_bricks=16)
    gpu.update_nodes(codes, depths, ops, vals)
    assert gpu.stats()["regrows"] > 0
    cpu = OracleMap(RES)
    cpu.update_nodes(codes, depths, ops, vals)
    assert_value_fields_equal(gpu.value_field(), cpu.value_field(), what="OracleMap")
    o, e = rays(20000, seed=5, r=15.0)
    gpu = Map(RES, initial_bricks=16)
    gpu.insert_rays(o, e, hit_end=True)
    assert gpu.stats()["regrows"] > 0
    cpu = OracleMap(RES)
    cpu.insert_rays(o, e, hit_end=True)
    assert_value_fields_equal(gpu.value_field(), cpu.value_field(), what="OracleMap")


def test_repeatable_and_async():
    codes, depths, ops, vals = mixed_batch(100_000, seed=6)
    o, e = rays(8192, seed=7)
    fields = []
    for async_ in (False, False, True):
        m = prefilled(Map)
        m.update_nodes(codes, depths, ops, vals, async_=async_)
        m.insert_rays(o, e, depth=1, hit_end=True, async_=async_)
        m.wait()
        fields.append(m.value_field())
        m.close()
    for f in fields[1:]:
        assert_value_fields_equal(fields[0], f, what="repeat")


def test_writes_interleaved_with_async_scans():
    gpu = Map(RES)
    cpu = OracleMap(RES)
    for k in range(3):
        o, p = scans.velodyne64(k=k, rings=16, azimuths=256)
        codes, depths, ops, vals = mixed_batch(20_000, seed=10 + k)
        ro, re = rays(4096, seed=20 + k)
        gpu.insert(o, p, max_range=20.0, async_=True)
        gpu.update_nodes(codes, depths, ops, vals, async_=True)
        gpu.insert_rays(ro, re, depth=k, hit_end=k != 1, async_=True)
        cpu.insert(o, p, max_range=20.0)
        cpu.update_nodes(codes, depths, ops, vals)
        cpu.insert_rays(ro, re, depth=k, hit_end=k != 1)
    gpu.wait()
    compare(gpu, [cpu])


@pytest.mark.skipif(not have_ref(), reason="the compiled reference did not travel")
def test_change_set_and_change_box():
    """Depth-0 writes: the change set equals the reference's changes_; depth-3 writes into untouched
    space: changed_codes(3) equals it too.  Neither call moves the min/max change box."""
    codes, depths, ops, vals = mixed_batch(50_000, seed=8, ops=False, depth_p=(1, 0, 0, 0, 0, 0, 0))
    gpu = prefilled(Map)
    ref = prefilled(RefMap)
    box = gpu.change_bbox()
    for m in (gpu, ref):
        m.enable_change_detection(True)
        m.update_nodes(codes, depths, ops, vals)
    assert np.array_equal(gpu.changed_codes(0), np.unique(ref.changed_codes()[0]))
    o, e = rays(4096, seed=9)
    for m in (gpu, ref):
        m.reset_change_detection()
        m.insert_rays(o, e, hit_end=True)
    assert np.array_equal(gpu.changed_codes(0), np.unique(ref.changed_codes()[0]))
    gbox = gpu.change_bbox()
    assert np.array_equal(box[0], gbox[0]) and np.array_equal(box[1], gbox[1])
    gpu, ref = Map(RES), RefMap(RES)
    rng = np.random.default_rng(11)
    keys = np.unique(rng.integers(32768 - 400, 32768 + 400, size=(3000, 3)) >> 3, axis=0) << 3
    c3 = codes_of(keys, np.full(len(keys), 3))
    for m in (gpu, ref):
        m.enable_change_detection(True)
        m.update_nodes(c3, 3, 0, VALUES[0])
    assert np.array_equal(gpu.changed_codes(3), np.unique(ref.changed_codes()[0]))


def test_rejections_leave_the_map_unchanged():
    gpu = prefilled(Map)
    before = gpu.value_field()
    c = gpu.to_code([0.3, 0.2, 0.1])
    out = np.uint64(1 << 48)  # key x = 2^16: outside a 16-level tree
    cases = [
        (E_UNSUPPORTED, lambda: gpu.update_nodes([c, c], [0, 7], 0, 0.5)),
        (E_INVALID, lambda: gpu.update_nodes([c, out], [0, 0], 0, 0.5)),
        (E_UNSUPPORTED, lambda: gpu.insert_rays([0, 0, 0], [[1, 0, 0]], depth=7)),
        (E_INVALID, lambda: gpu.insert_rays([0, 0, 0], [[1, 0, 0], [5000.0, 0, 0]])),
        (E_INVALID, lambda: gpu.insert_rays([[0, 0, 0], [-5000.0, 0, 0]], [[1, 0, 0], [1, 0, 0]])),
    ]
    for status, call in cases:
        with pytest.raises(UfoError) as e:
            call()
        assert e.value.status == status
        assert_value_fields_equal(before, gpu.value_field(), what="after a rejected batch")
    col = Map(RES, color=True)
    with pytest.raises(UfoError) as e:
        col.update_nodes([c], [1], [1], 0.5)
    assert e.value.status == E_UNSUPPORTED and col.value_field_count() == 0
    sh = Map(RES)
    sh.set_shard(0, 2)
    for call in (lambda: sh.update_nodes([c], 0, 0, 0.5), lambda: sh.insert_rays([0, 0, 0], [[1, 0, 0]])):
        with pytest.raises(UfoError) as e:
            call()
        assert e.value.status == E_UNSUPPORTED
    assert sh.value_field_count() == 0


def test_write_cost_does_not_depend_on_the_map_size():
    """A batch touching K bricks reports touched_bricks == K on a small and on a large map."""
    rng = np.random.default_rng(12)
    keys = rng.integers(32768 - 300, 32768 + 300, size=(20000, 3))
    codes = codes_of(keys, np.zeros(len(keys)))
    k = len(np.unique(codes >> np.uint64(12)))
    for prefill in (0, 6):
        m = Map(RES, initial_bricks=1 << 16)
        for j in range(prefill):
            o, p = scans.velodyne64(k=j, rings=32, azimuths=1024)
            shift = np.array([100.0 * (j + 1), 0.0, 0.0])
            m.insert(o + shift, p + shift, max_range=30.0)
        m.update_nodes(codes, 0, 0, VALUES[1])
        st = m.stats()
        assert st["touched_bricks"] == k, (prefill, st["touched_bricks"], k)
        m.close()


def test_config2_rays_full_length():
    """BASELINE config #2 at 2 cm, every 16th ray of the 131 072-point scan (rays of up to 30 m), as
    insertRay; the CPU side integrates in a background thread while the GPU runs."""
    o, p = scans.velodyne64(k=0)
    ends = p[::16]
    origins = np.broadcast_to(o, ends.shape)
    cpu = RefMap(0.02) if have_ref() else OracleMap(0.02)
    with cf.ThreadPoolExecutor(1) as ex:
        fut = ex.submit(cpu.insert_rays, origins, ends, 30.0, 0, True)
        gpu = Map(0.02)
        gpu.insert_rays(origins, ends, max_range=30.0, hit_end=True)
        gfield = sorted_field_large(gpu)
        fut.result()
    cfield = cpu.value_field()
    assert_value_fields_equal(gfield, cfield, what=type(cpu).__name__)
    check_inner_sampled(gpu, cfield, cpu.sensor_model())
