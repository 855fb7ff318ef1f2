"""Early stopping on the device (ufo_early.cuh) against the compiled reference and the C oracle.

A map that opted in with set_early_stopping(True) must produce the reference's map for
insertPointCloud[Discrete](..., early_stopping=E): the value field bit for bit, inner aggregates
as pure functions of it.  Maps that did not opt in, and routed passes, keep rejecting the option.
"""
import numpy as np
import pytest

from helpers import assert_value_fields_equal, check_inner_against_field, check_inner_sampled, sorted_field_large
from oracle_lib import OracleMap, RefMap, have_ref
from ufomap_b200 import capi, scans
from ufomap_b200.capi import E_UNSUPPORTED, Map, UfoError

pytestmark = pytest.mark.gpu


def _early_map(color=False, initial_blocks=1 << 14, **kw):
    m = Map(color=color, initial_blocks=initial_blocks, **kw)
    m.set_early_stopping(True)
    return m


def _run(map_kw, inserts, color=False, oracle=True, levels=(1, 2, 3, 4, 5, 6, 9), initial_blocks=1 << 14):
    """Every insert on the device and on the CPU checkers; returns the device map's last early stats."""
    gpu = _early_map(color=color, initial_blocks=initial_blocks, **map_kw)
    cpus = [RefMap(color=color, **map_kw)] if have_ref() else []
    if oracle or not cpus:
        cpus.append(OracleMap(color=color, **map_kw))
    for ins in inserts:
        gpu.insert(**ins)
        for c in cpus:
            c.insert(**ins)
    field = gpu.value_field()
    for c in cpus:
        assert_value_fields_equal(field, c.value_field(), color_tol=0, what=type(c).__name__)
    check_inner_against_field(gpu, cpus[0].value_field(), cpus[0].sensor_model(), levels=levels)
    st = gpu.early_stats()
    gpu.close()
    return st


@pytest.mark.parametrize("discrete", [False, True])
@pytest.mark.parametrize("depth", [0, 1, 3, 5])
@pytest.mark.parametrize("simple", [False, True])
@pytest.mark.parametrize("stop", [1, 2, 3, 7, 10 ** 6])
def test_matrix(stop, simple, depth, discrete):
    o, p = scans.random_shell(n=1500, rmin=0.5, rmax=4.0)
    st = _run(dict(resolution=0.05), [dict(origin=o, xyz=p, max_range=3.0, depth=depth, simple=simple,
                                           discrete=discrete, early_stopping=stop)])
    assert st["rounds"] >= 1 and st["converged"] == 1


@pytest.mark.parametrize("res", [0.05, 0.02])
def test_velodyne_reduced(res):
    o, p = scans.velodyne64(rings=16, azimuths=512)
    st = _run(dict(resolution=res), [dict(origin=o, xyz=p, max_range=30.0, early_stopping=3)], oracle=False)
    print("velodyne 16x512 @ %g m: %r" % (res, st))


def test_velodyne_full_5cm():
    """64 x 2048 returns: one ring-major scan, the order the rounds have to resolve (the same scan at
    2 cm is test_full_size_config[2])."""
    o, p = scans.velodyne64()
    st = _run(dict(resolution=0.05), [dict(origin=o, xyz=p, max_range=30.0, early_stopping=3)], oracle=False,
              levels=(1, 2, 4, 5, 9))
    print("velodyne 64x2048 @ 5 cm: %r" % st)


def test_rgbd_color_discrete():
    o, p, c = scans.rgbd(width=160, height=120)
    o2, p2, c2 = scans.rgbd(k=2, width=160, height=120)
    _run(dict(resolution=0.02), [dict(origin=o, xyz=p, rgb=c, max_range=3.0, discrete=True, early_stopping=2),
                                 dict(origin=o2, xyz=p2, rgb=c2, max_range=3.0, discrete=True, early_stopping=5)],
         color=True)


def test_random_shell_stream():
    ins = []
    for k in range(4):
        o, p = scans.random_shell(n=3000, seed=42 + k, origin=(0.013 + 0.3 * k, 0.021, 0.007))
        ins.append(dict(origin=o, xyz=p, max_range=5.0, early_stopping=1 + k, simple=k == 3))
    _run(dict(resolution=0.05), ins)


def test_velodyne_stream_async_and_growth():
    """4 scans enqueued with async = 1 into a map created far too small: the pools and the
    early-stopping buffers grow mid-scan and the scans are repeated."""
    ins = [dict(origin=o, xyz=p, max_range=20.0, early_stopping=2)
           for o, p in (scans.velodyne64(k=k, rings=8, azimuths=512) for k in range(4))]
    gpu = _early_map(resolution=0.05, initial_blocks=64)
    sync = _early_map(resolution=0.05)
    for ins_k in ins:
        gpu.insert(async_=True, **ins_k)
        sync.insert(**ins_k)
    gpu.wait()
    assert gpu.stats()["bricks_in_map"] > 16
    assert_value_fields_equal(gpu.value_field(), sync.value_field(), what="async vs sync")
    _run(dict(resolution=0.05), ins, oracle=False, initial_blocks=64)


def test_never_triggering_stop_equals_the_plain_path():
    o, p = scans.velodyne64(rings=16, azimuths=512)
    for kw in (dict(), dict(discrete=True), dict(depth=3), dict(simple=True)):
        a = _early_map(resolution=0.05)
        b = Map(0.05)
        a.insert(o, p, max_range=20.0, early_stopping=10 ** 6, **kw)
        b.insert(o, p, max_range=20.0, **kw)
        assert_value_fields_equal(a.value_field(), b.value_field(), what=repr(kw))


def test_shards_union_equals_the_single_map():
    world = 3
    full = _early_map(resolution=0.05)
    shards = [_early_map(resolution=0.05) for _ in range(world)]
    for r, m in enumerate(shards):
        m.set_shard(r, world)
    for k in range(2):
        o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
        for m in [full] + shards:
            m.insert(o, p, max_range=20.0, early_stopping=2)
    fields = [m.value_field() for m in shards]
    codes = np.concatenate([f[0] for f in fields])
    assert len(np.unique(codes)) == len(codes), "shards overlap"
    order = np.argsort(codes, kind="stable")
    union = (codes[order], np.concatenate([f[1] for f in fields])[order], np.concatenate([f[2] for f in fields])[order])
    assert_value_fields_equal(union, full.value_field(), what="union of shards")


def test_rays_leaving_through_plus_faces_alias():
    rng = np.random.default_rng(7)
    o = np.array([0.3, -0.2, 0.1])
    p = np.concatenate([np.array([[15.99, 15.99, 15.99], [16.0, 0.1, 0.1], [0.5, 16.0, 0.5]]),
                        rng.uniform(-40, 40.0, size=(3000, 3))]).astype(np.float32).astype(np.float64)
    for disc in (False, True):
        _run(dict(resolution=0.5, depth_levels=6), [dict(origin=o, xyz=p, max_range=-1.0, discrete=disc,
                                                         early_stopping=2)] * 2, levels=(1, 2, 3, 4, 5, 6))


def test_frame_and_pointcloud2_entry_points():
    o, p = scans.velodyne64(rings=8, azimuths=512)
    pose = capi.pose_from_rpy(0.4, -0.2, 0.1, 0.03, -0.02, 0.9)
    local = capi.transform_points(np.array([-0.4, 0.2, -0.1, 1.0, 0.0, 0.0, 0.0]), p)  # any cloud will do
    local = local.astype(np.float32).astype(np.float64)
    world_pts = capi.transform_points(pose, local)
    ref = _early_map(resolution=0.05)
    ref.insert(o, world_pts, max_range=20.0, early_stopping=3)
    a = _early_map(resolution=0.05)
    a.insert_frame(o, local, pose, max_range=20.0, early_stopping=3)
    assert_value_fields_equal(a.value_field(), ref.value_field(), what="frame")
    rec = np.zeros((len(local), 16), np.uint8)
    rec[:, :12] = local.astype(np.float32).view(np.uint8).reshape(-1, 12)
    b = _early_map(resolution=0.05)
    b.insert_pointcloud2(o, rec, 16, frame_pose=pose, max_range=20.0, early_stopping=3)
    assert_value_fields_equal(b.value_field(), ref.value_field(), what="PointCloud2")


def test_device_resident_cloud():
    torch = pytest.importorskip("torch")
    o, p = scans.random_shell(n=2000)
    buf, layout = capi.pack_points(p, None, np.float32)
    d = torch.from_numpy(buf).cuda()
    a = _early_map(resolution=0.05)
    a.insert_packed(o, d.data_ptr(), len(buf), layout, max_range=5.0, on_device=True, early_stopping=2)
    torch.cuda.synchronize()
    b = _early_map(resolution=0.05)
    b.insert(o, p, max_range=5.0, early_stopping=2, dtype=np.float32)
    assert_value_fields_equal(a.value_field(), b.value_field(), what="device cloud")


@pytest.mark.skipif(not have_ref(), reason="needs the compiled reference")
@pytest.mark.parametrize("simple", [False, True])
def test_stats_match_the_reference_free_set(simple):
    o, p = scans.random_shell(n=4000, rmin=1.0, rmax=5.0)
    for stop in (1, 3):
        m = _early_map(resolution=0.05)
        m.set_profiling(1)
        m.insert(o, p, max_range=-1.0, simple=simple, early_stopping=stop)
        st = m.early_stats()
        ref = RefMap(resolution=0.05).free_set(o, p, simple=simple, early_stopping=stop)
        assert st["rounds"] >= 1 and st["converged"] == 1
        assert st["free_nodes"] == len(ref)
        assert st["nodes"] >= st["free_nodes"] and st["visits"] >= st["nodes"]
        assert st["table_bytes"] > 0 and st["id_bytes"] >= 4 * st["visits"]
        assert st["ms_walk"] > 0 and st["ms_rounds"] > 0 and st["ms_mark"] > 0
        m.insert(o, p, max_range=-1.0, simple=simple)
        assert m.early_stats()["rounds"] == 0  # a plain insert reports no early-stopping work


def test_rejected_without_opt_in_and_in_routed_mode():
    m = Map(0.1)
    with pytest.raises(UfoError) as e:
        m.insert([0, 0, 0], [[1.0, 0, 0]], early_stopping=3)
    assert e.value.status == E_UNSUPPORTED
    m.set_early_stopping(True)
    m.insert([0, 0, 0], [[1.0, 0, 0]], early_stopping=3)
    m.set_early_stopping(False)
    with pytest.raises(UfoError) as e:
        m.insert([0, 0, 0], [[1.0, 0, 0]], early_stopping=3)
    assert e.value.status == E_UNSUPPORTED
    maps = [Map(0.05, initial_bricks=1 << 12) for _ in range(2)]
    ptrs = [mm.route_setup(r, 2) for r, mm in enumerate(maps)]
    for mm in maps:
        mm.route_connect(ptrs)
        mm.set_early_stopping(True)
    o, p = scans.velodyne64(rings=8, azimuths=128)
    buf, layout = capi.pack_points(p, None, np.float32)
    for mm in maps:
        with pytest.raises(UfoError) as e:
            mm.route_mark_ex(o, buf.ctypes.data, len(buf), layout, max_range=10.0, early_stopping=2)
        assert e.value.status == E_UNSUPPORTED


@pytest.mark.skipif(not have_ref(), reason="needs the compiled reference")
@pytest.mark.parametrize("config", [2, 4])
def test_full_size_config(config):
    """One full 131 072-point scan of config #2 (2 cm, 30 m) or #4 (5 cm, 100 m) with E = 3."""
    res, rng = (0.02, 30.0) if config == 2 else (0.05, 100.0)
    o, p = scans.velodyne64(k=0)
    gpu = _early_map(resolution=res, initial_bricks=1 << 18)
    gpu.insert(o, p, max_range=rng, early_stopping=3)
    ref = RefMap(resolution=res)
    ref.insert(o, p, max_range=rng, early_stopping=3)
    field = sorted_field_large(gpu)
    rf = ref.value_field()
    assert_value_fields_equal(field, rf, what="config #%d" % config)
    check_inner_sampled(gpu, rf, ref.sensor_model())
    print("config #%d: %r" % (config, gpu.early_stats()))
