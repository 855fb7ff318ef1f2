"""Replays the committed fixtures (tests/golden/*.npz, generated from the unmodified
reference by tests/golden/make_golden.py) through
  * the CPU oracle restatement            (no GPU needed), and
  * the CUDA path via the C ABI            (-m gpu),
so both are pinned to reference outputs even where /root/reference is absent."""
import glob
import os

import numpy as np
import pytest

from helpers import assert_value_fields_equal
from oracle_lib import OracleMap

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
SCAN_CASES = sorted(os.path.basename(f)[:-4] for f in glob.glob(os.path.join(GOLD, "*.npz"))
                    if not f.endswith("indexing.npz")
                    and not os.path.basename(f).startswith(("frame_", "fileimage_")))


def _load_case(name):
    z = np.load(os.path.join(GOLD, name + ".npz"))
    map_kw = {k[4:]: z[k].item() for k in z.files if k.startswith("map_")}
    map_kw = {k: (bool(v) if k == "automatic_pruning" else v) for k, v in map_kw.items()}
    inserts = []
    for i in range(int(z["n_inserts"])):
        pre = "ins%d_" % i
        ins = {k[len(pre):]: z[k] for k in z.files if k.startswith(pre)}
        for k in ("max_range", "depth", "simple", "discrete", "early_stopping"):
            if k in ins:
                ins[k] = ins[k].item()
        inserts.append(ins)
    return z, map_kw, inserts, bool(z["color"])


def _replay(cls, name, **extra):
    z, map_kw, inserts, color = _load_case(name)
    m = cls(color=color, **map_kw, **extra)
    for ins in inserts:
        m.insert(**ins)
    return z, m


def test_fixture_inventory():
    assert len(SCAN_CASES) >= 4


@pytest.mark.parametrize("name", SCAN_CASES)
def test_oracle_matches_golden(name):
    z, m = _replay(OracleMap, name)
    assert_value_fields_equal(m.value_field(), (z["codes"], z["occ"], z["rgb"]), what=name)
    ic, idp, iocc, irgb, ifl = m.walk(False)
    ka, kb = np.lexsort((ic, idp)), np.lexsort((z["inner_codes"], z["inner_depths"]))
    assert np.array_equal(ic[ka], z["inner_codes"][kb])
    assert np.array_equal(iocc[ka].view(np.uint32), z["inner_occ"][kb].view(np.uint32))
    assert np.array_equal(ifl[ka], z["inner_flags"][kb])
    assert np.array_equal(irgb[ka], z["inner_rgb"][kb])
    mn, mx = m.change_bbox()
    assert np.array_equal(mn, z["bbox_min"]) and np.array_equal(mx, z["bbox_max"])
    assert np.array_equal(m.sensor_model(), z["sensor_model"])


def _check_indexing(m):
    z = np.load(os.path.join(GOLD, "indexing.npz"))
    for i, d in enumerate(z["depths"]):
        for j, p in enumerate(z["pts"]):
            k = m.to_key(p, int(d))
            assert np.array_equal(k, z["keys"][i, j])
            assert m.to_code(p, int(d)) == int(z["codes"][i, j])
            assert m.key_to_code(k, int(d)) == int(z["codes"][i, j])
            assert np.array_equal(m.key_to_coord(k, int(d)), z["coords"][i, j])
            assert np.array_equal(m.code_to_key(int(z["codes"][i, j]), int(d)), k)
    for si, (d, mr) in enumerate(z["ray_specs"]):
        flat, lens = z["ray%d_codes" % si], z["ray%d_lens" % si]
        off = 0
        for a, b, n in zip(z["ray_a"], z["ray_b"], lens):
            assert np.array_equal(m.compute_ray(a, b, float(mr), int(d)), flat[off:off + n])
            off += n
    return z


def test_oracle_indexing_and_rays_match_golden():
    m = OracleMap(0.05)
    z = _check_indexing(m)
    for fi, (d, simple) in enumerate(z["free_specs"]):
        got = np.sort(m.free_set(z["free_origin"], z["free_ends"], int(d), bool(simple)))
        assert np.array_equal(got, z["free%d" % fi])


def test_cuda_library_host_geometry_matches_golden():
    """The C-ABI's host-side helpers (toKey/toCode/toCoord/computeRay) need no GPU:
    checked here through a geometry-only handle."""
    from ufomap_b200.capi import Map
    m = Map(0.05, device=-2)
    _check_indexing(m)
    m.close()


def _frame_fixture():
    return np.load(os.path.join(GOLD, "frame_velodyne_10cm.npz"))


def test_oracle_frame_transform_matches_golden():
    """Pose6(x,y,z,r,p,y) and PointCloud::transform outputs of the reference, bit for bit."""
    from oracle_lib import ORACLE_SO, _load
    api = _load(ORACLE_SO, "ufo_oracle_")
    z = _frame_fixture()
    m = OracleMap(float(z["resolution"]))
    for k in range(int(z["n_inserts"])):
        pose = np.empty(7)
        api["pose_from_rpy"](*[float(v) for v in z["pose%d" % k][:3]], *[float(v) for v in z["rpy%d" % k]],
                             pose.ctypes.data)
        assert pose.tobytes() == z["pose%d" % k].tobytes()
        local = np.ascontiguousarray(z["local%d" % k])
        world = np.empty_like(local)
        api["transform"](pose.ctypes.data, local.ctypes.data, len(local), world.ctypes.data)
        assert world.tobytes() == z["world%d" % k].tobytes()
        m.insert(origin=pose[:3], xyz=world, max_range=float(z["max_range"]))
    assert_value_fields_equal(m.value_field(), (z["codes"], z["occ"], z["rgb"]), what="frame")


def test_cuda_library_host_transform_matches_golden():
    """ufo_b200_pose_from_rpy / ufo_b200_transform_points are host code: no GPU needed."""
    from ufomap_b200 import capi
    z = _frame_fixture()
    for k in range(int(z["n_inserts"])):
        pose = capi.pose_from_rpy(*z["pose%d" % k][:3], *z["rpy%d" % k])
        assert pose.tobytes() == z["pose%d" % k].tobytes()
        for dt in (np.float64, np.float32):
            world = capi.transform_points(pose, z["local%d" % k], dtype=dt)
            assert world.tobytes() == z["world%d" % k].tobytes()


def _replay_file_image(cls, **extra):
    z = np.load(os.path.join(GOLD, "fileimage_rgbd_8cm.npz"))
    m = cls(float(z["resolution"]), color=True, automatic_pruning=False, **extra)
    for k in range(int(z["n_inserts"])):
        m.insert(origin=z["origin%d" % k], xyz=z["xyz%d" % k], rgb=z["rgb%d" % k],
                 max_range=float(z["max_range"]), discrete=True)
    return z["image"].tobytes(), m


def test_oracle_file_image_matches_golden():
    """The reference's own Octree::write output, byte for byte."""
    image, m = _replay_file_image(OracleMap)
    assert m.write() == image


@pytest.mark.gpu
def test_cuda_file_image_matches_golden():
    from ufomap_b200.capi import Map
    image, m = _replay_file_image(Map, initial_blocks=1 << 12)
    assert m.write() == image
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_cuda_frame_insert_matches_golden(dtype):
    """The fused device-side transform == the reference's host transform + insert."""
    from ufomap_b200.capi import Map
    z = _frame_fixture()
    m = Map(float(z["resolution"]), initial_blocks=1 << 12)
    for k in range(int(z["n_inserts"])):
        pose = z["pose%d" % k]
        m.insert_frame(pose[:3], z["local%d" % k], pose, max_range=float(z["max_range"]), dtype=dtype)
    assert_value_fields_equal(m.value_field(), (z["codes"], z["occ"], z["rgb"]), what="frame")
    m.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", SCAN_CASES)
def test_cuda_matches_golden(name):
    from ufomap_b200.capi import Map
    z, m = _replay(Map, name, initial_blocks=1 << 12)
    assert_value_fields_equal(m.value_field(), (z["codes"], z["occ"], z["rgb"]),
                              color_tol=0, what=name)
    # inner nodes of the reference tree == CUDA aggregates (intended getNode semantics)
    occ, flags, rgb = m.query(z["inner_codes"], z["inner_depths"])
    assert np.array_equal(occ.view(np.uint32), z["inner_occ"].view(np.uint32))
    assert np.array_equal(flags & 3, z["inner_flags"] & 3)
    if bool(z["color"]):
        assert np.array_equal(rgb, z["inner_rgb"])
    mn, mx = m.change_bbox()
    assert np.array_equal(mn, z["bbox_min"]) and np.array_equal(mx, z["bbox_max"])
    m.close()
