"""The mapping server's get_map, clear_volume and save_map bodies through the C++ facade
(include/ufomap_b200/ufomap.hpp, tests/cpp/facade_volumes.cpp): they compile unchanged, the shape
constructors give the reference's doubles, bad volumes are rejected, and known answers on a device."""
import os
import struct
import subprocess

import numpy as np
import pytest

import volumes_lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    """The facade program, built once per module outside the source tree (which may be read-only)."""
    path = str(tmp_path_factory.mktemp("facade") / "facade_volumes")
    lib_dir = os.path.join(ROOT, "ufomap_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_volumes.cpp"), "-o", path,
                           "-L" + lib_dir, "-lufomap_b200", "-Wl,-rpath," + lib_dir])
    return path


def _doubles(line):
    return np.array([struct.unpack("<d", struct.pack("<Q", int(h, 16)))[0] for h in line.split()[1:]])


def test_facade_volumes_compile_and_reject(exe):
    out = subprocess.run([exe, "--no-device"], capture_output=True, text=True)
    assert out.returncode == 0 and "facade volumes ok (no device)" in out.stdout, (out.returncode, out.stdout, out.stderr)
    if not volumes_lib.have_ref():
        pytest.skip("reference volume checker not built: constructors not compared")
    got = {line.split()[0]: _doubles(line) for line in out.stdout.splitlines() if " " in line and "ok" not in line}
    want = {
        "frustum": volumes_lib.ref_frustum7([0.5, -1, 0.25], [0.5, 2, 0.25], [0, 0, 1], 0.7, 1.1, 0.1, 3.0),
        "plane": volumes_lib.ref_plane3([0.1, 0.2, 0.3], [1.3, -0.2, 0.7], [-0.4, 0.9, 1.1]),
        "ray": volumes_lib.ref_ray([0.1, 0.2, 0.3], [0.3, -0.7, 2.9]),
        "obb": volumes_lib.ref_quaternion_rpy(0.3, -0.2, 1.1),
    }
    for k, v in want.items():
        assert np.array_equal(got[k].view(np.uint64), v.view(np.uint64)), k


@pytest.mark.gpu
def test_facade_volumes_on_device(exe, tmp_path):
    out = subprocess.run([exe, str(tmp_path / "saved.ufo")], capture_output=True, text=True)
    assert out.returncode == 0 and "facade volumes ok" in out.stdout, (out.returncode, out.stdout, out.stderr)
