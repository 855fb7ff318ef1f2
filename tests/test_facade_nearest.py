"""beginNNTree / beginNNLeaves through the C++ facade (include/ufomap_b200/ufomap.hpp,
tests/cpp/facade_nearest.cpp): the program compiles for both map types and the argument checks of
ufo_b200_nearest hold without a device.  The run on a device is in tests/test_gpu_nearest.py."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_facade_nearest(directory):
    """The facade program, built outside the source tree (which may be read-only)."""
    path = os.path.join(str(directory), "facade_nearest")
    lib_dir = os.path.join(ROOT, "ufomap_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_nearest.cpp"), "-o", path,
                           "-L" + lib_dir, "-lufomap_b200", "-Wl,-rpath," + lib_dir])
    return path


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return build_facade_nearest(tmp_path_factory.mktemp("facade"))


def test_facade_nearest_compiles_and_rejects(exe):
    out = subprocess.run([exe, "--no-device"], capture_output=True, text=True)
    assert out.returncode == 0 and "facade nearest ok (no device)" in out.stdout, (out.returncode, out.stdout, out.stderr)
