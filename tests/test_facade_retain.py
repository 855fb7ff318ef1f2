"""retain / pageOut / pageIn through the C++ facade (include/ufomap_b200/ufomap.hpp,
tests/cpp/facade_retain.cpp): they compile for both map types and every volume form, and the argument
checks of the C ABI hold without a device.  The run on a device is in tests/test_gpu_retain.py."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_facade_retain(directory):
    """The facade program, built outside the source tree (which may be read-only)."""
    path = os.path.join(str(directory), "facade_retain")
    lib_dir = os.path.join(ROOT, "ufomap_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_retain.cpp"), "-o", path,
                           "-L" + lib_dir, "-lufomap_b200", "-Wl,-rpath," + lib_dir])
    return path


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return build_facade_retain(tmp_path_factory.mktemp("facade"))


def test_facade_retain_compiles_and_rejects(exe):
    out = subprocess.run([exe, "--no-device"], capture_output=True, text=True)
    assert out.returncode == 0 and "facade retain ok (no device)" in out.stdout, (out.returncode, out.stdout, out.stderr)
