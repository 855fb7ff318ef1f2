"""The colour map's writers through the C++ facade (include/ufomap_b200/ufomap.hpp): the reference's
calling code compiles unchanged, the rejection statuses come back without a device, and known
answers on a device."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    """The facade program, built once per module outside the source tree (which may be read-only)."""
    path = str(tmp_path_factory.mktemp("facade") / "facade_color_writes")
    lib_dir = os.path.join(ROOT, "ufomap_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_color_writes.cpp"), "-o", path,
                           "-L" + lib_dir, "-lufomap_b200", "-Wl,-rpath," + lib_dir])
    return path


def test_facade_colour_writes_compile_and_reject_without_a_device(exe):
    out = subprocess.run([exe, "--no-device"], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


@pytest.mark.gpu
def test_facade_colour_writes_on_device(exe):
    out = subprocess.run([exe], capture_output=True, text=True)
    assert out.returncode == 0 and "facade colour writes ok" in out.stdout, (out.returncode, out.stdout, out.stderr)
