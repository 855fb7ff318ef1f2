"""Opening a saved map through the C++ facade (include/ufomap_b200/ufomap.hpp, tests/cpp/facade_read.cpp):
the file constructors, read(std::istream&) and readType compile for both map types, readType needs
no device, and on a device a file the facade wrote opens and iterates."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    """The facade program, built outside the source tree (which may be read-only)."""
    path = str(tmp_path_factory.mktemp("facade") / "facade_read")
    lib_dir = os.path.join(ROOT, "ufomap_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_read.cpp"), "-o", path,
                           "-L" + lib_dir, "-lufomap_b200", "-Wl,-rpath," + lib_dir])
    return path


def test_facade_read_compiles_and_reads_types(exe):
    out = subprocess.run([exe, "--no-device"], capture_output=True, text=True)
    assert out.returncode == 0 and "facade read ok (no device)" in out.stdout, (out.returncode, out.stdout,
                                                                                out.stderr)


@pytest.mark.gpu
def test_facade_opens_a_saved_map(exe, tmp_path):
    out = subprocess.run([exe, str(tmp_path)], capture_output=True, text=True)
    assert out.returncode == 0 and "facade read ok:" in out.stdout, (out.returncode, out.stdout, out.stderr)
