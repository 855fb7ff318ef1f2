"""Per-node writes and ray insertion through the C++ facade (include/ufomap_b200/ufomap.hpp): every
overload of the reference compiles, depths above 6 are rejected, and known answers on a device."""
import os
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EXE = os.path.join(ROOT, "tests", "cpp", "facade_writes")


def _build():
    lib_dir = os.path.join(ROOT, "ufomap_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_writes.cpp"), "-o", EXE,
                           "-L" + lib_dir, "-lufomap_b200", "-Wl,-rpath," + lib_dir])


def test_facade_writes_compile_and_reject_deep_nodes():
    _build()
    out = subprocess.run([EXE, "--no-device"], capture_output=True, text=True)
    assert out.returncode == 0, out.stdout + out.stderr


@pytest.mark.gpu
def test_facade_writes_on_device():
    _build()
    out = subprocess.run([EXE], capture_output=True, text=True)
    assert out.returncode == 0 and "facade writes ok" in out.stdout, (out.returncode, out.stdout, out.stderr)
