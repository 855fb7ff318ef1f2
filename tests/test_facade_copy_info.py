"""Copies of facade maps and the RViz plugin's updateInfo call through the C++ facade
(include/ufomap_b200/ufomap.hpp, tests/cpp/facade_copy_info.cpp): copies inside a std::variant,
``auto snapshot = map;``, a copy assignment and a by-value parameter.  Without a device the program
compiles for both map types and the argument checks hold; on a device every copy reports the
source's counters, known box and sensor model, the counters equal those of ufo_b200_tree_info and of
the reference's copy, and a change to a copy leaves the source as it was."""
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def build_facade_copy_info(directory):
    """The facade program, built outside the source tree (which may be read-only)."""
    path = os.path.join(str(directory), "facade_copy_info")
    lib_dir = os.path.join(ROOT, "ufomap_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O1", "-Wall", "-I" + os.path.join(ROOT, "include"),
                           os.path.join(ROOT, "tests", "cpp", "facade_copy_info.cpp"), "-o", path,
                           "-L" + lib_dir, "-lufomap_b200", "-Wl,-rpath," + lib_dir])
    return path


@pytest.fixture(scope="module")
def exe(tmp_path_factory):
    return build_facade_copy_info(tmp_path_factory.mktemp("facade"))


def test_facade_copy_info_compiles_and_rejects(exe):
    out = subprocess.run([exe, "--no-device"], capture_output=True, text=True)
    assert out.returncode == 0 and "facade copy info ok (no device)" in out.stdout, (out.returncode, out.stdout, out.stderr)


def _lines(stdout):
    info = {}
    for line in stdout.splitlines():
        if line.startswith("info "):
            f = line.split()
            info[f[1]] = f[2:]
    return info


@pytest.mark.gpu
@pytest.mark.parametrize("color", [False, True])
def test_facade_copies_on_device(exe, tmp_path, color):
    from ufomap_b200 import scans
    from ufomap_b200.capi import Map
    import info_lib

    res, levels = 0.08, 16
    src = Map(res, levels, color=color, device=0)
    for k in range(2):
        o, p = scans.velodyne64(k=k, rings=16, azimuths=256)
        rgb = np.random.default_rng(k).integers(0, 256, (len(p), 3)).astype(np.uint8) if color else None
        src.insert(o, p, rgb=rgb, max_range=12.0)
    data = src.write_data()
    path = tmp_path / "map.data"
    path.write_bytes(bytes(data))
    out = subprocess.run([exe, str(path), str(res), str(levels), str(int(color))], capture_output=True, text=True)
    assert out.returncode == 0 and "facade copy info ok" in out.stdout, (out.returncode, out.stdout, out.stderr)
    info = _lines(out.stdout)
    for name in ("variant_copy", "variant_assign", "snapshot", "assigned", "by_value", "source_after"):
        assert info[name][:10] == info["source"][:10], name
    assert info["snapshot_after"][:4] != info["source"][:4]

    twin = Map(res, levels, color=color, device=0)
    twin.read_data(bytes(data))
    t = twin.tree_info()
    leaf, inner, size, mem = (int(x) for x in info["source"][:4])
    assert (leaf, inner, size) == (t["num_leaf_nodes"], t["num_inner_nodes"], t["size"])
    assert mem == inner * (24 if color else 16) + leaf * (8 if color else 4)
    upd = [line.split() for line in out.stdout.splitlines() if line.startswith("updateInfo")][0]
    assert (int(upd[2]), int(upd[3]), int(upd[4])) == (leaf, inner, mem)

    # the sensor model of a copy: the reference's copy constructor, toLogit(toProb(x)), bit for bit
    info_lib.build()
    if info_lib.have_ref():
        ref = info_lib.InfoRefMap(res, levels, color=color, prob_hit=0.7123456789)
        ref.read_data(bytes(data))
        rt = ref.tree_info()
        assert (leaf, inner, size, mem) == (rt["num_leaf_nodes"], rt["num_inner_nodes"], rt["size"], rt["memory_usage"])
        centre = [int(x, 16) for x in info["source"][4:10]]
        assert centre == list(np.concatenate([rt["center"], rt["half_size"]]).view(np.uint64))
        model = [int(x, 16) for x in info["snapshot"][10:16]]
        assert model == list(ref.copy().sensor_model().view(np.uint64))
