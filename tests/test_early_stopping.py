"""Early stopping without a device: the new C-ABI entry points and their argument checks, and the
free set that the device is compared against, pinned between the C oracle and the reference."""
import ctypes as C

import numpy as np
import pytest

from oracle_lib import OracleMap, RefMap, have_ref
from ufomap_b200 import capi, scans


def test_symbols_resolve():
    lib = capi.load()
    for name in ("ufo_b200_set_early_stopping", "ufo_b200_last_early_stats"):
        assert hasattr(lib, name)
    assert C.sizeof(capi.EarlyStats) == 7 * 8 + 3 * 4 + 4  # trailing padding to 8-byte alignment


def test_set_early_stopping_validates_its_arguments():
    lib = capi.load()
    m = capi.Map(0.1, device=-2)
    m.set_early_stopping(True)
    m.set_early_stopping(False)
    for bad in (2, -1, 7):
        with pytest.raises(capi.UfoError) as e:
            m.set_early_stopping(bad)
        assert e.value.status == capi.E_INVALID
    assert lib.ufo_b200_set_early_stopping(None, 1) == capi.E_INVALID
    assert lib.ufo_b200_last_early_stats(m.h, None) == capi.E_INVALID
    # opting in does not make a CPU path appear: a handle without a device still refuses to insert
    m.set_early_stopping(True)
    with pytest.raises(capi.UfoError) as e:
        m.insert([0, 0, 0], [[1.0, 0, 0]], early_stopping=3)
    assert e.value.status == capi.E_CUDA
    m.close()


@pytest.mark.skipif(not have_ref(), reason="needs the compiled reference (oracle/_ref)")
@pytest.mark.parametrize("depth", [0, 2, 5])
@pytest.mark.parametrize("simple", [False, True])
@pytest.mark.parametrize("stop", [1, 2, 3, 7])
def test_oracle_free_set_matches_the_reference(stop, simple, depth):
    o, p = scans.random_shell(n=1500, seed=11 + stop, rmin=0.3, rmax=2.5)
    ref = RefMap(0.05).free_set(o, p, depth=depth, simple=simple, early_stopping=stop)
    orc = OracleMap(0.05).free_set(o, p, depth=depth, simple=simple, early_stopping=stop)
    assert np.array_equal(np.sort(ref), np.sort(orc))
    # at depth 0 the option does something here: the free set without it is larger
    full = RefMap(0.05).free_set(o, p, depth=depth, simple=simple, early_stopping=0)
    assert len(ref) < len(full) if depth == 0 else len(ref) <= len(full)


def test_facade_setter_compiles(tmp_path):
    """OccupancyMap::setEarlyStoppingExact(bool) next to lastStatus(), with a plain host compiler."""
    import os
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = tmp_path / "early.cpp"
    src.write_text(
        "#include <ufo/map/occupancy_map.h>\n"
        "int configure(ufo::map::OccupancyMap& map, unsigned early_stopping) {\n"
        "  map.setEarlyStoppingExact(early_stopping != 0);\n"
        "  return map.lastStatus();\n"
        "}\n")
    subprocess.check_call(["g++", "-std=c++17", "-Wall", "-Werror", "-c", "-I" + os.path.join(root, "include"),
                           str(src), "-o", str(tmp_path / "early.o")])
