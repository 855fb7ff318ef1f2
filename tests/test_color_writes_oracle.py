"""CPU: the C restatement of the colour map's writers (oracle/ufo_oracle_color_writes.c) equals the
compiled, unmodified reference (oracle/_ref/libufo_ref_color_writes.so): every voxel's log-odds bits
and colour, the file image and the change set."""
import numpy as np
import pytest

import color_writes_lib
from color_writes_lib import ColorWritesOracleMap as OracleMap, ColorWritesRefMap as RefMap, have_ref
from color_writes_lib import mixed_color_batch
from ufomap_b200 import scans

color_writes_lib.build()
pytestmark = pytest.mark.skipif(not have_ref(), reason="the compiled reference is not available")

RES = 0.04


def _both(scanned):
    maps = [RefMap(RES, color=True), OracleMap(RES, color=True)]
    if scanned:
        for k in range(3):
            o, p, c = scans.rgbd(k=k, width=48, height=36)
            for m in maps:
                m.insert(o, p, rgb=c, max_range=3.0, discrete=True)
    maps[0].enable_change_detection(True)
    return maps


def _same(ref, orc):
    a, b = ref.value_field(), orc.value_field()
    assert np.array_equal(a[0], b[0])
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
    assert np.array_equal(a[2], b[2])
    assert ref.write() == orc.write()


def _run(ref, orc, batch):
    ref.reset_change_detection()
    ref.update_nodes_color(*batch)
    changed = orc.update_nodes_color(*batch)
    _same(ref, orc)
    codes, depths = ref.changed_codes()
    assert np.array_equal(np.unique(codes[depths == 0]), changed)


@pytest.mark.parametrize("scanned", [False, True])
@pytest.mark.parametrize("seed", [1, 2])
def test_mixed_colour_batches(scanned, seed):
    """ADD at depths 0..6 interleaved with ADD_COLOR and SET_COLOR, one voxel hit 200 times, black
    colours, entries into untouched space."""
    ref, orc = _both(scanned)
    _run(ref, orc, mixed_color_batch(4000, seed=seed + 10 * scanned))


def test_colour_cases_one_by_one():
    """The cases the blend rule singles out, each checked after its own call."""
    ref, orc = _both(True)
    c = ref.key_to_code([32768 + 5, 32768 + 1, 32768 - 2], 0)
    v = np.float32(0.8473)
    steps = [
        (3, 0.0, (200, 10, 30)),   # setColor on untouched space
        (2, v, (10, 250, 90)),     # blend into a set colour
        (0, v, (0, 0, 0)),         # ADD, colour unchanged
        (2, v, (10, 250, 90)),     # the blend now reads the larger log-odds
        (2, -2.5, (0, 0, 0)),      # (0,0,0) onto a set colour blends towards black
        (3, 0.0, (0, 0, 0)),       # setColor (0,0,0) unsets
        (2, v, (7, 8, 9)),         # an unset colour takes the update
        (2, v, (7, 8, 9)),         # an equal colour returns early; the add still happens
    ]
    for op, val, rgb in steps:
        _run(ref, orc, ([c], 0, op, val, [rgb]))


def test_reference_refuses_what_it_cannot_compile():
    ref = RefMap(RES, color=True)
    c = ref.key_to_code([32768, 32768, 32768], 0)
    with pytest.raises(RuntimeError):
        ref.update_nodes_color([c], 0, 1, 0.5, [(1, 2, 3)])
    mono = RefMap(RES)
    with pytest.raises(RuntimeError):
        mono.update_nodes_color([c], 0, 2, 0.5, [(1, 2, 3)])
