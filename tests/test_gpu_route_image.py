"""One file image from several maps: Map.image_part / capi.assemble_image (ufo_b200_image_part_bv,
ufo_b200_image_assemble).

  * one map's part assembled alone == write_bv / write_data_bv / write_compressed_bv, byte for byte
    (mono and colour; no volume, an AABB, a sphere + frustum union, a volume missing the map;
    min_depth 0 / 2 / 4; expanded)
  * the parts of the ranks of a routed map, in any order, assemble to the single map's image and
    compressed image (2 and 4 ranks; mono plain, mono discrete at depths 0 / 3 / 6, colour
    discrete); the compiled reference writes the same file for the plain case
  * assembly refuses parts that do not belong together, malformed parts and a brick given twice
"""
import ctypes as C

import numpy as np
import pytest

from oracle_lib import RefMap, have_ref
from test_gpu_route_discrete import _barrier, _ranks
from ufomap_b200 import capi, scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu


def _volumes(color):
    s = 0.4 if color else 1.0
    return {
        "none": None,
        "aabb": capi.aabb(np.array([-2.1, -1.3, -0.9]) * s, np.array([1.7, 2.9, 0.6]) * s),
        "union": [capi.sphere(np.array([1.1, -0.7, 0.1]) * s, 1.9 * s),
                  capi.frustum7(np.array([-5.0, 0.5, 0.4]) * s, [0.0, 0.0, 0.0], [0, 0, 1], 0.5, 0.8, 0.3 * s,
                                6.0 * s)],
        "miss": capi.sphere([1.0e6, 0.0, 0.0], 1.0),
    }


def _mapped(color):
    if color:
        m = Map(0.02, color=True, initial_bricks=1 << 14)
        for k in range(2):
            o, p, rgb = scans.rgbd(k=k, width=96, height=72)
            m.insert(o, p, rgb=rgb, max_range=4.0, discrete=True, dtype=np.float32)
        return m
    m = Map(0.05, initial_bricks=1 << 14)
    for k in range(2):
        o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
        m.insert(o, p, max_range=10.0, dtype=np.float32)
    return m


@pytest.mark.parametrize("color", [False, True], ids=["mono", "color"])
def test_one_part_assembles_to_the_writers(color):
    m = _mapped(color)
    for name, vol in _volumes(color).items():
        for min_depth in (0, 2, 4):
            for expanded in (False, True):
                part = m.image_part(volume=vol, min_depth=min_depth, expanded=expanded)
                what = (name, min_depth, expanded)
                assert capi.assemble_image([part]) == m.write_bv(vol, min_depth, expanded), what
                if expanded:
                    continue
                assert capi.assemble_image([part], with_header=False) == m.write_data_bv(vol, min_depth), what
                for data_only in (False, True):
                    want = m.write_compressed_bv(vol, min_depth, data_only=data_only)
                    got = capi.assemble_image([part], with_header=not data_only, compressed=True)
                    assert got == want, what + (data_only,)


# (name, colour, depth, discrete, plain route_mark)
CASES = [
    ("mono-plain", False, 0, False, True),
    ("mono-discrete-d0", False, 0, True, False),
    ("mono-discrete-d3", False, 3, True, False),
    ("mono-discrete-d6", False, 6, True, False),
    ("color-discrete-d0", True, 0, True, False),
]


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_routed_union_image_equals_single_map(case, world):
    _, color, depth, discrete, plain = case
    res = 0.02 if color else 0.05
    maps = _ranks(world, res, color=color)
    single = Map(res, color=color, initial_bricks=1 << 15)
    ref = RefMap(res) if plain and have_ref() else None
    for k in range(3):
        if color:
            o, p, rgb = scans.rgbd(k=k, width=96, height=72)
            rng_max = 4.0
        else:
            o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
            rgb, rng_max = None, 10.0
        single.insert(o, p, rgb=rgb, max_range=rng_max, depth=depth, discrete=discrete, dtype=np.float32)
        if ref is not None:
            ref.insert(o, p, max_range=rng_max)
        buf, layout = capi.pack_points(p, rgb, np.float32)
        keep = []
        for r, m in enumerate(maps):
            part = np.ascontiguousarray(buf[r::world])
            keep.append(part)
            if plain:
                m.route_mark(o, part.ctypes.data, len(part), layout, max_range=rng_max)
            else:
                m.route_mark_ex(o, part.ctypes.data, len(part), layout, max_range=rng_max, depth=depth,
                                discrete=discrete, index_base=r, index_stride=world)
        _barrier(maps)
        for m in maps:
            m.route_apply(0, world, True)
        _barrier(maps)
    rng = np.random.default_rng(world)
    for name, vol in _volumes(color).items():
        for min_depth in (0, 2):
            parts = [m.image_part(volume=vol, min_depth=min_depth) for m in maps]
            shuffled = [parts[i] for i in rng.permutation(world)]
            what = (name, min_depth)
            assert capi.assemble_image(parts) == single.write_bv(vol, min_depth), what
            assert capi.assemble_image(shuffled) == single.write_bv(vol, min_depth), what
            assert capi.assemble_image(shuffled, with_header=False) == single.write_data_bv(vol, min_depth), what
            got = capi.assemble_image(shuffled, compressed=True)
            assert got == single.write_compressed_bv(vol, min_depth), what
    parts = [m.image_part(expanded=True) for m in maps]
    assert capi.assemble_image(parts[::-1]) == single.write_bv(expanded=True)
    if ref is not None:
        assert capi.assemble_image([m.image_part() for m in maps]) == ref.write()


def _assemble_status(parts):
    with pytest.raises(capi.UfoError) as e:
        capi.assemble_image(parts)
    return e.value.status


def test_assembly_rejects_parts_that_do_not_belong_together():
    m = _mapped(False)
    part = m.image_part()
    assert len(part) > 56
    # parts of empty maps hold no bricks: only their header can make them not belong
    empty = Map(0.05, initial_bricks=1 << 10)
    assert capi.assemble_image([empty.image_part(), part]) == m.write()
    box = capi.aabb([-1.0, -1.0, -1.0], [1.0, 1.0, 1.0])
    other = {
        "resolution": Map(0.04, initial_bricks=1 << 10).image_part(),
        "depth_levels": Map(0.05, depth_levels=15, initial_bricks=1 << 10).image_part(),
        "colour": Map(0.05, color=True, initial_bricks=1 << 10).image_part(),
        "volume": empty.image_part(volume=box),
        "min_depth": empty.image_part(min_depth=2),
        "expanded": empty.image_part(expanded=True),
    }
    for name, p in other.items():
        assert _assemble_status([part, p]) == capi.E_INVALID, name
    # the same part twice: every brick twice
    assert _assemble_status([part, part]) == capi.E_INVALID
    # truncated, wrong magic, wrong version, trailing bytes, empty, no parts
    bad = {
        "truncated": part[:-1],
        "header only": part[:56],
        "magic": b"XFIP" + part[4:],
        "version": part[:4] + (2).to_bytes(4, "little") + part[8:],
        "trailing": part + b"\0",
        "empty": b"",
    }
    for name, b in bad.items():
        assert _assemble_status([b]) == capi.E_INVALID, name
    assert _assemble_status([]) == capi.E_INVALID


def test_too_small_buffer_only_reports_the_size():
    m = _mapped(False)
    part = np.frombuffer(m.image_part(), np.uint8)
    lib = capi.load()
    ptrs = (C.c_void_p * 1)(part.ctypes.data)
    sizes = (C.c_size_t * 1)(len(part))
    n, u = C.c_size_t(), C.c_size_t()
    assert lib.ufo_b200_image_assemble(ptrs, sizes, 1, 1, 0, 1, 0, None, 0, C.byref(n), C.byref(u)) == capi.OK
    want = m.write()
    assert n.value == len(want)
    out = np.full(n.value, 0xAB, np.uint8)
    assert lib.ufo_b200_image_assemble(ptrs, sizes, 1, 1, 0, 1, 0, out.ctypes.data, n.value - 1, C.byref(n),
                                       C.byref(u)) == capi.OK
    assert n.value == len(want) and (out == 0xAB).all()
    assert lib.ufo_b200_image_assemble(ptrs, sizes, 1, 1, 0, 1, 0, out.ctypes.data, n.value, C.byref(n),
                                       C.byref(u)) == capi.OK
    assert out.tobytes() == want
    # the part itself follows the same convention
    k = C.c_size_t()
    small = np.full(len(part), 0xCD, np.uint8)
    assert lib.ufo_b200_image_part_bv(m.h, None, 0, 0, 0, small.ctypes.data, len(part) - 1, C.byref(k)) == capi.OK
    assert k.value == len(part) and (small == 0xCD).all()
