"""The page blob's header and size formula, and the new entry points of the binding, without a
device."""
import struct

import numpy as np
import pytest

from ufomap_b200 import capi

MAGIC = int.from_bytes(b"UFOPAGE1", "little")


def _header(n_bricks, color=0, resolution=0.1, depth_levels=16, magic=MAGIC, version=1):
    bits = struct.unpack("<Q", struct.pack("<d", resolution))[0]
    return struct.pack("<QIIQIIQ24x", magic, version, color, bits, depth_levels, 0, n_bricks)


@pytest.mark.parametrize("color", [0, 1])
@pytest.mark.parametrize("n", [0, 1, 7, 244000])
def test_header_parse_and_size_formula(color, n):
    hdr = _header(n, color=color, resolution=0.02, depth_levels=17)
    assert len(hdr) == 64
    info = capi.page_info(hdr)
    assert info == dict(version=1, color=color, depth_levels=17, resolution=0.02, n_bricks=n,
                        bytes=64 + n * (8 + 4096 * 4 + 64 + color * 4096 * 4))


def test_page_keys_reads_the_key_section():
    keys = np.array([5 | (6 << 21) | (7 << 42), 1 << 20], np.uint64)
    blob = _header(2) + keys.tobytes()
    assert capi.page_keys(blob).tolist() == [[5, 6, 7], [1 << 20, 0, 0]]


def test_foreign_headers_are_refused():
    for bad in (_header(1, magic=MAGIC ^ 1), _header(1, version=2), _header(1, color=2), _header(1 << 40), _header(1)[:63], b""):
        with pytest.raises(capi.UfoError) as e:
            capi.page_info(bad)
        assert e.value.status == capi.E_INVALID


def test_entry_points_bind_and_fail_loudly_without_a_device():
    """Every new wrapper reaches the library with a well-formed call and, on a geometry-only handle,
    fails with UFO_B200_E_CUDA instead of falling back to anything."""
    m = capi.Map(0.1, device=-2)
    box = (np.zeros(3), np.ones(3))
    calls = [
        lambda: m.retain(), lambda: m.retain([capi.sphere([0, 0, 0], 1.0)]), lambda: m.retain(box=box),
        lambda: m.page_out(), lambda: m.page_out([capi.aabb(*box)]), lambda: m.page_out(box=box),
        lambda: m.page_in(_header(0)), lambda: m.page_in(np.frombuffer(_header(0), np.uint8)), lambda: m.pool_stats(),
    ]
    for i, call in enumerate(calls):
        with pytest.raises(capi.UfoError) as e:
            call()
        assert e.value.status == capi.E_CUDA, i
    bad = capi.volume_record(99, [0.0])
    with pytest.raises(capi.UfoError) as e:
        m.retain(bad)
    assert e.value.status == capi.E_INVALID
    m.close()
