"""Routed-mode inbox sizes and the new entry points' argument checks, without a device."""
import pytest

from ufomap_b200 import capi


def test_colour_inbox_carries_16_byte_hit_records():
    for world, cap_m, cap_h in [(2, 1, 1), (2, 1 << 16, 1 << 18), (4, 1000, 3000), (16, 7, 1 << 20)]:
        mono = capi.route_inbox_bytes(world, cap_m, cap_h)
        color = capi.route_inbox_bytes(world, cap_m, cap_h, color=True)
        # per (parity, source) region: 256 B header, brick records (8 + 64 * 8 B), hit records; 256 B aligned
        region = lambda hit_bytes: 256 + (cap_m * 65 * 8 + 255) // 256 * 256 + (cap_h * hit_bytes + 255) // 256 * 256
        assert mono == 2 * world * region(8)
        assert color == 2 * world * region(16)


def test_inbox_size_rejects_bad_capacities():
    for args in [(1, 1, 1), (17, 1, 1), (2, 0, 1), (2, 1, 0)]:
        for color in (False, True):
            with pytest.raises(capi.UfoError):
                capi.route_inbox_bytes(*args, color=color)


def test_route_mark_ex_binds_and_fails_loudly_without_a_device():
    m = capi.Map(0.1, device=-2)
    buf, layout = capi.pack_points([[1.0, 0.0, 0.0]], [[1, 2, 3]])
    calls = [
        lambda: m.route_mark_ex([0, 0, 0], buf.ctypes.data, 1, layout, depth=6, discrete=True, index_base=3,
                                index_stride=2),
        lambda: m.route_sent(),
    ]
    for call in calls:
        with pytest.raises(capi.UfoError) as e:
            call()
        assert e.value.status == capi.E_CUDA  # no CPU fallback
    m.close()
