"""A map in bounded memory: ufo_b200_retain_bv removes the bricks a bounding volume does not keep and
gives their memory back, ufo_b200_page_out_bv writes them into a page blob first and ufo_b200_page_in
puts them back.  Checked against the map's own earlier state (value field, file image, tree dump,
queries), against a twin map that never retained, and -- for what a retained map does next -- against
the reference fed with the retained map's file image."""
import math
import struct

import numpy as np
import pytest

from helpers import assert_value_fields_equal
from oracle_lib import OracleMap, RefMap, have_ref
from test_gpu_parity import _boundary_cloud
from ufomap_b200 import capi, scans
from ufomap_b200.capi import E_INVALID, E_UNSUPPORTED, Map, UfoError

pytestmark = pytest.mark.gpu

COLORS = [False, True]
BRICK_BYTES = {False: 8 + 16384 + 64, True: 8 + 2 * 16384 + 64}


def _inserts(color, first=0, count=3):
    """Scans at the small sizes of tests/test_gpu_export.py: (map kwargs, insert kwargs)."""
    ins = []
    if color:
        for k in range(first, first + count):
            o, p, c = scans.rgbd(k=k, width=48, height=36)
            ins.append(dict(origin=o, xyz=p, rgb=c, max_range=3.0, discrete=bool(k & 1)))
        return dict(resolution=0.04), ins
    for k in range(first, first + count):
        o, p = scans.velodyne64(k=k, rings=8, azimuths=128)
        ins.append(dict(origin=o, xyz=p, max_range=25.0))
    return dict(resolution=0.2), ins


def _build(color, count=3, bricks=128):
    mkw, ins = _inserts(color, count=count)
    m = Map(color=color, initial_bricks=bricks, **mkw)
    for i in ins:
        m.insert(**i)
    return m, mkw


def _volumes(m):
    mn, mx = m.change_bbox()
    mid, span = (mn + mx) / 2, float(np.min((mx - mn)[:2]))
    s = 0.5 * span
    box = capi.aabb(mid - 0.4 * s, mid + np.array([0.3, 0.5, 0.4]) * s)
    sph = capi.sphere(mid + 0.2 * s, 0.45 * s)
    fru = capi.frustum7(mid, mid + np.array([s, 0.3 * s, 0]), [0, 0, 1], math.pi / 6, math.pi / 5, 0.05 * s, 0.8 * s)
    return {"aabb": [box], "sphere": [sph], "frustum": [fru], "union": [box, capi.sphere(mid - 0.5 * s, 0.3 * s)],
            "none": [], "miss": [capi.sphere([1e4, 1e4, 1e4], 1.0)]}


def _kept(m, codes, volume):
    """The keep rule, restated: per depth-0 code, whether every cube on the path of its brick from the
    root down to the brick's own depth-4 cube passes the volume."""
    L = m.depth_levels
    if len(capi.as_volume(volume)) == 0:
        return np.ones(len(codes), bool)
    half = [m.resolution / 2.0, m.resolution]
    while len(half) <= L:
        half.append(half[-1] * 2.0)
    bricks, inv = np.unique(codes >> np.uint64(12), return_inverse=True)
    c = np.zeros((len(bricks), 3))
    ok = capi.volume_intersects(volume, c, half[L])
    for d in range(L, 4, -1):
        i = (bricks >> np.uint64(3 * (d - 5))) & np.uint64(7)
        for k in range(3):
            c[:, k] = c[:, k] + np.where((i >> np.uint64(k)) & np.uint64(1), half[d - 1], -half[d - 1])
        ok &= capi.volume_intersects(volume, c, half[d - 1])
    return ok[inv]


def _dump(m):
    """beginTree with the contains forms of the filters: every node of the canonical tree."""
    return m.iterate(leaves=False, occupied=True, free=True, unknown=True, contains=True)


def _same_dump(a, b, what=""):
    for x, y, name in zip(a, b, ("codes", "depths", "logodds", "flags", "rgb")):
        if x.dtype == np.float32:
            x, y = x.view(np.uint32), y.view(np.uint32)
        assert x.shape == y.shape and np.array_equal(x, y), "%s: %s differ" % (what, name)


def _restrict(field, mask):
    return tuple(a[mask] for a in field)


def _n_bricks(codes):
    return len(np.unique(codes >> np.uint64(12)))


# -- 1. retain is exact ------------------------------------------------------------------------------
@pytest.mark.parametrize("color", COLORS)
@pytest.mark.parametrize("shape", ["aabb", "sphere", "frustum", "union", "none", "miss"])
def test_retain_is_exact(color, shape):
    m, mkw = _build(color)
    vol = _volumes(m)[shape]
    before = m.value_field()
    image = m.write()
    keep = _kept(m, before[0], vol)
    st = m.retain(vol)
    assert_value_fields_equal(m.value_field(), _restrict(before, keep), what=shape)
    assert st["bricks_kept"] == _n_bricks(before[0][keep])
    if shape == "none":
        assert keep.all() and st["bricks_removed"] == 0 and m.write() == image
    elif shape == "miss":
        assert not keep.any() and m.pool_stats()["bricks"] == 0 and m.pool_stats()["upper_nodes"] == 0
    else:
        assert 0 < keep.sum() < len(keep), "the shape is meant to split the map"
    # the rebuilt levels above the bricks: a fresh map that reads the retained map's node stream
    fresh = Map(color=color, **mkw)
    fresh.read_data(m.write_data())
    _same_dump(_dump(m), _dump(fresh), shape)
    assert m.write() == fresh.write()
    fresh.close()
    m.close()


def test_retain_box_form_is_the_aabb_volume():
    a, _ = _build(False)
    b, _ = _build(False)
    mn, mx = a.change_bbox()
    lo, hi = mn + 0.3 * (mx - mn), mx - 0.25 * (mx - mn)
    sa, sb = a.retain(box=(lo, hi)), b.retain([capi.aabb(lo, hi)])
    assert sa["bricks_kept"] == sb["bricks_kept"] > 0 and sa["bricks_removed"] > 0
    assert a.write() == b.write()


# -- 2. memory comes back ----------------------------------------------------------------------------
@pytest.mark.parametrize("color", COLORS)
def test_memory_comes_back(color):
    m, _ = _build(color, count=4, bricks=16)
    before = m.value_field()
    p0 = m.pool_stats()
    assert p0["bricks"] >= _n_bricks(before[0]) and p0["bricks"] <= p0["brick_cap"]
    mn, mx = m.change_bbox()
    mid = (mn + mx) / 2
    vol = [capi.sphere(mid, 0.12 * float(np.min((mx - mn)[:2])))]
    keep = _kept(m, before[0], vol)
    st = m.retain(vol)
    p1 = m.pool_stats()
    assert st["bricks_before"] == p0["bricks"] and st["bricks_kept"] == p1["bricks"] == _n_bricks(before[0][keep])
    assert st["bricks_removed"] == p0["bricks"] - p1["bricks"] > p0["bricks"] // 2
    assert (st["brick_cap_before"], st["brick_cap_after"]) == (p0["brick_cap"], p1["brick_cap"])
    assert (st["device_bytes_before"], st["device_bytes_after"]) == (p0["device_bytes"], p1["device_bytes"])
    assert p1["brick_cap"] < p0["brick_cap"] and p1["device_bytes"] < p0["device_bytes"]
    assert p1["brick_cap"] >= 2 * p1["bricks"]
    # a later scan that needs the pools to grow again, against a twin that starts from the retained image
    twin = Map(color=color, initial_bricks=16, **_inserts(color)[0])
    twin.read_data(m.write_data())
    _, more = _inserts(color, first=4, count=1)
    m.insert(**more[0])
    twin.insert(**more[0])
    assert_value_fields_equal(m.value_field(), twin.value_field())
    assert m.stats()["regrows"] >= 1 and m.pool_stats()["brick_cap"] > p1["brick_cap"]
    twin.close()


# -- 3. round trip -----------------------------------------------------------------------------------
@pytest.mark.parametrize("color", COLORS)
def test_page_round_trip(color):
    m, mkw = _build(color)
    twin, _ = _build(color)
    vol = _volumes(m)["union"]
    field, image, dump = m.value_field(), m.write(), _dump(m)
    rng = np.random.default_rng(3)
    codes = np.concatenate([field[0][rng.integers(0, len(field[0]), 400)], rng.integers(0, 1 << 48, 100).astype(np.uint64)])
    depths = rng.integers(0, 7, len(codes)).astype(np.uint32)
    answers = m.query(codes, depths)
    blob = m.page_out(vol)
    assert m.write() == image, "page_out leaves the map alone"
    info = capi.page_info(blob)
    keep = _kept(m, field[0], vol)
    assert info["n_bricks"] == _n_bricks(field[0][~keep]) > 0
    assert info["bytes"] == len(blob) == 64 + info["n_bricks"] * BRICK_BYTES[color]
    assert (info["color"], info["depth_levels"], info["resolution"]) == (int(color), 16, mkw["resolution"])
    assert np.array_equal(blob, twin.page_out(vol)), "equal maps give equal blobs"
    st = m.retain(vol)
    assert st["bricks_removed"] >= info["n_bricks"]
    back = m.page_in(blob.tobytes())
    assert back["bricks_kept"] == back["bricks_before"] + info["n_bricks"]
    assert m.write() == image
    assert_value_fields_equal(m.value_field(), field)
    _same_dump(_dump(m), dump)
    for got, want in zip(m.query(codes, depths), answers):
        assert np.array_equal(got.view(np.uint8), want.view(np.uint8))
    m.close()
    twin.close()


# -- 4. the map keeps working like the reference ------------------------------------------------------
@pytest.mark.skipif(not have_ref(), reason="reference harness not built")
@pytest.mark.parametrize("color", COLORS)
@pytest.mark.parametrize("reenter", [False, True])
def test_scans_after_a_retain_match_the_reference(color, reenter):
    m, mkw = _build(color)
    mn, mx = m.change_bbox()
    span = float(np.min((mx - mn)[:2]))
    # reenter: the later scans reach into removed space; otherwise their range stays inside the kept sphere
    reach = (3.0 if color else 25.0) if reenter else 0.2 * span
    vol = [capi.sphere(scans.sensor_origin(0) if not color else np.zeros(3), 0.35 * span)]
    st = m.retain(vol)
    assert st["bricks_removed"] > 0 and st["bricks_kept"] > 0
    ref = RefMap(color=color, **mkw)
    assert ref.read(m.write())
    m.reset_change_bbox()
    ref.reset_change_bbox()
    _, later = _inserts(color, first=3, count=3)
    later[1].update(discrete=True, depth=2)
    for ins in later:
        ins["max_range"] = reach
        m.insert(**ins)
        ref.insert(**ins)
    assert_value_fields_equal(m.value_field(), ref.value_field(), what="after retain")
    a, b = m.change_bbox(), ref.change_bbox()
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    m.close()


# -- 5. a window that follows the sensor ---------------------------------------------------------------
@pytest.mark.parametrize("color", COLORS)
def test_window_follows_the_sensor(color):
    res, reach, half, step, bricks = (0.05, 2.5, 2.8, 1.8, 128) if color else (0.1, 8.0, 10.0, 3.0, 512)
    kw = dict(resolution=res, color=color, initial_bricks=bricks)
    win, twin = Map(**kw), Map(**kw)
    blobs, peak = {}, 0

    def scan(k):
        o = np.array([0.013 + step * k, 0.021, 0.007])
        if color:
            o, p, c = scans.rgbd(k=k, width=48, height=36, origin=o, room_lo=(-1.0, -1.2, -1.0), room_hi=(25.0, 1.2, 1.0))
            return dict(origin=o, xyz=p, rgb=c, max_range=reach)
        o, p = scans.velodyne64(k=k, rings=8, azimuths=256, origin=o)
        return dict(origin=o, xyz=p, max_range=reach)

    for k in range(12):
        ins = scan(k)
        box = [capi.aabb(ins["origin"] - half, ins["origin"] + half)]  # wider than the sensor's reach
        for key in [key for key, blob in blobs.items() if _blob_touches(win, blob, box)]:
            win.page_in(blobs.pop(key))
        win.insert(**ins)
        twin.insert(**ins)
        peak = max(peak, win.pool_stats()["device_bytes"])
        blob = win.page_out(box)
        if capi.page_info(blob)["n_bricks"]:
            blobs[k] = blob
        win.retain(box)
        peak = max(peak, win.pool_stats()["device_bytes"])
    assert len(blobs) >= 3, "the window is meant to leave pages behind"
    assert peak < twin.pool_stats()["device_bytes"]
    assert win.pool_stats()["bricks"] < twin.pool_stats()["bricks"]
    for blob in blobs.values():
        win.page_in(blob)
    assert win.write() == twin.write()
    assert_value_fields_equal(win.value_field(), twin.value_field())
    win.close()
    twin.close()


def _blob_touches(m, blob, volume):
    """Whether the volume keeps any brick of the blob."""
    k = capi.page_keys(blob).astype(np.uint64) << np.uint64(4)
    codes = np.array([m.key_to_code(x) for x in k], np.uint64)
    return bool(_kept(m, codes, volume).any())


# -- 6. thresholds changed while paged out --------------------------------------------------------------
@pytest.mark.parametrize("color", COLORS)
def test_thresholds_change_while_paged_out(color):
    m, _ = _build(color)
    twin, _ = _build(color)
    vol = _volumes(m)["sphere"]
    blob = m.page_out(vol)
    m.retain(vol)
    for x in (m, twin):
        x.set_sensor_model_field(0, 0.8)
        x.set_sensor_model_field(1, 0.35)
    m.page_in(blob)
    _same_dump(_dump(m), _dump(twin))
    assert m.write() == twin.write()
    m.close()
    twin.close()


# -- 7. refusals, nothing applied ------------------------------------------------------------------------
def _refused(m, call, status, state=lambda m: m.write()):
    before = state(m)
    with pytest.raises(UfoError) as e:
        call()
    assert e.value.status == status, str(e.value)
    assert state(m) == before


@pytest.mark.parametrize("color", COLORS)
def test_page_in_refusals(color):
    m, mkw = _build(color)
    vol = _volumes(m)["aabb"]
    blob = m.page_out(vol)
    _refused(m, lambda: m.page_in(blob), E_INVALID)  # its bricks exist
    m.retain(vol)
    bad = blob.copy()
    bad[0] ^= 0xFF
    _refused(m, lambda: m.page_in(bad), E_INVALID)
    bad = blob.copy()
    bad[8] = 2  # format version
    _refused(m, lambda: m.page_in(bad), E_INVALID)
    _refused(m, lambda: m.page_in(blob[:-16]), E_INVALID)
    _refused(m, lambda: m.page_in(blob[:40]), E_INVALID)
    bad = blob.copy()
    bad[64:72], bad[72:80] = blob[72:80], blob[64:72]  # keys out of order
    _refused(m, lambda: m.page_in(bad), E_INVALID)
    other = Map(color=not color, **mkw)
    _refused(other, lambda: other.page_in(blob), E_INVALID)
    other.close()
    other = Map(color=color, resolution=mkw["resolution"] * 2)
    _refused(other, lambda: other.page_in(blob), E_INVALID)
    other.close()
    other = Map(color=color, depth_levels=15, **mkw)
    _refused(other, lambda: other.page_in(blob), E_INVALID)
    other.close()
    m.page_in(blob)
    twin, _ = _build(color)
    assert m.write() == twin.write()
    m.close()
    twin.close()


def test_unsupported_maps_are_refused():
    o, p = scans.random_shell(n=500, rmin=0.3, rmax=1.5)
    box = (np.full(3, -0.5), np.full(3, 0.5))
    small = Map(0.25, depth_levels=4)
    small.insert(o, p, max_range=1.5)
    def state(m):
        return [a.tobytes() for a in m.value_field()] + [m.pool_stats()]

    for call in (lambda: small.retain(box=box), lambda: small.page_out(box=box)):
        _refused(small, call, E_UNSUPPORTED, state)
    hdr = struct.pack("<QIIQIIQ24x", int.from_bytes(b"UFOPAGE1", "little"), 1, 0, struct.unpack("<Q", struct.pack("<d", 0.25))[0], 4, 0, 0)
    _refused(small, lambda: small.page_in(hdr), E_UNSUPPORTED, state)
    small.close()
    routed = Map(0.1, initial_bricks=1 << 10)
    routed.route_setup(0, 2, cap_bricks=64, cap_hits=64)
    for call in (lambda: routed.retain(box=box), lambda: routed.page_out(box=box), lambda: routed.page_in(hdr)):
        _refused(routed, call, E_UNSUPPORTED, state)
    routed.close()


# -- 8. change detection and alias state survive -----------------------------------------------------------
def test_recorded_changes_move_with_their_bricks():
    mkw, ins = _inserts(False)
    m = Map(initial_blocks=1 << 12, **mkw)
    m.enable_change_detection()
    for i in ins:
        m.insert(**i)
    vol = _volumes(m)["union"]
    changed = m.changed_codes(0)
    assert len(changed)
    m.retain(vol)
    assert np.array_equal(m.changed_codes(0), changed[_kept(m, changed, vol)])
    # a paged-in brick records nothing
    blob = m.page_out([capi.sphere([1e4, 1e4, 1e4], 1.0)])
    m.retain([capi.sphere([1e4, 1e4, 1e4], 1.0)])
    assert len(m.changed_codes(0)) == 0
    m.page_in(blob)
    assert len(m.changed_codes(0)) == 0
    m.close()


def test_out_of_tree_marks_after_a_retain():
    """A map that has seen keys outside the tree (tests/test_gpu_parity.py,
    test_rays_leaving_through_plus_faces_alias) retains -- every brick that owns voxels is kept, the
    bricks that only collect such marks go -- and takes one more such scan."""
    o, p = _boundary_cloud(40.0)
    kw = dict(resolution=0.5, depth_levels=6)
    ins = dict(origin=o, xyz=p, max_range=-1.0)
    m, cpu = Map(initial_blocks=1 << 14, **kw), OracleMap(**kw)
    m.insert(**ins)
    cpu.insert(**ins)
    everything = [capi.aabb([-17.0] * 3, [17.0] * 3)]
    bricks = _n_bricks(m.value_field()[0])
    st = m.retain(everything)
    assert st["bricks_kept"] == bricks and st["bricks_removed"] > 0
    assert_value_fields_equal(m.value_field(), cpu.value_field())
    m.insert(**ins)
    cpu.insert(**ins)
    assert_value_fields_equal(m.value_field(), cpu.value_field())
    m.close()


def test_facade_round_trip(tmp_path):
    """tests/cpp/facade_retain.cpp: page out, retain and page in through the C++ facade, both map types."""
    import subprocess
    from test_facade_retain import build_facade_retain
    out = subprocess.run([build_facade_retain(tmp_path)], capture_output=True, text=True)
    assert out.returncode == 0 and "facade retain ok" in out.stdout, (out.returncode, out.stdout, out.stderr)
