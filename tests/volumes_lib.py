"""ctypes wrapper of the CPU checker of the bounding-volume paths (TEST INFRASTRUCTURE ONLY), built
by oracle/volumes.mk into oracle/_ref/libufo_ref_volumes.so from the unmodified reference
(ref_volumes.cpp).

* ``VolumesRefMap``      every method of RefMap plus the BoundingVolume forms of writeData / write /
                         readData / setValueVolume / beginLeaves
* ``ref_intersects``     BoundingVolume::intersects(AABB) of the reference for a batch of cubes
* ``ref_frustum7`` ...   the geometry constructors whose arithmetic decides a shape's doubles

Volumes are arrays of ufomap_b200.capi.VOLUME_DTYPE records, the layout of the C ABI.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_lib import ORACLE_DIR, RefMap, _f64
from ufomap_b200.capi import as_volume

REF_VOLUMES_SO = os.path.join(ORACLE_DIR, "_ref", "libufo_ref_volumes.so")
_SOURCES = ("ref_harness.cpp", "ref_volumes.cpp", "volumes.mk")


def build():
    """Compile the library when it is missing or older than its sources (where the reference
    sources exist)."""
    newest = max(os.path.getmtime(os.path.join(ORACLE_DIR, s)) for s in _SOURCES)
    if os.path.isdir("/root/reference/ufomap/include") and (
            not os.path.exists(REF_VOLUMES_SO) or os.path.getmtime(REF_VOLUMES_SO) < newest):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "volumes.mk", "ref"], stdout=subprocess.DEVNULL)


def have_ref():
    return os.path.exists(REF_VOLUMES_SO)


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(REF_VOLUMES_SO)
        vp, sz, dbl, u32, i32 = C.c_void_p, C.c_size_t, C.c_double, C.c_uint, C.c_int
        for name, res, args in (
                ("vol_intersects", None, [vp, sz, vp, vp, sz, vp]),
                ("write_data_bv", sz, [vp, vp, sz, u32, vp, sz]),
                ("write_bv", sz, [vp, vp, sz, u32, i32, i32, i32, vp, sz]),
                ("read_data_bv", i32, [vp, vp, sz, vp, sz]),
                ("set_value_volume_bv", None, [vp, vp, dbl, u32]),
                ("leaves_bv", sz, [vp, i32, i32, i32, vp, sz, u32, vp, vp, vp, sz]),
                ("frustum7", None, [vp, vp, vp, dbl, dbl, dbl, dbl, vp]),
                ("quaternion_rpy", None, [dbl, dbl, dbl, vp]),
                ("ray", None, [vp, vp, vp]),
                ("plane3", None, [vp, vp, vp, vp])):
            f = getattr(lib, "ufo_ref_" + name)
            f.restype = res
            f.argtypes = args
        _lib = lib
    return _lib


def _bv(volume):
    bv = as_volume(volume)
    return bv, (bv.ctypes.data if len(bv) else None), len(bv)


def ref_intersects(volume, centres, half_sizes):
    bv, bp, nb = _bv(volume)
    c = _f64(centres).reshape(-1, 3)
    h = np.asarray(half_sizes, np.float64)
    h = np.ascontiguousarray(np.broadcast_to(h.reshape(-1, 1) if h.ndim <= 1 else h, c.shape))
    out = np.zeros(len(c), np.uint8)
    _load().ufo_ref_vol_intersects(bp, nb, c.ctypes.data, h.ctypes.data, len(c), out.ctypes.data)
    return out.astype(bool)


def ref_frustum7(pos, target, up, vertical_angle, horizontal_angle, near, far):
    out = np.empty(24)
    pos, target, up = _f64(pos), _f64(target), _f64(up)  # kept alive across the call
    _load().ufo_ref_frustum7(pos.ctypes.data, target.ctypes.data, up.ctypes.data,
                             float(vertical_angle), float(horizontal_angle), float(near), float(far), out.ctypes.data)
    return out


def ref_quaternion_rpy(roll, pitch, yaw):
    out = np.empty(4)
    _load().ufo_ref_quaternion_rpy(float(roll), float(pitch), float(yaw), out.ctypes.data)
    return out


def ref_ray(origin, direction):
    out = np.empty(6)
    origin, direction = _f64(origin), _f64(direction)
    _load().ufo_ref_ray(origin.ctypes.data, direction.ctypes.data, out.ctypes.data)
    return out


def ref_plane3(v1, v2, v3):
    out = np.empty(4)
    v1, v2, v3 = _f64(v1), _f64(v2), _f64(v3)
    _load().ufo_ref_plane3(v1.ctypes.data, v2.ctypes.data, v3.ctypes.data, out.ctypes.data)
    return out


class VolumesRefMap(RefMap):
    _path = REF_VOLUMES_SO

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        self.vl = _load()

    def write_data_bv(self, volume=None, min_depth=0):
        bv, bp, nb = _bv(volume)
        n = self.vl.ufo_ref_write_data_bv(self.h, bp, nb, int(min_depth), None, 0)
        buf = np.empty(max(n, 1), np.uint8)
        self.vl.ufo_ref_write_data_bv(self.h, bp, nb, int(min_depth), buf.ctypes.data, n)
        return buf[:n].tobytes()

    def write_bv(self, volume=None, min_depth=0, compress=False, acceleration=1, level=0):
        bv, bp, nb = _bv(volume)
        args = (int(min_depth), int(compress), int(acceleration), int(level))
        n = self.vl.ufo_ref_write_bv(self.h, bp, nb, *args, None, 0)
        buf = np.empty(max(n, 1), np.uint8)
        self.vl.ufo_ref_write_bv(self.h, bp, nb, *args, buf.ctypes.data, n)
        return buf[:n].tobytes()

    def read_data_bv(self, data, volume=None):
        bv, bp, nb = _bv(volume)
        buf = np.frombuffer(data, np.uint8)
        return bool(self.vl.ufo_ref_read_data_bv(self.h, bp, nb, buf.ctypes.data if len(buf) else None, len(buf)))

    def set_value_volume_bv(self, shape, occupancy, min_depth=0):
        bv = as_volume(shape)
        assert len(bv) == 1
        self.vl.ufo_ref_set_value_volume_bv(self.h, bv.ctypes.data, float(occupancy), int(min_depth))

    def leaves_bv(self, volume=None, occupied=True, free=True, unknown=False, min_depth=0):
        """(codes, depths, occ) of beginLeaves(BoundingVolume, ...)."""
        bv, bp, nb = _bv(volume)
        flt = (int(occupied), int(free), int(unknown))
        n = self.vl.ufo_ref_leaves_bv(self.h, *flt, bp, nb, int(min_depth), None, None, None, 0)
        codes, depths, occ = np.empty(n, np.uint64), np.empty(n, np.uint32), np.empty(n, np.float32)
        if n:
            self.vl.ufo_ref_leaves_bv(self.h, *flt, bp, nb, int(min_depth), codes.ctypes.data, depths.ctypes.data,
                                      occ.ctypes.data, n)
        return codes, depths, occ
