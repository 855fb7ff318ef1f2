"""ctypes wrapper of the CPU checkers of the nearest-first iteration (TEST INFRASTRUCTURE ONLY), built
by oracle/nearest.mk into oracle/_ref/libufo_ref_nearest.so from the unmodified reference
(ref_nearest.cpp, which includes the bounding-volume checker).  The reference's own beginNN* are never
run: beginNNTree does not compile and beginNNLeaves reads past its queue.

* ``NearestRefMap``  every method of RefMap plus ``nearest``: beginTree / beginLeaves stable-sorted by
                     the reference's squared distance (kind="sorted"), or the reference's best-first
                     search with the popped-node test fixed (kind="bestfirst")
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_lib import ORACLE_DIR, RefMap
from volumes_lib import _bv

REF_NEAREST_SO = os.path.join(ORACLE_DIR, "_ref", "libufo_ref_nearest.so")
_SOURCES = ("ref_harness.cpp", "ref_volumes.cpp", "ref_nearest.cpp", "nearest.mk")


def build():
    """Compile the library when it is missing or older than its sources (where the reference
    sources exist)."""
    newest = max(os.path.getmtime(os.path.join(ORACLE_DIR, s)) for s in _SOURCES)
    if os.path.isdir("/root/reference/ufomap/include") and (
            not os.path.exists(REF_NEAREST_SO) or os.path.getmtime(REF_NEAREST_SO) < newest):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "nearest.mk", "ref"], stdout=subprocess.DEVNULL)


def have_ref():
    return os.path.exists(REF_NEAREST_SO)


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(REF_NEAREST_SO)
        vp, sz, u32, i32 = C.c_void_p, C.c_size_t, C.c_uint, C.c_int
        for f in (lib.ufo_ref_nearest_sorted, lib.ufo_ref_nearest_bestfirst):
            f.restype = sz
            f.argtypes = [vp, vp, i32, i32, i32, i32, i32, u32, vp, sz, vp, vp, vp, vp, vp, vp, vp, sz]
        _lib = lib
    return _lib


class NearestRefMap(RefMap):
    _path = REF_NEAREST_SO

    def nearest(self, point, volume=None, leaves=True, occupied=True, free=True, unknown=False, contains=False,
                min_depth=0, kind="sorted"):
        """(codes, depths u8, logodds f32, flags u8, rgb u8[n,3], centres f64[n,3], d2 f64) in non-decreasing d2.
        flags: bit0 containsFree, bit1 containsUnknown, bit2 isLeaf."""
        lib = _load()
        fn = lib.ufo_ref_nearest_sorted if kind == "sorted" else lib.ufo_ref_nearest_bestfirst
        bv, bp, nb = _bv(volume)
        pt = np.ascontiguousarray(point, np.float64).reshape(3)
        args = (pt.ctypes.data, int(bool(leaves)), int(bool(occupied)), int(bool(free)), int(bool(unknown)),
                int(bool(contains)), int(min_depth), bp, nb)
        n = fn(self.h, *args, None, None, None, None, None, None, None, 0)
        codes, depths = np.empty(n, np.uint64), np.empty(n, np.uint8)
        occ, flags = np.empty(n, np.float32), np.empty(n, np.uint8)
        rgb, centres, d2 = np.zeros((n, 3), np.uint8), np.empty((n, 3), np.float64), np.empty(n, np.float64)
        if n:
            fn(self.h, *args, codes.ctypes.data, depths.ctypes.data, occ.ctypes.data, flags.ctypes.data, rgb.ctypes.data,
               centres.ctypes.data, d2.ctypes.data, n)
        return codes, depths, occ, flags, rgb, centres, d2
