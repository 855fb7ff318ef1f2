"""ctypes wrapper of the CPU checker of the iteration (TEST INFRASTRUCTURE ONLY), built by
oracle/iterate.mk into oracle/_ref/libufo_ref_iterate.so from the unmodified reference
(ref_iterate.cpp, which includes the bounding-volume checker).

* ``IterateRefMap``  every method of RefMap plus ``iterate``: the reference's own beginTree /
                     beginLeaves over a bounding volume, node by node
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_lib import ORACLE_DIR, RefMap
from volumes_lib import _bv

REF_ITERATE_SO = os.path.join(ORACLE_DIR, "_ref", "libufo_ref_iterate.so")
_SOURCES = ("ref_harness.cpp", "ref_volumes.cpp", "ref_iterate.cpp", "iterate.mk")


def build():
    """Compile the library when it is missing or older than its sources (where the reference
    sources exist)."""
    newest = max(os.path.getmtime(os.path.join(ORACLE_DIR, s)) for s in _SOURCES)
    if os.path.isdir("/root/reference/ufomap/include") and (
            not os.path.exists(REF_ITERATE_SO) or os.path.getmtime(REF_ITERATE_SO) < newest):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "iterate.mk", "ref"], stdout=subprocess.DEVNULL)


def have_ref():
    return os.path.exists(REF_ITERATE_SO)


_lib = None


def _load():
    global _lib
    if _lib is None:
        lib = C.CDLL(REF_ITERATE_SO)
        vp, sz, u32, i32 = C.c_void_p, C.c_size_t, C.c_uint, C.c_int
        lib.ufo_ref_iterate.restype = sz
        lib.ufo_ref_iterate.argtypes = [vp, i32, i32, i32, i32, i32, u32, vp, sz, vp, vp, vp, vp, vp, vp, vp, sz]
        _lib = lib
    return _lib


class IterateRefMap(RefMap):
    _path = REF_ITERATE_SO

    def iterate(self, volume=None, leaves=True, occupied=True, free=True, unknown=False, contains=False, min_depth=0):
        """(codes, depths u8, logodds f32, flags u8, rgb u8[n,3], centres f64[n,3], getOccupancy f64) of the reference's
        beginLeaves (leaves=True) / beginTree.  flags: bit0 containsFree, bit1 containsUnknown,
        bit2 isLeaf, bit3 isOccupied, bit4 isFree, bit5 isUnknown, bit6 containsOccupied."""
        lib = _load()
        bv, bp, nb = _bv(volume)
        args = (int(bool(leaves)), int(bool(occupied)), int(bool(free)), int(bool(unknown)), int(bool(contains)),
                int(min_depth), bp, nb)
        n = lib.ufo_ref_iterate(self.h, *args, None, None, None, None, None, None, None, 0)
        codes, depths = np.empty(n, np.uint64), np.empty(n, np.uint8)
        occ, flags = np.empty(n, np.float32), np.empty(n, np.uint8)
        rgb, centres, probs = np.zeros((n, 3), np.uint8), np.empty((n, 3), np.float64), np.empty(n, np.float64)
        if n:
            lib.ufo_ref_iterate(self.h, *args, codes.ctypes.data, depths.ctypes.data, occ.ctypes.data,
                                flags.ctypes.data, rgb.ctypes.data, centres.ctypes.data, probs.ctypes.data, n)
        return codes, depths, occ, flags, rgb, centres, probs
