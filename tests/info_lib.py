"""ctypes wrapper of the CPU checker of the tree counters, the known box and the copy constructor
(TEST INFRASTRUCTURE ONLY), built by oracle/info.mk into oracle/_ref/libufo_ref_info.so from the
unmodified reference (ref_info.cpp, which includes the colour-writes checker).

* ``InfoRefMap``  every method of ColorWritesRefMap plus ``tree_info`` (getNumLeafNodes,
                  getNumInnerNodes, size, memoryUsage, getKnownBBX) and ``copy`` (the copy constructor)
"""
import ctypes as C
import os
import subprocess

import numpy as np

from color_writes_lib import ColorWritesRefMap
from oracle_lib import ORACLE_DIR

REF_INFO_SO = os.path.join(ORACLE_DIR, "_ref", "libufo_ref_info.so")
_SOURCES = ("ref_harness.cpp", "ref_writes.cpp", "ref_color_writes.cpp", "ref_info.cpp", "info.mk")


def build():
    """Compile the library when it is missing or older than its sources (where the reference
    sources exist)."""
    newest = max(os.path.getmtime(os.path.join(ORACLE_DIR, s)) for s in _SOURCES)
    if os.path.isdir("/root/reference/ufomap/include") and (
            not os.path.exists(REF_INFO_SO) or os.path.getmtime(REF_INFO_SO) < newest):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "info.mk", "ref"], stdout=subprocess.DEVNULL)


def have_ref():
    return os.path.exists(REF_INFO_SO)


class InfoRefMap(ColorWritesRefMap):
    _path = REF_INFO_SO

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        if "tree_info" not in self.api:
            lib = C.CDLL(self._path)
            f = lib.ufo_ref_tree_info
            f.restype = None
            f.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
            g = lib.ufo_ref_copy
            g.restype = C.c_void_p
            g.argtypes = [C.c_void_p]
            self.api["tree_info"] = f
            self.api["copy"] = g

    def tree_info(self):
        """dict: num_leaf_nodes, num_inner_nodes, size, memory_usage, and getKnownBBX() as the AABB
        holds it (centre, half_size: f64[3] each)."""
        out = np.zeros(4, np.uint64)
        box = np.zeros(6, np.float64)
        self.api["tree_info"](self.h, out.ctypes.data, box.ctypes.data)
        return dict(num_leaf_nodes=int(out[0]), num_inner_nodes=int(out[1]), size=int(out[2]),
                    memory_usage=int(out[3]), center=box[:3].copy(), half_size=box[3:].copy())

    def copy(self):
        """A new InfoRefMap holding OccupancyMap[Color](*this)."""
        h = self.api["copy"](self.h)
        if not h:
            raise RuntimeError("the reference's copy constructor threw")
        other = InfoRefMap.__new__(InfoRefMap)
        other.api, other.h = self.api, h
        other.color, other.resolution, other.depth_levels = self.color, self.resolution, self.depth_levels
        return other
