"""ctypes wrappers of the CPU checkers of the per-node writes and ray insertion (TEST INFRASTRUCTURE
ONLY), built by oracle/writes.mk:

* ``WritesRefMap``    -> oracle/_ref/libufo_ref_writes.so  (the unmodified reference, ref_writes.cpp)
* ``WritesOracleMap`` -> oracle/libufo_oracle_writes.so    (the C restatement, ufo_oracle_writes.c)

Each library carries the whole shim of its oracle_lib counterpart, so these classes offer every
method of RefMap / OracleMap plus ``update_nodes`` and ``insert_rays``.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_lib import ORACLE_DIR, OracleMap, RefMap, _f64

REF_WRITES_SO = os.path.join(ORACLE_DIR, "_ref", "libufo_ref_writes.so")
ORACLE_WRITES_SO = os.path.join(ORACLE_DIR, "libufo_oracle_writes.so")
_SOURCES = ("ufo_oracle.c", "ufo_oracle_writes.c", "ref_harness.cpp", "ref_writes.cpp", "writes.mk")


def build():
    """Compile the two libraries when they are missing or older than their sources (the reference
    one only where the reference sources exist)."""
    newest = max(os.path.getmtime(os.path.join(ORACLE_DIR, s)) for s in _SOURCES)
    if not os.path.exists(ORACLE_WRITES_SO) or os.path.getmtime(ORACLE_WRITES_SO) < newest:
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "writes.mk", "libufo_oracle_writes.so"],
                              stdout=subprocess.DEVNULL)
    if os.path.isdir("/root/reference/ufomap/include") and (
            not os.path.exists(REF_WRITES_SO) or os.path.getmtime(REF_WRITES_SO) < newest):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "writes.mk", "ref"], stdout=subprocess.DEVNULL)


def have_ref():
    return os.path.exists(REF_WRITES_SO)


class _Writes:
    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        if "update_nodes" not in self.api:
            lib = C.CDLL(self._path)
            vp, sz, dbl, u32, i32 = C.c_void_p, C.c_size_t, C.c_double, C.c_uint, C.c_int
            f = getattr(lib, self._prefix + "update_nodes")
            f.restype = i32 if self._prefix == "ufo_ref_" else None
            f.argtypes = [vp, vp, vp, vp, vp, sz]
            g = getattr(lib, self._prefix + "insert_rays")
            g.restype = None
            g.argtypes = [vp, vp, vp, sz, dbl, u32, i32]
            self.api["update_nodes"] = f
            self.api["insert_rays"] = g

    def update_nodes(self, codes, depths, ops, values):
        """Per-node writes in array order: op 0 updateValue(Code(code, depth), value), op 1
        setNodeValue as intended (the compiled reference has no form of it and raises)."""
        c = np.ascontiguousarray(codes, dtype=np.uint64).reshape(-1)
        n = len(c)
        d = np.ascontiguousarray(np.broadcast_to(depths, (n,)), dtype=np.uint32)
        o = np.ascontiguousarray(np.broadcast_to(ops, (n,)), dtype=np.uint8)
        v = np.ascontiguousarray(np.broadcast_to(values, (n,)), dtype=np.float32)
        rc = self.api["update_nodes"](self.h, c.ctypes.data, d.ctypes.data, o.ctypes.data, v.ctypes.data, n)
        if rc is not None and rc < 0:
            raise RuntimeError("setNodeValue does not compile in the reference")

    def insert_rays(self, origins, ends, max_range=-1.0, depth=0, hit_end=False):
        """insertMissOnRay (hit_end=False) / insertRay (hit_end=True) for every (origin, end)."""
        e = _f64(ends).reshape(-1, 3)
        o = np.ascontiguousarray(np.broadcast_to(_f64(origins).reshape(-1, 3), e.shape))
        self.api["insert_rays"](self.h, o.ctypes.data, e.ctypes.data, len(e), float(max_range), int(depth),
                                int(hit_end))


class WritesRefMap(_Writes, RefMap):
    _path = REF_WRITES_SO


class WritesOracleMap(_Writes, OracleMap):
    _path = ORACLE_WRITES_SO
