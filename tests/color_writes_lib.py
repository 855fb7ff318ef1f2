"""ctypes wrappers of the CPU checkers of the colour map's writers (TEST INFRASTRUCTURE ONLY), built by
oracle/color_writes.mk:

* ``ColorWritesRefMap``    -> oracle/_ref/libufo_ref_color_writes.so  (the unmodified reference,
                              ref_color_writes.cpp)
* ``ColorWritesOracleMap`` -> oracle/libufo_oracle_color_writes.so    (the C restatement,
                              ufo_oracle_color_writes.c)

Each library carries the whole shim of its writes_lib counterpart, so these classes offer every
method of WritesRefMap / WritesOracleMap plus ``update_nodes_color``.
"""
import ctypes as C
import os
import subprocess

import numpy as np

from oracle_lib import ORACLE_DIR
from writes_lib import WritesOracleMap, WritesRefMap

REF_COLOR_WRITES_SO = os.path.join(ORACLE_DIR, "_ref", "libufo_ref_color_writes.so")
ORACLE_COLOR_WRITES_SO = os.path.join(ORACLE_DIR, "libufo_oracle_color_writes.so")
_SOURCES = ("ufo_oracle.c", "ufo_oracle_writes.c", "ufo_oracle_color_writes.c", "ref_harness.cpp", "ref_writes.cpp",
            "ref_color_writes.cpp", "color_writes.mk")


def build():
    """Compile the two libraries when they are missing or older than their sources (the reference
    one only where the reference sources exist)."""
    newest = max(os.path.getmtime(os.path.join(ORACLE_DIR, s)) for s in _SOURCES)
    if not os.path.exists(ORACLE_COLOR_WRITES_SO) or os.path.getmtime(ORACLE_COLOR_WRITES_SO) < newest:
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "color_writes.mk", "libufo_oracle_color_writes.so"],
                              stdout=subprocess.DEVNULL)
    if os.path.isdir("/root/reference/ufomap/include") and (
            not os.path.exists(REF_COLOR_WRITES_SO) or os.path.getmtime(REF_COLOR_WRITES_SO) < newest):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-f", "color_writes.mk", "ref"], stdout=subprocess.DEVNULL)


def have_ref():
    return os.path.exists(REF_COLOR_WRITES_SO)


VALUES = np.float32([0.8473, -0.4055, 1.5, -2.5, 0.3, 3.0, -0.05])


def _spread(v):
    v = v.astype(np.uint64) & np.uint64(0x1fffff)
    out = np.zeros_like(v)
    for b in range(21):
        out |= ((v >> np.uint64(b)) & np.uint64(1)) << np.uint64(3 * b)
    return out


def codes_of(keys, depths):
    """Code of the depth-d node holding each key, with the centre bits a depth-d Key carries."""
    keys = np.asarray(keys, np.uint64)
    d = np.asarray(depths, np.uint64)[:, None]
    centre = np.where(d > 0, np.uint64(1) << (np.maximum(d, np.uint64(1)) - np.uint64(1)), np.uint64(0))
    k = ((keys >> d) << d) | centre
    return _spread(k[:, 0]) | (_spread(k[:, 1]) << np.uint64(1)) | (_spread(k[:, 2]) << np.uint64(2))


def mixed_color_batch(n, seed, half=40, set_ops=False, hot=200):
    """n entries around the map centre (keys 2^15 +- half): ADD at depths 0..6, ADD_COLOR and
    SET_COLOR at depth 0, SET at depth 0 when set_ops (the reference has no SET).  Every code comes
    about four times; one voxel takes `hot` entries of every op interleaved; one colour in ten is
    (0,0,0), which unsets (SET_COLOR) or blends towards black (ADD_COLOR)."""
    rng = np.random.default_rng(seed)
    keys = rng.integers(32768 - half, 32768 + half, size=(max(n // 4, 1), 3))
    keys = keys[rng.integers(0, len(keys), n)]
    keys[rng.choice(n, size=min(hot, n), replace=False)] = 32768 + half // 3
    ops = rng.choice(np.uint8([0, 1, 2, 3]), size=n, p=[0.35, 0.1, 0.35, 0.2] if set_ops else [0.4, 0, 0.4, 0.2])
    depths = np.zeros(n, np.uint32)
    add = ops == 0
    depths[add] = rng.choice(7, size=int(add.sum()), p=[0.7, 0.1, 0.08, 0.06, 0.04, 0.015, 0.005])
    codes = codes_of(keys, depths)
    vals = VALUES[rng.integers(0, len(VALUES), n)]
    rgb = rng.integers(0, 256, size=(n, 3)).astype(np.uint8)
    rgb[rng.random(n) < 0.1] = 0
    return codes, depths, ops.astype(np.uint8), vals, rgb


def batch_arrays(codes, depths, ops, values, rgb):
    c = np.ascontiguousarray(codes, dtype=np.uint64).reshape(-1)
    n = len(c)
    d = np.ascontiguousarray(np.broadcast_to(depths, (n,)), dtype=np.uint32)
    o = np.ascontiguousarray(np.broadcast_to(ops, (n,)), dtype=np.uint8)
    v = np.ascontiguousarray(np.broadcast_to(values, (n,)), dtype=np.float32)
    col = np.ascontiguousarray(np.broadcast_to(np.asarray(rgb, np.uint8).reshape(-1, 3), (n, 3)))
    return c, d, o, v, col


class ColorWritesRefMap(WritesRefMap):
    _path = REF_COLOR_WRITES_SO

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        if "update_nodes_color" not in self.api:
            f = getattr(C.CDLL(self._path), "ufo_ref_update_nodes_color")
            f.restype = C.c_int
            f.argtypes = [C.c_void_p] * 6 + [C.c_size_t]
            self.api["update_nodes_color"] = f

    def update_nodes_color(self, codes, depths, ops, values, rgb):
        """One reference call per entry in array order: op 0 updateValue(code, value), op 2
        updateValue(code, value, Color(rgb)), op 3 setColor(code, Color(rgb))."""
        c, d, o, v, col = batch_arrays(codes, depths, ops, values, rgb)
        rc = self.api["update_nodes_color"](self.h, c.ctypes.data, d.ctypes.data, o.ctypes.data, v.ctypes.data,
                                            col.ctypes.data, len(c))
        if rc < 0:
            raise RuntimeError("the batch has no form in the reference (SET, or a colour op on a mono map)")


class ColorWritesOracleMap(WritesOracleMap):
    _path = ORACLE_COLOR_WRITES_SO

    def __init__(self, *args, **kw):
        super().__init__(*args, **kw)
        if "update_nodes_color" not in self.api:
            f = getattr(C.CDLL(self._path), "ufo_oracle_update_nodes_color")
            f.restype = None
            f.argtypes = [C.c_void_p] * 6 + [C.c_size_t, C.c_void_p]
            self.api["update_nodes_color"] = f

    def update_nodes_color(self, codes, depths, ops, values, rgb):
        """The restatement of the same batch; returns the sorted codes whose log-odds a depth-0 op 0
        or op 2 changed (the reference's change detection records exactly those)."""
        c, d, o, v, col = batch_arrays(codes, depths, ops, values, rgb)
        changed = np.zeros(len(c), np.uint8)
        self.api["update_nodes_color"](self.h, c.ctypes.data, d.ctypes.data, o.ctypes.data, v.ctypes.data,
                                       col.ctypes.data, len(c), changed.ctypes.data)
        return np.unique(c[changed != 0])
