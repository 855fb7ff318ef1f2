"""Plain float64 restatement of the colour rules of OccupancyMapColor (test infrastructure).

* Leaf blend: updateNodeColor (occupancy_map_color.cpp:142-171), applied by updateValue
  (occupancy_map_color.h:269-287) BEFORE the occupancy update of the same hit.
* Inner colour: getAverageChildColor / getAverageColor (occupancy_map_color.cpp:177-222), the
  root-mean-square of the children whose colour is set (any channel != 0), truncated to uint8;
  0 when no child is set.  Every level is computed from the level below it: a root-mean-square of
  root-mean-squares is not the root-mean-square of the leaves.

toProb is evaluated with the C library's own expf (the reference's std::exp(float)), not numpy.
"""
import ctypes
import ctypes.util

import numpy as np

_libm = ctypes.CDLL(ctypes.util.find_library("m") or "libm.so.6")
_libm.expf.restype = ctypes.c_float
_libm.expf.argtypes = [ctypes.c_float]


def expf(x):
    return float(_libm.expf(ctypes.c_float(x)))


def to_prob(logit):
    """toProb(float) (occupancy_map_base.h:911): 1 / (1 + expf(-logit)) in double."""
    return 1.0 / (1.0 + expf(-float(np.float32(logit))))


def to_logit(prob):
    return float(np.log(prob / (1.0 - prob)))


def blend(cur, upd, hit_logit, cur_logit):
    """updateNodeColor(node, upd, toProb(hit)) on a leaf of colour `cur` and log-odds `cur_logit`.
    No isSet check on the update: a black update darkens a set colour."""
    cur = tuple(int(c) for c in cur)
    upd = tuple(int(c) for c in upd)
    if cur == upd:
        return cur
    if not any(cur):
        return upd
    prob = to_prob(hit_logit)
    prob = prob / (prob + to_prob(cur_logit))
    inv = 1.0 - prob
    return tuple(int(np.sqrt(((float(c) * float(c)) * inv) + ((float(u) * float(u)) * prob)))
                 for c, u in zip(cur, upd))


def apply_update(logit, upd, clamp_min_logit, clamp_max_logit):
    """Float add + clamp (occupancy_map_base.h:1139-1145)."""
    v = np.float32(np.float32(logit) + np.float32(upd))
    return np.float32(min(max(v, np.float32(clamp_min_logit)), np.float32(clamp_max_logit)))


def check_tree_colors(cpu_map, what=""):
    """Every node of a checker's tree (inner nodes and leaves above depth 0) holds the restated
    colour of its value field."""
    codes, occ, rgb = cpu_map.value_field()
    levels = inner_colors(codes, rgb, cpu_map.depth_levels)
    for leaves in (False, True):
        nc, nd, _, nrgb, _ = cpu_map.walk(leaves)
        sel = nd > 0
        want, _ = node_colors_at(levels, nc[sel], nd[sel])
        bad = np.nonzero((want != nrgb[sel]).any(axis=1))[0]
        assert len(bad) == 0, "%s: %d %s colours differ from the restatement, first code %x depth %d: %r vs %r" % (
            what, len(bad), "leaf" if leaves else "inner", int(nc[sel][bad[0]]), int(nd[sel][bad[0]]),
            tuple(nrgb[sel][bad[0]]), tuple(want[bad[0]]))


# -- scenes ------------------------------------------------------------------------------
# The + face: depth_levels=6 at 0.5 m, half size 16 m.  isInside is inclusive (octree.h:1297-1304),
# so a point with a coordinate of exactly +16 is inside and toKey gives 2^6 there: an out-of-tree
# key that the tree's code walk wraps onto key 0 of that axis (the voxel at -16..-15.5).
FACE_RES, FACE_LEVELS, FACE_HALF = 0.5, 6, 16.0
_IN = -15.9  # key 0 on its axis: the voxel every +face point on that axis wraps onto


def _face_scan(k, reverse=False):
    """One discrete colour scan that hits wrapped voxels from the + faces: single-face aliases,
    corner points whose several out-of-tree codes all wrap onto one voxel, and in-tree points in the
    same wrapped voxels with a lower and with a higher cloud index."""
    H = FACE_HALF
    pts, cols = [], []

    def add(p, c):
        pts.append(p)
        cols.append(c)

    sh = 1.5 * k
    add((_IN, 3.2, 1.1 + sh), (200, 10 + k, 10))         # in-tree point, lowest index
    add((H, -7.3, 2.2 + sh), (5 + 40 * k, 250, 1))       # its alias on another voxel: in-tree later
    add((H, 3.2, 1.1 + sh), (0, 0, 255 - k))              # alias of the first voxel, higher index
    add((H, H, H), (255, 255, 255))                       # corner: 3 axes out of tree -> (0, 0, 0)
    add((H, _IN, _IN), (255, 0, 0))                       # 1 axis -> (0, 0, 0)
    add((_IN, _IN, _IN), (30 + k, 220, 40))               # the in-tree point of (0, 0, 0), mid index
    add((_IN, H, _IN), (0, 255, 0))
    add((_IN, _IN, H), (0, 0, 255))
    add((H, H, _IN), (17, 17, 200 + k))
    add((_IN, -7.3, 2.2 + sh), (90, 90, 90))              # in-tree point of the second voxel
    add((H, H, H), (1, 2, 3))                             # duplicate out-of-tree code: dropped
    add((5.3, H, -4.4 - sh), (0, 0, 0) if k else (9, 9, 9))  # black update into a set colour
    add((5.3, _IN, -4.4 - sh), (9, 9, 9))
    add((2.1, -3.3, H), (255, 255, 255))
    add((2.1, -3.3, _IN), (255, 255, 255))                # equal update
    add((-6.2, H, H), (0, 77, 0))                         # single channel, edge of two + faces
    if reverse:
        pts, cols = pts[::-1], cols[::-1]
    rng = np.random.default_rng(100 + k)
    # interior points so that the wrapped voxels sit among ordinary ones
    inner = rng.uniform(-15.0, 15.0, (200, 3)).astype(np.float32).astype(np.float64)
    icol = rng.integers(0, 256, (200, 3)).astype(np.uint8)
    origin = np.array([0.013 + 0.3 * k, 0.021 - 0.2 * k, 0.007])
    return dict(origin=origin, xyz=np.concatenate([np.array(pts, np.float64), inner]),
                rgb=np.concatenate([np.array(cols, np.uint8), icol]))


def face_scans(n=4, discrete=True):
    """A stream of + face scans (the first colours the wrapped voxels with in-tree points only)."""
    out = []
    for k in range(n):
        s = _face_scan(k, reverse=(k % 2 == 1))
        if k == 0:
            keep = (s["xyz"] < FACE_HALF).all(axis=1)
            s = dict(origin=s["origin"], xyz=s["xyz"][keep], rgb=s["rgb"][keep])
        s["discrete"] = discrete
        out.append(s)
    return out


def clipped_face_scans(n=3):
    """Non-discrete colour scans whose rays leave the map through the + faces: moveLineInside clips
    their ends onto the face, where they become out-of-tree hits."""
    out = []
    for k in range(n):
        rng = np.random.default_rng(200 + k)
        far = rng.uniform(-30.0, 30.0, (300, 3))
        far[:100, 0] = rng.uniform(17.0, 40.0, 100)
        far[100:150, 1] = rng.uniform(17.0, 40.0, 50)
        far[150:200, 2] = rng.uniform(17.0, 40.0, 50)
        inner = rng.uniform(-15.0, 15.0, (100, 3))
        xyz = np.concatenate([far, inner]).astype(np.float32).astype(np.float64)
        rgb = rng.integers(0, 256, (len(xyz), 3)).astype(np.uint8)
        origin = np.array([0.013 + 0.5 * k, 0.021, 0.007 - 0.25 * k])
        out.append(dict(origin=origin, xyz=xyz, rgb=rgb))
    return out


def inner_colors(codes, rgb, max_level):
    """{level: (parent codes (code >> 3*level), rgb u8[n,3])} for levels 1..max_level of a value
    field (codes sorted, rgb of every listed depth-0 voxel; absent voxels are unset)."""
    out = {}
    codes = np.asarray(codes, np.uint64)
    col = np.asarray(rgb, np.uint8).reshape(-1, 3)
    for lvl in range(1, max_level + 1):
        parents = codes >> np.uint64(3)
        uniq, inv = np.unique(parents, return_inverse=True)
        is_set = col.any(axis=1)
        sq = np.zeros((len(uniq), 3), np.float64)
        cnt = np.zeros(len(uniq), np.float64)
        c64 = col.astype(np.float64)
        np.add.at(sq, inv[is_set], c64[is_set] * c64[is_set])
        np.add.at(cnt, inv[is_set], 1.0)
        res = np.zeros((len(uniq), 3), np.uint8)
        nz = cnt > 0
        # getAverageColor sums the squares child by child in child order; the sums are exact
        # (integers below 2^53), so the order of np.add.at does not matter
        res[nz] = np.sqrt(sq[nz] / cnt[nz, None]).astype(np.uint8)
        out[lvl] = (uniq, res)
        codes, col = uniq, res
    return out


def node_colors_at(levels_map, codes, depths):
    """Restated colour of the nodes (code at depth); depth 0 is not handled here."""
    codes = np.asarray(codes, np.uint64)
    depths = np.asarray(depths)
    out = np.zeros((len(codes), 3), np.uint8)
    found = np.zeros(len(codes), bool)
    for d in np.unique(depths):
        sel = np.nonzero(depths == d)[0]
        uniq, col = levels_map[int(d)]
        key = codes[sel] >> np.uint64(3 * int(d))
        pos = np.searchsorted(uniq, key)
        pos_c = np.minimum(pos, max(len(uniq) - 1, 0))
        hit = (pos < len(uniq)) & (uniq[pos_c] == key) if len(uniq) else np.zeros(len(sel), bool)
        out[sel[hit]] = col[pos_c[hit]]
        found[sel] = hit
    return out, found
