"""Shared comparison helpers for the parity tests."""
import numpy as np

from color_lib import inner_colors
from oracle_lib import aggregate_level


def assert_value_fields_equal(a, b, color_tol=0, what=""):
    ca, va, ga = a
    cb, vb, gb = b
    assert len(ca) == len(cb), "%s: %d vs %d voxels" % (what, len(ca), len(cb))
    assert np.array_equal(ca, cb), "%s: voxel code sets differ" % what
    # float log-odds: bit-exact (the north star allows +-1 ULP; we hold 0)
    bad = np.nonzero(va.view(np.uint32) != vb.view(np.uint32))[0]
    assert len(bad) == 0, "%s: %d log-odds differ, first code %x: %r vs %r" % (
        what, len(bad), int(ca[bad[0]]), va[bad[0]], vb[bad[0]])
    if color_tol == 0:
        bad = np.nonzero((ga != gb).any(axis=1))[0]
        assert len(bad) == 0, "%s: %d colours differ, first code %x: %r vs %r" % (
            what, len(bad), int(ca[bad[0]]), tuple(int(x) for x in ga[bad[0]]), tuple(int(x) for x in gb[bad[0]]))
    else:
        d = np.abs(ga.astype(np.int32) - gb.astype(np.int32))
        assert d.max(initial=0) <= color_tol, "%s: colour error %d" % (what, d.max())


def check_inner_against_field(gpu_map, field, model, levels=(1, 2, 3, 4, 5, 6, 9), max_nodes=200000):
    """Inner aggregates of the CUDA map == pure function of the value field (max, flags and, on
    colour maps, the restated inner colour)."""
    codes, occ, rgb = field
    levels = [lvl for lvl in levels if lvl <= gpu_map.depth_levels]
    colors = inner_colors(codes, rgb, max(levels)) if gpu_map.color and levels else None
    for lvl in levels:
        parents, mx, free, unk = aggregate_level(codes, occ, rgb, lvl, model)
        col = None
        if colors is not None:
            assert np.array_equal(colors[lvl][0], parents)
            col = colors[lvl][1]
        if len(parents) > max_nodes:
            sel = np.linspace(0, len(parents) - 1, max_nodes).astype(np.int64)
            parents, mx, free, unk = parents[sel], mx[sel], free[sel], unk[sel]
            col = None if col is None else col[sel]
        q = parents << np.uint64(3 * lvl)
        o, f, g = gpu_map.query(q, lvl)
        assert np.array_equal(o.view(np.uint32), mx.view(np.uint32)), "level %d max mismatch" % lvl
        assert np.array_equal((f & 1).astype(bool), free), "level %d contains_free mismatch" % lvl
        assert np.array_equal(((f >> 1) & 1).astype(bool), unk), "level %d contains_unknown mismatch" % lvl
        if col is not None:
            bad = np.nonzero((g != col).any(axis=1))[0]
            assert len(bad) == 0, "level %d: %d inner colours differ, first node %x: %r vs %r" % (
                lvl, len(bad), int(q[bad[0]]), tuple(g[bad[0]]), tuple(col[bad[0]]))


def sorted_field_large(gpu_map):
    """value_field() of a map with ~10^8 voxels: the sort runs on the GPU through torch."""
    import torch
    codes, occ, rgb = gpu_map.value_field(sort=False)
    order = torch.argsort(torch.from_numpy(codes.view(np.int64)).cuda()).cpu().numpy()
    torch.cuda.empty_cache()
    return codes[order], occ[order], rgb[order]


def check_inner_sampled(gpu_map, field, model, levels=(1, 2, 3, 4, 5, 6, 9, 16), n=20000, seed=5):
    """check_inner_against_field on a random sample of the parents of each level, evaluated on
    ranges of the sorted field (the full aggregate_level needs minutes on 10^8 voxels)."""
    codes, occ, _ = field
    occ_thr, free_thr = model[0], model[1]
    rng = np.random.default_rng(seed)
    o64 = occ.astype(np.float64)
    is_free = o64 < free_thr
    is_unk = (o64 >= free_thr) & (o64 <= occ_thr)
    default_unknown = (0.0 >= free_thr) and (0.0 <= occ_thr)
    default_free = 0.0 < free_thr
    for lvl in levels:
        if lvl > gpu_map.depth_levels:
            continue
        sh = np.uint64(3 * lvl)
        pick = codes[rng.integers(0, len(codes), n)] >> sh
        parents = np.unique(pick)
        lo = np.searchsorted(codes, parents << sh, side="left")
        hi = np.searchsorted(codes, (parents + np.uint64(1)) << sh, side="left")
        assert (hi > lo).all()
        full = (hi - lo) == (1 << (3 * lvl)) if lvl < 21 else np.zeros(len(lo), bool)
        # reduceat over [lo, hi): interleave the boundaries, keep the even segments
        idx = np.stack([lo, hi], axis=1).reshape(-1)
        last = idx[-1] == len(codes)
        if last:
            idx = idx[:-1]

        def seg(ufunc, arr):
            r = ufunc.reduceat(arr, idx)
            return r[::2]
        mx = seg(np.maximum, occ)
        mx = np.where(full, mx, np.maximum(mx, np.float32(0)))
        free = seg(np.logical_or, is_free) | ((~full) & default_free)
        unk = seg(np.logical_or, is_unk) | ((~full) & default_unknown)
        o, f, _ = gpu_map.query(parents << sh, lvl)
        assert np.array_equal(o.view(np.uint32), mx.astype(np.float32).view(np.uint32)), "level %d max mismatch" % lvl
        assert np.array_equal((f & 1).astype(bool), free), "level %d contains_free mismatch" % lvl
        assert np.array_equal(((f >> 1) & 1).astype(bool), unk), "level %d contains_unknown mismatch" % lvl
