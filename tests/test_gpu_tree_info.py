"""The reference's node counters and known box on the device (ufo_b200_tree_info) against the
reference compiled from its unmodified sources (tests/info_lib.py): getNumLeafNodes,
getNumInnerNodes, size and memoryUsage equal, and getKnownBBX bit for bit, after the same history --
scans (mono and colour, insert depth 0 / 3 / 6, discrete and plain), setValueVolume, write batches,
readData of a collapsed stream, read of a file image, the empty map and a cleared map.  The
reference's tree after colour batches is not canonical, so there, and for a retained map (which has
no reference counterpart), the comparison is with a map that read this map's image."""
import numpy as np
import pytest

import info_lib
from ufomap_b200 import scans
from ufomap_b200.capi import E_UNSUPPORTED, Map, UfoError

pytestmark = [pytest.mark.gpu, pytest.mark.skipif(not info_lib.have_ref(), reason="reference info checker not built")]

NODE_BYTES = {False: (16, 4), True: (24, 8)}  # sizeof inner / leaf node of the reference, LP64


def expect_same(gpu, ref, what):
    """gpu: a Map; ref: an InfoRefMap holding the same tree."""
    t, r = gpu.tree_info(), ref.tree_info()
    inner, leaf = NODE_BYTES[gpu.color]
    assert (t["num_leaf_nodes"], t["num_inner_nodes"], t["size"]) == (r["num_leaf_nodes"], r["num_inner_nodes"], r["size"]), what
    assert t["num_inner_nodes"] * inner + t["num_leaf_nodes"] * leaf == r["memory_usage"], what
    if t["known"]:
        # AABB(min, max) as the reference's and the facade's constructor build it
        half = (t["known_max"] - t["known_min"]) / 2.0
        centre = t["known_min"] + half
    else:
        half, centre = np.zeros(3), np.zeros(3)
    assert np.array_equal(centre.view(np.uint64), r["center"].view(np.uint64)), (what, centre, r["center"])
    assert np.array_equal(half.view(np.uint64), r["half_size"].view(np.uint64)), (what, half, r["half_size"])
    return t


def collapsible(ref):
    """Nodes of the reference's tree whose eight children are leaves with one payload: its update
    order can leave them behind (updateParents stops at the first unchanged aggregate), and the file
    writer and the iterators of this library never have them."""
    codes, depths, occ, rgb, _ = ref.walk(False)
    lc, ld, lo, lr, _ = ref.walk(True)
    inner = set(zip(codes.tolist(), depths.tolist()))
    kids = {}
    for c, d, o, r in zip(np.concatenate([codes, lc]).tolist(), np.concatenate([depths, ld]).tolist(),
                          np.concatenate([occ, lo]).view(np.uint32).tolist(), [tuple(x) for x in np.concatenate([rgb, lr])]):
        key = (c & ~((1 << (3 * (d + 1))) - 1), d + 1)
        kids.setdefault(key, []).append(((c, d) in inner, o, r))
    return sum(1 for k in inner if not any(x[0] for x in kids[k]) and len({x[1:] for x in kids[k]}) == 1)


def expect_replay(gpu, ref, what):
    """The reference that replayed the same history, where its tree is the pruned tree; where its
    update order left collapsible nodes behind, the reference that read this map's image."""
    t, r = gpu.tree_info(), ref.tree_info()
    if (t["num_leaf_nodes"], t["num_inner_nodes"]) == (r["num_leaf_nodes"], r["num_inner_nodes"]):
        return expect_same(gpu, ref, what)
    assert collapsible(ref) > 0, (what, "the counters differ from a canonical reference tree")
    return expect_same(gpu, image_twin(gpu), (what, "image"))


def image_twin(gpu, **kw):
    ref = info_lib.InfoRefMap(gpu.resolution, gpu.depth_levels, color=gpu.color, **kw)
    assert ref.read(gpu.write())
    return ref


def _scans(color, k_max=2):
    out = []
    for k in range(k_max):
        if color:
            o, p, c = scans.rgbd(k=k, width=48, height=36)
            out.append(dict(origin=o, xyz=p, rgb=c, max_range=3.0))
        else:
            o, p = scans.velodyne64(k=k, rings=8, azimuths=128)
            out.append(dict(origin=o, xyz=p, max_range=12.0))
    return out


def _pair(color, resolution=None, **model):
    res = resolution or (0.04 if color else 0.1)
    return (Map(res, 16, color=color, device=0, initial_bricks=1 << 10, **model),
            info_lib.InfoRefMap(res, 16, color=color, **model))


@pytest.mark.parametrize("color", [False, True])
@pytest.mark.parametrize("depth", [0, 3, 6])
@pytest.mark.parametrize("discrete", [False, True])
def test_scans(color, depth, discrete):
    gpu, ref = _pair(color)
    for s in _scans(color):
        if not discrete:
            s.pop("rgb", None)  # the reference's colour map integrates coloured clouds only discretely
        gpu.insert(depth=depth, discrete=discrete, **s)
        ref.insert(depth=depth, discrete=discrete, **s)
    t = expect_replay(gpu, ref, (color, depth, discrete))
    assert t["known"] and t["num_leaf_nodes"] > 0
    expect_same(gpu, image_twin(gpu), "image")


def test_thresholds_and_empty_space_known():
    # occupied_thres below 0.5: never-touched space (log-odds 0) is occupied, so the whole map is known
    gpu, ref = _pair(False, occupied_thres=0.45, free_thres=0.3)
    t = expect_same(gpu, ref, "empty")
    assert t["known"]
    for s in _scans(False, 1):
        gpu.insert(**s)
        ref.insert(**s)
    expect_same(gpu, ref, "scanned")


def test_set_value_volume_and_write_batches():
    gpu, ref = _pair(False)
    for s in _scans(False):
        gpu.insert(**s)
        ref.insert(**s)
    box = (np.array([-1.0, -2.0, -0.5]), np.array([2.0, 1.5, 0.7]))
    gpu.set_value_volume(box, 0.2, 0)
    ref.set_value_volume(box, 0.2, 0)
    expect_same(gpu, ref, "setValueVolume")
    # a volume that collapses whole bricks into coarse free leaves
    box = (np.array([-6.4, -6.4, -3.2]), np.array([0.0, 0.0, 3.2]))
    gpu.set_value_volume(box, 0.1, 0)
    ref.set_value_volume(box, 0.1, 0)
    expect_same(gpu, ref, "coarse setValueVolume")
    rng = np.random.default_rng(5)
    pts = rng.uniform(-4, 4, size=(300, 3))
    depths = rng.integers(0, 4, size=300).astype(np.uint32)
    codes = np.array([gpu.to_code(p, int(d)) for p, d in zip(pts, depths)], np.uint64)
    vals = rng.choice([0.85, -0.4, 1.3, -2.0], size=300).astype(np.float32)
    gpu.update_nodes(codes, depths, 0, vals)
    ref.update_nodes(codes, depths, 0, vals)
    expect_replay(gpu, ref, "write batch")


def test_color_batches_against_the_image():
    from color_writes_lib import mixed_color_batch
    gpu, _ = _pair(True)
    for s in _scans(True):
        gpu.insert(**s)
    codes, depths, ops, vals, rgb = mixed_color_batch(2000, seed=3)
    gpu.update_nodes_color(codes, depths, ops, vals, rgb)
    expect_same(gpu, image_twin(gpu), "colour batches")


@pytest.mark.parametrize("color", [False, True])
def test_read_data_of_a_collapsed_stream_and_read(color):
    src, _ = _pair(color)
    for s in _scans(color):
        src.insert(**s)
    data = src.write_data(min_depth=3)
    gpu, ref = _pair(color)
    gpu.read_data(data)
    assert ref.read_data(data)
    expect_same(gpu, ref, "readData min_depth 3")
    image = src.write()
    gpu, ref = _pair(color)
    gpu.read(image)
    assert ref.read(image)
    expect_same(gpu, ref, "read")


def test_empty_and_cleared():
    for color in (False, True):
        gpu, ref = _pair(color)
        t = expect_same(gpu, ref, "empty")
        assert (t["num_leaf_nodes"], t["num_inner_nodes"], t["known"]) == (0, 1, False)
        for s in _scans(color, 1):
            gpu.insert(**s)
        gpu.clear()
        t = expect_same(gpu, ref, "cleared")
        assert (t["num_leaf_nodes"], t["num_inner_nodes"], t["known"]) == (0, 1, False)


def test_retained_map_against_its_image():
    gpu, _ = _pair(False)
    for s in _scans(False, 3):
        gpu.insert(**s)
    mn, mx = gpu.change_bbox()
    gpu.retain(box=(mn, (mn + mx) / 2))
    twin = Map(gpu.resolution, 16, device=0)
    twin.read(gpu.write())
    t = expect_same(gpu, image_twin(gpu), "retained")
    tt = twin.tree_info()
    for k in ("num_leaf_nodes", "num_inner_nodes", "with_children"):
        assert t[k] == tt[k], k
    assert np.array_equal(t["known_min"], tt["known_min"]) and np.array_equal(t["known_max"], tt["known_max"])


def test_shallow_maps_are_refused():
    m = Map(0.1, 4, device=0)
    with pytest.raises(UfoError) as e:
        m.tree_info()
    assert e.value.status == E_UNSUPPORTED
