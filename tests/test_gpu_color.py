"""Colour maps on the device against the compiled reference (RefMap) and the plain-C oracle, exactly:
leaf colours bit for bit, and every node of the checker's tree (inner nodes and leaves above depth 0)
against Map.query at that node's depth -- colour, occupancy and flags -- plus the float64 restatement
of the inner colours (color_lib) through check_inner_against_field.

Covers every path that writes colour state: the first-hit blend of k_hits, the wrapped voxels of
out-of-tree hits on the + faces, the depth 1-4 aggregates, the upper levels, pool growth, import,
per-node writes, volumes and the routed / sharded passes."""
import numpy as np
import pytest

import color_lib as cl
from helpers import assert_value_fields_equal, check_inner_against_field
from oracle_lib import OracleMap, RefMap, build_oracle, have_ref
from ufomap_b200 import capi, scans
from ufomap_b200.capi import E_UNSUPPORTED, Map, UfoError

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _oracles():
    build_oracle()


def _cpus(ref=True, oracle=True, **kw):
    out = []
    if ref and have_ref():
        out.append(RefMap(color=True, **kw))
    if oracle or not out:
        out.append(OracleMap(color=True, **kw))
    return out


def check_tree(gpu, cpu, max_depth=None, occupancy=True, what=""):
    """Every node of the checker's tree above depth 0 == Map.query at that depth.  occupancy=False
    compares colour only: after a free-space update at depth > 0 the checkers leave the updated
    inner node's own occupancy as it was (updateAllChildren, occupancy_map_base.h:1085-1120) while
    Map.query returns the aggregate of its children; check_inner_against_field covers those."""
    max_depth = cpu.depth_levels if max_depth is None else max_depth
    for leaves in (False, True):
        codes, depths, occ, rgb, flags = cpu.walk(leaves)
        sel = (depths > 0) & (depths <= max_depth)
        codes, depths, occ, rgb, flags = codes[sel], depths[sel], occ[sel], rgb[sel], flags[sel]
        o, f, g = gpu.query(codes, depths)
        kind = "%s %s" % (what, "leaf" if leaves else "inner")
        bad = np.nonzero((g != rgb).any(axis=1))[0]
        assert len(bad) == 0, "%s: %d colours differ, first code %x depth %d: %r vs %r" % (
            kind, len(bad), int(codes[bad[0]]), int(depths[bad[0]]), tuple(g[bad[0]]), tuple(rgb[bad[0]]))
        if occupancy:
            assert np.array_equal(o.view(np.uint32), occ.view(np.uint32)), "%s: occupancy differs" % kind
            assert np.array_equal(f & 3, flags & 3), "%s: flags differ" % kind


def compare(gpu, cpus, levels=(1, 2, 3, 4, 5, 6, 7, 9), occupancy=True):
    field = gpu.value_field()
    for c in cpus:
        assert_value_fields_equal(field, c.value_field(), color_tol=0, what=type(c).__name__)
        check_tree(gpu, c, occupancy=occupancy, what=type(c).__name__)
    check_inner_against_field(gpu, cpus[-1].value_field(), cpus[-1].sensor_model(), levels=levels)
    return field


def _stream(n=4, width=96, height=72, **kw):
    ins = []
    for k in range(n):
        o, p, c = scans.rgbd(k=k, width=width, height=height)
        ins.append(dict(origin=o, xyz=p, rgb=c, max_range=4.0, discrete=True, **kw))
    return ins


def _run(map_kw, inserts, gpu_kw=None, **cmp):
    gpu = Map(color=True, **(gpu_kw or dict(initial_blocks=1 << 12)), **map_kw)
    cpus = _cpus(**map_kw)
    for ins in inserts:
        gpu.insert(**ins)
        for c in cpus:
            # float32 inputs hold float32-representable coordinates: the checkers get the same points
            c.insert(**{k: v for k, v in ins.items() if k != "dtype"})
    compare(gpu, cpus, **cmp)
    return gpu, cpus


# -- a. discrete streams from moving poses, every input form ------------------------------
@pytest.mark.parametrize("dtype", [np.float64, np.float32])
def test_stream_xyzrgb(dtype):
    gpu, _ = _run(dict(resolution=0.03), [dict(ins, dtype=dtype) for ins in _stream()])
    gpu.close()


def test_stream_frame_and_pointcloud2():
    res = 0.03
    gpu_f = Map(res, color=True)
    cpus = _cpus(resolution=res)
    for k in range(4):
        o, p, c = scans.rgbd(k=k, width=96, height=72)
        pose = capi.pose_from_rpy(0.05 * k, -0.02 * k, 0.01, 0.01 * k, 0.02, -0.03 * k)
        world = capi.transform_points(pose, p)
        gpu_f.insert_frame(o, p, pose, rgb=c, max_range=4.0, discrete=True)
        for m in cpus:
            m.insert(o, world, rgb=c, max_range=4.0, discrete=True)
    compare(gpu_f, cpus)
    # PointCloud2 records: x y z f32, packed rgb (b g r at offsets 16..18)
    cpus32 = _cpus(resolution=res)
    gpu_p = Map(res, color=True)
    for k in range(4):
        o, p, c = scans.rgbd(k=k, width=96, height=72)
        pose = capi.pose_from_rpy(0.05 * k, -0.02 * k, 0.01, 0.01 * k, 0.02, -0.03 * k)
        world = capi.transform_points(pose, p).astype(np.float32).astype(np.float64)
        rec = np.zeros((len(p), 32), np.uint8)
        rec[:, 0:12] = world.astype(np.float32).view(np.uint8).reshape(-1, 12)
        rec[:, 16], rec[:, 17], rec[:, 18] = c[:, 2], c[:, 1], c[:, 0]
        gpu_p.insert_pointcloud2(o, rec, 32, off_rgb=16, max_range=4.0, discrete=True)
        for m in cpus32:
            m.insert(o, world, rgb=c, max_range=4.0, discrete=True)
    compare(gpu_p, cpus32)
    gpu_f.close()
    gpu_p.close()


# -- b. insert depths and simple ray casting ------------------------------------------------
@pytest.mark.parametrize("depth", [1, 2, 3, 4, 5, 6])
def test_insert_depths(depth):
    ins = _stream(n=3, width=64, height=48)
    ins[1] = dict(ins[1], depth=depth)
    ins[2] = dict(ins[2], depth=depth, simple=True)
    gpu, _ = _run(dict(resolution=0.02), ins, occupancy=False)
    gpu.close()


# -- c. early stopping on a colour map that opted in ---------------------------------------
def test_early_stopping():
    gpu = Map(0.03, color=True)
    gpu.set_early_stopping(True)
    cpus = _cpus(resolution=0.03)
    for ins in _stream(n=4, width=64, height=48):
        ins = dict(ins, early_stopping=2)
        gpu.insert(**ins)
        for c in cpus:
            c.insert(**ins)
    compare(gpu, cpus)
    gpu.close()


# -- d. pool growth in the middle of a scan -----------------------------------------------
def test_pool_growth_blends_once():
    gpu = Map(0.02, color=True, initial_blocks=16, initial_bricks=4)
    cpus = _cpus(resolution=0.02)
    grew = 0
    for k, ins in enumerate(_stream(n=5, width=96, height=72)):
        # later scans move away so that the pools grow while coloured blocks sit untouched
        shift = np.array([0.0, 0.0, 0.6 * k])
        ins = dict(ins, origin=ins["origin"] + shift, xyz=ins["xyz"] + shift)
        gpu.insert(**ins)
        for c in cpus:
            c.insert(**ins)
        grew += gpu.stats()["regrows"] > 0
    assert grew >= 2
    compare(gpu, cpus)
    gpu.close()


# -- e. async inserts -----------------------------------------------------------------------
def test_async_inserts():
    gpu = Map(0.03, color=True)
    cpus = _cpus(resolution=0.03)
    for ins in _stream(n=4):
        gpu.insert(async_=True, **ins)
        for c in cpus:
            c.insert(**ins)
    gpu.wait()
    compare(gpu, cpus)
    gpu.close()


# -- f. volumes and per-node writes on colour maps -----------------------------------------
def test_volumes_and_writes_keep_leaf_colours():
    import volumes_lib
    import writes_lib
    volumes_lib.build()
    writes_lib.build()
    res = 0.04
    gpu = Map(res, color=True)
    cpus = [volumes_lib.VolumesRefMap(res, color=True)] if volumes_lib.have_ref() else []
    cpus.append(OracleMap(res, color=True))
    wcpus = [writes_lib.WritesOracleMap(res, color=True)]
    for ins in _stream(n=3):
        for m in [gpu] + cpus + wcpus:
            m.insert(**ins)
    before = gpu.value_field()
    box = (np.array([0.5, -0.8, -0.5]), np.array([2.0, 0.4, 0.7]))
    for m in [gpu] + cpus + wcpus:
        m.set_value_volume(box, 0.3)
    shape = capi.sphere([1.5, 0.5, 0.2], 0.6)
    gpu.set_value_volume_bv(shape, 0.8)
    if len(cpus) == 2:
        cpus[0].set_value_volume_bv(shape, 0.8)
        field = compare(gpu, cpus[:1])
        keep = np.isin(before[0], field[0])
        assert np.array_equal(field[2][np.isin(field[0], before[0])], before[2][keep]), "leaf colours changed"
    for call in (lambda: gpu.set_value_volume(box, 0.3, 1), lambda: gpu.set_value_volume_bv(shape, 0.3, 1)):
        with pytest.raises(UfoError) as e:
            call()
        assert e.value.status == E_UNSUPPORTED
    with pytest.raises(UfoError) as e:
        gpu.update_nodes([gpu.to_code([1.0, 0.0, 0.0], 1)], [1], [1], 0.5)
    assert e.value.status == E_UNSUPPORTED
    # per-node writes and rays against the oracle's restatement of the writes
    w = Map(res, color=True)
    for ins in _stream(n=3):
        w.insert(**ins)
    w.set_value_volume(box, 0.3)
    before = w.value_field()
    rng = np.random.default_rng(5)
    pick = before[0][rng.integers(0, len(before[0]), 3000)]
    depths = rng.integers(0, 3, len(pick)).astype(np.uint32)
    codes = (pick >> (np.uint64(3) * depths.astype(np.uint64))) << (np.uint64(3) * depths.astype(np.uint64))
    ops = np.zeros(len(pick), np.uint8)
    ops[(depths == 0) & (rng.random(len(pick)) < 0.3)] = 1
    vals = rng.uniform(-2.0, 2.0, len(pick)).astype(np.float32)
    o = np.array([0.013, 0.021, 0.007])
    ends = scans.rgbd(k=5, width=48, height=36)[1]
    origins = np.ascontiguousarray(np.broadcast_to(o, ends.shape))
    for m in (w, wcpus[0]):
        m.update_nodes(codes, depths, ops, vals)
        m.insert_rays(origins, ends, max_range=3.0, hit_end=True)
    field = compare(w, wcpus, occupancy=False)
    assert np.array_equal(field[2][np.isin(field[0], before[0])], before[2][np.isin(before[0], field[0])])
    gpu.close()
    w.close()


# -- g. readData into a coloured map, then scans on top ------------------------------------
@pytest.mark.parametrize("kind", ["whole", "min_depth2", "box"])
def test_read_data_into_coloured_map(kind):
    res = 0.03
    src = RefMap(res, color=True) if have_ref() else OracleMap(res, color=True)
    for ins in _stream(n=2, width=80, height=60):
        src.insert(**ins)
    kw = dict(min_depth=2) if kind == "min_depth2" else {}
    box = (np.array([0.5, -1.0, -0.6]), np.array([2.5, 0.8, 0.9])) if kind == "box" else None
    data = src.write_data(box=box, **kw)
    gpu = Map(res, color=True)
    cpus = _cpus(resolution=res)
    stream = _stream(n=5, width=80, height=60)
    for ins in stream[2:4]:
        for m in [gpu] + cpus:
            m.insert(**ins)
    for m in [gpu] + cpus:
        m.read_data(data, box=box)
    compare(gpu, cpus)
    for m in [gpu] + cpus:
        m.insert(**stream[4])
    compare(gpu, cpus)
    gpu.close()


# -- h. shards and routed colour passes -----------------------------------------------------
def test_routed_and_sharded_colour():
    res, world = 0.02, 2
    maps = [Map(res, color=True, initial_bricks=1 << 14) for _ in range(world)]
    ptrs = [m.route_setup(r, world) for r, m in enumerate(maps)]
    for m in maps:
        m.route_connect(ptrs)
    shards = [Map(res, color=True, initial_bricks=1 << 14) for _ in range(world)]
    for r, m in enumerate(shards):
        m.set_shard(r, world)
    single = Map(res, color=True, initial_bricks=1 << 14)
    ref = _cpus(resolution=res)[0]
    keep = []
    for ins in _stream(n=4, width=96, height=72):
        single.insert(**ins)
        ref.insert(**ins)
        for m in shards:
            m.insert(**ins)
        buf, layout = capi.pack_points(ins["xyz"], ins["rgb"], np.float64)
        keep.append(buf)
        n = len(buf)
        for r, m in enumerate(maps):
            # rank r marks the contiguous sector [r n / world, (r + 1) n / world)
            a, b = r * n // world, (r + 1) * n // world
            m.route_mark_ex(ins["origin"], buf[a:].ctypes.data, b - a, layout, max_range=4.0, discrete=True,
                            index_base=a, index_stride=1)
        for m in maps:
            m.wait()
        for m in maps:
            m.route_apply(0, world, True)
        for m in maps:
            m.wait()
    want = single.value_field()
    compare(single, [ref])
    for group, what in ((maps, "routed"), (shards, "sharded")):
        parts = [m.value_field() for m in group]
        codes = np.concatenate([p[0] for p in parts])
        order = np.argsort(codes, kind="stable")
        field = (codes[order], np.concatenate([p[1] for p in parts])[order], np.concatenate([p[2] for p in parts])[order])
        assert_value_fields_equal(field, want, what=what)
        # depth 1-4 nodes lie inside one brick, so inside one rank: compare them on the owner
        c, d, _, _, _ = ref.walk(False)
        cl_, dl, _, _, _ = ref.walk(True)
        c, d = np.concatenate([c, cl_]), np.concatenate([d, dl])
        sel = (d >= 1) & (d <= 4)
        c, d = c[sel], d[sel]
        so, sf, sg = single.query(c, d)
        owner = np.zeros(len(c), np.int64) - 1
        for r, m in enumerate(group):
            o, f, g = m.query(c, d)
            mine = np.isin(c >> np.uint64(12), np.unique(parts[r][0] >> np.uint64(12)))
            owner[mine] = r
            assert np.array_equal(g[mine], sg[mine]), "%s rank %d: inner colours differ" % (what, r)
            assert np.array_equal(o[mine].view(np.uint32), so[mine].view(np.uint32)), "%s rank %d" % (what, r)
            assert np.array_equal(f[mine] & 3, sf[mine] & 3), "%s rank %d: flags" % (what, r)
        assert (owner >= 0).mean() > 0.9
    for m in maps + shards + [single]:
        m.close()


# -- i. edge colours --------------------------------------------------------------------------
def test_duplicate_hits_lowest_index_in_later_warp():
    """Many points per voxel, the cloud reversed: the lowest cloud index of each voxel sits in a
    later warp and CTA than the other points of the voxel."""
    res = 0.05
    rng = np.random.default_rng(9)
    centres = (np.floor(rng.uniform(-2.0, 2.0, (300, 3)) / res) + 0.5) * res
    reps = np.repeat(centres, 40, axis=0) + rng.uniform(-0.02, 0.02, (12000, 3))
    cols = rng.integers(0, 256, (len(reps), 3)).astype(np.uint8)
    ins = []
    for k in range(3):
        perm = rng.permutation(len(reps)) if k == 1 else np.arange(len(reps))[::-1]
        ins.append(dict(origin=np.array([0.013, 0.021, 0.007]), xyz=reps[perm], rgb=cols[perm], discrete=True))
    gpu, _ = _run(dict(resolution=res), ins)
    gpu.close()


def test_edge_colour_values():
    """Black updates into set colours, updates equal to the current colour, saturated and
    single-channel colours, voxels held at the clamping bounds."""
    res = 0.05
    rng = np.random.default_rng(4)
    pts = (np.floor(rng.uniform(-1.5, 1.5, (500, 3)) / res) + 0.5) * res
    palette = np.array([[0, 0, 0], [255, 255, 255], [255, 0, 0], [0, 255, 0], [0, 0, 255], [254, 255, 253],
                        [1, 0, 0], [255, 255, 0]], np.uint8)
    ins = []
    for k in range(14):
        c = palette[(np.arange(len(pts)) + k * (k % 3)) % len(palette)]
        if k % 4 == 3:
            c = ins[-1]["rgb"]  # equal updates
        ins.append(dict(origin=np.array([0.013, 0.021, 0.007]), xyz=pts, rgb=c, discrete=True))
    gpu, cpus = _run(dict(resolution=res, prob_hit=0.9), ins)
    occ = gpu.value_field()[1]
    assert (occ == occ.max()).sum() >= 100, "voxels held at the upper clamping bound"
    gpu.close()


def test_single_voxel_known_answer():
    """One voxel hit by a prescribed colour sequence over N scans == the numpy blend with the
    voxel's log-odds before each scan."""
    seq = [(200, 100, 50), (200, 100, 50), (0, 0, 0), (255, 255, 255), (255, 0, 0), (0, 255, 0), (255, 255, 255),
           (255, 255, 255), (12, 0, 0), (0, 0, 7), (255, 255, 255), (128, 128, 128), (3, 250, 3)]
    gpu = Map(0.1, color=True, prob_hit=0.9)
    target = np.array([[1.03, 0.51, 0.22]])
    code = np.array([gpu.to_code(target[0])], np.uint64)
    cur = (0, 0, 0)
    for c in seq:
        logit, _, rgb0 = gpu.query(code, 0)
        assert tuple(rgb0[0]) == cur
        gpu.insert([0.013, 0.021, 0.007], target, rgb=np.array([c], np.uint8), discrete=True)
        cur = cl.blend(cur, c, np.float32(cl.to_logit(0.9)), logit[0])
        assert tuple(gpu.query(code, 0)[2][0]) == cur, c
    gpu.close()


# -- j. the + face: out-of-tree hits wrapped onto in-tree voxels ----------------------------
def test_plus_face_wrapped_voxels():
    kw = dict(resolution=cl.FACE_RES, depth_levels=cl.FACE_LEVELS)
    gpu, cpus = _run(kw, cl.face_scans(), gpu_kw=dict(initial_blocks=16), levels=(1, 2, 3, 4, 5, 6))
    gpu.close()


# -- k. non-discrete colour inserts (the reference cannot build them) -------------------------
def test_non_discrete_clipped_rays():
    kw = dict(resolution=cl.FACE_RES, depth_levels=cl.FACE_LEVELS)
    gpu = Map(color=True, **kw)
    cpu = OracleMap(color=True, **kw)
    for ins in cl.clipped_face_scans() + [dict(s, discrete=False) for s in cl.face_scans()[1:]]:
        gpu.insert(**ins)
        cpu.insert(**ins)
    compare(gpu, [cpu], levels=(1, 2, 3, 4, 5, 6))
    res = 0.03
    gpu2, cpu2 = Map(res, color=True), OracleMap(res, color=True)
    for ins in _stream(n=4, width=80, height=60):
        ins = dict(ins, discrete=False)
        gpu2.insert(**ins)
        cpu2.insert(**ins)
    compare(gpu2, [cpu2])
    gpu.close()
    gpu2.close()
