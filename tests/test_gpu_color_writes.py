"""GPU: the colour map's writers (ufo_b200_update_nodes_color: setColor and the colour-weighted
updateValue) against the C restatement and, where the prebuilt harness travelled, the compiled
reference.  Value fields, colours included, are compared bit for bit, inner nodes against the pure
function of the field, and the file image byte for byte."""
import numpy as np
import pytest

import color_lib
import color_writes_lib
from color_writes_lib import ColorWritesOracleMap as OracleMap, ColorWritesRefMap as RefMap, have_ref
from color_writes_lib import VALUES, codes_of, mixed_color_batch
from helpers import assert_value_fields_equal, check_inner_against_field
from ufomap_b200 import scans
from ufomap_b200.capi import Map, UfoError, E_INVALID, E_UNSUPPORTED

pytestmark = pytest.mark.gpu
color_writes_lib.build()

LEVELS = (1, 2, 3, 4, 5, 6, 9, 16)
CMIN, CMAX = np.float32(np.log(0.1192 / 0.8808)), np.float32(np.log(0.971 / 0.029))


def _fill(m, scene):
    if scene == "rgbd_color_discrete":
        for k in range(2):
            o, p, c = scans.rgbd(k=k, width=48, height=36)
            m.insert(o, p, rgb=c, max_range=3.0, discrete=True)
    else:  # 2 cm Velodyne scan coloured by point index
        o, p = scans.velodyne64(k=0, rings=32, azimuths=512)
        i = np.arange(len(p))
        rgb = np.stack([i & 255, (i >> 3) & 255, (5 * i) & 255], axis=-1).astype(np.uint8)
        m.insert(o, p, rgb=rgb, max_range=20.0, discrete=True)
    return m


RES = {"rgbd_color_discrete": 0.04, "velodyne_2cm": 0.02}


def _maps(scene, with_ref=True):
    gpu = _fill(Map(RES[scene], color=True), scene)
    cpus = [_fill(OracleMap(RES[scene], color=True), scene)]
    if with_ref and have_ref():
        cpus.append(_fill(RefMap(RES[scene], color=True), scene))
    return gpu, cpus


def _compare(gpu, cpus, images=True):
    field = gpu.value_field()
    for c in cpus:
        assert_value_fields_equal(field, c.value_field(), color_tol=0, what=type(c).__name__)
    check_inner_against_field(gpu, field, cpus[0].sensor_model(), levels=LEVELS)
    # depth 0 through ufo_b200_query as well
    sel = np.linspace(0, len(field[0]) - 1, min(len(field[0]), 200000)).astype(np.int64)
    occ, _, rgb = gpu.query(field[0][sel], 0)
    assert np.array_equal(occ.view(np.uint32), field[1][sel].view(np.uint32))
    assert np.array_equal(rgb, field[2][sel])
    if images:
        # The device writes the canonical tree of its value field.  After these batches the
        # reference's own tree is not canonical (updateParents stops at the first unchanged node and
        # misses collapses further up), so the image is compared with the restatement's tree
        # collapsed to canonical form; the value fields above are the reference's.
        cpus[0].canonicalize()
        assert gpu.write() == cpus[0].write(), "file image differs from the canonical tree"
    return field


def test_known_answers():
    """setColor on untouched space, one ADD_COLOR onto a set colour, ADD then ADD_COLOR."""
    m = Map(0.02, color=True)
    c = m.to_code([0.5, 0.5, 0.5])
    m.update_nodes_color([c], 0, Map.SET_COLOR, 0.0, [(200, 10, 30)])
    codes, occ, rgb = m.value_field()
    assert codes.tolist() == [c] and occ.view(np.uint32).tolist() == [0] and rgb.tolist() == [[200, 10, 30]]
    hit = np.float32(0.8473)
    m.update_nodes_color([c], 0, Map.ADD_COLOR, hit, [(10, 250, 90)])
    want = color_lib.blend((200, 10, 30), (10, 250, 90), hit, 0.0)
    _, occ, rgb = m.value_field()
    assert occ.view(np.uint32).tolist() == [hit.view(np.uint32)] and tuple(rgb[0]) == want
    # ADD then ADD_COLOR in one batch: the blend reads the log-odds the ADD left
    m.update_nodes_color([c, c], 0, [Map.ADD, Map.ADD_COLOR], [1.5, hit], [(0, 0, 0), (0, 0, 0)])
    v1 = color_lib.apply_update(hit, 1.5, CMIN, CMAX)
    want2 = color_lib.blend(want, (0, 0, 0), hit, v1)
    v2 = color_lib.apply_update(v1, hit, CMIN, CMAX)
    _, occ, rgb = m.value_field()
    assert occ.view(np.uint32).tolist() == [v2.view(np.uint32)] and tuple(rgb[0]) == want2
    assert want2 != want and any(want2)  # (0,0,0) blends towards black, it does not unset
    assert want2 != color_lib.blend(want, (0, 0, 0), hit, hit)  # ADD_COLOR before the ADD differs
    # SET_COLOR (0,0,0) unsets: the voxel keeps its log-odds, the colour is gone
    m.update_nodes_color([c], 0, Map.SET_COLOR, 0.0, [(0, 0, 0)])
    _, occ, rgb = m.value_field()
    assert occ.view(np.uint32).tolist() == [v2.view(np.uint32)] and rgb.tolist() == [[0, 0, 0]]
    m.close()


@pytest.mark.parametrize("scene,n", [("rgbd_color_discrete", 10_000), ("rgbd_color_discrete", 200_000),
                                     ("velodyne_2cm", 1_000_000)])
def test_parity_with_the_reference(scene, n):
    """Seeded batches of ADD (depths 0..6), ADD_COLOR and SET_COLOR: one voxel hit 200 times,
    black colours, untouched space.  Then a depth-0 batch: its change set is the reference's."""
    gpu, cpus = _maps(scene)
    half = 40 if scene.startswith("rgbd") else 150
    batch = mixed_color_batch(n, seed=n % 97, half=half)
    gpu.update_nodes_color(*batch)
    for c in cpus:
        c.update_nodes_color(*batch)
    _compare(gpu, cpus)
    # the change set at depth 0 (an ADD above depth 0 changes every voxel below it on the device,
    # the reference records the node instead)
    codes, depths, ops, vals, rgb = mixed_color_batch(n // 4, seed=n % 89, half=half)
    d0 = depths == 0
    small = (codes[d0], depths[d0], ops[d0], vals[d0], rgb[d0])
    gpu.enable_change_detection(True)
    box = gpu.change_bbox()
    gpu.update_nodes_color(*small)
    changed = cpus[0].update_nodes_color(*small)
    for c in cpus[1:]:
        c.enable_change_detection(True)
        c.reset_change_detection()
        c.update_nodes_color(*small)
        assert np.array_equal(np.unique(c.changed_codes()[0]), changed)
    assert np.array_equal(gpu.changed_codes(0), changed)
    gbox = gpu.change_bbox()
    assert np.array_equal(box[0], gbox[0]) and np.array_equal(box[1], gbox[1])
    assert_value_fields_equal(gpu.value_field(), cpus[-1].value_field(), what=type(cpus[-1]).__name__)


def test_set_and_colour_ops_against_the_restatement():
    """SET (depth 0) mixed in: the reference has no form of it, the restatement does."""
    gpu, cpus = _maps("rgbd_color_discrete", with_ref=False)
    batch = mixed_color_batch(100_000, seed=3, set_ops=True)
    gpu.update_nodes_color(*batch)
    cpus[0].update_nodes_color(*batch)
    _compare(gpu, cpus)


def test_ordering_with_async_scans_and_repeats():
    """Batches interleaved with async scans equal the sequential checker; the same batch submitted
    with and without async gives the same map."""
    gpu = Map(0.04, color=True)
    cpu = OracleMap(0.04, color=True)
    for k in range(3):
        o, p, c = scans.rgbd(k=k, width=48, height=36)
        batch = mixed_color_batch(20_000, seed=40 + k, set_ops=True)
        gpu.insert(o, p, rgb=c, max_range=3.0, discrete=True, async_=True)
        gpu.update_nodes_color(*batch, async_=True)
        cpu.insert(o, p, rgb=c, max_range=3.0, discrete=True)
        cpu.update_nodes_color(*batch)
    gpu.wait()
    _compare(gpu, [cpu], images=False)
    batch = mixed_color_batch(50_000, seed=44)
    fields = []
    for async_ in (False, True):
        m = _fill(Map(0.04, color=True), "rgbd_color_discrete")
        m.update_nodes_color(*batch, async_=async_)
        m.update_nodes_color(*batch, async_=async_)
        m.wait()
        fields.append(m.value_field())
        m.close()
    assert_value_fields_equal(fields[0], fields[1], what="async")


def test_pool_growth_applies_every_colour_op_once():
    """A map created with 16 bricks grows while expanding the batch; blending twice would change the
    colours, so equality with the checker shows every colour op ran exactly once."""
    batch = mixed_color_batch(200_000, seed=5, half=300)
    gpu = Map(0.04, color=True, initial_bricks=16)
    gpu.update_nodes_color(*batch)
    assert gpu.stats()["regrows"] > 0
    cpu = OracleMap(0.04, color=True)
    cpu.update_nodes_color(*batch)
    _compare(gpu, [cpu], images=False)


def test_ops_0_and_1_are_update_nodes():
    """A batch without colour ops gives exactly what ufo_b200_update_nodes gives, on both map kinds."""
    codes, depths, ops, vals, rgb = mixed_color_batch(50_000, seed=6, set_ops=True)
    keep = ops <= 1
    keep &= ~((ops == 1) & (depths > 0))
    codes, depths, ops, vals, rgb = codes[keep], depths[keep], ops[keep], vals[keep], rgb[keep]
    for color in (False, True):
        a, b = [_fill(Map(0.04, color=True), "rgbd_color_discrete") if color else Map(0.04) for _ in range(2)]
        a.update_nodes(codes, depths, ops, vals)
        b.update_nodes_color(codes, depths, ops, vals, None)
        assert_value_fields_equal(a.value_field(), b.value_field(), what="update_nodes")
        assert a.write() == b.write()


def test_rejections_leave_the_map_unchanged():
    gpu = _fill(Map(0.04, color=True), "rgbd_color_discrete")
    mono = Map(0.04)
    before = gpu.value_field()
    c = gpu.to_code([0.3, 0.2, 0.1])
    out = np.uint64(1 << 48)  # key x = 2^16: outside a 16-level tree
    rgb = [(1, 2, 3), (4, 5, 6)]
    cases = [
        (E_INVALID, lambda: gpu.update_nodes_color([c, c], 0, [2, 4], 0.5, rgb)),
        (E_INVALID, lambda: gpu.update_nodes_color([c, c], 0, [0, 3], 0.5, None)),
        (E_INVALID, lambda: gpu.update_nodes_color([c, out], 0, [3, 2], 0.5, rgb)),
        (E_UNSUPPORTED, lambda: gpu.update_nodes_color([c, c], [0, 1], [2, 2], 0.5, rgb)),
        (E_UNSUPPORTED, lambda: gpu.update_nodes_color([c, c], [0, 2], [2, 3], 0.5, rgb)),
        (E_UNSUPPORTED, lambda: gpu.update_nodes_color([c, c], [0, 7], [2, 0], 0.5, rgb)),
        (E_UNSUPPORTED, lambda: gpu.update_nodes_color([c, c], [0, 1], [2, 1], 0.5, rgb)),
    ]
    for status, call in cases:
        with pytest.raises(UfoError) as e:
            call()
        assert e.value.status == status
        assert_value_fields_equal(before, gpu.value_field(), what="after a rejected batch")
    for op in (2, 3):
        with pytest.raises(UfoError) as e:
            mono.update_nodes_color([c], 0, op, 0.5, [(1, 2, 3)])
        assert e.value.status == E_INVALID and mono.value_field_count() == 0
    sh = Map(0.04, color=True)
    sh.set_shard(0, 2)
    with pytest.raises(UfoError) as e:
        sh.update_nodes_color([c], 0, 3, 0.0, [(1, 2, 3)])
    assert e.value.status == E_UNSUPPORTED and sh.value_field_count() == 0


def test_colour_write_cost_does_not_depend_on_the_map_size():
    """A colour batch touching K bricks reports touched_bricks == K on a small and on a large map."""
    rng = np.random.default_rng(12)
    keys = rng.integers(32768 - 300, 32768 + 300, size=(20000, 3))
    codes = codes_of(keys, np.zeros(len(keys)))
    k = len(np.unique(codes >> np.uint64(12)))
    ops = rng.choice(np.uint8([0, 2, 3]), size=len(codes))
    rgb = rng.integers(0, 256, size=(len(codes), 3)).astype(np.uint8)
    for prefill in (0, 4):
        m = Map(0.05, color=True, initial_bricks=1 << 16)
        for j in range(prefill):
            o, p = scans.velodyne64(k=j, rings=32, azimuths=1024)
            shift = np.array([100.0 * (j + 1), 0.0, 0.0])
            m.insert(o + shift, p + shift, rgb=np.full((len(p), 3), 99, np.uint8), max_range=30.0)
        m.update_nodes_color(codes, 0, ops, VALUES[1], rgb)
        st = m.stats()
        assert st["touched_bricks"] == k, (prefill, st["touched_bricks"], k)
        m.close()
