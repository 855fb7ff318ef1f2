"""CPU: the C restatement of the per-node writes and ray insertion (oracle/ufo_oracle_writes.c) equals the
compiled, unmodified reference (oracle/_ref/libufo_ref_writes.so), node for node through the file image."""
import numpy as np
import pytest

import writes_lib
from writes_lib import WritesOracleMap as OracleMap, WritesRefMap as RefMap, have_ref
from ufomap_b200 import scans

writes_lib.build()
pytestmark = pytest.mark.skipif(not have_ref(), reason="the compiled reference is not available")

RES = 0.1
HIT, MISS = np.float32(np.log(0.7 / 0.3)), np.float32(np.log(0.4 / 0.6))


def _both(scanned):
    maps = [RefMap(RES), OracleMap(RES)]
    if scanned:
        o, p = scans.velodyne64(k=0, rings=16, azimuths=256)
        for m in maps:
            m.insert(o, p, max_range=10.0)
    return maps


def _codes(ref, keys, depths):
    return np.array([ref.key_to_code(k, int(d)) for k, d in zip(keys, depths)], np.uint64)


def _same(ref, orc):
    a, b = ref.value_field(), orc.value_field()
    assert np.array_equal(a[0], b[0])
    assert np.array_equal(a[1].view(np.uint32), b[1].view(np.uint32))
    assert ref.write() == orc.write()


@pytest.mark.parametrize("scanned", [False, True])
def test_mixed_add_batches(scanned):
    """Repeated codes and values large enough to hit both clamps: order matters."""
    ref, orc = _both(scanned)
    rng = np.random.default_rng(1 + scanned)
    keys = rng.integers(32768 - 12, 32768 + 12, size=(300, 3)).astype(np.uint32)
    keys = keys[rng.integers(0, len(keys), 3000)]
    depths = rng.choice(7, size=len(keys), p=[0.5, 0.15, 0.1, 0.1, 0.1, 0.04, 0.01])
    keys = (keys >> depths[:, None].astype(np.uint32)) << depths[:, None].astype(np.uint32)
    keys |= np.where(depths > 0, 1 << np.maximum(depths - 1, 0), 0)[:, None].astype(np.uint32)
    codes = _codes(ref, keys, depths)
    vals = rng.choice(np.float32([HIT, MISS, 2.5, -3.0, 0.01]), size=len(codes))
    for m in (ref, orc):
        m.update_nodes(codes, depths, 0, vals)
    _same(ref, orc)


@pytest.mark.parametrize("depth", [0, 3])
@pytest.mark.parametrize("hit_end", [False, True])
def test_ray_batches(depth, hit_end):
    ref, orc = _both(True)
    rng = np.random.default_rng(depth + 7 * hit_end)
    o = rng.uniform(-0.5, 0.5, size=(400, 3))
    e = o + rng.normal(size=(400, 3)) * 3.0
    for m in (ref, orc):
        m.insert_rays(o, e, max_range=4.0 if hit_end else -1.0, depth=depth, hit_end=hit_end)
    _same(ref, orc)


def test_set_has_no_reference_form():
    ref = RefMap(RES)
    with pytest.raises(RuntimeError):
        ref.update_nodes([ref.key_to_code([32768, 32768, 32768], 0)], 0, 1, 0.5)


def test_change_set_after_depth0_writes():
    """The reference records a depth-0 voxel when ANY of its updates changed the value: an ADD that
    lands on a clamp it already holds is not a change."""
    ref = RefMap(RES)
    ref.enable_change_detection(True)
    rng = np.random.default_rng(3)
    keys = rng.integers(32768 - 5, 32768 + 5, size=(40, 3)).astype(np.uint32)
    keys = keys[rng.integers(0, len(keys), 400)]
    codes = _codes(ref, keys, np.zeros(len(keys)))
    vals = rng.choice(np.float32([HIT, 5.0, -5.0]), size=len(codes))
    # restated change rule: value before != value after for at least one update
    lo, hi = np.float32(np.log(0.1192 / 0.8808)), np.float32(np.log(0.971 / 0.029))
    state, expect = {}, set()
    for c, v in zip(codes.tolist(), vals):
        old = state.get(c, np.float32(0))
        new = np.float32(min(max(np.float32(old + v), lo), hi))
        if new != old:
            expect.add(c)
        state[c] = new
    ref.update_nodes(codes, 0, 0, vals)
    got, depths = ref.changed_codes()
    assert (depths == 0).all()
    assert sorted(set(got.tolist())) == sorted(expect)
