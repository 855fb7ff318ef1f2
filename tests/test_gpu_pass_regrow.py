"""GPU: a readData whose bricks fit the pool but whose upper nodes do not.  The import is repeated
after each growth of the upper-node pool and has to keep the nodes the failed attempt created:
the grown hash already holds them, so handing their slots out again would give two nodes one slot."""
import numpy as np
import pytest

from helpers import assert_value_fields_equal, check_inner_against_field
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu

RES = 0.05
N_BRICKS = 3000  # scattered over a 16-level tree: 23 567 upper nodes (depth 5..16) above them
# The stream lists the seven empty siblings of each brick as depth-4 leaves, and the import creates
# them: 24 000 bricks, which this pool holds, while its upper-node pool (2^15 / 2) does not hold
# the levels above them.
DST_BRICKS = 1 << 15
VALUES = np.float32([0.8473, -0.4055, 1.5, -2.5, 0.3, 3.0])


@pytest.mark.parametrize("color", [False, True])
def test_import_regrows_only_the_upper_pool(color):
    rng = np.random.default_rng(31)
    codes = rng.integers(0, 1 << 48, size=N_BRICKS, dtype=np.uint64)  # depth-0 codes anywhere in the tree
    assert len(np.unique(codes >> np.uint64(12))) == N_BRICKS
    vals = VALUES[rng.integers(0, len(VALUES), N_BRICKS)]
    src = Map(RES, color=color, initial_bricks=1 << 16)
    if color:
        rgb = rng.integers(0, 256, size=(N_BRICKS, 3), dtype=np.uint8)
        ops = np.concatenate([np.full(N_BRICKS, Map.SET, np.uint8), np.full(N_BRICKS, Map.SET_COLOR, np.uint8)])
        src.update_nodes_color(np.tile(codes, 2), 0, ops, np.tile(vals, 2), np.tile(rgb, (2, 1)))
    else:
        src.update_nodes(codes, 0, Map.SET, vals)
    ps = src.pool_stats()
    assert ps["bricks"] == N_BRICKS and ps["upper_nodes"] > DST_BRICKS // 2

    dst = Map(RES, color=color, initial_bricks=DST_BRICKS)
    p0 = dst.pool_stats()
    dst.read_data(src.write_data())
    p1 = dst.pool_stats()
    assert p1["brick_cap"] == p0["brick_cap"] and p1["up_cap"] > p0["up_cap"], "only the upper-node pool grew"
    assert p1["upper_nodes"] == ps["upper_nodes"]
    field = src.value_field()
    assert len(field[0]) == N_BRICKS
    assert_value_fields_equal(dst.value_field(), field)
    check_inner_against_field(dst, field, src.sensor_model(), levels=(1, 2, 3, 4, 5, 6, 9, 12, 16))
    src.close()
    dst.close()
