"""GPU: consecutive asynchronous scans share one leaf update (a paired pass).  Every case inserts a
seeded scan stream with async_=True and compares the whole map -- value field, file image (inner
nodes included) and each scan's counters -- with the same stream run with wait() after every insert,
which updates the leaves scan by scan, and the value field with the CPU oracle."""
import numpy as np
import pytest

from helpers import assert_value_fields_equal
import oracle_lib
from ufomap_b200 import scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu
oracle_lib.build_oracle()

RES = 0.1
COUNTERS = ("points", "rays", "touched_voxels", "hit_voxels", "touched_octets", "touched_blocks",
            "touched_d3", "touched_bricks", "upper_nodes", "blocks_in_map", "bricks_in_map")


def _stream(n, seed=0, step=0.27):
    rng = np.random.default_rng(seed)
    out = []
    for k in range(n):
        o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
        p = p + rng.normal(0.0, 0.02, p.shape)
        out.append((o + [step * k, 0.0, 0.0], p))
    return out


def _counters(st):
    return tuple(int(st[k]) for k in COUNTERS)


def _run(stream, paired, between=None, **kw):
    m = Map(RES, **kw)
    per_scan = []
    for i, (o, p) in enumerate(stream):
        m.insert(o, p, max_range=30.0, async_=paired)
        if not paired:
            per_scan.append(_counters(m.stats()))
        if between is not None:
            between(m, i)
    m.wait()
    return m, per_scan


def _same_map(a, b):
    assert_value_fields_equal(a.value_field(), b.value_field())
    assert a.write() == b.write(), "file images (inner nodes) differ"


@pytest.mark.parametrize("n", [4, 5])
def test_paired_stream_matches_scan_by_scan(n):
    stream = _stream(n)
    single, counts = _run(stream, False)
    m = Map(RES)
    seen = []
    for o, p in stream:
        m.insert(o, p, max_range=30.0, async_=True)
        seen.append(m.completed_stats())
    m.wait()
    last = m.stats()
    _same_map(m, single)
    # every scan's own counters, whether it was the first or the second of a pass
    assert _counters(last) == counts[-1]
    got = [_counters(c) for c in seen if c["points"]]
    for c in got:
        assert c in counts
    assert len(set(got)) >= n - 2
    # the scans did pair: a pass's lines count for its last scan, so a first scan reports none, and the
    # last scan of an even stream reports the lines of both
    assert any(c["points"] and c["touched_lines"] == 0 for c in seen)
    single.close()
    ref = Map(RES)
    for o, p in stream:
        ref.insert(o, p, max_range=30.0)
    if n % 2 == 0:
        assert last["touched_lines"] > ref.stats()["touched_lines"]
    else:
        assert last["touched_lines"] == ref.stats()["touched_lines"]
    cpu = oracle_lib.OracleMap(RES)
    for o, p in stream:
        cpu.insert(o, p, max_range=30.0)
    assert_value_fields_equal(m.value_field(), cpu.value_field())


def test_hit_then_miss_and_miss_then_hit():
    """A voxel hit by one scan of a pair and crossed by the other, both ways round, and hit by both."""
    o = np.zeros(3)
    wall = np.array([[3.05, y, 0.05] for y in np.arange(-1.0, 1.0, 0.1)])
    far = wall * 2.0
    stream = [(o, wall), (o, far), (o, far), (o, wall), (o, wall), (o, wall)]
    single, counts = _run(stream, False)
    paired, _ = _run(stream, True)
    _same_map(paired, single)
    assert _counters(paired.stats()) == counts[-1]


def test_lines_saturate_inside_a_pair():
    o, p = scans.velodyne64(k=0, rings=16, azimuths=512)
    stream = [(o, p)] * 14  # the free space of the first scans reaches clamping_thres_min in a pair
    single, counts = _run(stream, False)
    paired, _ = _run(stream, True)
    _same_map(paired, single)
    assert _counters(paired.stats()) == counts[-1]


FLUSHES = {
    "query": lambda m: m.query(np.zeros(1, np.uint64), np.zeros(1, np.uint32)),
    "export": lambda m: m.value_field(),
    "write": lambda m: m.write(),
    "write_batch": lambda m: m.update_nodes(np.zeros(1, np.uint64), np.zeros(1, np.uint32),
                                            np.zeros(1, np.uint8), np.zeros(1, np.float32)),
    "set_value_volume": lambda m: m.set_value_volume(([50.0] * 3, [50.5] * 3), 0.9),
    "done": lambda m: [m.done() for _ in range(3)],
    "clone": lambda m: m.clone().close(),
    "iterate": lambda m: m.iterate(),
    "nearest": lambda m: m.nearest([0.0, 0.0, 0.0]),
    "retain": lambda m: m.retain(box=([-100.0] * 3, [100.0] * 3)),
    "sync_insert": lambda m: m.insert(np.zeros(3), np.array([[1.0, 1.0, 0.0]]), max_range=30.0),
    "ineligible_insert": lambda m: m.insert(np.zeros(3), np.array([[1.0, 1.0, 0.0]]), max_range=30.0,
                                            discrete=True, async_=True),
}


@pytest.mark.parametrize("call", sorted(FLUSHES))
def test_deferred_scan_flushed_by_any_call(call):
    stream = _stream(3, seed=1)

    def between(m, i):
        if i == 0:  # the first scan is deferred here
            FLUSHES[call](m)

    single, _ = _run(stream, False, between)
    paired, _ = _run(stream, True, between)
    _same_map(paired, single)


def test_pool_growth_while_the_second_scan_marks():
    """The first scan (about 3.2 k bricks) fits the pool of 4096 bricks, the second one, 100 m away,
    does not: the pair's marking overflows in its second scan, the brick pool grows 4x and the upper
    pool with it, after the first scan's K4 created upper nodes."""
    o, p = scans.velodyne64(k=0, rings=16, azimuths=512)
    far = np.array([100.0, 0.0, 0.0])
    stream = [(o, p), (o + far, p + far), (o + far + [0.27, 0, 0], p + far), (o + [0.27, 0, 0], p)]
    regrows = {}

    def between(m, i):
        if i == 1:
            regrows[m] = m.stats()["regrows"]  # completes the pair (stats() waits)

    single, counts = _run(stream, False, between, initial_bricks=4096)
    assert single.pool_stats()["brick_cap"] > 4096
    paired, _ = _run(stream, True, between, initial_bricks=4096)
    assert regrows[single] >= 1 and regrows[paired] >= 1, "the second scan did not overflow the pool"
    st = paired.pool_stats()
    assert st["brick_cap"] > 4096 and st["up_cap"] > 4096, "the pools did not grow"
    _same_map(paired, single)
    assert _counters(paired.stats()) == counts[-1]
    first = Map(RES, initial_bricks=4096)
    first.insert(o, p, max_range=30.0)
    assert first.stats()["regrows"] == 0, "the first scan alone already overflowed the pool"
