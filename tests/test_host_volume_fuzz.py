"""The node-vs-volume predicate the kernels run (ufo_volume.cuh), called on the host through
ufo_b200_volume_intersects, against the reference's own intersects(AABB, X) compiled from its
unmodified sources: the same boolean for every cube, for each of the eight BoundingVar types, on
random cubes and on the cases where a tie or a NaN decides."""
import math

import numpy as np
import pytest

import volumes_lib
from ufomap_b200 import capi

pytestmark = pytest.mark.skipif(not volumes_lib.have_ref(), reason="reference volume checker not built")

N_CUBES = 10_000


def _cubes(rng, n=N_CUBES, span=4.0):
    """Random node-like cubes: centres on a 1/64 grid (ties with the shapes below are frequent),
    half sizes 2^-k."""
    c = np.round(rng.uniform(-span, span, (n, 3)) * 64.0) / 64.0
    hs = 2.0 ** -rng.integers(1, 7, n).astype(np.float64)
    return c, np.repeat(hs[:, None], 3, 1)


def _check(volume, c, h):
    got = capi.volume_intersects(volume, c, h)
    want = volumes_lib.ref_intersects(volume, c, h)
    bad = np.nonzero(got != want)[0]
    assert not len(bad), (capi.as_volume(volume), c[bad[:5]], h[bad[:5]], got[bad[:5]])
    return got


def _rand_shape(rng, kind):
    p = lambda: np.round(rng.uniform(-3, 3, 3) * 32) / 32  # noqa: E731
    if kind == capi.AABB:
        a, b = p(), p()
        return capi.aabb(np.minimum(a, b), np.maximum(a, b))
    if kind == capi.FRUSTUM:
        pos = p()
        tgt = pos + rng.normal(size=3)
        return capi.frustum(volumes_lib.ref_frustum7(pos, tgt, [0, 0, 1], rng.uniform(0.3, 1.5), rng.uniform(0.3, 2.0),
                                                     rng.uniform(0.05, 0.5), rng.uniform(1.0, 5.0)))
    if kind == capi.LINE_SEGMENT:
        return capi.line_segment(p(), p())
    if kind == capi.OBB:
        q = rng.normal(size=4)
        return capi.obb(p(), rng.uniform(0.05, 1.5, 3), q / np.linalg.norm(q))
    if kind == capi.PLANE:
        n = rng.normal(size=3)
        return capi.plane(n / np.linalg.norm(n), rng.uniform(-2, 2))
    if kind == capi.POINT:
        return capi.point(p())
    if kind == capi.RAY:
        return capi.volume_record(capi.RAY, volumes_lib.ref_ray(p(), rng.normal(size=3)))
    return capi.sphere(p(), rng.uniform(0.01, 1.5))


@pytest.mark.parametrize("kind", range(8))
def test_random_cubes(kind):
    rng = np.random.default_rng(100 + kind)
    hits = 0
    for _ in range(20):
        c, h = _cubes(rng, N_CUBES // 20 * 2)
        hits += _check(_rand_shape(rng, kind), c, h).sum()
    assert hits > 0


def test_unions_and_the_empty_volume():
    rng = np.random.default_rng(7)
    c, h = _cubes(rng)
    for _ in range(20):
        kinds = rng.integers(0, 8, rng.integers(2, 5))
        _check([_rand_shape(rng, int(k)) for k in kinds], c, h)
    assert _check(None, c, h).all()


def test_faces_on_cube_faces_and_tangent_spheres():
    g = np.arange(-8, 9) * 0.25
    c = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + 0.125
    h = np.full_like(c, 0.125)
    for lo, hi in (([0, 0, 0], [1, 1, 1]), ([0.25, -0.5, 0], [0.25, 0.5, 0.75]), ([-1, -1, -1], [-1, -1, -1])):
        _check(capi.aabb(lo, hi), c, h)
    for r in (0.125, 0.25, 0.375, 1.0):
        # tangent to the faces and the edges of the grid's cubes
        _check(capi.sphere([0.0, 0.0, 0.0], r), c, h)
        _check(capi.sphere([0.125, 0.0, 0.0], r), c, h)
    for q in ([0, 0, 0], [0.25, 0.25, 0.25], [0.25, 0.1, 0.0]):
        _check(capi.point(q), c, h)


def test_axis_parallel_and_degenerate_lines():
    g = np.arange(-4, 5) * 0.25
    c = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + 0.125
    h = np.full_like(c, 0.125)
    for o in ([0.0, 0.0, 0.0], [0.25, 0.5, 0.1], [0.125, 0.125, 0.125]):
        for d in ([1, 0, 0], [0, -1, 0], [0, 0, 1], [1, 1, 0], [0, 1, -1], [1, 1, 1]):
            _check(capi.volume_record(capi.RAY, volumes_lib.ref_ray(o, d)), c, h)
            _check(capi.line_segment(o, np.add(o, d)), c, h)
        # a zero-length segment: 0/0 directions, whose NaN decides as in the reference
        _check(capi.line_segment(o, o), c, h)


def test_obb_identity_and_right_angles():
    rng = np.random.default_rng(3)
    c, h = _cubes(rng, 4000, span=2.0)
    s = math.sqrt(0.5)
    quats = [[1, 0, 0, 0], [s, s, 0, 0], [s, 0, s, 0], [s, 0, 0, s], [0, 1, 0, 0], [0.5, 0.5, 0.5, 0.5]]
    quats += [volumes_lib.ref_quaternion_rpy(*rpy) for rpy in
              ((math.pi / 2, 0, 0), (0, math.pi / 2, 0), (0, 0, math.pi / 2), (math.pi, 0, 0), (0.3, -0.2, 1.1))]
    for q in quats:
        for centre, half in (([0, 0, 0], [0.5, 0.5, 0.5]), ([0.25, 0.5, 0.0], [0.25, 1.0, 0.125])):
            _check(capi.obb(centre, half, q), c, h)


def test_planes_through_cube_corners():
    g = np.arange(-4, 5) * 0.25
    c = np.stack(np.meshgrid(g, g, g, indexing="ij"), -1).reshape(-1, 3) + 0.125
    h = np.full_like(c, 0.125)
    for n in ([1, 0, 0], [0, 1, 0], [0, 0, -1], [1, 1, 0], [1, 1, 1], [1, -2, 3]):
        n = np.asarray(n, np.float64)
        n = n / np.sqrt((n[0] * n[0] + n[1] * n[1]) + n[2] * n[2])
        for corner in ([0, 0, 0], [0.25, 0.25, 0.25], [0.5, -0.25, 0.75]):
            d = (n[0] * corner[0] + n[1] * corner[1]) + n[2] * corner[2]
            _check(capi.plane(n, d), c, h)
            _check(capi.volume_record(capi.PLANE, volumes_lib.ref_plane3(corner, np.add(corner, [0.25, 0, 0]),
                                                                         np.add(corner, [0, 0.25, 0.25]))), c, h)


def test_frustums_from_the_seven_argument_constructor():
    rng = np.random.default_rng(11)
    c, h = _cubes(rng, 4000, span=3.0)
    for pos, tgt, up in (([0, 0, 0], [1, 0, 0], [0, 0, 1]), ([0.5, -1, 0.25], [0.5, 2, 0.25], [0, 0, 1]),
                         ([0, 0, 2], [0, 0, 0], [0, 1, 0])):
        for va, ha in ((math.pi / 4, math.pi / 3), (1.0, 1.0)):
            _check(capi.frustum(volumes_lib.ref_frustum7(pos, tgt, up, va, ha, 0.1, 3.0)), c, h)


@pytest.mark.parametrize("resolution,depth_levels", [(0.05, 16), (0.1, 12), (0.2, 10), (0.037, 16)])
def test_node_cubes_accumulated_from_the_root(resolution, depth_levels):
    """The cubes the recursions test: centres accumulated top-down like getChildCenter."""
    rng = np.random.default_rng(int(resolution * 1000) + depth_levels)
    half = [resolution / 2.0, resolution]
    while len(half) <= depth_levels:
        half.append(half[-1] * 2.0)
    n = 400
    cs, hs = [], []
    c = np.zeros((n, 3))
    for d in range(depth_levels, 0, -1):
        if d > 8:
            # stay near the origin, where the shapes are: the child towards it
            idx = (c[:, 0] <= 0) * 1 + (c[:, 1] <= 0) * 2 + (c[:, 2] <= 0) * 4
        else:
            idx = rng.integers(0, 8, n)
        step = np.stack([np.where(idx & 1, half[d - 1], -half[d - 1]), np.where(idx & 2, half[d - 1], -half[d - 1]),
                         np.where(idx & 4, half[d - 1], -half[d - 1])], 1)
        c = c + step
        if d <= 8:
            cs.append(c.copy())
            hs.append(np.full((n, 3), half[d - 1]))
    c, h = np.concatenate(cs), np.concatenate(hs)
    hits = 0
    for kind in range(8):
        for _ in range(4):
            hits += _check(_rand_shape(rng, kind), c, h).sum()
    assert hits > 0


def test_ray_constructor_matches_the_reference():
    rng = np.random.default_rng(5)
    for _ in range(200):
        o, d = rng.normal(size=3), rng.normal(size=3) * 10 ** rng.uniform(-3, 3)
        got = capi.as_volume(capi.ray(o, d))["v"][0, :6]
        assert np.array_equal(got.view(np.uint64), volumes_lib.ref_ray(o, d).view(np.uint64))


def test_unknown_type_is_rejected():
    bad = capi.volume_record(8, [0, 0, 0])
    with pytest.raises(capi.UfoError):
        capi.volume_intersects(bad, [[0, 0, 0]], 0.5)


def test_library_constructors_match_the_reference():
    """The constructors the facade's Frustum, Plane and OBB (roll, pitch, yaw) use, run in the library."""
    rng = np.random.default_rng(21)
    for _ in range(50):
        pos, tgt = rng.normal(size=3), rng.normal(size=3) * 4
        up = rng.normal(size=3)
        va, ha, near, far = rng.uniform(0.2, 2.0), rng.uniform(0.2, 2.5), rng.uniform(0.01, 1), rng.uniform(1, 50)
        got = capi.as_volume(capi.frustum7(pos, tgt, up, va, ha, near, far))["v"][0]
        assert np.array_equal(got.view(np.uint64), volumes_lib.ref_frustum7(pos, tgt, up, va, ha, near, far).view(np.uint64))
        v = rng.normal(size=(3, 3))
        got = capi.as_volume(capi.plane3(*v))["v"][0, :4]
        assert np.array_equal(got.view(np.uint64), volumes_lib.ref_plane3(*v).view(np.uint64))
        rpy = rng.uniform(-3.2, 3.2, 3)
        q = capi.pose_from_rpy(0, 0, 0, *rpy)[3:]
        assert np.array_equal(np.asarray(q, np.float64).view(np.uint64),
                              volumes_lib.ref_quaternion_rpy(*rpy).view(np.uint64))
