"""The float64 restatement of the colour rules (color_lib) against the compiled reference and the
plain-C oracle: inner-node colours of their trees, and the leaf blend step by step."""
import numpy as np
import pytest

import color_lib as cl
from oracle_lib import OracleMap, RefMap, build_oracle, have_ref
from ufomap_b200 import scans


@pytest.fixture(scope="module", autouse=True)
def _oracles():
    build_oracle()


def _checkers():
    return [OracleMap] + ([RefMap] if have_ref() else [])


def _stream(depth, n=4, width=64, height=48):
    ins = []
    for k in range(n):
        o, p, c = scans.rgbd(k=k, width=width, height=height)
        ins.append(dict(origin=o, xyz=p, rgb=c, max_range=4.0, discrete=True, depth=depth))
    return ins


@pytest.mark.parametrize("depth", [0, 1, 2, 3, 4, 5, 6])
def test_inner_colors_match_checker_trees(depth):
    """Discrete colour streams at every insert depth: the restated inner colours equal the colour
    of every inner node and of every leaf above depth 0 of both checkers' trees."""
    for cls in _checkers():
        m = cls(0.04, color=True)
        for ins in _stream(depth):
            m.insert(**ins)
        cl.check_tree_colors(m, what="%s depth %d" % (cls.__name__, depth))
        m.close()


def test_inner_colors_match_checker_trees_plus_face():
    fields = []
    for cls in _checkers():
        m = cls(cl.FACE_RES, depth_levels=cl.FACE_LEVELS, color=True)
        for ins in cl.face_scans():
            m.insert(**ins)
        cl.check_tree_colors(m, what="%s +face" % cls.__name__)
        fields.append(m.value_field())
        m.close()
    # the oracle applies the wrapped voxels' hits like the reference: in cloud order
    if len(fields) == 2:
        (ca, va, ga), (cb, vb, gb) = fields
        assert np.array_equal(ca, cb)
        assert np.array_equal(va.view(np.uint32), vb.view(np.uint32))
        assert np.array_equal(ga, gb)


def test_inner_colors_non_discrete_clipped_rays():
    """insertPointCloud on a colour map (the reference cannot instantiate it): the oracle's tree."""
    m = OracleMap(cl.FACE_RES, depth_levels=cl.FACE_LEVELS, color=True)
    for ins in cl.clipped_face_scans():
        m.insert(**ins)
    cl.check_tree_colors(m, what="oracle non-discrete")
    m.close()


def test_restatement_small_cases():
    # rms over the SET children only, truncated; an all-unset parent is 0
    codes = np.array([0, 1, 2, 8, 9], np.uint64)
    rgb = np.array([[255, 0, 1], [254, 0, 0], [0, 0, 0], [0, 0, 0], [0, 0, 0]], np.uint8)
    lv = cl.inner_colors(codes, rgb, 2)
    u, c = lv[1]
    assert list(u) == [0, 1]
    # sqrt((255^2 + 254^2) / 2) = 254.50..., sqrt(1/2) = 0.707
    assert tuple(c[0]) == (254, 0, 0) and tuple(c[1]) == (0, 0, 0)
    assert tuple(lv[2][1][0]) == (254, 0, 0)
    # level 2 from level 1, not from the leaves: rms(254 and three unset) = 254
    # black update darkens; equal update is a no-op; unset takes the update
    hit = cl.to_logit(0.7)
    assert cl.blend((10, 20, 30), (10, 20, 30), hit, 0.0) == (10, 20, 30)
    assert cl.blend((0, 0, 0), (10, 20, 30), hit, 0.0) == (10, 20, 30)
    assert cl.blend((100, 100, 100), (0, 0, 0), hit, 0.0)[0] < 100


@pytest.mark.parametrize("cls", [OracleMap, RefMap])
def test_leaf_blend_known_answer(cls):
    """One voxel hit by a prescribed colour sequence over many scans, up to the clamping bound:
    every step equals the restated blend with the voxel's log-odds before the scan."""
    if cls is RefMap and not have_ref():
        pytest.skip("reference harness not built")
    seq = [(200, 100, 50), (200, 100, 50), (0, 0, 0), (255, 255, 255), (255, 0, 0), (0, 255, 0),
           (255, 255, 255), (255, 255, 255), (12, 0, 0), (12, 0, 0), (0, 0, 7), (255, 255, 255),
           (128, 128, 128), (3, 250, 3)]
    m = cls(0.1, color=True, prob_hit=0.9)
    target = np.array([[1.03, 0.51, 0.22]])
    code = m.to_code(target[0])
    cur, saw_clamp = (0, 0, 0), False
    for c in seq:
        _, logit, rgb0, _, _ = m.node(code, 0)
        assert rgb0 == cur
        m.insert([0.013, 0.021, 0.007], target, rgb=np.array([c], np.uint8), discrete=True)
        cur = cl.blend(cur, c, np.float32(cl.to_logit(0.9)), logit)
        _, after, rgb1, _, _ = m.node(code, 0)
        assert rgb1 == cur, (c, rgb1, cur)
        saw_clamp |= after == logit  # held at the upper clamping bound
    assert saw_clamp
    m.close()
