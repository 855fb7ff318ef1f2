"""Opening saved maps: ufo_b200_read / ufo_b200_read_file (Octree::read) and the node-stream parser
behind them and ufo_b200_read_data (k_import_parse, one CTA per depth-4 sub-stream).

  * read(write()) into a fresh map of another geometry, mono and colour: min_depth 0 / 2 / 4, LZ4,
    AABB / sphere / frustum + OBB images -- value field, inner nodes, re-written image
  * the committed reference image through Map.read and Map.open
  * header cases: comments and unknown tokens, each missing or invalid field, the wrong tree type,
    another geometry, a truncated body
  * parser cases against the CPU checker's readData: merges into scanned maps, collapsed nodes of
    depth 1-7, volumes whose boundary cuts through voxels, a stream of several upload chunks read
    into pools that must grow
  * routed maps of 2 and 4 ranks reading one file
"""
import os

import numpy as np
import pytest

from helpers import assert_value_fields_equal, check_inner_against_field
from oracle_lib import OracleMap, RefMap, have_ref
from test_gpu_route_discrete import _barrier, _ranks
from test_gpu_route_read import _bricks, _check, _close, _volumes
from ufomap_b200 import capi, scans
from ufomap_b200.capi import Map

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def _res(color):
    return 0.04 if color else 0.08


def _source(color, ks=(0, 1)):
    m = Map(_res(color), color=color, initial_bricks=1 << 14)
    for k in ks:
        if color:
            o, p, rgb = scans.rgbd(k=k, width=96, height=72)
            m.insert(origin=o, xyz=p, rgb=rgb, max_range=4.0, discrete=True)
        else:
            o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
            m.insert(origin=o, xyz=p, max_range=12.0)
    return m


def _model():
    return OracleMap(0.1).sensor_model()


def _state(m):
    return [a.tobytes() for a in m.value_field()] + [m.pool_stats(), m.resolution, m.depth_levels]


def _images(src, color):
    """(name, image, rewrite, volume): rewrite(map) writes the image again with the arguments it was
    written with."""
    out = [("min_depth %d" % d, src.write(min_depth=d), lambda m, d=d: m.write(min_depth=d), None) for d in (0, 2, 4)]
    packed, _ = src.write_compressed()
    out.append(("lz4", packed, lambda m: m.write_compressed()[0], None))
    for name, vol in _volumes(color).items():
        out.append((name, src.write_bv(vol), lambda m, vol=vol: m.write_bv(vol), vol))
    return out


@pytest.mark.parametrize("color", [False, True], ids=["mono", "color"])
def test_read_round_trip(color):
    """Octree::read takes no volume, and a writer skips the children outside its volume without
    clearing their bits: an image written with a volume is read back through readData with that
    volume (the mapping server's get_map / msgToUfo pairing), here after its header."""
    src = _source(color)
    whole = src.value_field()
    for name, image, rewrite, vol in _images(src, color):
        m = Map(0.1, color=color, initial_bricks=1 << 8)  # the file's geometry replaces this one
        if vol is None:
            m.read(image)
        else:
            ok, h = capi.read_header(image)
            assert ok
            m.clear_resize(h["resolution"], h["depth_levels"])
            m.read_data_bv(image[h["data_offset"]:], vol)
        assert (m.resolution, m.depth_levels) == (_res(color), 16), name
        field = m.value_field()
        if name in ("min_depth 0", "lz4"):
            assert rewrite(m) == image, name
        else:
            # leaves above depth 0 or cut by the volume may merge into larger canonical leaves when
            # written again: the rewritten image reads back to the same map
            again = Map(0.1, color=color)
            if vol is None:
                again.read(rewrite(m))
            else:
                again.clear_resize(_res(color), 16)
                img = rewrite(m)
                again.read_data_bv(img[capi.read_header(img)[1]["data_offset"]:], vol)
            assert_value_fields_equal(again.value_field(), field, what="%s: rewritten" % name)
            again.close()
        if name in ("min_depth 0", "lz4"):
            assert_value_fields_equal(field, whole, what=name)
        check_inner_against_field(m, field, _model(), levels=(1, 2, 3, 4, 5, 6, 9, 16))
        if have_ref() and vol is None and name != "lz4":  # the reference cannot read its own compressed files
            ref = RefMap(_res(color), color=color)
            assert ref.read(image), name
            assert_value_fields_equal(field, ref.value_field(), what="%s: reference" % name)
        m.close()
    src.close()


def test_reference_reads_compressed_files_twice_decompressed():
    """DESIGN.md section 7: the reference's read decompresses a compressed file a second time and
    fails on it; this library reads it."""
    if not have_ref():
        pytest.skip("reference harness not built")
    src = _source(False, (0,))
    packed, _ = src.write_compressed()
    assert not RefMap(_res(False)).read(packed)
    m = Map(_res(False))
    m.read(packed)
    assert m.write() == src.write()
    _close([m, src])


def test_golden_image_opens(tmp_path):
    image = np.load(os.path.join(GOLD, "fileimage_rgbd_8cm.npz"))["image"].tobytes()
    m = Map(0.1, color=True)
    m.read(image)
    assert m.write() == image
    path = tmp_path / "rgbd.um"
    path.write_bytes(image)
    opened = Map.open(str(path))
    assert opened.color and opened.resolution == 0.08
    assert opened.write() == image
    again = Map(0.08, color=True)
    again.read_file(str(path))
    assert again.write() == image
    _close([m, opened, again])


def _with_header(image, header):
    ok, h = capi.read_header(image)
    assert ok
    return header.encode() + image[h["data_offset"]:]


GOOD = ("# UFOMap file\n# (feel free to add / change comments, but leave the first line as it is!)\n#\n"
        "version 1.0.0\nid occupancy_map\nresolution 0.08\ndepth_levels 16\ncompressed 0\n"
        "uncompressed_data_size 0\ndata\n")  # the writers put the stream's size into uncompressed_data_size


def test_header_cases():
    src = _source(False, (0,))
    image = src.write()
    assert image.startswith(GOOD.split("uncompressed_data_size")[0].encode())
    # comments, unknown tokens, fields in another order and on one line
    variants = [GOOD.replace("#\n", "# another comment\nfoo bar baz\n#x y\n"),
                "# UFOMap file v2\nid occupancy_map depth_levels 16\nversion 2\nresolution 0.08 colour red\n"
                "uncompressed_data_size 7 compressed 0\n# done\ndata  trailing words\n"]
    for v in variants:
        m = Map(0.08)
        m.read(_with_header(image, v))
        assert m.write() == image, v
        m.close()
    # each missing or invalid field: refused, nothing changed
    bad = [GOOD.replace("# UFOMap file", "# UFOmap file"), GOOD.replace("data\n", "dat\n"),
           GOOD.replace("version 1.0.0\n", ""), GOOD.replace("id occupancy_map\n", ""),
           GOOD.replace("resolution 0.08", "resolution 0"), GOOD.replace("resolution 0.08", "resolution -0.08"),
           GOOD.replace("resolution 0.08", "resolution x"), GOOD.replace("depth_levels 16", "depth_levels 0"),
           GOOD.replace("uncompressed_data_size 0", "uncompressed_data_size -1"),
           GOOD.replace("uncompressed_data_size 0\n", ""), GOOD.replace("compressed 0", "compressed 2"),
           GOOD.replace("depth_levels 16", "depth_levels 22")]
    m = _source(False, (1,))
    before = _state(m)
    for h in bad:
        with pytest.raises(capi.UfoError) as e:
            m.read(_with_header(image, h))
        assert e.value.status == capi.E_INVALID, h
        assert _state(m) == before, h
    # depth_levels < 5: the node stream is not readable here
    with pytest.raises(capi.UfoError) as e:
        m.read(_with_header(image, GOOD.replace("depth_levels 16", "depth_levels 4")))
    assert e.value.status == capi.E_UNSUPPORTED
    # a mono file into a colour map and back
    c = Map(0.08, color=True)
    cb = _state(c)
    with pytest.raises(capi.UfoError) as e:
        c.read(image)
    assert e.value.status == capi.E_INVALID and _state(c) == cb
    with pytest.raises(capi.UfoError) as e:
        m.read(_source(True, (0,)).write())
    assert e.value.status == capi.E_INVALID and _state(m) == before
    # truncated body: refused before anything is cleared, even with another geometry
    for dst in (m, Map(0.1, depth_levels=12)):
        b = _state(dst)
        with pytest.raises(capi.UfoError) as e:
            dst.read(image[:-3])
        assert e.value.status == capi.E_INVALID and _state(dst) == b
    # another geometry: the map is re-created with the file's
    for res, depth in ((0.1, 16), (0.08, 14), (0.2, 10)):
        dst = Map(res, depth_levels=depth)
        dst.insert(**dict(zip(("origin", "xyz"), scans.velodyne64(k=3, rings=8, azimuths=128))), max_range=5.0)
        dst.read(image)
        assert (dst.resolution, dst.depth_levels) == (0.08, 16)
        assert dst.write() == image
        dst.close()
    # the same geometry merges, like readData
    oracle = OracleMap(0.08)
    o, p = scans.velodyne64(k=1, rings=16, azimuths=512)
    oracle.insert(o, p, max_range=12.0)
    body = image[capi.read_header(image)[1]["data_offset"]:]
    assert oracle.read_data(body)
    m.read(image)
    assert_value_fields_equal(m.value_field(), oracle.value_field(), what="merge")
    _close([m, c, src])


def test_read_header_matches_readType():
    image = GOOD.encode() + b"\x00"
    ok, h = capi.read_header(image)
    assert ok and h == dict(version="1.0.0", id="occupancy_map", resolution=0.08, depth_levels=16, compressed=False,
                            uncompressed_data_size=0, data_offset=len(GOOD))
    # readType returns the id even when another field is invalid
    ok, h = capi.read_header(GOOD.replace("version 1.0.0\n", "").encode())
    assert not ok and h["id"] == "occupancy_map"
    ok, h = capi.read_header(b"# UFOMap fil\nid occupancy_map\n")
    assert not ok and h["id"] == ""


def _node_box(depth, corner_key, res, L=16):
    """(min, max) strictly inside the node of `depth` whose first voxel has key `corner_key`."""
    lo = (np.asarray(corner_key, np.float64) - 2 ** (L - 1)) * res
    size = res * 2 ** depth
    e = 0.25 * res
    return lo + e, lo + size - e


def test_collapsed_nodes_of_every_depth():
    res = 0.05
    src = Map(res, initial_bricks=1 << 12)
    base = 2 ** 15
    for d in range(1, 8):
        key = [base + 256 * d, base + 128, base - 256]
        src.set_value_volume(_node_box(d, key, res), 0.3 + 0.08 * d, 0)
    # and a node of depth 3 inside a refined brick
    src.set_value_volume(_node_box(0, [base + 3, base + 5, base + 7], res), 0.8, 0)
    src.set_value_volume(_node_box(3, [base + 8, base, base], res), 0.6, 0)
    image = src.write()
    m = Map(res)
    m.read(image)
    assert m.write() == image
    assert_value_fields_equal(m.value_field(), src.value_field(), what="collapsed")
    oracle = OracleMap(res)
    assert oracle.read_data(src.write_data())
    assert_value_fields_equal(m.value_field(), oracle.value_field(), what="oracle")
    _close([m, src])


@pytest.mark.parametrize("color", [False, True], ids=["mono", "color"])
def test_merge_and_volume_cuts(color):
    res = _res(color)
    other = _source(color, (2,))
    # boxes whose faces lie inside voxels
    boxes = [(np.array([-1.37, -0.93, -0.41]), np.array([1.13, 0.77, 0.29])),
             (np.array([0.011, -2.5, -0.7]), np.array([3.3, 0.013, 0.5]))]
    for box in boxes:
        m = _source(color, (0, 1))
        oracle = OracleMap(res, color=color)
        for k in (0, 1):
            if color:
                o, p, rgb = scans.rgbd(k=k, width=96, height=72)
                oracle.insert(o, p, rgb=rgb, max_range=4.0, discrete=True)
            else:
                o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
                oracle.insert(o, p, max_range=12.0)
        data = other.write_data(box=box)
        m.read_data(data, box=box)
        assert oracle.read_data(data, box=box)
        assert_value_fields_equal(m.value_field(), oracle.value_field(), what="box %r" % (box,))
        check_inner_against_field(m, m.value_field(), oracle.sensor_model())
        if have_ref():
            ref = RefMap(res, color=color)
            for k in (0, 1):
                if color:
                    o, p, rgb = scans.rgbd(k=k, width=96, height=72)
                    ref.insert(o, p, rgb=rgb, max_range=4.0, discrete=True)
                else:
                    o, p = scans.velodyne64(k=k, rings=16, azimuths=512)
                    ref.insert(o, p, max_range=12.0)
            assert ref.read_data(data, box=box)
            assert_value_fields_equal(m.value_field(), ref.value_field(), what="reference")
        _close([m])
    other.close()


def test_stream_of_several_chunks_into_growing_pools():
    """~1300 bricks of distinct values: a node stream of about 21 MB, more than one 16 MB upload
    chunk, read into a map created with 16 bricks."""
    res = 0.05
    src = Map(res, initial_bricks=1 << 12)
    base = np.uint64(7) << np.uint64(42)
    n = 1300 * 4096
    codes = base + np.arange(n, dtype=np.uint64)
    rng = np.random.default_rng(3)
    values = rng.uniform(-2.0, 2.0, n).astype(np.float32)
    src.update_nodes(codes, 0, Map.SET, values)
    data = src.write_data()
    assert len(data) > 16 << 20
    m = Map(res, initial_bricks=16)
    m.read_data(data)
    assert m.pool_stats()["brick_cap"] >= 1300
    assert m.write_data() == data
    assert_value_fields_equal(m.value_field(), src.value_field(), what="chunks")
    image = src.write()
    f = Map(0.1, initial_bricks=16)
    f.read(image)
    assert f.write() == image
    _close([m, f, src])


@pytest.mark.parametrize("world", [2, 4])
@pytest.mark.parametrize("color", [False, True], ids=["mono", "color"])
def test_routed_ranks_read_one_file(color, world, tmp_path):
    res = _res(color)
    src = _source(color, (0, 1))
    path = tmp_path / "map.um"
    src.write_file(str(path))
    image = path.read_bytes()
    maps = _ranks(world, res, bricks=1 << 14, color=color)
    single = Map(res, color=color, initial_bricks=1 << 14)
    before = _bricks(maps + [single])
    for m in maps + [single]:
        m.read_file(str(path))
    _barrier(maps)
    _check(maps, single, "read_file", before)
    assert single.write() == image
    # another geometry: refused on every rank, nothing changed
    other = Map(res * 2, color=color)
    foreign = other.write()
    states = [_state(m) for m in maps]
    for m in maps:
        with pytest.raises(capi.UfoError) as e:
            m.read(foreign)
        assert e.value.status == capi.E_UNSUPPORTED
    assert [_state(m) for m in maps] == states
    _close(maps + [single, src, other])
