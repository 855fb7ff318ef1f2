"""ctypes binding of libufomap_b200.so (include/ufomap_b200.h).

This is plumbing for tests/, bench.py and __graft_entry__: the product is the
shared library and its C ABI; the reference-facing host API is the C++ facade in
include/ufomap_b200/ufomap.hpp.  Loading fails loudly when the library has not
been built -- there is no CPU fallback.
"""
import ctypes as C
import math
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# UFOMAP_B200_LIB selects an experimental build of the same library (kernel variants)
LIB_PATH = os.environ.get("UFOMAP_B200_LIB") or os.path.join(HERE, "libufomap_b200.so")

OK, E_INVALID, E_CUDA, E_NOMEM, E_UNSUPPORTED = 0, 1, 2, 3, 4
XYZ_F64, XYZ_F32, XYZRGB_F64, XYZRGB_F32 = 0, 1, 2, 3


class Params(C.Structure):
    _fields_ = [
        ("resolution", C.c_double),
        ("depth_levels", C.c_uint32),
        ("automatic_pruning", C.c_int32),
        ("occupied_thres", C.c_double),
        ("free_thres", C.c_double),
        ("prob_hit", C.c_double),
        ("prob_miss", C.c_double),
        ("clamping_thres_min", C.c_double),
        ("clamping_thres_max", C.c_double),
        ("color", C.c_int32),
        ("device", C.c_int32),
        ("initial_blocks", C.c_uint64),
        ("initial_bricks", C.c_uint64),
    ]


class ScanStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "points", "rays", "visits", "touched_voxels", "hit_voxels", "touched_octets",
        "touched_blocks", "touched_d3", "touched_bricks", "upper_nodes", "blocks_in_map", "bricks_in_map",
        "device_bytes", "regrows", "launches", "result_bytes", "touched_lines")] + [(n, C.c_float) for n in (
            "ms_total", "ms_h2d", "ms_points", "ms_rays", "ms_scatter", "ms_update", "ms_propagate")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class WalkStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("records", "mask_reductions", "words_marked", "dirty_reductions")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class UpdateStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("saturated_octets", "saturated_lines", "clean_sectors")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class EarlyStats(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in (
        "rounds", "converged", "visits", "nodes", "free_nodes", "table_bytes", "id_bytes")] + [
            (n, C.c_float) for n in ("ms_walk", "ms_rounds", "ms_mark")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class RetainStats(C.Structure):
    """ufo_b200_retain_stats (retain and page_in)."""
    _fields_ = [(n, C.c_uint64) for n in (
        "bricks_before", "bricks_kept", "bricks_removed", "brick_cap_before", "brick_cap_after",
        "device_bytes_before", "device_bytes_after")] + [(n, C.c_float) for n in (
            "ms_classify", "ms_compact", "ms_upper")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class PageHeader(C.Structure):
    """ufo_b200_page_header: what ufo_b200_page_info reads from a blob."""
    _fields_ = [("version", C.c_uint32), ("color", C.c_uint32), ("depth_levels", C.c_uint32),
                ("reserved", C.c_uint32), ("resolution", C.c_double), ("n_bricks", C.c_uint64),
                ("bytes", C.c_uint64)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_ if n != "reserved"}


class FileHeader(C.Structure):
    """ufo_b200_file_header: the text header of a UFOMap file image."""
    _fields_ = [("version", C.c_char * 32), ("id", C.c_char * 32), ("resolution", C.c_double),
                ("depth_levels", C.c_uint32), ("compressed", C.c_int32), ("uncompressed_data_size", C.c_int64),
                ("data_offset", C.c_uint64)]


class PoolCounts(C.Structure):
    _fields_ = [(n, C.c_uint64) for n in ("bricks", "brick_cap", "upper_nodes", "up_cap", "device_bytes")]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


class TreeStats(C.Structure):
    """ufo_b200_tree_stats: the reference's node counters and known box of the pruned tree."""
    _fields_ = [("num_leaf_nodes", C.c_uint64), ("num_inner_nodes", C.c_uint64), ("with_children", C.c_uint64 * 22),
                ("known", C.c_int32), ("reserved", C.c_int32), ("known_min", C.c_double * 3),
                ("known_max", C.c_double * 3), ("ms_device", C.c_float), ("reserved2", C.c_float)]


class NearestStats(C.Structure):
    """ufo_b200_nearest_stats: the work of the last nearest-first shell."""
    _fields_ = [("bricks_visited", C.c_uint64), ("upper_visited", C.c_uint64), ("shells", C.c_uint32),
                ("rebuilt", C.c_int32), ("revision", C.c_uint64), ("ms_device", C.c_float), ("ms_rebuild", C.c_float)]

    def as_dict(self):
        return {n: getattr(self, n) for n, _ in self._fields_}


# every symbol include/ufomap_b200.h declares
SYMBOLS = [
    "ufo_b200_default_params", "ufo_b200_create", "ufo_b200_destroy", "ufo_b200_last_error",
    "ufo_b200_set_stream", "ufo_b200_insert_pointcloud", "ufo_b200_insert_device", "ufo_b200_wait",
    "ufo_b200_done", "ufo_b200_compute_ray", "ufo_b200_to_key", "ufo_b200_to_code",
    "ufo_b200_key_to_coord", "ufo_b200_key_to_code", "ufo_b200_code_to_key", "ufo_b200_query",
    "ufo_b200_export_leaves", "ufo_b200_set_sensor_model", "ufo_b200_sensor_model_logit",
    "ufo_b200_change_bbox", "ufo_b200_reset_change_bbox", "ufo_b200_last_scan_stats",
    "ufo_b200_set_profiling", "ufo_b200_clear", "ufo_b200_version", "ufo_b200_set_shard",
    "ufo_b200_insert_pointcloud_frame", "ufo_b200_transform_points", "ufo_b200_pose_from_rpy",
    "ufo_b200_insert_pointcloud2", "ufo_b200_write", "ufo_b200_write_file",
    "ufo_b200_write_data", "ufo_b200_set_value_volume", "ufo_b200_clear_resize",
    "ufo_b200_completed_scan_stats", "ufo_b200_set_sensor_model_field",
    "ufo_b200_route_inbox_bytes", "ufo_b200_route_setup", "ufo_b200_route_connect", "ufo_b200_route_mark",
    "ufo_b200_route_apply", "ufo_b200_ipc_export", "ufo_b200_ipc_open", "ufo_b200_ipc_close",
    "ufo_b200_write_compressed", "ufo_b200_cast_rays", "ufo_b200_export_nodes", "ufo_b200_read_data", "ufo_b200_enable_change_detection", "ufo_b200_reset_change_detection", "ufo_b200_changed_codes",
    "ufo_b200_update_nodes", "ufo_b200_insert_rays",
    "ufo_b200_route_inbox_bytes_color", "ufo_b200_route_mark_ex", "ufo_b200_route_sent",
    "ufo_b200_last_walk_stats",
    "ufo_b200_write_bv", "ufo_b200_write_data_bv", "ufo_b200_write_compressed_bv", "ufo_b200_read_data_bv",
    "ufo_b200_export_nodes_bv", "ufo_b200_set_value_volume_bv", "ufo_b200_volume_intersects",
    "ufo_b200_geometry_frustum", "ufo_b200_geometry_plane", "ufo_b200_geometry_ray",
    "ufo_b200_set_early_stopping", "ufo_b200_last_early_stats",
    "ufo_b200_iterate", "ufo_b200_update_nodes_color",
    "ufo_b200_retain_bv", "ufo_b200_retain", "ufo_b200_page_out_bv", "ufo_b200_page_in", "ufo_b200_page_info",
    "ufo_b200_pool_stats", "ufo_b200_last_update_stats", "ufo_b200_image_part_bv", "ufo_b200_image_assemble",
    "ufo_b200_read_header", "ufo_b200_read", "ufo_b200_read_file", "ufo_b200_clone", "ufo_b200_tree_info",
    "ufo_b200_nearest", "ufo_b200_last_nearest_stats",
]

# ufo_b200_volume: one shape of a bounding volume (type in BoundingVar order, members in v)
VOLUME_DTYPE = np.dtype([("type", "<u4"), ("reserved", "<u4"), ("v", "<f8", (24,))])
AABB, FRUSTUM, LINE_SEGMENT, OBB, PLANE, POINT, RAY, SPHERE = range(8)


def volume_record(kind, values):
    """One ufo_b200_volume: kind = AABB .. SPHERE, values = the shape's members in the reference's
    order (see include/ufomap_b200.h)."""
    r = np.zeros(1, VOLUME_DTYPE)
    v = np.asarray(values, np.float64).reshape(-1)
    r["type"] = kind
    r["v"][0, :len(v)] = v
    return r


def aabb(mn, mx):
    """AABB(min, max): half = (max - min) / 2, centre = min + half (geometry/aabb.h)."""
    mn, mx = np.asarray(mn, np.float64), np.asarray(mx, np.float64)
    half = (mx - mn) / 2.0
    return volume_record(AABB, np.concatenate([mn + half, half]))


def sphere(centre, radius):
    return volume_record(SPHERE, np.concatenate([np.asarray(centre, np.float64), [radius]]))


def obb(centre, half_size, quaternion_wxyz):
    return volume_record(OBB, np.concatenate([np.asarray(centre, np.float64), np.asarray(half_size, np.float64),
                                              np.asarray(quaternion_wxyz, np.float64)]))


def plane(normal, distance):
    return volume_record(PLANE, np.concatenate([np.asarray(normal, np.float64), [distance]]))


def point(xyz):
    return volume_record(POINT, np.asarray(xyz, np.float64))


def line_segment(start, end):
    return volume_record(LINE_SEGMENT, np.concatenate([np.asarray(start, np.float64), np.asarray(end, np.float64)]))


def ray(origin, direction):
    """Ray(origin, direction): the direction is normalised like the Ray constructor does (each
    component divided by sqrt((x*x + y*y) + z*z))."""
    d = [float(x) for x in direction]
    n = math.sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2])
    return volume_record(RAY, list(origin) + [d[0] / n, d[1] / n, d[2] / n])


def frustum(planes):
    """Frustum from its six planes (top, bottom, left, right, near, far), each (normal xyz, distance)."""
    return volume_record(FRUSTUM, np.asarray(planes, np.float64).reshape(24))


def frustum7(pos, target, up, vertical_angle, horizontal_angle, near_distance, far_distance):
    """Frustum(pos, target, up, vertical_angle, horizontal_angle, near, far), computed by the library."""
    out = np.empty(24)
    args = [np.ascontiguousarray(v, np.float64) for v in (pos, target, up)]
    load().ufo_b200_geometry_frustum(*(a.ctypes.data for a in args), float(vertical_angle), float(horizontal_angle),
                                     float(near_distance), float(far_distance), out.ctypes.data)
    return volume_record(FRUSTUM, out)


def plane3(v1, v2, v3):
    """Plane(v1, v2, v3), computed by the library."""
    out = np.empty(4)
    args = [np.ascontiguousarray(v, np.float64) for v in (v1, v2, v3)]
    load().ufo_b200_geometry_plane(*(a.ctypes.data for a in args), out.ctypes.data)
    return volume_record(PLANE, out)


def as_volume(volume):
    """A bounding volume as a contiguous array of ufo_b200_volume records: None / [] (the whole
    map), one record, or a sequence of records (their union)."""
    if volume is None:
        return np.zeros(0, VOLUME_DTYPE)
    if isinstance(volume, np.ndarray) and volume.dtype == VOLUME_DTYPE:
        return np.ascontiguousarray(volume.reshape(-1))
    parts = [as_volume(v) for v in volume]
    return np.ascontiguousarray(np.concatenate(parts)) if parts else np.zeros(0, VOLUME_DTYPE)


def volume_intersects(volume, centres, half_sizes):
    """The device's node-vs-volume predicate, run on the host: bool per cube (centres [n, 3],
    half_sizes [n, 3] or [n] for cubes)."""
    lib = load()
    bv = as_volume(volume)
    c = np.ascontiguousarray(centres, np.float64).reshape(-1, 3)
    h = np.asarray(half_sizes, np.float64)
    h = np.ascontiguousarray(np.broadcast_to(h.reshape(-1, 1) if h.ndim <= 1 else h, c.shape))
    out = np.zeros(len(c), np.uint8)
    rc = lib.ufo_b200_volume_intersects(bv.ctypes.data if len(bv) else None, len(bv), c.ctypes.data, h.ctypes.data,
                                        len(c), out.ctypes.data)
    if rc != OK:
        raise UfoError(rc, "invalid bounding volume")
    return out.astype(bool)

class Cloud2(C.Structure):
    """ufo_b200_cloud2: a sensor_msgs/PointCloud2 data buffer + field offsets."""
    _fields_ = [("data", C.c_void_p), ("n", C.c_size_t), ("point_step", C.c_uint32),
                ("off_x", C.c_uint32), ("off_y", C.c_uint32), ("off_z", C.c_uint32),
                ("off_r", C.c_int32), ("off_g", C.c_int32), ("off_b", C.c_int32),
                ("on_device", C.c_int32)]


_lib = None


def load():
    """Load the CUDA library; raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "ufomap_b200: %s is missing -- build it with `python -m ufomap_b200.build` "
            "(there is no CPU fallback)" % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    vp, sz, dbl, u32, i32, u64p = C.c_void_p, C.c_size_t, C.c_double, C.c_uint32, C.c_int, C.c_void_p
    lib.ufo_b200_default_params.argtypes = [C.POINTER(Params)]
    lib.ufo_b200_default_params.restype = None
    lib.ufo_b200_create.argtypes = [C.POINTER(Params), C.POINTER(vp)]
    lib.ufo_b200_destroy.argtypes = [vp]
    lib.ufo_b200_destroy.restype = None
    lib.ufo_b200_last_error.argtypes = [vp]
    lib.ufo_b200_last_error.restype = C.c_char_p
    lib.ufo_b200_set_stream.argtypes = [vp, vp]
    for f in (lib.ufo_b200_insert_pointcloud, lib.ufo_b200_insert_device):
        f.argtypes = [vp, vp, vp, sz, i32, dbl, u32, i32, u32, i32, i32]
    lib.ufo_b200_insert_pointcloud_frame.argtypes = [vp, vp, vp, sz, i32, vp, dbl, u32, i32, u32, i32,
                                                     i32]
    lib.ufo_b200_insert_pointcloud2.argtypes = [vp, vp, C.POINTER(Cloud2), vp, dbl, u32, i32, u32, i32, i32]
    lib.ufo_b200_write.argtypes = [vp, vp, u32, i32, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_write_file.argtypes = [vp, C.c_char_p, vp, u32, i32]
    lib.ufo_b200_clear_resize.argtypes = [vp, dbl, u32]
    lib.ufo_b200_set_value_volume.argtypes = [vp, vp, dbl, u32]
    lib.ufo_b200_update_nodes.argtypes = [vp, vp, vp, vp, vp, sz, i32]
    lib.ufo_b200_update_nodes_color.argtypes = [vp, vp, vp, vp, vp, vp, sz, i32]
    lib.ufo_b200_insert_rays.argtypes = [vp, vp, vp, sz, dbl, u32, i32, i32]
    lib.ufo_b200_write_data.argtypes = [vp, vp, u32, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_transform_points.argtypes = [vp, vp, sz, i32, vp]
    lib.ufo_b200_pose_from_rpy.argtypes = [dbl, dbl, dbl, dbl, dbl, dbl, vp]
    lib.ufo_b200_wait.argtypes = [vp]
    lib.ufo_b200_done.argtypes = [vp, C.POINTER(C.c_int)]
    lib.ufo_b200_compute_ray.argtypes = [vp, vp, vp, dbl, u32, u64p, sz, C.POINTER(sz)]
    lib.ufo_b200_to_key.argtypes = [vp, vp, u32, vp]
    lib.ufo_b200_to_code.argtypes = [vp, vp, u32, C.POINTER(C.c_uint64)]
    lib.ufo_b200_key_to_coord.argtypes = [vp, vp, u32, vp]
    lib.ufo_b200_key_to_code.argtypes = [vp]
    lib.ufo_b200_key_to_code.restype = C.c_uint64
    lib.ufo_b200_code_to_key.argtypes = [C.c_uint64, vp]
    lib.ufo_b200_code_to_key.restype = None
    lib.ufo_b200_query.argtypes = [vp, vp, vp, sz, vp, vp, vp]
    lib.ufo_b200_export_leaves.argtypes = [vp, vp, vp, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_set_sensor_model.argtypes = [vp, vp]
    lib.ufo_b200_sensor_model_logit.argtypes = [vp, vp]
    lib.ufo_b200_change_bbox.argtypes = [vp, vp, vp]
    lib.ufo_b200_reset_change_bbox.argtypes = [vp]
    lib.ufo_b200_last_scan_stats.argtypes = [vp, C.POINTER(ScanStats)]
    lib.ufo_b200_completed_scan_stats.argtypes = [vp, C.POINTER(ScanStats)]
    lib.ufo_b200_last_walk_stats.argtypes = [vp, C.POINTER(WalkStats)]
    lib.ufo_b200_last_update_stats.argtypes = [vp, C.POINTER(UpdateStats)]
    lib.ufo_b200_set_sensor_model_field.argtypes = [vp, i32, dbl]
    lib.ufo_b200_set_profiling.argtypes = [vp, i32]
    lib.ufo_b200_write_compressed.argtypes = [vp, vp, u32, i32, i32, i32, vp, sz, C.POINTER(sz), C.POINTER(sz)]
    lib.ufo_b200_read_data.argtypes = [vp, vp, vp, sz, i32, sz]
    lib.ufo_b200_export_nodes.argtypes = [vp, u32, i32, i32, i32, vp, vp, vp, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_cast_rays.argtypes = [vp, vp, vp, sz, i32, dbl, u32, vp, vp]
    lib.ufo_b200_enable_change_detection.argtypes = [vp, i32]
    lib.ufo_b200_reset_change_detection.argtypes = [vp]
    lib.ufo_b200_changed_codes.argtypes = [vp, u32, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_route_inbox_bytes.argtypes = [u32, u32, u32, C.POINTER(sz)]
    lib.ufo_b200_route_setup.argtypes = [vp, u32, u32, u32, u32, C.POINTER(vp)]
    lib.ufo_b200_route_connect.argtypes = [vp, C.POINTER(vp)]
    lib.ufo_b200_route_mark.argtypes = [vp, vp, vp, sz, i32, dbl, i32, i32]
    lib.ufo_b200_route_apply.argtypes = [vp, u32, u32, i32]
    lib.ufo_b200_route_inbox_bytes_color.argtypes = [u32, u32, u32, C.POINTER(sz)]
    lib.ufo_b200_route_mark_ex.argtypes = [vp, vp, vp, sz, i32, dbl, u32, i32, u32, i32, C.c_uint64, u32, i32, i32]
    lib.ufo_b200_route_sent.argtypes = [vp, C.POINTER(C.c_uint32 * 3)]
    lib.ufo_b200_ipc_export.argtypes = [vp, vp]
    lib.ufo_b200_ipc_open.argtypes = [vp, C.POINTER(vp)]
    lib.ufo_b200_ipc_close.argtypes = [vp]
    lib.ufo_b200_write_bv.argtypes = [vp, vp, sz, u32, i32, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_write_data_bv.argtypes = [vp, vp, sz, u32, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_write_compressed_bv.argtypes = [vp, vp, sz, u32, i32, i32, i32, vp, sz, C.POINTER(sz), C.POINTER(sz)]
    lib.ufo_b200_read_data_bv.argtypes = [vp, vp, sz, vp, sz, i32, sz]
    lib.ufo_b200_read_header.argtypes = [vp, sz, C.POINTER(FileHeader)]
    lib.ufo_b200_read.argtypes = [vp, vp, sz]
    lib.ufo_b200_read_file.argtypes = [vp, C.c_char_p]
    lib.ufo_b200_image_part_bv.argtypes = [vp, vp, sz, u32, i32, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_image_assemble.argtypes = [C.POINTER(vp), C.POINTER(sz), sz, i32, i32, i32, i32, vp, sz,
                                            C.POINTER(sz), C.POINTER(sz)]
    lib.ufo_b200_export_nodes_bv.argtypes = [vp, u32, i32, i32, i32, vp, sz, vp, vp, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_iterate.argtypes = [vp, i32, i32, i32, i32, i32, u32, vp, sz, vp, vp, vp, vp, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_set_value_volume_bv.argtypes = [vp, vp, dbl, u32]
    lib.ufo_b200_volume_intersects.argtypes = [vp, sz, vp, vp, sz, vp]
    lib.ufo_b200_geometry_frustum.argtypes = [vp, vp, vp, dbl, dbl, dbl, dbl, vp]
    lib.ufo_b200_geometry_plane.argtypes = [vp, vp, vp, vp]
    lib.ufo_b200_geometry_ray.argtypes = [vp, vp, vp]
    lib.ufo_b200_clear.argtypes = [vp]
    lib.ufo_b200_set_shard.argtypes = [vp, u32, u32]
    lib.ufo_b200_set_early_stopping.argtypes = [vp, i32]
    lib.ufo_b200_last_early_stats.argtypes = [vp, C.POINTER(EarlyStats)]
    lib.ufo_b200_retain_bv.argtypes = [vp, vp, sz, C.POINTER(RetainStats)]
    lib.ufo_b200_retain.argtypes = [vp, vp, C.POINTER(RetainStats)]
    lib.ufo_b200_page_out_bv.argtypes = [vp, vp, sz, vp, sz, C.POINTER(sz)]
    lib.ufo_b200_page_in.argtypes = [vp, vp, sz, C.POINTER(RetainStats)]
    lib.ufo_b200_page_info.argtypes = [vp, sz, C.POINTER(PageHeader)]
    lib.ufo_b200_pool_stats.argtypes = [vp, C.POINTER(PoolCounts)]
    lib.ufo_b200_clone.argtypes = [vp, C.POINTER(vp)]
    lib.ufo_b200_tree_info.argtypes = [vp, C.POINTER(TreeStats)]
    lib.ufo_b200_nearest.argtypes = [vp, vp, vp, sz, i32, i32, i32, i32, i32, u32, dbl, sz, vp, vp, vp, vp, vp, vp, sz,
                                     C.POINTER(sz), C.POINTER(C.c_double)]
    lib.ufo_b200_last_nearest_stats.argtypes = [vp, C.POINTER(NearestStats)]
    lib.ufo_b200_version.restype = C.c_char_p
    _lib = lib
    return lib


class UfoError(RuntimeError):
    def __init__(self, status, msg):
        super().__init__("ufomap_b200 status %d: %s" % (status, msg))
        self.status = status


def pack_points(xyz, rgb=None, dtype=np.float64):
    """Pack points into one of the C-ABI layouts; returns (buffer, layout)."""
    xyz = np.asarray(xyz)
    n = len(xyz)
    if rgb is None:
        buf = np.ascontiguousarray(xyz, dtype=dtype).reshape(n, 3)
        return buf, (XYZ_F64 if dtype == np.float64 else XYZ_F32)
    rgb = np.asarray(rgb, dtype=np.uint8).reshape(n, 3)
    if dtype == np.float64:
        buf = np.zeros((n, 32), np.uint8)
        buf[:, :24] = np.ascontiguousarray(xyz, dtype=np.float64).reshape(n, 3).view(np.uint8).reshape(n, 24)
        buf[:, 24:27] = rgb
        return buf, XYZRGB_F64
    buf = np.zeros((n, 16), np.uint8)
    buf[:, :12] = np.ascontiguousarray(xyz, dtype=np.float32).reshape(n, 3).view(np.uint8).reshape(n, 12)
    buf[:, 12:15] = rgb
    return buf, XYZRGB_F32


def read_header(image):
    """Octree::readHeader of a file image (bytes, or a prefix holding the header): (ok, fields).
    fields: version, id, resolution, depth_levels, compressed, uncompressed_data_size and
    data_offset (the node stream's first byte), as far as they were read; id is what
    Octree::readType returns."""
    buf = np.frombuffer(image, np.uint8)
    h = FileHeader()
    rc = load().ufo_b200_read_header(buf.ctypes.data if len(buf) else None, len(buf), C.byref(h))
    fields = dict(version=h.version.decode(), id=h.id.decode(), resolution=h.resolution,
                  depth_levels=int(h.depth_levels), compressed=bool(h.compressed),
                  uncompressed_data_size=int(h.uncompressed_data_size), data_offset=int(h.data_offset))
    return rc == OK, fields


class Map:
    """Thin object wrapper over the C ABI (one map = one device + one stream)."""

    def __init__(self, resolution, depth_levels=16, automatic_pruning=True, color=False,
                 device=-1, initial_blocks=0, initial_bricks=0, **model):
        self.lib = load()
        p = Params()
        self.lib.ufo_b200_default_params(C.byref(p))
        p.resolution = resolution
        p.depth_levels = depth_levels
        p.automatic_pruning = int(automatic_pruning)
        p.color = int(color)
        p.device = device
        p.initial_blocks = int(initial_blocks)
        p.initial_bricks = int(initial_bricks)
        for k, v in model.items():
            setattr(p, k, v)
        self.color = bool(color)
        self.resolution = resolution
        self.depth_levels = depth_levels
        self.h = C.c_void_p()
        rc = self.lib.ufo_b200_create(C.byref(p), C.byref(self.h))
        if rc == E_INVALID:
            raise ValueError("invalid map parameters (depth_levels has to be [2, 21])")
        if rc != OK:
            raise UfoError(rc, "ufo_b200_create failed (no usable CUDA device?)")

    def close(self):
        if getattr(self, "h", None):
            self.lib.ufo_b200_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _check(self, rc):
        if rc != OK:
            raise UfoError(rc, (self.lib.ufo_b200_last_error(self.h) or b"").decode())

    # -- integration --------------------------------------------------------
    def insert(self, origin, xyz, rgb=None, max_range=-1.0, depth=0, simple=False,
               early_stopping=0, discrete=False, async_=False, dtype=np.float64):
        buf, layout = pack_points(xyz, rgb, dtype)
        o = np.ascontiguousarray(origin, dtype=np.float64)
        self._keep = (buf, o)
        self._check(self.lib.ufo_b200_insert_pointcloud(
            self.h, o.ctypes.data, buf.ctypes.data, len(buf), layout, float(max_range), int(depth),
            int(simple), int(early_stopping), int(discrete), int(async_)))

    def insert_frame(self, origin, xyz, frame_pose, rgb=None, max_range=-1.0, depth=0, simple=False,
                     discrete=False, async_=False, dtype=np.float64, early_stopping=0):
        """insertPointCloud(sensor_origin, cloud, frame_origin, ...): the cloud is moved into the
        map frame on the device.  frame_pose = (tx, ty, tz, qw, qx, qy, qz)."""
        buf, layout = pack_points(xyz, rgb, dtype)
        o = np.ascontiguousarray(origin, dtype=np.float64)
        f = np.ascontiguousarray(frame_pose, dtype=np.float64)
        assert f.shape == (7,)
        self._keep = (buf, o, f)
        self._check(self.lib.ufo_b200_insert_pointcloud_frame(
            self.h, o.ctypes.data, buf.ctypes.data, len(buf), layout, f.ctypes.data,
            float(max_range), int(depth), int(simple), int(early_stopping), int(discrete), int(async_)))

    def insert_pointcloud2(self, origin, data, point_step, off_xyz=(0, 4, 8), off_rgb=None,
                           frame_pose=None, max_range=-1.0, depth=0, simple=False, discrete=False,
                           async_=False, early_stopping=0):
        """Insert a raw sensor_msgs/PointCloud2 data buffer (numpy uint8 array); NaN points are
        skipped on the device like rosToUfo does."""
        buf = np.ascontiguousarray(data, dtype=np.uint8).reshape(-1)
        assert len(buf) % point_step == 0
        o = np.ascontiguousarray(origin, dtype=np.float64)
        f = None if frame_pose is None else np.ascontiguousarray(frame_pose, dtype=np.float64)
        r, g, b = (-1, -1, -1) if off_rgb is None else (off_rgb + 2, off_rgb + 1, off_rgb)
        c = Cloud2(buf.ctypes.data, len(buf) // point_step, point_step, off_xyz[0], off_xyz[1], off_xyz[2],
                   r, g, b, 0)
        self._keep = (buf, o, f, c)
        self._check(self.lib.ufo_b200_insert_pointcloud2(
            self.h, o.ctypes.data, C.byref(c), None if f is None else f.ctypes.data, float(max_range),
            int(depth), int(simple), int(early_stopping), int(discrete), int(async_)))

    def insert_packed(self, origin, buf_ptr, n, layout, max_range=-1.0, depth=0, simple=False,
                      discrete=False, async_=False, on_device=False, early_stopping=0):
        """Insert from an already packed buffer (host pointer, or device pointer when
        on_device=True)."""
        o = np.ascontiguousarray(origin, dtype=np.float64)
        f = self.lib.ufo_b200_insert_device if on_device else self.lib.ufo_b200_insert_pointcloud
        self._check(f(self.h, o.ctypes.data, buf_ptr, int(n), int(layout), float(max_range),
                      int(depth), int(simple), int(early_stopping), int(discrete), int(async_)))

    def wait(self):
        self._check(self.lib.ufo_b200_wait(self.h))

    def done(self):
        d = C.c_int()
        self._check(self.lib.ufo_b200_done(self.h, C.byref(d)))
        return bool(d.value)

    def set_stream(self, stream_ptr):
        self._check(self.lib.ufo_b200_set_stream(self.h, stream_ptr))

    def set_profiling(self, enable=True):
        self._check(self.lib.ufo_b200_set_profiling(self.h, int(enable)))

    def stats(self):
        st = ScanStats()
        self._check(self.lib.ufo_b200_last_scan_stats(self.h, C.byref(st)))
        return st.as_dict()

    def completed_stats(self):
        """Statistics of the last COMPLETED scan (no wait for the scan in flight)."""
        st = ScanStats()
        self._check(self.lib.ufo_b200_completed_scan_stats(self.h, C.byref(st)))
        return st.as_dict()

    def walk_stats(self):
        """What the fused walk of the last insert sent to the scan volume (profiling level 2):
        records pushed, mask reductions issued, words they found empty, dirty-bit reductions."""
        st = WalkStats()
        self._check(self.lib.ufo_b200_last_walk_stats(self.h, C.byref(st)))
        return st.as_dict()

    def update_stats(self):
        """What the leaf update of the last insert left out (profiling level 2): touched octets of
        saturated lines, leaf lines not read because of them, sectors not written back."""
        st = UpdateStats()
        self._check(self.lib.ufo_b200_last_update_stats(self.h, C.byref(st)))
        return st.as_dict()

    def set_early_stopping(self, exact):
        """exact=True: inserts with early_stopping != 0 compute the reference's sequential result on
        the device (extra work and memory); False: they are rejected with E_UNSUPPORTED (the
        default)."""
        self._check(self.lib.ufo_b200_set_early_stopping(self.h, int(exact)))

    def early_stats(self):
        """The last insert's early-stopping work: rounds, converged, visits, nodes, free_nodes,
        table_bytes, id_bytes and, at profiling level >= 1, ms_walk / ms_rounds / ms_mark."""
        st = EarlyStats()
        self._check(self.lib.ufo_b200_last_early_stats(self.h, C.byref(st)))
        return st.as_dict()

    def set_sensor_model_field(self, index, probability):
        """One parameter, like the reference's setProbHit/... (the other stored log-odds stay)."""
        self._check(self.lib.ufo_b200_set_sensor_model_field(self.h, int(index), float(probability)))

    def clear(self):
        self._check(self.lib.ufo_b200_clear(self.h))

    def set_shard(self, rank, world):
        """Keep only the bricks this rank owns (spatial sharding over several GPUs)."""
        self._check(self.lib.ufo_b200_set_shard(self.h, int(rank), int(world)))

    # -- routed multi-GPU mode ----------------------------------------------
    def route_setup(self, rank, world, cap_bricks=1 << 16, cap_hits=1 << 18):
        """Allocate this rank's inbox; returns its device pointer (int)."""
        ptr = C.c_void_p()
        self._check(self.lib.ufo_b200_route_setup(self.h, int(rank), int(world), int(cap_bricks), int(cap_hits),
                                                  C.byref(ptr)))
        self.route_world = world
        return ptr.value

    def route_connect(self, peer_ptrs):
        arr = (C.c_void_p * len(peer_ptrs))(*[C.c_void_p(p) for p in peer_ptrs])
        self._check(self.lib.ufo_b200_route_connect(self.h, arr))

    def route_mark(self, origin, buf_ptr, n, layout, max_range=-1.0, on_device=False, self_too=False):
        o = np.ascontiguousarray(origin, dtype=np.float64)
        self._check(self.lib.ufo_b200_route_mark(self.h, o.ctypes.data, buf_ptr, int(n), int(layout),
                                                 float(max_range), int(on_device), int(self_too)))

    def route_mark_ex(self, origin, buf_ptr, n, layout, max_range=-1.0, depth=0, simple=False,
                      early_stopping=0, discrete=False, index_base=0, index_stride=1, on_device=False,
                      self_too=False):
        """route_mark with the options of insert (mono and colour maps).  Local point i is point
        index_base + i * index_stride of the whole cloud: (offset, 1) for a contiguous sector,
        (rank, world) for buf[rank::world]."""
        o = np.ascontiguousarray(origin, dtype=np.float64)
        self._check(self.lib.ufo_b200_route_mark_ex(
            self.h, o.ctypes.data, buf_ptr, int(n), int(layout), float(max_range), int(depth), int(simple),
            int(early_stopping), int(discrete), int(index_base), int(index_stride), int(on_device), int(self_too)))

    def route_sent(self):
        """Records this rank wrote into inboxes in its last mark pass (waits for the map's stream)."""
        c = (C.c_uint32 * 3)()
        self._check(self.lib.ufo_b200_route_sent(self.h, C.byref(c)))
        return {"brick_records": c[0], "full_brick_records": c[1], "hit_records": c[2]}

    def route_apply(self, first=0, count=None, last=True):
        count = self.route_world if count is None else count
        self._check(self.lib.ufo_b200_route_apply(self.h, int(first), int(count), int(last)))

    # -- file / wire format -------------------------------------------------
    @staticmethod
    def _box6(box):
        """(min xyz, max xyz) -> the AABB's centre / half size, like its (min, max) constructor."""
        if box is None:
            return None
        mn, mx = np.asarray(box[0], np.float64), np.asarray(box[1], np.float64)
        half = (mx - mn) / 2.0
        return np.ascontiguousarray(np.concatenate([mn + half, half]), np.float64)

    def write(self, expanded=False, box=None, min_depth=0):
        """The map as a UFOMap file image (bytes), Octree::write with compress=False."""
        b = self._box6(box)
        bp = None if b is None else b.ctypes.data
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_write(self.h, bp, int(min_depth), int(expanded), None, 0, C.byref(n)))
        buf = np.empty(n.value, np.uint8)
        self._check(self.lib.ufo_b200_write(self.h, bp, int(min_depth), int(expanded), buf.ctypes.data, n.value,
                                            C.byref(n)))
        assert n.value == len(buf)
        return buf.tobytes()

    def write_compressed(self, box=None, min_depth=0, data_only=False, acceleration=1, level=0):
        """Octree::write / writeData with compress=True: (bytes, uncompressed_data_size)."""
        b = self._box6(box)
        bp = None if b is None else b.ctypes.data
        n, u = C.c_size_t(), C.c_size_t()
        self._check(self.lib.ufo_b200_write_compressed(self.h, bp, int(min_depth), int(data_only), int(acceleration),
                                                       int(level), None, 0, C.byref(n), C.byref(u)))
        buf = np.empty(max(n.value, 1), np.uint8)
        self._check(self.lib.ufo_b200_write_compressed(self.h, bp, int(min_depth), int(data_only), int(acceleration),
                                                       int(level), buf.ctypes.data, n.value, C.byref(n), C.byref(u)))
        return buf[:n.value].tobytes(), int(u.value)

    def read_data(self, data, box=None, compressed=False, uncompressed_size=0):
        """Octree::readData: merge a node stream (bytes) into the map; box = (min xyz, max xyz)."""
        b = self._box6(box)
        buf = np.frombuffer(data, np.uint8)
        self._check(self.lib.ufo_b200_read_data(self.h, None if b is None else b.ctypes.data,
                                                buf.ctypes.data if len(buf) else None, len(buf), int(compressed),
                                                int(uncompressed_size)))

    def read(self, image):
        """Octree::read of a file image (bytes): a file of another resolution / depth_levels
        re-creates the map with the file's, one of the same merges into it."""
        buf = np.frombuffer(image, np.uint8)
        self._check(self.lib.ufo_b200_read(self.h, buf.ctypes.data if len(buf) else None, len(buf)))
        self._geometry_from(image[:1 << 16])

    def read_file(self, filename):
        """Octree::read(filename)."""
        self._check(self.lib.ufo_b200_read_file(self.h, os.fsencode(filename)))
        with open(filename, "rb") as f:
            self._geometry_from(f.read(1 << 16))

    def _geometry_from(self, head):
        ok, h = read_header(head)
        if ok:
            self.resolution, self.depth_levels = h["resolution"], h["depth_levels"]

    @classmethod
    def open(cls, filename, device=-1, **kwargs):
        """A new map of the file's tree type, read from the file (the file constructors
        OccupancyMap(filename) / OccupancyMapColor(filename))."""
        with open(filename, "rb") as f:
            ok, h = read_header(f.read(1 << 16))
        if h["id"] not in ("occupancy_map", "occupancy_map_color"):
            raise ValueError("%s: not a UFOMap file of a known tree type" % filename)
        m = cls(h["resolution"] if ok else 0.1, h["depth_levels"] if ok and 5 <= h["depth_levels"] <= 21 else 16,
                color=h["id"] == "occupancy_map_color", device=device, **kwargs)
        try:
            m.read_file(filename)
        except Exception:
            m.close()
            raise
        return m

    def write_file(self, filename, expanded=False, box=None, min_depth=0):
        b = self._box6(box)
        self._check(self.lib.ufo_b200_write_file(self.h, os.fsencode(filename),
                                                 None if b is None else b.ctypes.data, int(min_depth),
                                                 int(expanded)))

    def clear_resize(self, resolution, depth_levels):
        """Octree::clear(resolution, depth_levels)."""
        self._check(self.lib.ufo_b200_clear_resize(self.h, float(resolution), int(depth_levels)))
        self.resolution, self.depth_levels = resolution, depth_levels

    def set_value_volume(self, box, occupancy, min_depth=0):
        """setValueVolume(AABB(min, max), occupancy probability, min_depth); box = (min xyz, max xyz)."""
        b = self._box6(box)
        self._check(self.lib.ufo_b200_set_value_volume(self.h, b.ctypes.data, float(occupancy), int(min_depth)))

    # -- per-node writes ----------------------------------------------------
    ADD, SET = 0, 1

    def update_nodes(self, codes, depths, ops, values, async_=False):
        """Ordered batch of node writes: op 0 adds values[i] (float log-odds) to every voxel below
        the node (updateValue), op 1 sets them to it (setNodeValue); clamped after every update."""
        c = np.ascontiguousarray(codes, dtype=np.uint64).reshape(-1)
        n = len(c)
        d = np.ascontiguousarray(np.broadcast_to(depths, (n,)), dtype=np.uint32)
        o = np.ascontiguousarray(np.broadcast_to(ops, (n,)), dtype=np.uint8)
        v = np.ascontiguousarray(np.broadcast_to(values, (n,)), dtype=np.float32)
        self._check(self.lib.ufo_b200_update_nodes(self.h, c.ctypes.data, d.ctypes.data, o.ctypes.data,
                                                   v.ctypes.data, n, int(async_)))

    ADD_COLOR, SET_COLOR = 2, 3

    def update_nodes_color(self, codes, depths, ops, values, rgb, async_=False):
        """update_nodes plus the colour map's writers, one ordered batch: op 2 blends rgb[i] into the
        voxel's colour and then adds values[i] (updateValue(code, value, Color)), op 3 sets the
        colour (setColor); both at depth 0.  rgb: [n][3] uint8 or one colour, or None for a batch
        without ops 2 and 3."""
        c = np.ascontiguousarray(codes, dtype=np.uint64).reshape(-1)
        n = len(c)
        d = np.ascontiguousarray(np.broadcast_to(depths, (n,)), dtype=np.uint32)
        o = np.ascontiguousarray(np.broadcast_to(ops, (n,)), dtype=np.uint8)
        v = np.ascontiguousarray(np.broadcast_to(values, (n,)), dtype=np.float32)
        col = None
        if rgb is not None:
            col = np.ascontiguousarray(np.broadcast_to(np.asarray(rgb, np.uint8).reshape(-1, 3), (n, 3)))
        self._check(self.lib.ufo_b200_update_nodes_color(self.h, c.ctypes.data, d.ctypes.data, o.ctypes.data,
                                                         v.ctypes.data, None if col is None else col.ctypes.data,
                                                         n, int(async_)))

    def insert_rays(self, origins, ends, max_range=-1.0, depth=0, hit_end=False, async_=False):
        """insertMissOnRay (hit_end=False) / insertRay (hit_end=True) for every (origin, end)."""
        e = np.ascontiguousarray(ends, dtype=np.float64).reshape(-1, 3)
        o = np.ascontiguousarray(np.broadcast_to(np.asarray(origins, np.float64).reshape(-1, 3), e.shape),
                                 dtype=np.float64)
        self._check(self.lib.ufo_b200_insert_rays(self.h, o.ctypes.data, e.ctypes.data, len(e), float(max_range),
                                                  int(depth), int(hit_end), int(async_)))

    def write_data(self, box=None, min_depth=0):
        """Octree::writeData(stream, AABB(min, max) or whole map, False, min_depth): node stream.
        box = (min xyz, max xyz); converted to the AABB's centre / half size like its constructor."""
        b = self._box6(box)
        bp = None if b is None else b.ctypes.data
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_write_data(self.h, bp, int(min_depth), None, 0, C.byref(n)))
        buf = np.empty(max(n.value, 1), np.uint8)
        self._check(self.lib.ufo_b200_write_data(self.h, bp, int(min_depth), buf.ctypes.data, n.value,
                                                 C.byref(n)))
        return buf[:n.value].tobytes()

    # -- bounding volumes (volume: see as_volume) -----------------------------
    @staticmethod
    def _bv(volume):
        bv = as_volume(volume)
        return bv, (bv.ctypes.data if len(bv) else None), len(bv)

    def write_bv(self, volume=None, min_depth=0, expanded=False):
        """Octree::write(stream, BoundingVolume, compress=False, min_depth): file image (bytes)."""
        bv, bp, nb = self._bv(volume)
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_write_bv(self.h, bp, nb, int(min_depth), int(expanded), None, 0, C.byref(n)))
        buf = np.empty(max(n.value, 1), np.uint8)
        self._check(self.lib.ufo_b200_write_bv(self.h, bp, nb, int(min_depth), int(expanded), buf.ctypes.data, n.value,
                                               C.byref(n)))
        return buf[:n.value].tobytes()

    def write_data_bv(self, volume=None, min_depth=0):
        """Octree::writeData(stream, BoundingVolume, compress=False, min_depth): node stream (bytes)."""
        bv, bp, nb = self._bv(volume)
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_write_data_bv(self.h, bp, nb, int(min_depth), None, 0, C.byref(n)))
        buf = np.empty(max(n.value, 1), np.uint8)
        self._check(self.lib.ufo_b200_write_data_bv(self.h, bp, nb, int(min_depth), buf.ctypes.data, n.value, C.byref(n)))
        return buf[:n.value].tobytes()

    def write_compressed_bv(self, volume=None, min_depth=0, data_only=False, acceleration=1, level=0):
        """Octree::write / writeData with a BoundingVolume and compress=True: (bytes, uncompressed size)."""
        bv, bp, nb = self._bv(volume)
        n, u = C.c_size_t(), C.c_size_t()
        args = (int(min_depth), int(data_only), int(acceleration), int(level))
        self._check(self.lib.ufo_b200_write_compressed_bv(self.h, bp, nb, *args, None, 0, C.byref(n), C.byref(u)))
        buf = np.empty(max(n.value, 1), np.uint8)
        self._check(self.lib.ufo_b200_write_compressed_bv(self.h, bp, nb, *args, buf.ctypes.data, n.value, C.byref(n),
                                                          C.byref(u)))
        return buf[:n.value].tobytes(), int(u.value)

    def image_part(self, volume=None, box=None, min_depth=0, expanded=False):
        """This map's part of the file image for (volume or box = (min xyz, max xyz), min_depth,
        expanded) as bytes; assemble_image() of the parts of maps holding disjoint bricks (the ranks
        of a routed map) is the image of their union."""
        bv, bp, nb = self._bv(aabb(*box) if box is not None else volume)
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_image_part_bv(self.h, bp, nb, int(min_depth), int(expanded), None, 0, C.byref(n)))
        buf = np.empty(n.value, np.uint8)
        self._check(self.lib.ufo_b200_image_part_bv(self.h, bp, nb, int(min_depth), int(expanded), buf.ctypes.data,
                                                    n.value, C.byref(n)))
        assert n.value == len(buf)
        return buf.tobytes()

    def read_data_bv(self, data, volume=None, compressed=False, uncompressed_size=0):
        """Octree::readData(stream, BoundingVolume, ...): merge a node stream into the map."""
        bv, bp, nb = self._bv(volume)
        buf = np.frombuffer(data, np.uint8)
        self._check(self.lib.ufo_b200_read_data_bv(self.h, bp, nb, buf.ctypes.data if len(buf) else None, len(buf),
                                                   int(compressed), int(uncompressed_size)))

    def export_nodes_bv(self, volume=None, depth=0, occupied=True, free=True, unknown=False):
        """beginLeaves(BoundingVolume, occupied, free, unknown, false, depth) as a batch: (codes sorted,
        occ, rgb) of the depth-`depth` nodes whose whole path from the root passes the volume."""
        bv, bp, nb = self._bv(volume)
        flt = (int(depth), int(occupied), int(free), int(unknown))
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_export_nodes_bv(self.h, *flt, bp, nb, None, None, None, 0, C.byref(n)))
        cnt = n.value
        codes = np.empty(cnt, np.uint64)
        occ = np.empty(cnt, np.float32)
        rgb = np.zeros((cnt, 3), np.uint8)
        if cnt:
            self._check(self.lib.ufo_b200_export_nodes_bv(self.h, *flt, bp, nb, codes.ctypes.data, occ.ctypes.data,
                                                          rgb.ctypes.data if self.color else None, cnt, C.byref(n)))
        order = np.argsort(codes, kind="stable")
        return codes[order], occ[order], rgb[order]

    def iterate(self, volume=None, leaves=True, occupied=True, free=True, unknown=False, contains=False, min_depth=0):
        """beginLeaves (leaves=True) / beginTree (occupancy_map_base.h:93-163) over a bounding volume
        (None: the whole map): (codes, depths u8, logodds f32, flags u8, rgb u8[n,3]) in the
        reference iterator's order.  flags: bit0 contains_free, bit1 contains_unknown, bit2 isLeaf."""
        bv, bp, nb = self._bv(volume)
        args = (int(bool(leaves)), int(bool(occupied)), int(bool(free)), int(bool(unknown)), int(bool(contains)),
                int(min_depth), bp, nb)
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_iterate(self.h, *args, None, None, None, None, None, 0, C.byref(n)))
        cnt = n.value
        codes = np.empty(cnt, np.uint64)
        depths = np.empty(cnt, np.uint8)
        occ = np.empty(cnt, np.float32)
        flags = np.empty(cnt, np.uint8)
        rgb = np.zeros((cnt, 3), np.uint8)
        if cnt:
            self._check(self.lib.ufo_b200_iterate(self.h, *args, codes.ctypes.data, depths.ctypes.data, occ.ctypes.data,
                                                  flags.ctypes.data, rgb.ctypes.data if self.color else None, cnt,
                                                  C.byref(n)))
            assert n.value == cnt
        return codes, depths, occ, flags, rgb

    def nearest(self, point, volume=None, leaves=True, occupied=True, free=True, unknown=False, contains=False,
                min_depth=0, d2_from=0.0, want=1):
        """One shell of beginNNLeaves (leaves=True) / beginNNTree from `point`: the nodes of iterate()
        with d2_from <= d2 < d2_next, sorted by (d2, iterate's order), at least `want` of them unless
        fewer remain.  Returns (codes, depths u8, logodds f32, flags u8, rgb u8[n,3], d2 f64, d2_next);
        d2_next is +inf when the iteration is done.  Two library calls: one counts, one fills the arrays
        (it repeats the search on the kept tree shape); last_nearest_stats() reports the first."""
        bv, bp, nb = self._bv(volume)
        pt = np.ascontiguousarray(point, np.float64).reshape(3)
        args = (pt.ctypes.data, bp, nb, int(bool(leaves)), int(bool(occupied)), int(bool(free)), int(bool(unknown)),
                int(bool(contains)), int(min_depth), float(d2_from), int(want))
        n, nxt = C.c_size_t(), C.c_double()
        self._check(self.lib.ufo_b200_nearest(self.h, *args, None, None, None, None, None, None, 0, C.byref(n),
                                              C.byref(nxt)))
        self._near_stats = NearestStats()
        self._check(self.lib.ufo_b200_last_nearest_stats(self.h, C.byref(self._near_stats)))
        cnt = n.value
        codes, depths = np.empty(cnt, np.uint64), np.empty(cnt, np.uint8)
        occ, flags = np.empty(cnt, np.float32), np.empty(cnt, np.uint8)
        rgb, d2 = np.zeros((cnt, 3), np.uint8), np.empty(cnt, np.float64)
        if cnt:
            self._check(self.lib.ufo_b200_nearest(self.h, *args, codes.ctypes.data, depths.ctypes.data, occ.ctypes.data,
                                                  flags.ctypes.data, rgb.ctypes.data if self.color else None,
                                                  d2.ctypes.data, cnt, C.byref(n), C.byref(nxt)))
            assert n.value == cnt
        return codes, depths, occ, flags, rgb, d2, nxt.value

    def nearest_shells(self, point, volume=None, want=1, **kw):
        """Every shell of nearest() from d2 = 0 on, in order (a generator)."""
        d2_from = 0.0
        while d2_from != math.inf:
            *shell, d2_from = self.nearest(point, volume, d2_from=d2_from, want=want, **kw)
            yield tuple(shell)

    def last_nearest_stats(self):
        """ufo_b200_last_nearest_stats of the counting call of the last nearest()."""
        return self._near_stats.as_dict()

    def set_value_volume_bv(self, shape, occupancy, min_depth=0):
        """setValueVolume(BoundingVar, occupancy probability, min_depth) for one shape record."""
        bv = as_volume(shape)
        if len(bv) != 1:
            raise ValueError("set_value_volume_bv takes exactly one shape")
        self._check(self.lib.ufo_b200_set_value_volume_bv(self.h, bv.ctypes.data, float(occupancy), int(min_depth)))

    # -- bounded memory: retain / page out / page in ---------------------------
    def retain(self, volume=None, box=None):
        """Remove every brick the volume does not keep and give the memory back; returns the
        retain stats.  volume: see as_volume (None / []: keep everything); box = (min xyz, max xyz)
        instead of a volume: the AABB form."""
        st = RetainStats()
        if box is not None:
            b = self._box6(box)
            self._check(self.lib.ufo_b200_retain(self.h, b.ctypes.data, C.byref(st)))
        else:
            bv, bp, nb = self._bv(volume)
            self._check(self.lib.ufo_b200_retain_bv(self.h, bp, nb, C.byref(st)))
        return st.as_dict()

    def page_out(self, volume=None, box=None):
        """The bricks retain() would remove for the same volume, as a page blob (numpy uint8); the
        map is not changed."""
        bv, bp, nb = self._bv(aabb(*box) if box is not None else volume)
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_page_out_bv(self.h, bp, nb, None, 0, C.byref(n)))
        buf = np.empty(n.value, np.uint8)
        self._check(self.lib.ufo_b200_page_out_bv(self.h, bp, nb, buf.ctypes.data, len(buf), C.byref(n)))
        assert n.value == len(buf)
        return buf

    def page_in(self, blob):
        """Put the bricks of a page blob (bytes or numpy uint8) back; returns the stats."""
        buf = np.ascontiguousarray(np.frombuffer(blob, np.uint8))
        st = RetainStats()
        self._check(self.lib.ufo_b200_page_in(self.h, buf.ctypes.data if len(buf) else None, len(buf), C.byref(st)))
        return st.as_dict()

    def pool_stats(self):
        """Live bricks / upper nodes, pool capacities and device bytes of the map right now."""
        st = PoolCounts()
        self._check(self.lib.ufo_b200_pool_stats(self.h, C.byref(st)))
        return st.as_dict()

    def clone(self):
        """A new Map on the same device holding this map's content (ufo_b200_clone): sensor model,
        leaves, colours and everything derived; change detection, the change box, the early-stopping
        opt-in, profiling and a set stream start as on a new map."""
        h = C.c_void_p()
        self._check(self.lib.ufo_b200_clone(self.h, C.byref(h)))
        other = Map.__new__(Map)
        other.lib, other.h = self.lib, h
        other.color, other.resolution, other.depth_levels = self.color, self.resolution, self.depth_levels
        return other

    def tree_info(self):
        """The reference's counters and known box of the pruned tree (ufo_b200_tree_info): dict with
        num_leaf_nodes, num_inner_nodes, size, with_children (list by depth), known (bool), known_min,
        known_max (getKnownBBX()'s min / max; zeros when nothing is known) and ms_device."""
        st = TreeStats()
        self._check(self.lib.ufo_b200_tree_info(self.h, C.byref(st)))
        return dict(num_leaf_nodes=st.num_leaf_nodes, num_inner_nodes=st.num_inner_nodes,
                    size=st.num_leaf_nodes + st.num_inner_nodes, with_children=list(st.with_children),
                    known=bool(st.known), known_min=np.array(st.known_min[:]), known_max=np.array(st.known_max[:]),
                    ms_device=st.ms_device)

    # -- state ----------------------------------------------------------------
    def value_field(self, sort=True):
        """(codes sorted, occ f32, rgb u8[n,3]): every voxel with a non-default payload.
        sort=False returns them in the device's emission order."""
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_export_leaves(self.h, None, None, None, 0, C.byref(n)))
        cnt = n.value
        codes = np.empty(cnt, np.uint64)
        occ = np.empty(cnt, np.float32)
        rgb = np.zeros((cnt, 3), np.uint8)
        if cnt:
            self._check(self.lib.ufo_b200_export_leaves(
                self.h, codes.ctypes.data, occ.ctypes.data, rgb.ctypes.data if self.color else None,
                cnt, C.byref(n)))
            assert n.value == cnt
        if not sort:
            return codes, occ, rgb
        order = np.argsort(codes, kind="stable")
        return codes[order], occ[order], rgb[order]

    def value_field_count(self):
        """Number of voxels value_field() would return."""
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_export_leaves(self.h, None, None, None, 0, C.byref(n)))
        return int(n.value)

    def query(self, codes, depths):
        codes = np.ascontiguousarray(codes, dtype=np.uint64)
        depths = np.ascontiguousarray(np.broadcast_to(depths, codes.shape), dtype=np.uint32)
        n = len(codes)
        occ = np.empty(n, np.float32)
        flags = np.empty(n, np.uint8)
        rgb = np.zeros((n, 3), np.uint8)
        self._check(self.lib.ufo_b200_query(self.h, codes.ctypes.data, depths.ctypes.data, n,
                                            occ.ctypes.data, flags.ctypes.data,
                                            rgb.ctypes.data if self.color else None))
        return occ, flags, rgb

    def export_nodes(self, depth=0, occupied=True, free=True, unknown=False, box=None):
        """Filtered leaf iteration as a batch: (codes sorted, occ, rgb) of the depth-`depth` nodes
        whose state passes the filter and whose cube intersects box = (min xyz, max xyz)."""
        b = self._box6(box)
        bp = None if b is None else b.ctypes.data
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_export_nodes(self.h, int(depth), int(occupied), int(free), int(unknown), bp,
                                                   None, None, None, 0, C.byref(n)))
        cnt = n.value
        codes = np.empty(cnt, np.uint64)
        occ = np.empty(cnt, np.float32)
        rgb = np.zeros((cnt, 3), np.uint8)
        if cnt:
            self._check(self.lib.ufo_b200_export_nodes(self.h, int(depth), int(occupied), int(free), int(unknown), bp,
                                                       codes.ctypes.data, occ.ctypes.data,
                                                       rgb.ctypes.data if self.color else None, cnt, C.byref(n)))
        order = np.argsort(codes, kind="stable")
        return codes[order], occ[order], rgb[order]

    def cast_rays(self, origins, directions, ignore_unknown=False, max_range=-1.0, depth=0):
        """Batched castRay: (hit bool[n], code u64[n])."""
        o = np.ascontiguousarray(origins, dtype=np.float64).reshape(-1, 3)
        d = np.ascontiguousarray(directions, dtype=np.float64).reshape(-1, 3)
        assert o.shape == d.shape
        codes = np.zeros(len(o), np.uint64)
        hit = np.zeros(len(o), np.uint8)
        self._check(self.lib.ufo_b200_cast_rays(self.h, o.ctypes.data, d.ctypes.data, len(o), int(ignore_unknown),
                                                float(max_range), int(depth), codes.ctypes.data, hit.ctypes.data))
        return hit.astype(bool), codes

    # -- geometry -----------------------------------------------------------
    def compute_ray(self, origin, end, max_range=-1.0, depth=0):
        o = np.ascontiguousarray(origin, dtype=np.float64)
        e = np.ascontiguousarray(end, dtype=np.float64)
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_compute_ray(self.h, o.ctypes.data, e.ctypes.data,
                                                  float(max_range), int(depth), None, 0, C.byref(n)))
        out = np.empty(n.value, np.uint64)
        if n.value:
            self._check(self.lib.ufo_b200_compute_ray(self.h, o.ctypes.data, e.ctypes.data,
                                                      float(max_range), int(depth), out.ctypes.data,
                                                      n.value, C.byref(n)))
        return out

    def to_key(self, xyz, depth=0):
        p = np.ascontiguousarray(xyz, dtype=np.float64)
        k = np.empty(3, np.uint32)
        self._check(self.lib.ufo_b200_to_key(self.h, p.ctypes.data, int(depth), k.ctypes.data))
        return k

    def to_code(self, xyz, depth=0):
        p = np.ascontiguousarray(xyz, dtype=np.float64)
        c = C.c_uint64()
        self._check(self.lib.ufo_b200_to_code(self.h, p.ctypes.data, int(depth), C.byref(c)))
        return int(c.value)

    def key_to_code(self, key, depth=0):
        k = np.ascontiguousarray(key, dtype=np.uint32)
        return int(self.lib.ufo_b200_key_to_code(k.ctypes.data))

    def code_to_key(self, code, depth=0):
        k = np.empty(3, np.uint32)
        self.lib.ufo_b200_code_to_key(int(code), k.ctypes.data)
        return k

    def key_to_coord(self, key, depth=0):
        k = np.ascontiguousarray(key, dtype=np.uint32)
        p = np.empty(3, np.float64)
        self._check(self.lib.ufo_b200_key_to_coord(self.h, k.ctypes.data, int(depth), p.ctypes.data))
        return p

    def change_bbox(self):
        mn, mx = np.empty(3), np.empty(3)
        self._check(self.lib.ufo_b200_change_bbox(self.h, mn.ctypes.data, mx.ctypes.data))
        return mn, mx

    def enable_change_detection(self, enable=True):
        self._check(self.lib.ufo_b200_enable_change_detection(self.h, int(enable)))

    def reset_change_detection(self):
        self._check(self.lib.ufo_b200_reset_change_detection(self.h))

    def changed_codes(self, depth=0):
        """Sorted codes (at `depth`) of the nodes whose value changed since the last reset."""
        n = C.c_size_t()
        self._check(self.lib.ufo_b200_changed_codes(self.h, int(depth), None, 0, C.byref(n)))
        out = np.empty(n.value, np.uint64)
        if n.value:
            self._check(self.lib.ufo_b200_changed_codes(self.h, int(depth), out.ctypes.data, n.value, C.byref(n)))
        return np.sort(out[:n.value])

    def reset_change_bbox(self):
        self._check(self.lib.ufo_b200_reset_change_bbox(self.h))

    def sensor_model(self):
        out = np.empty(6)
        self._check(self.lib.ufo_b200_sensor_model_logit(self.h, out.ctypes.data))
        return out

    def set_sensor_model(self, occupied_thres=0.5, free_thres=0.5, prob_hit=0.7, prob_miss=0.4,
                         clamping_thres_min=0.1192, clamping_thres_max=0.971):
        p = np.array([occupied_thres, free_thres, prob_hit, prob_miss, clamping_thres_min,
                      clamping_thres_max], dtype=np.float64)
        self._check(self.lib.ufo_b200_set_sensor_model(self.h, p.ctypes.data))


def assemble_image(parts, with_header=True, compressed=False, acceleration=1, level=0):
    """The file image (with_header) or node stream of the union of image parts (Map.image_part,
    any order), on the host.  compressed: (bytes, uncompressed node-stream size) as
    Map.write_compressed_bv with data_only = not with_header; otherwise bytes."""
    lib = load()
    bufs = [np.ascontiguousarray(np.frombuffer(p, np.uint8)) for p in parts]
    ptrs = (C.c_void_p * max(len(bufs), 1))(*[b.ctypes.data for b in bufs])
    sizes = (C.c_size_t * max(len(bufs), 1))(*[len(b) for b in bufs])
    args = (ptrs, sizes, len(bufs), int(with_header), int(compressed), int(acceleration), int(level))
    n, u = C.c_size_t(), C.c_size_t()
    rc = lib.ufo_b200_image_assemble(*args, None, 0, C.byref(n), C.byref(u))
    if rc != OK:
        raise UfoError(rc, "ufo_b200_image_assemble failed")
    out = np.empty(max(n.value, 1), np.uint8)
    rc = lib.ufo_b200_image_assemble(*args, out.ctypes.data, n.value, C.byref(n), C.byref(u))
    if rc != OK:
        raise UfoError(rc, "ufo_b200_image_assemble failed")
    data = out[:n.value].tobytes()
    return (data, int(u.value)) if compressed else data


def page_info(blob):
    """Header of a page blob (no map needed): version, color, depth_levels, resolution, n_bricks and
    bytes, the size of the whole blob the header describes."""
    buf = np.ascontiguousarray(np.frombuffer(blob, np.uint8))
    h = PageHeader()
    rc = load().ufo_b200_page_info(buf.ctypes.data if len(buf) else None, len(buf), C.byref(h))
    if rc != OK:
        raise UfoError(rc, "not a page blob of this library's format version")
    return h.as_dict()


def page_keys(blob):
    """Brick coordinates (key >> 4 per axis) [n, 3] of the bricks a page blob holds, ascending by
    packed key."""
    n = page_info(blob)["n_bricks"]
    k = np.frombuffer(blob, np.uint8)[64:64 + 8 * n].view(np.uint64)
    m = np.uint64(0x1fffff)
    return np.stack([k & m, (k >> np.uint64(21)) & m, (k >> np.uint64(42)) & m], axis=1).astype(np.uint32)


def transform_points(frame_pose, xyz, dtype=np.float64):
    """Pose6::transform on the host (bit-identical to the device path)."""
    lib = load()
    buf, layout = pack_points(xyz, None, dtype)
    f = np.ascontiguousarray(frame_pose, dtype=np.float64)
    out = np.empty((len(buf), 3), np.float64)
    rc = lib.ufo_b200_transform_points(f.ctypes.data, buf.ctypes.data, len(buf), layout,
                                       out.ctypes.data)
    if rc != 0:
        raise RuntimeError("ufo_b200_transform_points failed: %d" % rc)
    return out


def pose_from_rpy(x, y, z, roll, pitch, yaw):
    """Pose6(x, y, z, roll, pitch, yaw) as (tx, ty, tz, qw, qx, qy, qz)."""
    lib = load()
    out = np.empty(7, np.float64)
    lib.ufo_b200_pose_from_rpy(float(x), float(y), float(z), float(roll), float(pitch), float(yaw),
                               out.ctypes.data)
    return out


def route_inbox_bytes(world, cap_bricks=1 << 16, cap_hits=1 << 18, color=False):
    """Device bytes of one rank's inbox (Map.route_setup with the same capacities); colour maps
    carry 16-byte hit records instead of 8."""
    lib = load()
    out = C.c_size_t()
    f = lib.ufo_b200_route_inbox_bytes_color if color else lib.ufo_b200_route_inbox_bytes
    rc = f(int(world), int(cap_bricks), int(cap_hits), C.byref(out))
    if rc != 0:
        raise UfoError(rc, "invalid routed-mode capacities")
    return out.value


def ipc_export(dev_ptr):
    """cudaIpcMemHandle (64 bytes) of a device allocation of this process."""
    lib = load()
    h = (C.c_ubyte * 64)()
    rc = lib.ufo_b200_ipc_export(C.c_void_p(dev_ptr), h)
    if rc != 0:
        raise UfoError(rc, "cudaIpcGetMemHandle failed")
    return bytes(h)


def ipc_open(handle):
    """Map another process's allocation; returns the device pointer (int) valid in this process."""
    lib = load()
    buf = (C.c_ubyte * 64).from_buffer_copy(handle)
    p = C.c_void_p()
    rc = lib.ufo_b200_ipc_open(buf, C.byref(p))
    if rc != 0:
        raise UfoError(rc, "cudaIpcOpenMemHandle failed")
    return p.value


def ipc_close(dev_ptr):
    """Unmap a pointer obtained from ipc_open."""
    lib = load()
    rc = lib.ufo_b200_ipc_close(C.c_void_p(dev_ptr))
    if rc != 0:
        raise UfoError(rc, "cudaIpcCloseMemHandle failed")
