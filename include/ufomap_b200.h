/* ufomap_b200.h -- C ABI of the H100-native UFOMap point-cloud integration path.
 *
 * The reference (UFOMap) has no FFI or plugin layer: its boundary for this path
 * is the C++ class API of libMap (ufo::map::OccupancyMap / OccupancyMapColor,
 * mostly header templates).  Each entry point below names the reference member
 * it stands in for (paths relative to /root/reference/ufomap/include/ufo/map/).
 * The source-compatible C++ facade in include/ufomap_b200/ufomap.hpp forwards to
 * these functions; INTEGRATION.md shows the binding a maintainer would add.
 *
 * Conventions: plain pointers and sizes only; every function returns a
 * ufo_b200_status (0 = OK) unless stated otherwise; a map is bound to one CUDA
 * device and one CUDA stream and is not thread-safe (same as the reference).
 * The library never falls back to a CPU implementation: without a usable
 * device ufo_b200_create fails with UFO_B200_E_CUDA.
 */
#ifndef UFOMAP_B200_H
#define UFOMAP_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ufo_b200_map ufo_b200_map;

typedef enum {
	UFO_B200_OK = 0,
	UFO_B200_E_INVALID = 1,     /* bad argument (e.g. depth_levels outside [2,21], octree.h:931-935) */
	UFO_B200_E_CUDA = 2,        /* CUDA runtime error; see ufo_b200_last_error() */
	UFO_B200_E_NOMEM = 3,       /* device pool could not grow */
	UFO_B200_E_UNSUPPORTED = 4  /* documented out-of-scope option (see DESIGN.md) */
} ufo_b200_status;

/* Point buffer layouts accepted by ufo_b200_insert_*: tightly packed AoS. */
typedef enum {
	UFO_B200_XYZ_F64 = 0,     /* double x,y,z             (PointCloud,      point_cloud.h:277) */
	UFO_B200_XYZ_F32 = 1,     /* float  x,y,z             (ROS PointCloud2 payload)            */
	UFO_B200_XYZRGB_F64 = 2,  /* double x,y,z + u8 r,g,b + 5 pad = 32 B (Point3Color, types.h:60-102) */
	UFO_B200_XYZRGB_F32 = 3   /* float  x,y,z + u8 r,g,b + 1 pad = 16 B                        */
} ufo_b200_layout;

/* Constructor arguments of OccupancyMap / OccupancyMapColor (occupancy_map.h:60-63,
 * occupancy_map_base.h:859-876) plus device-side sizing hints. */
typedef struct {
	double resolution;
	uint32_t depth_levels;       /* 2..21, default 16 */
	int32_t automatic_pruning;   /* accepted for API parity; pruning is representational only */
	double occupied_thres;       /* 0.5 */
	double free_thres;           /* 0.5 */
	double prob_hit;             /* 0.7 */
	double prob_miss;            /* 0.4 */
	double clamping_thres_min;   /* 0.1192 */
	double clamping_thres_max;   /* 0.971 */
	int32_t color;               /* 0: OccupancyMap, 1: OccupancyMapColor */
	int32_t device;              /* CUDA device ordinal, -1 = current, -2 = geometry-only handle
	                              * (host indexing / computeRay helpers only, no device state) */
	uint64_t initial_blocks;     /* capacity hint: 4^3-voxel blocks (0 = default) */
	uint64_t initial_bricks;     /* capacity hint: 16^3-voxel bricks (0 = default) */
} ufo_b200_params;

/* Fills *p with the reference's default constructor arguments. */
void ufo_b200_default_params(ufo_b200_params* p);

/* OccupancyMap::OccupancyMap(...)  occupancy_map.h:60-63 */
int ufo_b200_create(const ufo_b200_params* p, ufo_b200_map** out);
void ufo_b200_destroy(ufo_b200_map* m);
const char* ufo_b200_last_error(const ufo_b200_map* m);

/* Run all work of this map on an externally owned CUDA stream (cudaStream_t as
 * void*).  NULL restores the map's own stream. */
int ufo_b200_set_stream(ufo_b200_map* m, void* cuda_stream);

/* insertPointCloud          occupancy_map_base.h:270-327, occupancy_map_color.h:87-160
 * insertPointCloudDiscrete  occupancy_map_base.h:340-417, occupancy_map_color.h:177-267
 *
 * `points` is HOST memory holding n points in `layout`; it is copied before the
 * call returns (the reference takes the cloud by value).  max_range < 0 means
 * unlimited.  depth = insert depth of the free-space rays.  async != 0 returns
 * after the work is enqueued; ufo_b200_wait / ufo_b200_done mirror
 * insertPointCloudWait / insertPointCloudDone (occupancy_map_base.h:430-443).
 * early_stopping != 0 is order-dependent in the reference: it is rejected with
 * UFO_B200_E_UNSUPPORTED unless the map opted in with ufo_b200_set_early_stopping(m, 1),
 * which computes the reference's sequential result exactly (at the cost of extra device
 * work and memory; see ufo_b200_last_early_stats). */
int ufo_b200_insert_pointcloud(ufo_b200_map* m, const double origin[3], const void* points,
                               size_t n, int layout, double max_range, uint32_t depth,
                               int simple_ray_casting, uint32_t early_stopping, int discrete,
                               int async);

/* Same, but `points` is DEVICE memory on the map's device (no copy is made; the
 * buffer must stay valid until the call's work has finished). */
int ufo_b200_insert_device(ufo_b200_map* m, const double origin[3], const void* d_points,
                           size_t n, int layout, double max_range, uint32_t depth,
                           int simple_ray_casting, uint32_t early_stopping, int discrete,
                           int async);

/* insertPointCloud[Discrete](sensor_origin, cloud, frame_origin, ...) -- the overloads that
 * first move the cloud into the map frame (occupancy_map_base.h:313-327, 403-417;
 * occupancy_map_color.h:146-160, 253-267 -> PointCloudT::transform point_cloud.h:157-166 ->
 * Pose6::transform math/pose6.h:115-125).  frame_pose = {tx, ty, tz, qw, qx, qy, qz}.
 * The transform runs on the device while the points are read (bit-identical to the
 * reference's double arithmetic), so the raw sensor buffer crosses PCIe once. */
int ufo_b200_insert_pointcloud_frame(ufo_b200_map* m, const double origin[3], const void* points,
                                     size_t n, int layout, const double frame_pose[7],
                                     double max_range, uint32_t depth, int simple_ray_casting,
                                     uint32_t early_stopping, int discrete, int async);

/* A sensor_msgs/PointCloud2 buffer exactly as ROS delivers it: n = width*height records of
 * point_step bytes, x/y/z FLOAT32 fields at the given byte offsets, colour bytes at off_r/g/b
 * (for the usual packed "rgb" field at offset o: r = o+2, g = o+1, b = o; -1 = no colour).
 * Replaces rosToUfo (ufomap_ros/ufomap_ros/src/conversions.cpp:77-138): records with a NaN
 * coordinate are skipped, float32 is widened to double, on the device -- the raw buffer is the
 * only thing that crosses PCIe.  frame_pose may be NULL (cloud already in the map frame);
 * otherwise it is the transform the server applies next (server.cpp:116). */
typedef struct ufo_b200_cloud2 {
	const void* data;
	size_t n;
	uint32_t point_step;
	uint32_t off_x, off_y, off_z;
	int32_t off_r, off_g, off_b;
	int32_t on_device; /* != 0: data is device memory on the map's device */
} ufo_b200_cloud2;
int ufo_b200_insert_pointcloud2(ufo_b200_map* m, const double origin[3], const ufo_b200_cloud2* cloud,
                                const double* frame_pose, double max_range, uint32_t depth,
                                int simple_ray_casting, uint32_t early_stopping, int discrete, int async);

/* Host helpers (no device needed).  ufo_b200_transform_points: Pose6::transform of n points of
 * the given layout into out_xyz[n][3].  ufo_b200_pose_from_rpy: Pose6(x, y, z, roll, pitch,
 * yaw) math/pose6.h:71-74 with Quaternion(roll, pitch, yaw) math/quaternion.h:69-93. */
int ufo_b200_transform_points(const double frame_pose[7], const void* points, size_t n, int layout,
                              double* out_xyz);
int ufo_b200_pose_from_rpy(double x, double y, double z, double roll, double pitch, double yaw,
                           double frame_pose[7]);

int ufo_b200_wait(ufo_b200_map* m);           /* insertPointCloudWait */
int ufo_b200_done(ufo_b200_map* m, int* done); /* insertPointCloudDone; never blocks while device work is in flight (completes a scan that ran into a full pool once the device is idle) */

/* Octree::computeRay  octree.h:449-496 -- forward walk, origin voxel included,
 * end voxel excluded.  Writes up to cap codes, *n receives the full count. */
int ufo_b200_compute_ray(const ufo_b200_map* m, const double origin[3], const double end[3],
                         double max_range, uint32_t depth, uint64_t* codes, size_t cap, size_t* n);

/* Octree::toKey / toCode / toCoord  octree.h:299-394, Code <-> Key code.h:183-230 */
int ufo_b200_to_key(const ufo_b200_map* m, const double xyz[3], uint32_t depth, uint32_t key[3]);
int ufo_b200_to_code(const ufo_b200_map* m, const double xyz[3], uint32_t depth, uint64_t* code);
int ufo_b200_key_to_coord(const ufo_b200_map* m, const uint32_t key[3], uint32_t depth,
                          double xyz[3]);
uint64_t ufo_b200_key_to_code(const uint32_t key[3]);
void ufo_b200_code_to_key(uint64_t code, uint32_t key[3]);

/* Node state at (code, depth) with the INTENDED semantics of getOccupancy /
 * getColor / containsFree / containsUnknown (occupancy_map_base.h:599-728; the
 * reference's own Code-based getters read the depth-1 parent, octree.h:974-985).
 * logodds[i]: float log-odds (max over the subtree for depth > 0);
 * flags[i]: bit0 contains_free, bit1 contains_unknown; rgb: 3 bytes per query or NULL.
 * Host pointers. */
int ufo_b200_query(ufo_b200_map* m, const uint64_t* codes, const uint32_t* depths, size_t n,
                   float* logodds, uint8_t* flags, uint8_t* rgb);

/* Dump of the value field: every depth-0 voxel whose payload differs from the
 * default (log-odds 0, colour unset).  Call with codes == NULL to get the count
 * in *n; then with buffers of that capacity (host pointers; rgb may be NULL). */
int ufo_b200_export_leaves(ufo_b200_map* m, uint64_t* codes, float* logodds, uint8_t* rgb,
                           size_t cap, size_t* n);

/* setValueVolume(AABB, occupancy probability, min_depth)  occupancy_map_base.h:492-518 -- the
 * other map writer the mapping server uses (robot clearing server.cpp:152-154, clear_volume
 * service :354).  box6 = the AABB's centre xyz and half_size xyz (geometry/aabb.h:49-70).  Every
 * node of depth min_depth whose cube -- and every ancestor cube -- intersects the box is set to
 * clamp(float(logit(occupancy))) (setOccupancy, :1151-1157), i.e. all voxels below it.
 * min_depth 0..4; colour maps at min_depth 0 only (deeper, the reference also replaces the
 * voxels' colours by the node's mean colour).  On a routed map (ufo_b200_route_setup) every rank
 * takes the same call and sets the bricks it owns; the union of the ranks is the single map.
 * Between ufo_b200_route_mark and the last ufo_b200_route_apply of a pass: UFO_B200_E_INVALID,
 * nothing written.  A sharded map: UFO_B200_E_UNSUPPORTED. */
int ufo_b200_set_value_volume(ufo_b200_map* m, const double box6[6], double occupancy, uint32_t min_depth);

/* Per-node writes as one ordered batch, the same as making the calls one after the other in array
 * order (DESIGN.md section 8 states the semantics):
 *   op[i] = 0  ADD value[i] (float log-odds): updateValue(code, value)  occupancy_map_base.h:1063-1120
 *              -- integrateHit / integrateMiss :565-593 (value = float(prob_hit_log) / float(prob_miss_log)),
 *              updateOccupancy :544-559 (value = float(toLogit(p))).  Every voxel below the node at
 *              (codes[i], depths[i]) becomes clamp(v + value), one clamp per update.
 *   op[i] = 1  SET value[i]: setOccupancy :524-538 -> setNodeValue :1037-1057 as intended (the
 *              reference's does not compile): every voxel below the node becomes clamp(value).
 * depths[i] 0..6.  Host arrays.  Rejected as a whole (nothing applied): a code whose depth-0 key lies
 * outside the map (UFO_B200_E_INVALID); depth > 6, a sharded map, SET at depth > 0 on a colour map
 * (UFO_B200_E_UNSUPPORTED).  Leaf colours are not changed.  The min/max change box is not
 * updated (the reference does not update it for these calls); change detection records the voxels
 * whose value changed.  async != 0 returns after the work is enqueued.
 * Routed maps: every rank takes the same batch and applies it to the bricks it owns (a node of
 * depth 5/6 to its share of the node's bricks), so the union of the ranks is the single map; each
 * voxel's updates are applied in batch order by its one owner.  A batch between
 * ufo_b200_route_mark and the last ufo_b200_route_apply of a pass is UFO_B200_E_INVALID.  The
 * rejections above depend on the arguments and the map's parameters only, so they are the same
 * on every rank. */
int ufo_b200_update_nodes(ufo_b200_map* m, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                          const float* values, size_t n, int async);

/* ufo_b200_update_nodes plus the two writers of a colour map, as one ordered batch (DESIGN.md
 * section 8); rgb[n][3] (host array) holds the colour of entry i, read for ops 2 and 3 only:
 *   op[i] = 0, 1  as ufo_b200_update_nodes; the colour is left as it is.
 *   op[i] = 2     ADD_COLOR: OccupancyMapColor::updateValue(code, value, Color(rgb))
 *                 occupancy_map_color.h:269-287 -- the voxel's colour blends towards rgb
 *                 (updateNodeColor, occupancy_map_color.cpp:142-171) weighted by toProb(value)
 *                 against toProb of the log-odds the batch's earlier entries left, then the
 *                 log-odds becomes clamp(v + value).  An unset colour takes rgb; rgb (0,0,0)
 *                 onto a set colour blends towards black.
 *   op[i] = 3     SET_COLOR: setColor(code, Color(rgb))  occupancy_map_color.cpp:74-81 -- the
 *                 voxel's colour becomes rgb ((0,0,0) unsets it); the log-odds is unchanged.
 * Ops 2 and 3 create the voxel like createNode does, and the inner colours up to the root are
 * recomputed after the batch.  Change detection records a voxel when an ADD_COLOR changed its
 * log-odds, never for SET_COLOR; the min/max change box is not updated.  Rejected as a whole,
 * before anything is applied: op > 3, ops 2 / 3 on a map without colour, rgb == NULL while the
 * batch holds op 2 or 3, a code outside the map (UFO_B200_E_INVALID); ops 2 / 3 at depth > 0 (the
 * reference's result depends on whether the node has children) and everything
 * ufo_b200_update_nodes rejects with UFO_B200_E_UNSUPPORTED.  These checks need no device. */
int ufo_b200_update_nodes_color(ufo_b200_map* m, const uint64_t* codes, const uint32_t* depths,
                                const uint8_t* ops, const float* values, const uint8_t* rgb, size_t n,
                                int async);

/* insertMissOnRay (hit_end = 0) / insertRay (hit_end = 1)  occupancy_map_base.h:251-268 for n rays,
 * origins / ends [n][3] (host arrays): integrateMiss on every node computeRay (octree.h:449-496, as
 * ufo_b200_compute_ray) walks at `depth`, then with hit_end integrateHit on the depth-0 voxel of the
 * GIVEN end point (not the one max_range truncates to).  Rays are applied in array order.  Rejected
 * as a whole: an origin or end outside the map (UFO_B200_E_INVALID); depth > 6, sharded maps
 * (UFO_B200_E_UNSUPPORTED).  Routed maps as ufo_b200_update_nodes: every rank walks every ray and
 * applies the nodes whose bricks it owns, the hit_end voxel included. */
int ufo_b200_insert_rays(ufo_b200_map* m, const double* origins, const double* ends, size_t n,
                         double max_range, uint32_t depth, int hit_end, int async);

/* Octree::write(std::ostream& / filename, bounding_volume, compress = false, min_depth)
 * (octree.h:776-864, writeNodes occupancy_map_base.h:1457-1533): the map as a UFOMap file image
 * -- text header, then the pre-order node stream -- which the reference's Octree::read / the RViz
 * plugin parse; the save_map service of the mapping server (server.cpp:381-392).  box6 (NULL =
 * whole map) and min_depth as for ufo_b200_write_data below.
 * expanded = 0: the canonical tree of the map's value field (a node whose eight children are
 * leaves with equal payload is a leaf).  The reference collapses such nodes itself (updateNode,
 * occupancy_map_base.h:1210-1212 -- logically even with automatic pruning off,
 * octree.h:1060-1066), so this is byte-identical to its own file unless its update order left a
 * collapsible node behind (updateParents stops at the first unchanged aggregate, :1126-1133);
 * then the two files differ in shape only and read back to the same map.  expanded != 0: every
 * octet that was ever touched is written as eight voxels (value-equivalent, larger).
 * ufo_b200_write: *size receives the image size; the image is copied when it fits into cap
 * (call with buf = NULL to size the buffer).  No LZ4. */
int ufo_b200_write(ufo_b200_map* m, const double* box6, uint32_t min_depth, int expanded, void* buf, size_t cap,
                   size_t* size);
int ufo_b200_write_file(ufo_b200_map* m, const char* filename, const double* box6, uint32_t min_depth,
                        int expanded);

/* Octree::writeData(stream, bounding_volume, compress = false, min_depth) (octree.h:885-917): the
 * node stream alone, as ufoToMsg puts it into a UFOMap message
 * (ufomap_ros/ufomap_msgs/include/ufomap_msgs/conversions.h:161-185; the mapping server publishes
 * the changed region at depths 0..publish_depth this way, server.cpp:184-199).  box6 = the
 * fields of a ufo::geometry::AABB: centre xyz, half_size xyz (geometry/aabb.h:49-70; for
 * AABB(min, max) that is half = (max - min) / 2, centre = min + half) or NULL for the whole map:
 * children whose cube misses the box are skipped (intersects(AABB, AABB),
 * collision_checks.cpp:256-264).  Children at min_depth are written as leaves carrying their aggregate
 * (max occupancy, mean colour); min_depth 0..4 is supported.  Canonical tree, see above.
 * *size = 0 when the box misses the map (the reference writes nothing then). */
int ufo_b200_write_data(ufo_b200_map* m, const double* box6, uint32_t min_depth, void* buf, size_t cap,
                        size_t* size);

/* castRay  occupancy_map_base.h:449-486, batched.  The reference's own version does not compile
 * (SURVEY.md G5); this is its intent (DESIGN.md section 8 states it; the CPU checker restates it): max_range < 0 -> the map's
 * diagonal; the ray origin + t * direction, clipped into the map, is walked forward at `depth`;
 * the first occupied node is the hit (hit[i] = 1, codes[i] = its Code), an unknown node ends the
 * ray unless ignore_unknown.  Node state follows the intended getNode semantics of ufo_b200_query. */
int ufo_b200_cast_rays(ufo_b200_map* m, const double* origins, const double* directions, size_t n,
                       int ignore_unknown, double max_range, uint32_t depth, uint64_t* codes, uint8_t* hit);

/* Leaf iteration with state and bounding-volume filters (beginLeaves(occupied, free, unknown,
 * contains = false, min_depth) and its bounding-volume form, occupancy_map_base.h:130-216; validity
 * rule iterator/occupancy_map.h:168-207), as a batch: every node of depth `depth` in the known
 * space whose own state passes the filter (occupied: value > occupied threshold; free: value <
 * free threshold; unknown: in between; an inner node carries the maximum of its subtree) and whose
 * cube intersects the AABB box6 (centre, half size; NULL: everywhere).  codes carry the depth's
 * centre bits; unordered.  A leaf the reference keeps collapsed above `depth` appears as its
 * depth-`depth` cells.  codes == NULL: count only. */
int ufo_b200_export_nodes(ufo_b200_map* m, uint32_t depth, int occupied, int free_space, int unknown, const double* box6,
                          uint64_t* codes, float* logodds, uint8_t* rgb, size_t cap, size_t* n);

/* Octree::write / writeData with compress = true (octree.h:812-917, :1428-1456): the node stream
 * as one LZ4 block (LZ4_compress_fast with acceleration_level when compression_level <= 0, else
 * LZ4_compress_HC), behind the text header with "compressed 1" unless data_only.  liblz4.so.1 is
 * loaded at run time, like the reference links it; UFO_B200_E_UNSUPPORTED if it is absent.
 * *uncompressed_size = what the header's uncompressed_data_size says (writeData's return value). */
int ufo_b200_write_compressed(ufo_b200_map* m, const double* box6, uint32_t min_depth, int data_only,
                              int acceleration_level, int compression_level, void* buf, size_t cap, size_t* size,
                              size_t* uncompressed_size);

/* Octree::readData (octree.h:733-770 -> readNodes, occupancy_map_base.h:1379-1456): merges a node
 * stream -- the body of a UFOMap file, or a UFOMap message the way the ROS layer applies it
 * (msgToUfo, ufomap_msgs/conversions.h:122-134) -- into the map: every leaf of the stream sets all
 * voxels below it to its payload, nodes whose cube misses the AABB box6 (centre, half size; NULL:
 * none) are skipped exactly like the writer skipped them.  The stream must have been written for
 * this map's resolution / depth_levels (the reference clears and resizes otherwise: call
 * ufo_b200_clear_resize first).  compressed != 0: `data` is one LZ4 block of uncompressed_size
 * bytes.  A collapsed non-default node above the brick level is expanded into bricks (at most 2^20
 * per call, else UFO_B200_E_UNSUPPORTED).
 * Routed maps (ufo_b200_route_setup): every rank takes the same call -- stream, box or volume,
 * compressed flag and sizes -- and applies the part of the stream that falls in the bricks it owns;
 * it creates no brick another rank owns.  The union of the ranks equals one map that read the same
 * stream after the same history, and ufo_b200_image_part_bv / ufo_b200_image_assemble of the ranks
 * give that map's image, so a map written by any number of ranks (or by one map) loads onto any
 * number of ranks.  The 2^20 limit counts every brick of a node, owned or not.  Every rejection --
 * a call between ufo_b200_route_mark and the last ufo_b200_route_apply of a pass, a truncated
 * stream, a failed decompression, an invalid volume (UFO_B200_E_INVALID), depth_levels < 5 or the
 * 2^20 limit (UFO_B200_E_UNSUPPORTED) -- is decided from the arguments before any device work, so
 * every rank returns the same status and none changes.  Pools grow as on one map.  Sharded maps
 * (ufo_b200_set_shard): UFO_B200_E_UNSUPPORTED. */
int ufo_b200_read_data(ufo_b200_map* m, const double* box6, const void* data, size_t size, int compressed,
                       size_t uncompressed_size);

/* The text header of a UFOMap file image (Octree::readHeader, octree.h:1338-1417).  Layout, 96 bytes:
 *   offset  0  char version[32]                 the version token, NUL-terminated (first 31 bytes)
 *   offset 32  char id[32]                      the id token (tree type), NUL-terminated (first 31 bytes)
 *   offset 64  double resolution
 *   offset 72  uint32_t depth_levels
 *   offset 76  int32_t compressed               0 or 1
 *   offset 80  int64_t uncompressed_data_size   -1 when the header has none
 *   offset 88  uint64_t data_offset             the byte offset of the node stream in the image; 0
 *                                               when no "data" line was found */
typedef struct {
	char version[32];
	char id[32];
	double resolution;
	uint32_t depth_levels;
	int32_t compressed;
	int64_t uncompressed_data_size;
	uint64_t data_offset;
} ufo_b200_file_header;

/* Octree::readHeader on an image (the whole file, or any prefix that holds its header); needs no
 * map and no device.  The first line must start with "# UFOMap file"; then whitespace-separated
 * tokens: a token starting with '#' and an unknown token skip to the end of their line, "data" ends
 * the header at the end of its line, and version, id, resolution, depth_levels, compressed (0 or 1)
 * and uncompressed_data_size take the token after them, numbers as an istream reads them.
 * UFO_B200_E_INVALID, as the reference returns false: a first line without the file mark, no "data"
 * line, an empty version or id, resolution <= 0, depth_levels 0, a negative or missing
 * uncompressed_data_size, or a value the stream cannot read.  *out holds what was read either way:
 * its id is what Octree::readType returns (empty when the first line is not the file mark). */
int ufo_b200_read_header(const void* image, size_t size, ufo_b200_file_header* out);

/* Octree::read (octree.h:690-729) of a file image -- header, then the node stream -- or of the file
 * `filename`.  The header's id must be the map's tree type ("occupancy_map" / "occupancy_map_color",
 * as the writers put it).  A file of another resolution or depth_levels re-creates the map with the
 * file's (ufo_b200_clear_resize), as the reference's readData does (octree.h:760-762); a file of the
 * same geometry merges into the map like ufo_b200_read_data.  A compressed file ("compressed 1") is
 * one LZ4 block, decompressed once (the reference decompresses it a second time and so cannot read
 * its own compressed files, DESIGN.md section 7).  Every rejection is decided before the map is
 * touched, so a rejected call changes nothing (the reference clears the map before it parses):
 * an invalid header, a tree type other than the map's, depth_levels above 21 (UFO_B200_E_INVALID);
 * depth_levels < 5 (UFO_B200_E_UNSUPPORTED); a file that cannot be opened or read, a failed
 * decompression, a truncated stream (UFO_B200_E_INVALID); the limits of ufo_b200_read_data.
 * Routed maps: every rank takes the same call as for ufo_b200_read_data; a file whose geometry
 * differs from the map's is refused on every rank (UFO_B200_E_UNSUPPORTED), since a rank cannot
 * re-create a routed map on its own. */
int ufo_b200_read(ufo_b200_map* m, const void* image, size_t size);
int ufo_b200_read_file(ufo_b200_map* m, const char* filename);

/* Bounding volumes (ufo::geometry::BoundingVolume, geometry/bounding_volume.h): a union of shapes,
 * each one ufo_b200_volume.  type follows the order of ufo::geometry::BoundingVar
 * (geometry/types.h); v holds the shape's members as the reference stores them:
 *   0 AABB         centre xyz, half_size xyz
 *   1 Frustum      six planes (top, bottom, left, right, near, far), each normal xyz, distance
 *   2 LineSegment  start xyz, end xyz
 *   3 OBB          centre xyz, half_size xyz, rotation w x y z
 *   4 Plane        normal xyz, distance
 *   5 Point        xyz
 *   6 Ray          origin xyz, direction xyz (already normalised, as the Ray constructor leaves it)
 *   7 Sphere       centre xyz, radius
 * A node's cube passes a shape as intersects(AABB, shape) of collision_checks.cpp:53-356 decides,
 * bit for bit; it passes the volume if it passes any of its shapes.  A node is inside the filter
 * iff every cube on its path from the root down passes (the reference's recursions and iterator
 * decide this way).  n_bv == 0: the whole map.  An unknown type: UFO_B200_E_INVALID.  reserved is
 * ignored (set it to 0).
 * Each *_bv entry point is its box6 twin with the volume in place of the AABB; the box6 forms are
 * the *_bv forms with one AABB record.  ufo_b200_set_value_volume_bv takes routed maps like
 * ufo_b200_set_value_volume: the descent is the same on every rank, each sets the bricks it owns. */
#define UFO_B200_VOLUME_AABB 0
#define UFO_B200_VOLUME_FRUSTUM 1
#define UFO_B200_VOLUME_LINE_SEGMENT 2
#define UFO_B200_VOLUME_OBB 3
#define UFO_B200_VOLUME_PLANE 4
#define UFO_B200_VOLUME_POINT 5
#define UFO_B200_VOLUME_RAY 6
#define UFO_B200_VOLUME_SPHERE 7
typedef struct {
	uint32_t type;
	uint32_t reserved;
	double v[24];
} ufo_b200_volume;

int ufo_b200_write_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, uint32_t min_depth, int expanded,
                      void* buf, size_t cap, size_t* size);
int ufo_b200_write_data_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, uint32_t min_depth, void* buf,
                           size_t cap, size_t* size);
int ufo_b200_write_compressed_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, uint32_t min_depth,
                                 int data_only, int acceleration_level, int compression_level, void* buf, size_t cap,
                                 size_t* size, size_t* uncompressed_size);
int ufo_b200_read_data_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, const void* data, size_t size,
                          int compressed, size_t uncompressed_size);
/* One file image from several maps that hold disjoint bricks -- the ranks of a routed map.  Every
 * level above the 16^3-voxel bricks of an image is a function of the bricks' own shapes and
 * payloads, so the image of the union is assembled from one part per rank:
 *   ufo_b200_image_part_bv  this map's part of the image for (bv[n_bv], min_depth, expanded), as
 *                           ufo_b200_write_bv would write it: an opaque, versioned blob holding
 *                           those arguments, the map's resolution, depth_levels and colour mode,
 *                           and per brick of the tree its code, shape and node stream.  *size =
 *                           the blob's bytes; copied when it fits into cap (buf = NULL sizes it).
 *                           Waits for a pending scan; between ufo_b200_route_mark and the last
 *                           ufo_b200_route_apply of a pass UFO_B200_E_INVALID.  Other rejections
 *                           as ufo_b200_write_bv.
 *   ufo_b200_image_assemble the image of the union of parts[0..n_parts) (sizes[i] bytes each, host
 *                           memory, any order) on the host; no map or device needed.  with_header:
 *                           the file image (ufo_b200_write_bv), else the bare node stream
 *                           (ufo_b200_write_data_bv); compress: the stream as one LZ4 block, as
 *                           ufo_b200_write_compressed_bv (data_only = !with_header), with
 *                           acceleration_level / compression_level as there.  *uncompressed_size
 *                           (may be NULL) = bytes of the node stream.  *size = the image's bytes;
 *                           copied only when it fits into cap.  UFO_B200_E_INVALID: no parts, a
 *                           truncated or malformed part, parts that differ in resolution,
 *                           depth_levels, colour, volume, min_depth or expanded, a brick in two
 *                           parts (two histories of one brick; also the same part given twice).
 * A single map's writers are its own part assembled alone, so assembling the ranks' parts gives
 * the bytes one map holding the union would write.  The parts travel however the caller's ranks
 * talk (e.g. an all-gather of byte tensors); for a change-box publish take the min / max of the
 * ranks' ufo_b200_change_bbox first and ask every rank for the part of that box. */
int ufo_b200_image_part_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, uint32_t min_depth, int expanded,
                           void* buf, size_t cap, size_t* size);
int ufo_b200_image_assemble(const void* const* parts, const size_t* sizes, size_t n_parts, int with_header, int compress,
                            int acceleration_level, int compression_level, void* buf, size_t cap, size_t* size,
                            size_t* uncompressed_size);
/* Leaf iteration as ufo_b200_export_nodes, with the reference iterator's rule: a node is returned
 * iff every cube on its path from the root passes the volume (ufo_b200_export_nodes tests the
 * node's own cube only). */
int ufo_b200_export_nodes_bv(ufo_b200_map* m, uint32_t depth, int occupied, int free_space, int unknown,
                             const ufo_b200_volume* bv, size_t n_bv, uint64_t* codes, float* logodds, uint8_t* rgb,
                             size_t cap, size_t* n);
/* Iteration: beginLeaves (leaves_only != 0) / beginTree (occupancy_map_base.h:93-163) with the
 * filters occupied / free_space / unknown / contains and min_depth, over the bounding volume bv[n_bv]
 * (n_bv == 0: the whole map).  The nodes come in the reference iterator's order (pre-order, children
 * 0..7) over the canonical tree of the file writer (a node whose eight children are leaves with equal
 * payload is a leaf; untouched space is a default leaf):
 *   codes[i]   the node's Code as the iterator builds it (Code::getChild from the root: the bits
 *              below 3 * depth are zero)
 *   depths[i]  its depth, 0..depth_levels
 *   logodds[i] a leaf's value, an inner node's aggregate (max over the subtree) -- ufo_b200_query's
 *   flags[i]   bit0 contains_free, bit1 contains_unknown (as ufo_b200_query), bit2 isLeaf
 *   rgb        3 bytes per node or NULL
 * *n is always the number of nodes; the arrays (host memory) are filled when it is <= cap.
 * min_depth > depth_levels, or a volume that misses the root: no nodes.  Waits for a pending scan.
 * depth_levels < 5 is UFO_B200_E_UNSUPPORTED; an unknown volume type UFO_B200_E_INVALID.  A sharded
 * or routed map iterates the part its own rank holds. */
int ufo_b200_iterate(ufo_b200_map* m, int leaves_only, int occupied, int free_space, int unknown, int contains,
                     uint32_t min_depth, const ufo_b200_volume* bv, size_t n_bv, uint64_t* codes, uint8_t* depths,
                     float* logodds, uint8_t* flags, uint8_t* rgb, size_t cap, size_t* n);
/* setValueVolume(BoundingVar, occupancy, min_depth) for one shape (the mapping server loops over the
 * shapes of a volume, server.cpp:345-354).  The bricks whose path passes are found by a descent on
 * the device, one level per kernel; more than 2^22 nodes at any level of it is UFO_B200_E_UNSUPPORTED
 * before anything is written.  Otherwise as ufo_b200_set_value_volume. */
int ufo_b200_set_value_volume_bv(ufo_b200_map* m, const ufo_b200_volume* bv, double occupancy, uint32_t min_depth);
/* The node-vs-volume predicate on the host (the code the kernels run): out[i] = 1 iff the cube of
 * centre centres[i] and half size half_sizes[i] (per axis; the node cubes of a map have three equal
 * ones) passes the volume.  No map needed. */
int ufo_b200_volume_intersects(const ufo_b200_volume* bv, size_t n_bv, const double* centres, const double* half_sizes,
                               size_t n, uint8_t* out);

/* Shape constructors whose arithmetic decides a shape's doubles, on the host in the library (no FMA
 * contraction, whatever flags the caller compiles with), as the facade's geometry types use them:
 *   ufo_b200_geometry_frustum: Frustum(pos, target, up, vertical_angle, horizontal_angle, near, far)
 *     (geometry/frustum.h) -> planes[24] = 6 x (normal xyz, distance), top bottom left right near far
 *   ufo_b200_geometry_plane:   Plane(v1, v2, v3) (geometry/plane.h) -> plane[4] = normal xyz, distance
 *   ufo_b200_geometry_ray:     Ray(origin, direction) (geometry/ray.h) -> ray[6] = origin, direction
 *     divided by its norm */
int ufo_b200_geometry_frustum(const double pos[3], const double target[3], const double up[3], double vertical_angle,
                              double horizontal_angle, double near_distance, double far_distance, double planes[24]);
int ufo_b200_geometry_plane(const double v1[3], const double v2[3], const double v3[3], double plane[4]);
int ufo_b200_geometry_ray(const double origin[3], const double direction[3], double ray[6]);

/* Sensor model  occupancy_map_base.h:734-773.  out6/in: occupied_thres,
 * free_thres, prob_hit, prob_miss, clamping_thres_min, clamping_thres_max as
 * probabilities (setters) or as stored double log-odds (ufo_b200_sensor_model_logit). */
int ufo_b200_set_sensor_model(ufo_b200_map* m, const double prob6[6]);
/* One sensor-model parameter, the way the reference's setters work (occupancy_map_base.h:748-773:
 * setProbHit / setProbMiss / setClampingThresMin / setClampingThresMax / setOccupiedFreeThres each
 * store toLogit(p) into ONE member and leave the others' stored log-odds untouched).
 * index: 0 occupied_thres, 1 free_thres, 2 prob_hit, 3 prob_miss, 4 clamping_thres_min,
 * 5 clamping_thres_max.  Changing a threshold (0, 1) re-derives the contains_free /
 * contains_unknown flags of every inner node, like the reference's write + read round trip. */
int ufo_b200_set_sensor_model_field(ufo_b200_map* m, int index, double probability);
int ufo_b200_sensor_model_logit(const ufo_b200_map* m, double logit6[6]);

/* min/max change detection  occupancy_map_base.h:792-822 (always enabled). */
int ufo_b200_change_bbox(ufo_b200_map* m, double min_change[3], double max_change[3]);
int ufo_b200_reset_change_bbox(ufo_b200_map* m);

/* Change detection  occupancy_map_base.h:779-790 (enableChangeDetection / resetChangeDetection /
 * changesBegin..changesEnd / numChangedDetected): the set of nodes whose occupancy value changed
 * since the last reset (updateOccupancy returned true, :1070, :1094, :1106).  Recorded per voxel on
 * the device; ufo_b200_changed_codes returns the set at `depth` -- the insert depth the caller
 * used, 0 for the server's default -- as Code values (with the centre bits a Code built from a
 * depth-d Key carries), unordered like the reference's CodeSet.  codes == NULL: count only. */
int ufo_b200_enable_change_detection(ufo_b200_map* m, int enable);
int ufo_b200_reset_change_detection(ufo_b200_map* m);
int ufo_b200_changed_codes(ufo_b200_map* m, uint32_t depth, uint64_t* codes, size_t cap, size_t* n);

/* Counters and timings of the most recent insert (waits for it to finish). */
typedef struct {
	uint64_t points;          /* N                                         */
	uint64_t rays;            /* rays cast                                 */
	uint64_t visits;          /* V: voxel visits of the ray walk (only when profiling) */
	uint64_t touched_voxels;  /* U: unique voxels that received an update  */
	uint64_t hit_voxels;      /* U_h                                       */
	uint64_t touched_octets;  /* D_1                                       */
	uint64_t touched_blocks;  /* D_2 (4^3 blocks)                          */
	uint64_t touched_d3;      /* D_3 (8^3 nodes)                           */
	uint64_t touched_bricks;  /* D_4 (16^3 bricks)                         */
	uint64_t upper_nodes;     /* sum of D_l, l >= 5                        */
	uint64_t blocks_in_map;   /* pool occupancy                            */
	uint64_t bricks_in_map;
	uint64_t device_bytes;    /* device memory held by the map             */
	uint64_t regrows;         /* pool growth events during this insert (routed: mark and apply phases of the pass) */
	uint64_t launches;        /* kernels launched by this insert           */
	uint64_t result_bytes;    /* bytes of per-scan counters copied device -> host by this insert */
	uint64_t touched_lines;   /* 128-byte lines of leaf data the update read (HBM moves whole lines): lines holding a touched octet, less saturated lines (ufo_b200_last_update_stats) */
	float ms_total;           /* CUDA-event time of the whole insert (device work) */
	float ms_h2d;
	float ms_points;          /* K1: discretise + hit marking              */
	float ms_rays;            /* K2: ray walk (k_rays)                     */
	float ms_scatter;         /* K2b: record lookup + mask marking (k_scatter) */
	float ms_update;          /* K3: leaf log-odds update + in-block aggregates */
	float ms_propagate;       /* K4: brick + upper-level aggregates        */
} ufo_b200_scan_stats;

int ufo_b200_last_scan_stats(ufo_b200_map* m, ufo_b200_scan_stats* out);
/* Statistics of the most recent scan whose integration is COMPLETE, without waiting for the scan
 * in flight: after an async insert of scan k this returns scan k-1 (its counters were read back
 * when scan k was enqueued).  For callers that stream scans with async = 1 and still want each
 * scan's result.  points == 0 in *out: no scan has completed yet. */
int ufo_b200_completed_scan_stats(ufo_b200_map* m, ufo_b200_scan_stats* out);

/* What the fused ray walk sent to the dense scan volume in the most recent insert (waits for it
 * to finish).  Counted at profiling level 2 only; all zero otherwise, and for scans that took
 * another marking path (generic record path, brick-hash probes, routed passes without a volume). */
typedef struct {
	uint64_t records;          /* block records pushed: a ray segment left a 4^3 block or ended */
	uint64_t mask_reductions;  /* global 64-bit OR reductions on block masks (records merged per word first) */
	uint64_t words_marked;     /* of those, the ones that found the word empty: distinct words the walk marked */
	uint64_t dirty_reductions; /* reductions on the bitmap of touched bricks */
} ufo_b200_walk_stats;
int ufo_b200_last_walk_stats(ufo_b200_map* m, ufo_b200_walk_stats* out);

/* What the leaf update of the most recent insert left out (waits for it to finish).  Counted at
 * profiling level 2 only; all zero otherwise, and always zero on colour maps, which read and write
 * every touched line.  A saturated line is a 128 B leaf line of four initialised octets that the
 * scan only marked free and whose 32 voxels already sit at clamping_thres_min: the update would
 * not change it, so it is neither read nor written. */
typedef struct {
	uint64_t saturated_octets; /* touched octets in saturated lines (part of touched_octets)          */
	uint64_t saturated_lines;  /* saturated lines with touched voxels: not read                        */
	uint64_t clean_sectors;    /* 32 B leaf sectors read and updated but left unchanged: not written back */
} ufo_b200_update_stats;
int ufo_b200_last_update_stats(ufo_b200_map* m, ufo_b200_update_stats* out);

/* Early stopping.  On the CPU, early_stopping = E > 0 makes a scan cheaper: a ray stops after E
 * nodes in a row that earlier rays (or its own earlier samples) already put into the scan's free
 * set.  The result depends on the order of the rays.  Here it costs more than a plain scan: every
 * ray's walk is stored and the prefixes are solved in parallel rounds until they reach the
 * reference's sequential answer.  So a map rejects early_stopping != 0 (UFO_B200_E_UNSUPPORTED)
 * until the caller opts in with exact = 1; exact = 0 restores the rejection.  Any other value:
 * UFO_B200_E_INVALID.  Needs no device.  Routed passes keep rejecting early_stopping. */
int ufo_b200_set_early_stopping(ufo_b200_map* m, int exact);

/* The most recent insert's early-stopping work (waits for it to finish); all zero when that
 * insert did not use early stopping.  The times are CUDA events at profiling level >= 1. */
typedef struct {
	uint64_t rounds;      /* rounds of the prefix solver, the last one without a change included */
	uint64_t converged;   /* 1: the rounds reached their fixed point                    */
	uint64_t visits;      /* node visits of all walks                                  */
	uint64_t nodes;       /* distinct nodes the walks visit                            */
	uint64_t free_nodes;  /* nodes in the scan's free set                              */
	uint64_t table_bytes; /* device memory of the scan-local node table                */
	uint64_t id_bytes;    /* device memory of the visit ids and per-ray arrays         */
	float ms_walk;        /* E1: walks, node ids                                       */
	float ms_rounds;      /* E2: prefix rounds                                         */
	float ms_mark;        /* E3: free set -> miss masks                                */
} ufo_b200_early_stats;
int ufo_b200_last_early_stats(ufo_b200_map* m, ufo_b200_early_stats* out);

/* Octree::clear(resolution, depth_levels)  octree.h:541-560 -- the server's reset service
 * (server.cpp:364-378): empties the map and changes its geometry. */
int ufo_b200_clear_resize(ufo_b200_map* m, double resolution, uint32_t depth_levels);

/* 0: off; 1: per-kernel CUDA-event timing; 2: additionally count ray-walk visits
 * (one extra atomic per ray). */
int ufo_b200_set_profiling(ufo_b200_map* m, int enable);

/* Spatial sharding over several GPUs (SURVEY.md 8(e), variant 1): every rank is given the same
 * scans (broadcast) and keeps only the bricks (16^3-voxel nodes) it owns -- ownership is a hash of
 * the brick key, so the touched space splits evenly wherever the sensor is.  The union of the
 * ranks' value fields is the single-GPU map; no state is exchanged.  Aggregates of depth >= 5 are
 * per rank (partial) in this mode.  Must be called on an empty map.  world <= 1 turns it off. */
int ufo_b200_set_shard(ufo_b200_map* m, uint32_t rank, uint32_t world);

/* Routed multi-GPU mode (SURVEY.md 8(e), variant 2; BASELINE configs #4 "octant shard" and #5
 * "one GPU per sensor with boundary merge").  The reference integrates on one thread
 * (occupancy_map_base.h:270-327); this is the multi-GPU form of the same insertPointCloud:
 * state is owned by space (rank = hash of the 16^3-voxel brick key, as in ufo_b200_set_shard),
 * marking is parallel over rays.  Every rank walks ITS rays -- a slice of one scan, or its own
 * sensor's scan -- and the per-brick free-space masks / hit voxels of bricks another rank owns
 * are written straight into that rank's inbox over NVLink peer memory; the only collective is a
 * barrier between the two calls below (the caller's: e.g. a 4-byte NCCL all-reduce on the map's
 * stream).  Every option of ufo_b200_insert_pointcloud except early_stopping: mono and colour
 * maps, discrete insertion, insert depth 0..6, simple_ray_casting (ufo_b200_route_mark_ex).
 *
 *   ufo_b200_route_setup    allocates this rank's inbox (cap_bricks brick records and cap_hits hit
 *                           records per source rank and parity) and returns its device pointer.
 *                           Colour maps use 16-byte hit records (voxel key, global cloud index,
 *                           rgb): ufo_b200_route_inbox_bytes_color gives their inbox size.  A hit
 *                           record is also what carries a whole brick below an insert-depth-5/6
 *                           free-space node
 *   ufo_b200_ipc_export/_open   cudaIpc handle of that pointer / mapping of a peer's handle, for
 *                           one-process-per-GPU launches (handles travel through the caller's
 *                           control plane, e.g. torch.distributed.all_gather_object)
 *   ufo_b200_route_connect  peer_inboxes[r] = device pointer of rank r's inbox as seen from this
 *                           process (its own for r == rank)
 *   ufo_b200_route_mark     H2D, K1, fused walk, then a wait for the marking kernels: if a pool ran
 *                           full, it grows and the marking runs again before anything is
 *                           published; then enqueues the forwarding of foreign marks.  self_too != 0:
 *                           the rank's own marks go through its inbox as well, which lets the
 *                           owner apply several sensors one after the other (clamping makes the
 *                           order matter).  Mono maps, insert depth 0, plain insertion; a colour
 *                           map returns UFO_B200_E_UNSUPPORTED
 *   ufo_b200_route_mark_ex  the same with the options of ufo_b200_insert_pointcloud.  Local point i
 *                           has the global cloud index index_base + i * index_stride (a contiguous
 *                           sector: (offset, 1); the interleaved split buf[r::world]: (r, world)).
 *                           On colour maps the point with the lowest global index of a hit voxel,
 *                           over all ranks, blends its colour, as on one map; indices have to stay
 *                           below 2^32 - 1 there.  early_stopping != 0 or depth > 6:
 *                           UFO_B200_E_UNSUPPORTED; index_stride == 0: UFO_B200_E_INVALID
 *   -- barrier across the ranks, ordered after route_mark on the map's stream --
 *   ufo_b200_route_apply    enqueue: marks received from sources [first_source, first_source +
 *                           n_sources) -> K3; last != 0 additionally runs the inner-node
 *                           propagation and ends the pass.  One scan split over the ranks:
 *                           route_apply(0, world, 1).  One sensor per rank, merged in sensor order:
 *                           route_apply(s, 1, s == world - 1) for s = 0..world-1.
 *   ufo_b200_route_sent     waits for the map's stream; counts[0..2] = brick-mask records,
 *                           whole-brick records and hit records this rank wrote into inboxes
 *                           (its own included) in its last mark pass
 * The union of the ranks' value fields equals the single-GPU map (tests/test_gpu_route.py,
 * tests/test_gpu_route_discrete.py).  Pools grow during a routed pass as on one map, so
 * initial_bricks is a starting size: route_mark grows them while marking (above), and an apply call
 * whose pool runs full backs off with the later calls of the pass, which are replayed in their order
 * after the growth at the rank's next synchronising call (the next route_mark, wait, a query or a
 * writer).  ufo_b200_last_scan_stats.regrows counts the growths of both phases of the last pass.
 * The inbox does not grow: a region too small for a pass is UFO_B200_E_NOMEM at the next
 * synchronising call.  Maps that have seen out-of-tree keys are rejected.  Between passes the ranks
 * also take setValueVolume, write batches and readData (each applies what it owns; pools grow there
 * as on one map), and ufo_b200_image_part_bv / ufo_b200_image_assemble give the union's file image. */
int ufo_b200_route_inbox_bytes(uint32_t world, uint32_t cap_bricks, uint32_t cap_hits, size_t* bytes);
int ufo_b200_route_inbox_bytes_color(uint32_t world, uint32_t cap_bricks, uint32_t cap_hits, size_t* bytes);
int ufo_b200_route_setup(ufo_b200_map* m, uint32_t rank, uint32_t world, uint32_t cap_bricks, uint32_t cap_hits,
                         void** inbox);
int ufo_b200_route_connect(ufo_b200_map* m, void* const* peer_inboxes);
int ufo_b200_route_mark(ufo_b200_map* m, const double origin[3], const void* points, size_t n, int layout,
                        double max_range, int on_device, int self_too);
int ufo_b200_route_mark_ex(ufo_b200_map* m, const double origin[3], const void* points, size_t n, int layout,
                           double max_range, uint32_t depth, int simple_ray_casting, uint32_t early_stopping,
                           int discrete, uint64_t index_base, uint32_t index_stride, int on_device, int self_too);
int ufo_b200_route_sent(ufo_b200_map* m, uint32_t counts[3]);
int ufo_b200_route_apply(ufo_b200_map* m, uint32_t first_source, uint32_t n_sources, int last);
int ufo_b200_ipc_export(void* dev_ptr, void* handle64);
int ufo_b200_ipc_open(const void* handle64, void** dev_ptr);
int ufo_b200_ipc_close(void* dev_ptr);

/* Forget everything (Octree::clear, octree.h:541-560): keeps device pools. */
int ufo_b200_clear(ufo_b200_map* m);

/* A map in bounded memory (no counterpart in the reference: pruneNode / deleteNodeChildren do not
 * compile, SURVEY.md G5, and a pointer tree on the host has no 80 GB ceiling).  A local map follows
 * the sensor; the rest lives with the caller, in host memory or on disk, as page blobs.
 *
 * One rule says which bricks (depth-4 nodes, 16^3 voxels) a volume KEEPS: a brick is kept iff every
 * cube on its path from the root down to its own depth-4 cube passes the volume -- the chain test of
 * ufo_b200_export_nodes_bv, stopped at depth 4.  Whole bricks only: a kept brick keeps all its
 * voxels, those outside the volume included.  n_bv == 0 keeps everything; a volume that misses the
 * map keeps nothing.  ufo_b200_retain is ufo_b200_retain_bv with one AABB record (box6: centre, half size).
 *
 * ufo_b200_retain_bv    removes every brick the volume does not keep and gives the memory back: the
 *                       survivors are compacted into pools of max(the map's initial capacity,
 *                       2 x survivors) bricks (peak: the old pools plus one array) and the levels
 *                       above the bricks are rebuilt from them; a removed brick is never-touched
 *                       space again.  Scan stamps move with their brick; the sensor model and the
 *                       min/max change box are unchanged; the recorded changes of removed bricks are
 *                       dropped with them.  out may be NULL.
 * ufo_b200_page_out_bv  writes the bricks ufo_b200_retain_bv would remove for the same volume into a
 *                       page blob and leaves the map as it is: page out, then retain.  *size receives
 *                       the blob's size; it is written when it fits into cap (buf = NULL sizes the
 *                       buffer).  Equal maps give equal blobs (bricks in ascending key order).
 * ufo_b200_page_in      puts the bricks of a blob back and recomputes everything derived under the
 *                       map's CURRENT sensor model.  Their scan stamps are 0 and change detection
 *                       records nothing for them.  The blob must come from a map of the same
 *                       resolution, depth_levels and colour mode, and NONE of its bricks may exist in
 *                       the map (merging two histories of one voxel has no sound meaning): otherwise
 *                       UFO_B200_E_INVALID and nothing is applied.  So a caller keeps the retained
 *                       volume wider than the sensor's reach (max_range) and brings a page in before
 *                       that reach enters it; a scan would otherwise re-create those bricks from
 *                       unknown.
 * ufo_b200_page_info    the header of a blob, on the host (no map needed); UFO_B200_E_INVALID when
 *                       the magic or the version is not this library's or size is below the header's.
 *
 * The blob is opaque and versioned, not an interchange format; no compression, no file variant (the
 * caller owns the bytes).  It holds nothing derived, so it stays valid when the thresholds change
 * while it is out.  Layout: a 64-byte header {u64 magic "UFOPAGE1", u32 version, u32 colour, u64
 * bits of the resolution double, u32 depth_levels, u32 0, u64 n bricks, 24 bytes 0}, then whole
 * sections: brick keys u64[n] (x | y << 21 | z << 42 of the brick coordinates, ascending), leaves
 * float[n][4096], octet-initialised bits u8[n][64], colour maps only: leaf colours u32[n][4096].
 *
 * Every call waits for a pending scan.  Rejected with nothing changed: routed maps
 * (ufo_b200_route_setup) and depth_levels < 5 (UFO_B200_E_UNSUPPORTED), a map whose scan failed
 * half-way (UFO_B200_E_INVALID).  A sharded map retains and pages within its own part. */
typedef struct {
	uint64_t bricks_before;
	uint64_t bricks_kept;          /* page_in: bricks in the map afterwards */
	uint64_t bricks_removed;       /* page_in: 0 */
	uint64_t brick_cap_before, brick_cap_after;
	uint64_t device_bytes_before, device_bytes_after;
	/* CUDA-event times on the map's stream, allocation and the waits between the steps included.
	 * retain: classify + prefix sum / compaction gather of every array / rebuild of the upper levels.
	 * page_in: existence check + brick creation / scatter of the sections / derived values + upper levels */
	float ms_classify, ms_compact, ms_upper;
} ufo_b200_retain_stats;

typedef struct {
	uint32_t version;
	uint32_t color;
	uint32_t depth_levels;
	uint32_t reserved;
	double resolution;
	uint64_t n_bricks;
	uint64_t bytes;   /* size of the whole blob the header describes */
} ufo_b200_page_header;

int ufo_b200_retain_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, ufo_b200_retain_stats* out);
int ufo_b200_retain(ufo_b200_map* m, const double box6[6], ufo_b200_retain_stats* out);
int ufo_b200_page_out_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, void* buf, size_t cap, size_t* size);
int ufo_b200_page_in(ufo_b200_map* m, const void* blob, size_t size, ufo_b200_retain_stats* out);
int ufo_b200_page_info(const void* blob, size_t size, ufo_b200_page_header* out);

/* What the map holds right now (waits for a pending scan): live bricks and upper nodes, the
 * capacities of their pools and the device memory of the map. */
typedef struct {
	uint64_t bricks, brick_cap;
	uint64_t upper_nodes, up_cap;
	uint64_t device_bytes;
} ufo_b200_pool_counts;
int ufo_b200_pool_stats(ufo_b200_map* m, ufo_b200_pool_counts* out);

/* ---- copies and tree size ----
 * ufo_b200_clone      a new map on the source's device holding the source's content, made on the
 *                     device without serialisation (the reference's copy constructor writes and reads
 *                     the map, occupancy_map_base.h:888-897).  Carried over: resolution, depth_levels,
 *                     colour mode, the six stored sensor-model log-odds bit for bit, every leaf, leaf
 *                     colour and octet-initialised bit, the values derived from them, and the alias state
 *                     of a map that has seen out-of-tree keys: the same later calls give the same
 *                     results on both maps.  Not carried over (a fresh map's defaults): change detection
 *                     and its changes, the min/max change box, the early-stopping opt-in, profiling and
 *                     a stream set with ufo_b200_set_stream (the copy has its own).  The brick pool's
 *                     capacity is max(initial capacity, 2 x bricks), as after ufo_b200_retain.  Waits for
 *                     a pending scan; the source is not changed.  Refused with nothing allocated: routed
 *                     maps (ufo_b200_route_setup) and sharded maps (UFO_B200_E_UNSUPPORTED), a map whose
 *                     scan failed half-way (UFO_B200_E_INVALID).  A device that cannot hold the copy gives
 *                     UFO_B200_E_NOMEM and *out = NULL.
 * ufo_b200_tree_info  the reference's node counters and getKnownBBX() of the pruned tree (the tree
 *                     ufo_b200_iterate and the file writer walk), computed on the device.  A node has
 *                     children iff it is not a leaf of that tree, so num_leaf_nodes = 8 x depth-1 nodes
 *                     with children and num_inner_nodes = 1 + 8 x nodes with children at depth >= 2
 *                     (getNumInnerNodes(): inner and inner-leaf nodes; the empty map has 1).  The known
 *                     box is the per-axis min / max of centre -/+ half_size over the leaves of
 *                     beginLeaves(occupied, free, !unknown), centres accumulated from the root as the
 *                     iterators accumulate them; AABB((0,0,0), 0) when there is none (known = 0).  A map
 *                     created with automatic_pruning = 0 reports the counters of the pruned tree.  A
 *                     routed or sharded map reports its own part: the counts of the ranks do not add up
 *                     to those of the union, whose upper levels and collapses differ.  Needs
 *                     depth_levels >= 5 (UFO_B200_E_UNSUPPORTED). */
int ufo_b200_clone(ufo_b200_map* src, ufo_b200_map** out);

typedef struct {
	uint64_t num_leaf_nodes;    /* getNumLeafNodes() */
	uint64_t num_inner_nodes;   /* getNumInnerNodes() */
	uint64_t with_children[22]; /* [d]: nodes of depth d that have children (d = 1 .. depth_levels) */
	int32_t known;              /* 1: the map has a free or occupied leaf */
	int32_t reserved;
	double known_min[3], known_max[3];  /* getKnownBBX() */
	float ms_device;            /* CUDA-event time of the brick pass on the map's stream */
	float reserved2;
} ufo_b200_tree_stats;
/* (a type cannot share the function's name in C) */
int ufo_b200_tree_info(ufo_b200_map* m, ufo_b200_tree_stats* out);

/* ---- nearest-first iteration ----
 * ufo_b200_nearest  one distance shell of beginNNLeaves (leaves_only != 0) / beginNNTree
 *                   (occupancy_map_base.h:169-245) from point[3]: the nodes that ufo_b200_iterate
 *                   returns for the same filters, contains, min_depth and volume, whose squared distance
 *                   d2 from the point satisfies d2_from <= d2 < hi, in non-decreasing d2; equal distances
 *                   keep ufo_b200_iterate's order (code ascending, depth descending).  d2 is the
 *                   reference's squaredDistance (iterator/octree_nearest.h:198-202): the point minus the
 *                   point clamped to the node's cube, (x*x + y*y) + z*z in doubles.  hi is chosen so that
 *                   at least `want` nodes come back, or all that remain; it never splits a group of equal
 *                   distances.  *d2_next = hi, where the next shell starts, or +inf when nothing is left.
 *                   Arrays as ufo_b200_iterate, plus d2[i]; *n is always the shell's size, the arrays are
 *                   filled when it is <= cap.  The shape of the tree above the bricks is kept on the map
 *                   and rebuilt by the first call after the map changed.  A non-finite point or a NaN
 *                   d2_from is UFO_B200_E_INVALID; depth_levels < 5 UFO_B200_E_UNSUPPORTED.  Waits for a
 *                   pending scan.  A sharded or routed map searches the part its own rank holds.
 * ufo_b200_last_nearest_stats  the work of the last ufo_b200_nearest call. */
int ufo_b200_nearest(ufo_b200_map* m, const double point[3], const ufo_b200_volume* bv, size_t n_bv, int leaves_only,
                     int occupied, int free_space, int unknown, int contains, uint32_t min_depth, double d2_from,
                     size_t want, uint64_t* codes, uint8_t* depths, float* logodds, uint8_t* flags, uint8_t* rgb,
                     double* d2, size_t cap, size_t* n, double* d2_next);

typedef struct {
	uint64_t bricks_visited;  /* CTAs of the brick kernel, summed over the shells tried */
	uint64_t upper_visited;   /* nodes above the bricks the host search visited */
	uint32_t shells;          /* brick kernel launches (a shell too small for `want` is doubled) */
	int32_t rebuilt;          /* 1: this call rebuilt the cached tree shape */
	uint64_t revision;        /* the map revision the call answered for; every write changes it */
	float ms_device;          /* CUDA-event time of the brick kernels and the sort */
	float ms_rebuild;         /* host time of the shape rebuild (0 when none) */
} ufo_b200_nearest_stats;
int ufo_b200_last_nearest_stats(ufo_b200_map* m, ufo_b200_nearest_stats* out);

const char* ufo_b200_version(void);

#ifdef __cplusplus
}
#endif
#endif /* UFOMAP_B200_H */
