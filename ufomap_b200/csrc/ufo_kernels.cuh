// ufo_kernels.cuh -- the integration kernels (sm_90a).
//
//   k_points   K1  per point: range test, BBX clip, hit voxel, ray end, change bbox
//                  (insertPointCloud front end, occupancy_map_base.h:281-309; discrete
//                  front end :354-399 / occupancy_map_color.h:195-246)
//   k_hits     K1b colour maps: first point per voxel blends its colour into the leaf
//                  (updateNodeColor, occupancy_map_color.cpp:142-171) and marks the hit
//   k_order_batches   sorts the batches of 32 rays by estimated walk length (load balance of K2)
//   k_rays     K2  one thread per ray, warp in lock-step: exact FP64 backward voxel walk
//                  (freeSpaceNormal, occupancy_map_base.h:1261-1301); visited voxels are
//                  OR-accumulated per 4^3 block in a register; leaving the block appends a
//                  16-byte (mask, voxel key) record to the warp's region of the record buffer
//   k_scatter  K2b one thread per record: brick hash probe -> atomicOr into the block's miss
//                  mask (set semantics of CodeMap::try_emplace, code.h:675-694)
//   k_rays_simple  fixed-step variant (freeSpaceSimple, occupancy_map_base.h:1303-1339)
//   k_update_brick (ufo_update.cuh)
//              K3  hit-then-miss float log-odds update of the marked voxels
//                  (updateOccupancy :1139-1145) and depth 1-4 aggregates per brick
//   k_brick_agg    depth-3/4 aggregates per brick (updateNode :1179-1224) when alias marks exist
//   k_split / k_walk_mark / k_gather* (ufo_walk.cuh): the fused marking path
//   k_alias_*      marks of keys outside the tree (octree.h:321), launched only when present
//   k_wrapped_colors  colour hits of keys outside the tree, in cloud order, on maps that met them
//   k_upper_*  K4  aggregates of the dirty nodes of depth >= 5 (seed, levels 5-6, one-CTA tail)
#pragma once

#include "ufo_device.cuh"
#include "ufo_update.cuh"

namespace ufo_b200
{
constexpr uint32_t kChunk = 256;  // records per k_scatter work item

struct QEntry {
	unsigned long long acc;  // visited-voxel bits of one 4^3 block (linear order)
	unsigned long long key;  // packed masked block coordinates (key >> 2)
};

// fused walk (ufo_walk.cuh): start state of one ray segment, and the per-ray constants
struct __align__(16) Item {
	double tx, ty, tz;        // t_max at the segment's first voxel
	uint32_t cx, cy, cz;      // first voxel (raw key, may lie outside the tree like the walk's own keys)
	uint32_t ex, ey, ez;      // end key: first voxel of the next segment, or the walk's end key
	uint32_t sgn;             // step signs, 2 bits per axis (1: +, 2: -, 0: none); 0xffffffff: no segment
	uint32_t pad[3];
};
static_assert(sizeof(Item) == 64, "Item is read as four 16-byte words");
struct __align__(16) RayConst {
	double dx, dy, dz;  // t_delta
	double dist;        // length of the (clipped) ray: the walk continues while min t_max <= dist
};
#ifndef UFO_SHELLS
#define UFO_SHELLS 16
#endif
constexpr uint32_t kShells = UFO_SHELLS;  // segments per ray at most

struct ScanArgs {
	Vec3 origin;       // sensor origin
	double max_range;  // < 0: unlimited
	uint32_t n;        // points
	uint32_t depth;    // insert depth of the free-space rays
	int layout;        // ufo_b200_layout
	int discrete;
	int use_color;     // colour map AND the cloud carries colour
	float miss;        // float(prob_miss_log / (2*depth+1)), occupancy_map_base.h:311
	const void* points;
	double* ray_end;   // [n][3], x = NaN when the point casts no ray
	// scan-local dedup table (discrete mode / colour hits)
	unsigned long long* tab_keys;
	uint32_t* tab_min;
	uint32_t tab_mask;
	uint32_t* hit_tab;  // [n] table position of the point's hit voxel or kNone
	int count_visits;
	// cloud frame applied while the points are read (insertPointCloud(..., frame_origin, ...),
	// occupancy_map_base.h:313-327 -> PointCloudT::transform, point_cloud.h:157-166)
	int has_frame;
	Frame frame;
	// layout 4 (sensor_msgs/PointCloud2 records): byte stride and field offsets; NaN points are
	// skipped like rosToUfo does (ufomap_ros/ufomap_ros/src/conversions.cpp:88-95, :115-137)
	uint32_t pc2_step, pc2_x, pc2_y, pc2_z;
	int pc2_r, pc2_g, pc2_b;
	// ray-walk output: (block key, visited-voxel mask) records, one region per warp of 32 rays
	struct QEntry* seg;
	unsigned long long seg_cap;  // records
	uint32_t* seg_base;          // [ceil(n/32)] first record of the warp's region
	uint32_t* seg_count;         // [ceil(n/32)] K1: capacity of the region, K2: records written
	uint32_t* order;             // [ceil(n/32)] ray batches sorted by estimated work, longest first
	// fused walk: segments by shell, [kShells][item_stride]; validity masks [kShells][ceil(n/32)]
	Item* items;
	size_t item_stride;
	uint32_t* vmask;
	RayConst* rc;                // [n]
	// insert depth 5/6: free-space nodes larger than a brick are collected here (deduplicated through
	// the scan-local table) and expanded into bricks by k_expand_nodes
	unsigned long long* nodes;   // [nodes_cap] packed (key >> depth)
	uint32_t nodes_cap;
};

// returns false for a point the ingestion drops (PointCloud2 records with a NaN coordinate)
__device__ __forceinline__ bool load_point(const ScanArgs& a, uint32_t i, Vec3& p, uint32_t& rgb)
{
	rgb = 0;
	switch (a.layout) {
		case 4: {
			const unsigned char* rec = reinterpret_cast<const unsigned char*>(a.points) + (size_t)a.pc2_step * i;
			const float x = *reinterpret_cast<const float*>(rec + a.pc2_x);
			const float y = *reinterpret_cast<const float*>(rec + a.pc2_y);
			const float z = *reinterpret_cast<const float*>(rec + a.pc2_z);
			p = {(double)x, (double)y, (double)z};
			if (x != x || y != y || z != z) return false;
			if (a.pc2_r >= 0) rgb = (uint32_t)rec[a.pc2_r] | ((uint32_t)rec[a.pc2_g] << 8) | ((uint32_t)rec[a.pc2_b] << 16);
		} break;
		case 0: {
			const double* q = reinterpret_cast<const double*>(a.points) + 3 * (size_t)i;
			p = {q[0], q[1], q[2]};
		} break;
		case 1: {
			const float* q = reinterpret_cast<const float*>(a.points) + 3 * (size_t)i;
			p = {(double)q[0], (double)q[1], (double)q[2]};
		} break;
		case 2: {
			const double* q = reinterpret_cast<const double*>(a.points) + 4 * (size_t)i;
			p = {q[0], q[1], q[2]};
			rgb = reinterpret_cast<const uint32_t*>(q + 3)[0] & 0xffffffu;
		} break;
		default: {
			const float4 q = reinterpret_cast<const float4*>(a.points)[i];
			p = {(double)q.x, (double)q.y, (double)q.z};
			rgb = __float_as_uint(q.w) & 0xffffffu;
		} break;
	}
	if (a.has_frame) p = frame_transform(a.frame, p);
	return true;
}

__device__ __forceinline__ void bbox_accumulate(const DeviceMap& M, double lo[3], double hi[3],
                                                bool any, bool cast)
{
	uint32_t rays = __ballot_sync(0xffffffffu, cast);
	if ((threadIdx.x & 31) == 0 && rays) atomicAdd(&M.ctr->n_rays, (uint32_t)__popc(rays));
	// warp-reduce, then one atomic per warp and component
	for (int c = 0; c < 3; ++c) {
		unsigned long long l = any ? encode_ordered(lo[c]) : ~0ull;
		unsigned long long h = any ? encode_ordered(hi[c]) : 0ull;
		for (int o = 16; o > 0; o >>= 1) {
			unsigned long long l2 = __shfl_xor_sync(0xffffffffu, l, o);
			unsigned long long h2 = __shfl_xor_sync(0xffffffffu, h, o);
			l = l2 < l ? l2 : l;
			h = h2 > h ? h2 : h;
		}
		if ((threadIdx.x & 31) == 0) {
			if (l != ~0ull) atomicMin(&M.ctr->bbox[c], l);
			if (h != 0ull) atomicMax(&M.ctr->bbox[3 + c], h);
		}
	}
}

// scan-local table: returns the slot of `key`; *first is true for the thread that
// inserted it.
__device__ __forceinline__ uint32_t table_insert(const ScanArgs& a, uint64_t key, bool* first)
{
	uint32_t i = hash_u64(key) & a.tab_mask;
	while (true) {
		unsigned long long k = ld_volatile_u64(&a.tab_keys[i]);
		if (k == kEmptyKey) {
			k = atomicCAS(&a.tab_keys[i], kEmptyKey, (unsigned long long)key);
			if (k == kEmptyKey) {
				*first = true;
				return i;
			}
		}
		if (k == key) {
			*first = false;
			return i;
		}
		i = (i + 1) & a.tab_mask;
	}
}

// Slow path for a voxel key (21 bits per axis, block coordinates bx..bz) with a component
// outside the tree: the mark is kept under the UNWRAPPED brick (own set semantics, like the
// reference's CodeSet/CodeMap) and the wrapped target brick is created right away so that
// the host's brick count is final after this kernel.  is_hit selects the mask array.
__device__ __noinline__ void mark_alias(const DeviceMap M, uint32_t bx, uint32_t by, uint32_t bz,
                                        unsigned long long bits, bool is_hit)
{
	if (!M.alias_miss) {
		atomicOr(&M.ctr->overflow, 32u);  // host allocates the alias arrays and re-runs
		return;
	}
	const uint32_t km = M.g.key_mask >> 2;
	// owned by the rank that owns the WRAPPED brick the mark lands in
	if (M.shard_world > 1 &&
	    brick_owner(pack_key((bx & km) >> 2, (by & km) >> 2, (bz & km) >> 2), M.shard_world) != M.shard_rank)
		return;
	const uint32_t src = brick_find_or_create(M, pack_key(bx >> 2, by >> 2, bz >> 2));
	const uint32_t dst = brick_find_or_create(M, pack_key((bx & km) >> 2, (by & km) >> 2, (bz & km) >> 2));
	if (src == kNone || dst == kNone) return;
	touch_brick(M, src);
	touch_brick(M, dst);
	atomicOr(&(is_hit ? M.alias_hit : M.alias_miss)[(size_t)src * 64 + morton2(bx, by, bz)], bits);
	atomicAdd(&M.ctr->alias_marks, 1u);
}

// Free-space node of depth 3 (8^3 voxels = 8 blocks) or 4 (16^3 = the whole brick): every
// voxel below it is marked.  (x, y, z) is any voxel key inside the node, 21 bits per axis.
// updateAllChildren (occupancy_map_base.h:1085-1120) applies the miss to every leaf below
// the node; in the value-field representation that is a full mask on each of its blocks.
__device__ __noinline__ void mark_node_miss(const DeviceMap M, uint32_t x, uint32_t y, uint32_t z,
                                               uint32_t depth)
{
	const uint32_t side = 1u << (depth - 2);  // blocks per axis: 2 or 4
	const uint32_t bx0 = (x >> depth) << (depth - 2), by0 = (y >> depth) << (depth - 2),
	               bz0 = (z >> depth) << (depth - 2);
	if ((x | y | z) & ~M.g.key_mask) {
		for (uint32_t k = 0; k < side; ++k)
			for (uint32_t j = 0; j < side; ++j)
				for (uint32_t i = 0; i < side; ++i) mark_alias(M, bx0 + i, by0 + j, bz0 + k, ~0ull, false);
		return;
	}
	if (M.shard_world > 1 && brick_owner(pack_key(bx0 >> 2, by0 >> 2, bz0 >> 2), M.shard_world) != M.shard_rank) return;
	const uint32_t brick = brick_find_or_create(M, pack_key(bx0 >> 2, by0 >> 2, bz0 >> 2));
	if (brick == kNone) return;
	touch_brick(M, brick);
	// the blocks of a depth-3 node are 8 consecutive Morton children, a depth-4 node is all 64
	const uint32_t first = depth == 3 ? (morton2(bx0, by0, bz0) & ~7u) : 0u;
	const uint32_t count = depth == 3 ? 8u : 64u;
	for (uint32_t c = 0; c < count; ++c) atomicOr(&M.miss_mask[(size_t)brick * 64 + first + c], ~0ull);
}

// Free-space node above the brick level (insert depth 5, 6): updateAllChildren
// (occupancy_map_base.h:1085-1120) reaches every voxel below it, i.e. every block of every brick
// below it.  Thousands of rays cross the same node, so the node goes into the scan's set first
// (the reference's CodeMap does the same) and k_expand_nodes marks its bricks once.
__device__ __noinline__ void collect_node(const DeviceMap M, const ScanArgs& a, uint32_t x, uint32_t y, uint32_t z,
                                          uint32_t depth)
{
	if ((x | y | z) & ~M.g.key_mask) {
		atomicOr(&M.ctr->overflow, 128u);  // out-of-tree node at this depth: not supported
		return;
	}
	const unsigned long long node = pack_key(x >> depth, y >> depth, z >> depth);
	bool first;
	table_insert(a, node | (3ull << 62), &first);
	if (!first) return;
	const uint32_t i = atomicAdd(&M.ctr->n_dirty, 1u);  // (the dense volume is not used on this path)
	if (i < a.nodes_cap) a.nodes[i] = node;
	else atomicOr(&M.ctr->overflow, 8u);
}

__device__ __noinline__ void scatter_slow(const DeviceMap M, const ScanArgs& a, uint32_t x, uint32_t y, uint32_t z,
                                          unsigned long long bits, uint32_t depth)
{
	if (depth >= 5) collect_node(M, a, x, y, z, depth);
	else if (depth >= 3) mark_node_miss(M, x, y, z, depth);
	else mark_alias(M, x >> 2, y >> 2, z >> 2, bits, false);
}

// routed mode: one hit-region record into the inbox of rank `owner` (ufo_route.cuh).  `rec` is a
// packed voxel key or a brick key | kFullBrick; colour maps add the global cloud index and rgb.
__device__ __forceinline__ void route_hit(const DeviceMap& M, uint32_t owner, unsigned long long rec, uint32_t index,
                                          uint32_t rgb)
{
	RouteTable* R = M.route;
	const uint32_t i = atomicAdd(&R->out_hit[owner], 1u);
	if (i >= R->cap_h) {
		atomicOr(&R->overflow, 1u);
		return;
	}
	if (M.color)
		*reinterpret_cast<ulonglong2*>(R->out[owner].hit + 2 * (size_t)i) = make_ulonglong2(rec, ((unsigned long long)rgb << 32) | index);
	else
		R->out[owner].hit[i] = rec;
}

// one thread per (collected node, brick below it): find-or-create the brick, full miss masks.
// Routed mode: a brick another rank owns (or every brick, with route_self) is not created here
// but sent to its owner as one whole-brick record.
__global__ void __launch_bounds__(256) k_expand_nodes(DeviceMap M, ScanArgs a)
{
	if (ld_volatile_u32(&M.ctr->overflow) & ~4u) return;
	const uint32_t per = 1u << (3 * (a.depth - 4));  // bricks per node
	const uint32_t side = 1u << (a.depth - 4);
	const size_t n = (size_t)min(ld_volatile_u32(&M.ctr->n_dirty), a.nodes_cap) * per;
	uint32_t sent = 0;
	for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
		uint32_t nx, ny, nz;
		unpack_key(a.nodes[e / per], nx, ny, nz);
		const uint32_t j = (uint32_t)(e % per);
		const uint32_t bx = nx * side + (j % side), by = ny * side + ((j / side) % side), bz = nz * side + j / (side * side);
		const unsigned long long bkey = pack_key(bx, by, bz);
		if (M.route_world > 1) {
			const uint32_t owner = brick_owner(bkey, M.route_world);
			if (owner != M.route_rank || M.route_self) {
				route_hit(M, owner, bkey | kFullBrick, kNone, 0u);
				++sent;
				continue;
			}
		}
		const uint32_t brick = brick_find_or_create(M, bkey);
		if (brick == kNone) continue;
		touch_brick(M, brick);
		ulonglong2* mm = reinterpret_cast<ulonglong2*>(M.miss_mask + (size_t)brick * 64);
		for (int c = 0; c < 32; ++c) mm[c] = make_ulonglong2(~0ull, ~0ull);
	}
	if (M.route_world > 1) {
		sent = __reduce_add_sync(0xffffffffu, sent);
		if ((threadIdx.x & 31) == 0 && sent) atomicAdd(&M.route->out_full, sent);
	}
}

// A brick received a mark: it joins the scan's touched list -- directly, or in dense mode through
// the volume's dirty bitmap (k_gather lists it together with the bricks the walk marked).
// (bx, by, bz) = brick coordinates (key >> 4).
__device__ __forceinline__ void touch_or_dirty(const DeviceMap& M, uint32_t brick, uint32_t bx, uint32_t by, uint32_t bz)
{
	if (M.dense) {
		const uint32_t vb = vol_brick(M, bx, by, bz);
		if (vb == kNone) atomicOr(&M.ctr->overflow, 64u);  // outside the volume: the host repeats the scan without it
		else vol_touch(M, vb);
	} else {
		touch_brick(M, brick);
	}
}

// mark a depth-0 hit voxel directly (mono maps)
__device__ __forceinline__ void mark_hit(const DeviceMap& M, Key3 k)
{
	k.x &= 0x1fffffu;  // a Code keeps 21 bits per axis (code.h:336-347)
	k.y &= 0x1fffffu;
	k.z &= 0x1fffffu;
	if ((k.x | k.y | k.z) & ~M.g.key_mask) {
		mark_alias(M, k.x >> 2, k.y >> 2, k.z >> 2, 1ull << linear2(k.x, k.y, k.z), true);
		return;
	}
	const uint64_t bkey = pack_key(k.x >> 4, k.y >> 4, k.z >> 4);
	if (M.shard_world > 1 && brick_owner(bkey, M.shard_world) != M.shard_rank) return;
	if (M.route_world > 1) {
		// routed mode: the hit voxel goes to the inbox of the rank that owns its brick
		const uint32_t owner = brick_owner(bkey, M.route_world);
		if (owner != M.route_rank || M.route_self) {
			route_hit(M, owner, pack_key(k.x, k.y, k.z), kNone, 0u);
			return;
		}
	}
	uint32_t brick = brick_find_or_create(M, bkey);
	if (brick == kNone) return;
	touch_or_dirty(M, brick, k.x >> 4, k.y >> 4, k.z >> 4);
	const size_t b = (size_t)brick * 64 + morton2(k.x >> 2, k.y >> 2, k.z >> 2);
	atomicOr(&M.hit_mask[b], 1ull << linear2(k.x, k.y, k.z));
	M.hit_stamp[brick] = M.scan_id;
}

// ---------------------------------------------------------------------------
// K1
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_points(DeviceMap M, ScanArgs a)
{
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	double lo[3], hi[3];
	bool contributes = false, cast = false;
	uint32_t bound = 0, span = 0;
	Vec3 end = {0.0, 0.0, 0.0};
	uint32_t rgb = 0;
	const bool valid = i < a.n && load_point(a, i, end, rgb);
	if (i < a.n && !valid) {
		// dropped by the ingestion: casts no ray, marks no hit
		a.ray_end[3 * (size_t)i] = __longlong_as_double(0x7ff8000000000000ll);
		if (a.hit_tab) a.hit_tab[i] = kNone;
	}
	if (valid) {
		const Geometry& g = M.g;
		const double bhi = node_half(g, g.depth_levels), blo = -bhi;
		uint32_t hit_slot = kNone;
		if (!a.discrete) {
			// occupancy_map_base.h:281-309
			Vec3 origin = a.origin;
			Vec3 dir = vsub(end, origin);
			double dist = vnorm(dir);
			if (move_line_inside(g, origin, end)) {
				if (0 > a.max_range || dist <= a.max_range) {
					Key3 k = point_to_key(g, end, 0);
					if (a.use_color) {
						bool first;
						hit_slot = table_insert(a, key_to_code(k), &first);
						atomicMin(&a.tab_min[hit_slot], i);
					} else {
						mark_hit(M, k);
					}
				} else {
					dir = vdiv(dir, dist);
					end = vadd(origin, vscale(dir, a.max_range));
				}
				cast = true;
				for (int c = 0; c < 3; ++c) {
					lo[c] = end[c] < origin[c] ? end[c] : origin[c];
					hi[c] = end[c] < origin[c] ? origin[c] : end[c];
				}
				contributes = true;
			}
		} else {
			// occupancy_map_base.h:354-399 / occupancy_map_color.h:195-246
			bool skip = false;
			double sq_max = dop::mul(a.max_range, a.max_range);
			if (0 > a.max_range || vsqnorm(vsub(end, a.origin)) < sq_max) {
				if (in_bbx(end, blo, bhi)) {
					Key3 k = point_to_key(g, end, 0);
					bool first;
					uint32_t slot = table_insert(a, key_to_code(k), &first);
					if (a.use_color) {
						hit_slot = slot;
						atomicMin(&a.tab_min[slot], i);
					} else if (first) {
						mark_hit(M, k);
					}
					// a later point in an already seen end voxel is dropped together with
					// its ray; the ray it would cast is identical to the first one's
					skip = !first;
				}
			} else {
				Vec3 dir = vsub(key_to_coord(g, point_to_key(g, end, a.depth), a.depth), a.origin);
				if (a.use_color) {
					double sq = vsqnorm(dir);
					if (0 <= a.max_range && sq > sq_max) {
						dir = vdiv(dir, dop::sqrt(sq));
						end = vadd(a.origin, vscale(dir, a.max_range));
					}
				} else {
					double nrm = vnorm(dir);
					dir = vdiv(dir, nrm);
					if (0 <= a.max_range && nrm > a.max_range) {
						end = vadd(a.origin, vscale(dir, a.max_range));
					}
				}
			}
			Vec3 cur = a.origin;
			if (!skip && move_line_inside(g, cur, end)) {
				Key3 ek = point_to_key(g, end, a.depth);
				// rays are deduplicated per end node (explicitly at depth > 0 in the
				// reference, implicitly by the set semantics at depth 0)
				bool first;
				table_insert(a, key_to_code(ek) | (1ull << 63), &first);
				Vec3 ec = key_to_coord(g, ek, a.depth);
				if (first) {
					end = ec;
					cast = true;
				}
				Vec3 cc = key_to_coord(g, point_to_key(g, cur, a.depth), a.depth);
				double t = node_half(g, a.depth);
				for (int c = 0; c < 3; ++c) {
					double e0 = dop::sub(ec[c], t), c0 = dop::sub(cc[c], t);
					double e1 = dop::add(ec[c], t), c1 = dop::add(cc[c], t);
					lo[c] = c0 < e0 ? c0 : e0;
					hi[c] = e1 < c1 ? c1 : e1;
				}
				contributes = true;
			}
		}
		double* r = a.ray_end + 3 * (size_t)i;
		if (cast) {
			r[0] = end.x;
			r[1] = end.y;
			r[2] = end.z;
		} else {
			r[0] = __longlong_as_double(0x7ff8000000000000ll);
		}
		if (a.hit_tab) a.hit_tab[i] = hit_slot;
		if (cast) {
			// upper bound of the 4^3 blocks this ray's walk can leave: one per block
			// boundary crossed on each axis, plus slack for the end-of-walk overshoot
			Vec3 from = a.origin, to = end;
			if (move_line_inside(g, from, to)) {
				Key3 kf = point_to_key(g, from, a.depth), kt = point_to_key(g, to, a.depth);
				// keys are u32 and may wrap below zero at the - faces (the walk wraps the same way)
				uint32_t dx = (uint32_t)abs((int)(kf.x - kt.x));
				uint32_t dy = (uint32_t)abs((int)(kf.y - kt.y));
				uint32_t dz = (uint32_t)abs((int)(kf.z - kt.z));
				bound = (dx >> 2) + (dy >> 2) + (dz >> 2) + 8u;
				span = max(dx, max(dy, dz)) >> a.depth;
			}
		}
	}
	bbox_accumulate(M, lo, hi, contributes, cast);
	if (a.items) {
		// longest ray in dominant-axis steps: sets the shell thickness of the fused walk
		for (int o = 16; o > 0; o >>= 1) span = max(span, __shfl_xor_sync(0xffffffffu, span, o));
		if ((threadIdx.x & 31) == 0 && span) atomicMax(&M.ctr->max_span, span);
	}
	if (a.seg_base) {
		for (int o = 16; o > 0; o >>= 1) bound += __shfl_xor_sync(0xffffffffu, bound, o);
		if ((threadIdx.x & 31) == 0 && i < a.n) {
			unsigned long long base = atomicAdd(&M.ctr->seg_total, (unsigned long long)bound);
			if (base + bound > a.seg_cap) {
				atomicOr(&M.ctr->overflow, 8u);  // record buffer too small: host grows it and re-runs
				base = 0;
				bound = 0;
			}
			a.seg_base[i >> 5] = (uint32_t)base;
			a.seg_count[i >> 5] = bound;
		}
	}
}

// updateNodeColor (occupancy_map_color.cpp:142-171): the colour of a leaf of colour `cur` and
// log-odds `occ` after an update of colour `upd` with hit probability `prob` (toProb of the
// update's log-odds; M.prob_hit for a scan's hits).  `hit` is taken by reference so that it is
// only read past the two early returns, as the scans' blends always did.
__device__ __forceinline__ uint32_t blended_color(uint32_t cur, uint32_t upd, const double& hit, float occ)
{
	if (cur == upd) return cur;
	if (cur == 0) return upd;
	double prob = hit;
	double total = prob + to_prob(occ);
	prob = prob / total;
	double inv = 1.0 - prob;
	uint32_t out = 0;
	for (int c = 0; c < 3; ++c) {
		double cc = (double)((cur >> (8 * c)) & 0xffu), uu = (double)((upd >> (8 * c)) & 0xffu);
		double r = dop::sqrt(dop::add(dop::mul(dop::mul(cc, cc), inv), dop::mul(dop::mul(uu, uu), prob)));
		out |= ((uint32_t)(int)r & 0xffu) << (8 * c);
	}
	return out;
}

// blends `upd` into leaf li, weighted by the leaf's occupancy before this scan's update
__device__ __forceinline__ void blend_color(const DeviceMap& M, size_t li, uint32_t upd)
{
	uint32_t cur = M.leaf_rgb[li];
	if (cur == upd) return;
	M.leaf_rgb[li] = blended_color(cur, upd, M.prob_hit, M.leaf[li]);
}

// slot of `key` in the scan-local table, kNone when absent
__device__ __forceinline__ uint32_t table_find(const ScanArgs& a, uint64_t key)
{
	for (uint32_t i = hash_u64(key) & a.tab_mask;; i = (i + 1) & a.tab_mask) {
		const unsigned long long k = a.tab_keys[i];
		if (k == key) return i;
		if (k == kEmptyKey) return kNone;
	}
}

// Out-of-tree hit keys: a point on a + face is inside the map (isInside is inclusive,
// octree.h:1297-1304) and toKey gives 2^L there; a ray end clipped onto a - face can give -1
// (2^21 - 1 in the 21-bit code).  The tree's code walk only reads L bits, so 2^L wraps onto
// key 0 and -1 onto key 2^L - 1 of that axis.  The wrapped key of an in-tree key (itself if none):
__device__ __forceinline__ uint32_t wrapped_alt(const DeviceMap& M, uint32_t c)
{
	if (M.g.key_mask == 0x1fffffu) return c;  // 21 levels: every 21-bit key is in the tree
	return c == 0u ? M.g.key_mask + 1u : (c == M.g.key_mask ? 0x1fffffu : c);
}

// Visits the table slots of the hits of in-tree voxel v (with_self) and of every out-of-tree key
// that wraps onto it (bit s of `sel` puts axis s at its wrapped key); f returns false to stop.
template <class F>
__device__ __forceinline__ void for_wrapped_hits(const DeviceMap& M, const ScanArgs& a, Key3 v, bool with_self, F f)
{
	const Key3 w = {wrapped_alt(M, v.x), wrapped_alt(M, v.y), wrapped_alt(M, v.z)};
	for (uint32_t sel = with_self ? 0u : 1u; sel < 8u; ++sel) {
		if (((sel & 1u) && w.x == v.x) || ((sel & 2u) && w.y == v.y) || ((sel & 4u) && w.z == v.z)) continue;
		const Key3 c = {(sel & 1u) ? w.x : v.x, (sel & 2u) ? w.y : v.y, (sel & 4u) ? w.z : v.z};
		const uint32_t ts = table_find(a, key_to_code(c));
		if (ts != kNone && !f(sel, a.tab_min[ts])) return;
	}
}

// K1b: colour maps.  The first point (lowest cloud index) of every hit voxel blends
// its colour into the leaf BEFORE the occupancy update of this scan
// (occupancy_map_color.h:269-287) and marks the hit bit.
__global__ void __launch_bounds__(256) k_hits(DeviceMap M, ScanArgs a)
{
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n) return;
	uint32_t t = a.hit_tab[i];
	if (t == kNone || a.tab_min[t] != i) return;
	Key3 k = code_to_key(a.tab_keys[t]);
	if ((k.x | k.y | k.z) & ~M.g.key_mask) {
		// out-of-tree hit voxel: occupancy goes through the alias path, colour through
		// k_wrapped_colors
		mark_alias(M, k.x >> 2, k.y >> 2, k.z >> 2, 1ull << linear2(k.x, k.y, k.z), true);
		return;
	}
	if (M.shard_world > 1 && brick_owner(pack_key(k.x >> 4, k.y >> 4, k.z >> 4), M.shard_world) != M.shard_rank) return;
	uint32_t brick = brick_find_or_create(M, pack_key(k.x >> 4, k.y >> 4, k.z >> 4));
	if (brick == kNone) return;
	touch_or_dirty(M, brick, k.x >> 4, k.y >> 4, k.z >> 4);
	const size_t slot = (size_t)brick * 64 + morton2(k.x >> 2, k.y >> 2, k.z >> 2);
	uint32_t v = morton2(k.x, k.y, k.z);
	const unsigned long long hbit = 1ull << linear2(k.x, k.y, k.z);
	unsigned long long old = atomicOr(&M.hit_mask[slot], hbit);
	M.hit_stamp[brick] = M.scan_id;
	if (old & hbit) return;  // re-run after a pool regrow: colour already blended
	if (wrapped_alt(M, k.x) != k.x || wrapped_alt(M, k.y) != k.y || wrapped_alt(M, k.z) != k.z) {
		// a voxel on the map's boundary may also receive out-of-tree hits: k_wrapped_colors blends
		// all of them in cloud order
		bool wrapped = false;
		for_wrapped_hits(M, a, k, false, [&](uint32_t, uint32_t) {
			wrapped = true;
			return false;
		});
		if (wrapped) return;
	}
	Vec3 p;
	uint32_t upd;
	load_point(a, i, p, upd);
	blend_color(M, slot * 64 + v, upd);
}

// The colour hits of a voxel that out-of-tree keys wrap onto, applied like the reference does: one
// at a time in cloud order, each blend with the occupancy the earlier hits of this scan left
// (occupancy_map_color.h:269-287).  One thread per such voxel: the lowest-index out-of-tree winner.
// Runs after marking and before any occupancy update of the scan, only in the scan's final run.
__global__ void __launch_bounds__(256) k_wrapped_colors(DeviceMap M, ScanArgs a)
{
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n || (__ldg(&M.ctr->overflow) & ~4u)) return;
	uint32_t t = a.hit_tab[i];
	if (t == kNone || a.tab_min[t] != i) return;
	Key3 k = code_to_key(a.tab_keys[t]);
	if (!((k.x | k.y | k.z) & ~M.g.key_mask)) return;
	k.x &= M.g.key_mask;
	k.y &= M.g.key_mask;
	k.z &= M.g.key_mask;
	if (M.shard_world > 1 && brick_owner(pack_key(k.x >> 4, k.y >> 4, k.z >> 4), M.shard_world) != M.shard_rank) return;
	uint32_t idx[8], n = 0;
	bool lead = true;
	for_wrapped_hits(M, a, k, true, [&](uint32_t sel, uint32_t j) {
		if (sel && j < i) {
			lead = false;
			return false;
		}
		idx[n++] = j;
		return true;
	});
	if (!lead) return;
	const uint32_t tb = brick_find(M, pack_key(k.x >> 4, k.y >> 4, k.z >> 4));
	if (tb == kNone) return;
	for (uint32_t x = 1; x < n; ++x)
		for (uint32_t y = x; y > 0 && idx[y - 1] > idx[y]; --y) {
			const uint32_t s = idx[y];
			idx[y] = idx[y - 1];
			idx[y - 1] = s;
		}
	const size_t tl = ((size_t)tb * 64 + morton2(k.x >> 2, k.y >> 2, k.z >> 2)) * 64 + morton2(k.x, k.y, k.z);
	float occ = M.leaf[tl];
	uint32_t rgb = M.leaf_rgb[tl];
	for (uint32_t x = 0; x < n; ++x) {
		Vec3 p;
		uint32_t upd;
		load_point(a, idx[x], p, upd);
		rgb = blended_color(rgb, upd, M.prob_hit, occ);
		occ = apply_update(M, occ, M.hit);
	}
	M.leaf_rgb[tl] = rgb;
}

// ---------------------------------------------------------------------------
// K2
// ---------------------------------------------------------------------------
template <int DEPTH>
__device__ __forceinline__ unsigned long long voxel_bits(Key3 k)
{
	if (DEPTH == 0) return 1ull << linear2(k.x, k.y, k.z);
	if (DEPTH == 1) return octet_mask_of(k.x, k.y, k.z);
	return ~0ull;
}

struct BrickCache {
	uint32_t bx, by, bz, slot;
};

// OR `bits` into the miss mask of the block that contains unmasked key k
__device__ __forceinline__ void flush_block(const DeviceMap& M, BrickCache& bc, uint32_t kx,
                                            uint32_t ky, uint32_t kz, unsigned long long bits)
{
	kx &= 0x1fffffu;
	ky &= 0x1fffffu;
	kz &= 0x1fffffu;
	if ((kx | ky | kz) & ~M.g.key_mask) {
		mark_alias(M, kx >> 2, ky >> 2, kz >> 2, bits, false);
		return;
	}
	uint32_t bx = kx >> 4, by = ky >> 4, bz = kz >> 4;
	if (M.shard_world > 1 && brick_owner(pack_key(bx, by, bz), M.shard_world) != M.shard_rank) return;
	if (bc.slot == kNone || bx != bc.bx || by != bc.by || bz != bc.bz) {
		bc.bx = bx;
		bc.by = by;
		bc.bz = bz;
		bc.slot = brick_find_or_create(M, pack_key(bx, by, bz));
		if (bc.slot != kNone) touch_brick(M, bc.slot);
	}
	if (bc.slot == kNone) return;
	atomicOr(&M.miss_mask[(size_t)bc.slot * 64 + morton2(kx >> 2, ky >> 2, kz >> 2)], bits);
}

// ---------------------------------------------------------------------------
// K2: ray walk
// ---------------------------------------------------------------------------
// k_rays is pure arithmetic: one thread per ray, the whole warp in lock-step, each lane
// ORs the voxels it visits into the 64-bit mask of the 4^3 block it is in and, when it
// leaves the block, appends a (block key, mask) record to the warp's region of a
// streaming buffer (ballot-compacted, so the warp's records of one step are contiguous).
// k_scatter then resolves every record (brick hash -> block slot) and ORs the mask into
// the block's per-scan miss mask with full memory-level parallelism.  Splitting the walk
// from the lookups keeps the latency-bound pointer chasing out of the FP64 loop.
#ifndef UFO_RAY_MINBLOCKS
#define UFO_RAY_MINBLOCKS 8
#endif
constexpr int kRayThreads = 128;

// One lock-step iteration of the ray walk for the whole warp, in PTX so that everything
// stays predicated (no divergent branches, no phi moves):
//   mark the current voxel; computeRayTakeStep (octree.h:1227-1233: argmin with <= and
//   x,y,z priority, vector3.h:244-251); loop condition of freeSpaceNormal
//   (occupancy_map_base.h:1300); when the lane left its 4^3 block or finished, append
//   (mask, voxel key of the old block) to the warp's record region via ballot compaction.
// `active` is 1 while the lane's walk continues.  Returns true while any lane is active.
__device__ __forceinline__ bool walk_iteration(double& tx, double& ty, double& tz, const double dx,
                                               const double dy, const double dz, const double dist,
                                               uint32_t& kx, uint32_t& ky, uint32_t& kz, const int sx,
                                               const int sy, const int sz, const uint32_t ex,
                                               const uint32_t ey, const uint32_t ez,
                                               unsigned long long& acc, const unsigned long long bits,
                                               uint32_t& active, uint32_t& cursor, const uint32_t cap,
                                               QEntry* out, const uint32_t lt_mask)
{
	uint32_t any;
	asm volatile(
	    "{\n\t"
	    ".reg .pred pa, px, py, pz, pt, pm, pn, pl, pp, pw;\n\t"
	    ".reg .u32 ox, oy, oz, vx, vy, vz, bal, rank, idx, cnt, klo, khi, t;\n\t"
	    ".reg .u64 key, addr;\n\t"
	    "setp.ne.u32 pa, %8, 0;\n\t"
	    "@pa or.b64 %7, %7, %22;\n\t"
	    "mov.u32 ox, %3;\n\t"
	    "mov.u32 oy, %4;\n\t"
	    "mov.u32 oz, %5;\n\t"
	    // axis selection
	    "setp.le.f64 px, %0, %1;\n\t"
	    "setp.le.and.f64 px, %0, %2, px;\n\t"
	    "setp.gt.f64 py, %0, %1;\n\t"
	    "setp.le.and.f64 py, %1, %2, py;\n\t"
	    "or.pred pt, px, py;\n\t"
	    "not.pred pz, pt;\n\t"
	    "and.pred px, px, pa;\n\t"
	    "and.pred py, py, pa;\n\t"
	    "and.pred pz, pz, pa;\n\t"
	    "@px add.rn.f64 %0, %0, %10;\n\t"
	    "@py add.rn.f64 %1, %1, %11;\n\t"
	    "@pz add.rn.f64 %2, %2, %12;\n\t"
	    "@px add.u32 %3, %3, %14;\n\t"
	    "@py add.u32 %4, %4, %15;\n\t"
	    "@pz add.u32 %5, %5, %16;\n\t"
	    // more = (cur != end) && (tx <= dist || ty <= dist || tz <= dist)
	    "setp.le.f64 pm, %0, %13;\n\t"
	    "setp.le.or.f64 pm, %1, %13, pm;\n\t"
	    "setp.le.or.f64 pm, %2, %13, pm;\n\t"
	    "setp.ne.u32 pn, %3, %17;\n\t"
	    "setp.ne.or.u32 pn, %4, %18, pn;\n\t"
	    "setp.ne.or.u32 pn, %5, %19, pn;\n\t"
	    "and.pred pm, pm, pn;\n\t"
	    // left = ((cur ^ old) >> 2) != 0 on any axis
	    "xor.b32 vx, ox, %3;\n\t"
	    "xor.b32 vy, oy, %4;\n\t"
	    "xor.b32 vz, oz, %5;\n\t"
	    "or.b32 vx, vx, vy;\n\t"
	    "or.b32 vx, vx, vz;\n\t"
	    "setp.gt.u32 pl, vx, 3;\n\t"
	    // push = active && (!more || left);  active' = active && more
	    "not.pred pt, pm;\n\t"
	    "or.pred pp, pt, pl;\n\t"
	    "and.pred pp, pp, pa;\n\t"
	    "and.pred pa, pa, pm;\n\t"
	    "selp.u32 %8, 1, 0, pa;\n\t"
	    // ballot-compacted append of {acc, voxel key of the block just left}
	    "vote.sync.ballot.b32 bal, pp, 0xffffffff;\n\t"
	    "and.b32 rank, bal, %21;\n\t"
	    "popc.b32 rank, rank;\n\t"
	    "add.u32 idx, %9, rank;\n\t"
	    "setp.lt.and.u32 pw, idx, %20, pp;\n\t"
	    "and.b32 ox, ox, 0x1fffff;\n\t"
	    "and.b32 oy, oy, 0x1fffff;\n\t"
	    "and.b32 oz, oz, 0x1fffff;\n\t"
	    "mad.lo.u32 klo, oy, 0x200000, ox;\n\t"
	    "shr.u32 t, oy, 11;\n\t"
	    "mad.lo.u32 khi, oz, 1024, t;\n\t"
	    "mov.b64 key, {klo, khi};\n\t"
	    "mad.wide.u32 addr, idx, 16, %23;\n\t"
	    "@pw st.global.v2.u64 [addr], {%7, key};\n\t"
	    "@pp mov.u64 %7, 0;\n\t"
	    "popc.b32 cnt, bal;\n\t"
	    "add.u32 %9, %9, cnt;\n\t"
	    "vote.sync.any.pred pt, pa, 0xffffffff;\n\t"
	    "selp.u32 %6, 1, 0, pt;\n\t"
	    "}"
	    : "+d"(tx), "+d"(ty), "+d"(tz), "+r"(kx), "+r"(ky), "+r"(kz), "=r"(any), "+l"(acc), "+r"(active),
	      "+r"(cursor)
	    : "d"(dx), "d"(dy), "d"(dz), "d"(dist), "r"(sx), "r"(sy), "r"(sz), "r"(ex), "r"(ey), "r"(ez),
	      "r"(cap), "r"(lt_mask), "l"(bits), "l"(out)
	    : "memory");
	return any != 0;
}

// Orders the batches of 32 rays by their estimated work (the record bound K1 computed,
// which is proportional to the walk length), longest first: a counting sort over 256
// work classes in one CTA.
__global__ void __launch_bounds__(1024) k_order_batches(const uint32_t* work, uint32_t n, uint32_t* order)
{
	__shared__ uint32_t hist[256];
	__shared__ uint32_t wmax;
	if (threadIdx.x < 256) hist[threadIdx.x] = 0;
	if (threadIdx.x == 0) wmax = 1;
	__syncthreads();
	uint32_t m = 0;
	for (uint32_t b = threadIdx.x; b < n; b += blockDim.x) m = max(m, work[b]);
	atomicMax(&wmax, m);
	__syncthreads();
	const uint32_t top = wmax;
	for (uint32_t b = threadIdx.x; b < n; b += blockDim.x)
		atomicAdd(&hist[255u - (uint32_t)(((unsigned long long)work[b] * 255ull) / top)], 1u);
	__syncthreads();
	if (threadIdx.x == 0) {
		uint32_t run = 0;
		for (int k = 0; k < 256; ++k) {
			uint32_t c = hist[k];
			hist[k] = run;
			run += c;
		}
	}
	__syncthreads();
	for (uint32_t b = threadIdx.x; b < n; b += blockDim.x)
		order[atomicAdd(&hist[255u - (uint32_t)(((unsigned long long)work[b] * 255ull) / top)], 1u)] = b;
}

// Warp w of CTA c walks the batches of rank c + gridDim.x * (w + 4 * round): every CTA
// gets one batch from each work quartile, so every SM receives the same amount of work
// whatever the hardware's CTA placement is.
template <int DEPTH, bool COUNT>
__global__ void __launch_bounds__(kRayThreads, UFO_RAY_MINBLOCKS) k_rays(DeviceMap M, ScanArgs a, uint32_t* batch_counter)
{
	const uint32_t lane = threadIdx.x & 31;
	constexpr uint32_t FULL = 0xffffffffu;
	const uint32_t lt_mask = (1u << lane) - 1u;
	const uint32_t n_batches = (a.n + 31) / 32;
	unsigned int visits = 0;
	(void)batch_counter;
	if (ld_volatile_u32(&M.ctr->overflow) & 8u) return;  // record buffer being regrown
	for (uint32_t v = (threadIdx.x >> 5) * gridDim.x + blockIdx.x; v < n_batches; v += gridDim.x * (kRayThreads / 32)) {
		const uint32_t batch = a.order[v];
		const uint32_t i = batch * 32 + lane;
		QEntry* out = a.seg + a.seg_base[batch];
		const uint32_t cap = a.seg_count[batch];
		uint32_t cursor = 0;
		Walk w;
		w.tx = w.ty = w.tz = 0.0;
		w.dx = w.dy = w.dz = 0.0;
		w.sx = w.sy = w.sz = 0;
		w.cur = {0, 0, 0};
		w.end = {0, 0, 0};
		double dist = 0.0;
		uint32_t active = 0;
		bool same = false;
		unsigned long long acc = 0;
		if (i < a.n) {
			const double* r = a.ray_end + 3 * (size_t)i;
			Vec3 to = {r[0], r[1], r[2]};
			Vec3 from = a.origin;
			// occupancy_map_base.h:1248-1251
			if (to.x == to.x && move_line_inside(M.g, from, to)) {
				// walked backwards: end point -> sensor (occupancy_map_base.h:1266-1279)
				Vec3 dir = vsub(from, to);
				dist = vnorm(dir);
				dir = vdiv(dir, dist);
				walk_init(M.g, to, from, dir, a.depth, w);  // DEPTH only selects the mark pattern
				same = w.same;
				active = same ? 0u : 1u;
			}
		}
		{
			// rays whose two ends share a voxel mark just that voxel (occupancy_map_base.h:1281-1284)
			const uint32_t pm = __ballot_sync(FULL, same);
			if (same) {
				const uint32_t idx = __popc(pm & lt_mask);
				if (idx < cap) {
					out[idx].acc = voxel_bits<DEPTH>(w.cur);
					out[idx].key = pack_key(w.cur.x & 0x1fffffu, w.cur.y & 0x1fffffu, w.cur.z & 0x1fffffu);
				}
				if (COUNT) ++visits;
			}
			cursor += __popc(pm);
		}
		bool any = __any_sync(FULL, active != 0u);
		while (any) {
			if (COUNT) visits += active;
			any = walk_iteration(w.tx, w.ty, w.tz, w.dx, w.dy, w.dz, dist, w.cur.x, w.cur.y, w.cur.z, w.sx,
			                     w.sy, w.sz, w.end.x, w.end.y, w.end.z, acc, voxel_bits<DEPTH>(w.cur),
			                     active, cursor, cap, out, lt_mask);
		}
		if (lane == 0) {
			if (cursor > cap) {
				atomicOr(&M.ctr->overflow, 16u);  // walk outran its bound: must never happen
				cursor = cap;
			}
			a.seg_count[batch] = cursor;
			atomicMax(&M.ctr->n_chunks, (cursor + kChunk - 1) / kChunk);  // longest region, in chunks
		}
	}
	if (COUNT && visits) atomicAdd(&M.ctr->visits, (unsigned long long)visits);
}

// K2b: one thread per record.  Resolves the brick (one probe of a two-entry hash bucket
// = one 32-byte sector in the common case), the block slot, and ORs the mask into the
// block's miss mask.  The upper half of a hash entry's value caches the scan stamp of the
// brick so that only the first records of a brick write brick_stamp.
// Work item (j, r) = the j-th kChunk-record slice COUNTED FROM THE END of region r, and
// items are visited j-major: the walks run from the end point towards the sensor, so the
// tails of all regions hold the records next to the sensor, which thousands of rays share
// -- visiting them together turns most of the mask atomics into L2 hits.
#ifndef UFO_SCATTER_MINBLOCKS
#define UFO_SCATTER_MINBLOCKS 8
#endif
// GENERIC = false is the common case (insert depth <= 2, no out-of-tree keys seen yet): the slow
// paths are compiled out so that the hot path stays small.  SHARD adds the ownership filter of a
// spatially sharded map (records of bricks another GPU owns are dropped before any memory access).
template <bool GENERIC, bool SHARD>
__device__ __forceinline__ void scatter_record(const DeviceMap& M, const ScanArgs& a, const ulonglong2 v)
{
	uint32_t x, y, z;
	unpack_key(v.y, x, y, z);
	if ((GENERIC && a.depth >= 3) || ((x | y | z) & ~M.g.key_mask)) {
		// rare: free-space nodes larger than a block, or a key outside the tree.  The lean
		// variant has no slow path: it asks the host for the alias arrays (bit 5), and the
		// re-run -- like every later scan of this map -- uses the generic variant.
		if (GENERIC) scatter_slow(M, a, x, y, z, v.x, a.depth);
		else atomicOr(&M.ctr->overflow, 32u);
		return;
	}
	x >>= 2;  // block coordinates
	y >>= 2;
	z >>= 2;
	const unsigned long long bkey = pack_key(x >> 2, y >> 2, z >> 2);
	if (SHARD && brick_owner(bkey, M.shard_world) != M.shard_rank) return;  // another GPU's brick
	const uint32_t hidx = hash_u64(bkey) & M.bh_mask & ~1u;
	// First entry of the two-entry bucket first (it holds the key three times out of four), the
	// second only on a mismatch: K2b is bound by L1 wavefronts of its scattered accesses as much
	// as by latency, and this drops a quarter of them.  L1-cached loads: thousands of records
	// near the sensor resolve to the same few bricks at the same time.
#ifdef UFO_SCATTER_BOTH_ENTRIES
	const ulonglong2 e0 = ld_cached_entry(&M.bh_tab[hidx]);
	const ulonglong2 e1 = ld_cached_entry(&M.bh_tab[hidx + 1]);
	const bool hit0 = e0.x == bkey, hit1 = e1.x == bkey;
	const ulonglong2 ent = hit0 ? e0 : e1;
	const uint32_t hpos = hit0 ? hidx : hidx + 1;
#else
	ulonglong2 ent = ld_cached_entry(&M.bh_tab[hidx]);
	const bool hit0 = ent.x == bkey;
	bool hit1 = false;
	uint32_t hpos = hidx;
	if (!hit0) {
		ent = ld_cached_entry(&M.bh_tab[hidx + 1]);
		hit1 = ent.x == bkey;
		hpos = hidx + 1;
	}
#endif
	uint32_t brick = (uint32_t)ent.y;
	if ((hit0 || hit1) && brick != kPending && brick != kFailed) {
		if ((uint32_t)(ent.y >> 32) != M.scan_id) {
			touch_brick(M, brick);
			reinterpret_cast<uint32_t*>(&M.bh_tab[hpos].y)[1] = M.scan_id;
		}
	} else {
		brick = brick_find_or_create_from(M, bkey, hidx);
		if (brick == kNone) return;
		touch_brick(M, brick);
	}
	atomicOr(&M.miss_mask[(size_t)brick * 64 + morton2(x, y, z)], v.x);
}

// The loop is software-pipelined over the CTA's items: while the record of item k is resolved
// (hash probe -> atomic), the record of item k+1 and the region length/base of item k+2 are
// already in flight, so an item exposes one dependent round trip instead of four.
template <bool GENERIC, bool SHARD>
__global__ void __launch_bounds__(kChunk, UFO_SCATTER_MINBLOCKS) k_scatter(DeviceMap M, ScanArgs a)
{
	if (ld_volatile_u32(&M.ctr->overflow) & 8u) return;
	const uint32_t n_regions = (a.n + 31) / 32;
	const uint32_t n_chunks = ld_volatile_u32(&M.ctr->n_chunks);
	// item (j, r), visited j-major; the iterator advances by gridDim.x items without dividing
	const uint32_t dj = gridDim.x / n_regions, dr = gridDim.x % n_regions;
	uint32_t jA = blockIdx.x / n_regions, rA = blockIdx.x % n_regions;
	// stage 1 (item k+1): region length and base known, record not yet requested
	uint32_t cnt1 = 0, base1 = 0, j1 = jA;
	bool v1 = jA < n_chunks;
	if (v1) {
		cnt1 = a.seg_count[rA];
		base1 = a.seg_base[rA];
	}
	rA += dr;
	jA += dj;
	if (rA >= n_regions) {
		rA -= n_regions;
		++jA;
	}
	// stage 0 (item k): record in registers
	ulonglong2 rec0 = make_ulonglong2(0ull, 0ull);
	bool ok0 = false;
	while (v1 || ok0) {
		// item k+2: region length and base
		const bool v2 = jA < n_chunks;
		const uint32_t j2 = jA;
		uint32_t cnt2 = 0, base2 = 0;
		if (v2) {
			cnt2 = a.seg_count[rA];
			base2 = a.seg_base[rA];
		}
		rA += dr;
		jA += dj;
		if (rA >= n_regions) {
			rA -= n_regions;
			++jA;
		}
		// item k+1: its record (slice j1 counted from the end of the region)
		ulonglong2 rec1 = make_ulonglong2(0ull, 0ull);
		bool ok1 = false;
		if (v1 && (unsigned long long)j1 * kChunk < cnt1) {
			const uint32_t hi = cnt1 - j1 * kChunk;  // one past the slice's last record
			const uint32_t lo = hi > kChunk ? hi - kChunk : 0u;
			ok1 = lo + threadIdx.x < hi;
			if (ok1) rec1 = *reinterpret_cast<const ulonglong2*>(&a.seg[(size_t)base1 + lo + threadIdx.x]);
		}
		// item k
		if (ok0) scatter_record<GENERIC, SHARD>(M, a, rec0);
		rec0 = rec1;
		ok0 = ok1;
		cnt1 = cnt2;
		base1 = base2;
		j1 = j2;
		v1 = v2;
	}
}

// freeSpaceSimple (occupancy_map_base.h:1303-1339): samples at fixed spacing
__global__ void __launch_bounds__(128) k_rays_simple(DeviceMap M, ScanArgs a)
{
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n) return;
	const double* r = a.ray_end + 3 * (size_t)i;
	Vec3 to = {r[0], r[1], r[2]};
	if (to.x != to.x) return;
	Vec3 from = a.origin;
	if (!move_line_inside(M.g, from, to)) return;
	Vec3 cur = to;
	Vec3 dir = vsub(from, to);
	double dist = vnorm(dir);
	dir = vdiv(dir, dist);
	const double size = node_size(M.g, a.depth);
	int num_steps = (int)dop::div(dist, size);
	Vec3 step = vscale(dir, size);
	BrickCache bc = {0, 0, 0, kNone};
	unsigned long long acc = 0;
	uint32_t ox = 0, oy = 0, oz = 0;
	bool have = false;
	unsigned int visits = 0;
	for (int s = 0; s <= num_steps; ++s) {
		Key3 k = point_to_key(M.g, cur, a.depth);
		if (a.depth >= 3) {
			if (a.depth >= 5) collect_node(M, a, k.x & 0x1fffffu, k.y & 0x1fffffu, k.z & 0x1fffffu, a.depth);
			else mark_node_miss(M, k.x & 0x1fffffu, k.y & 0x1fffffu, k.z & 0x1fffffu, a.depth);
			++visits;
			cur = vadd(cur, step);
			continue;
		}
		if (have && ((((k.x ^ ox) | (k.y ^ oy) | (k.z ^ oz)) >> 2) != 0)) {
			flush_block(M, bc, ox, oy, oz, acc);
			acc = 0;
			have = false;
		}
		if (!have) {
			ox = k.x;
			oy = k.y;
			oz = k.z;
			have = true;
		}
		acc |= a.depth == 0 ? voxel_bits<0>(k) : (a.depth == 1 ? voxel_bits<1>(k) : voxel_bits<2>(k));
		++visits;
		cur = vadd(cur, step);
	}
	if (have) flush_block(M, bc, ox, oy, oz, acc);
	if (a.count_visits) atomicAdd(&M.ctr->visits, (unsigned long long)visits);
}

// ---------------------------------------------------------------------------
// Out-of-tree keys (rare; launched only when a scan produced any)
// ---------------------------------------------------------------------------
// The reference applies to a voxel every hit of the scan first and every miss afterwards
// (occupancy_map_base.h:1351-1365).  With aliases a voxel can receive several of each, so
//   k_alias_apply(hits)   runs BEFORE k_update  (alias hits, then the voxel's own hit),
//   k_alias_apply(misses) runs AFTER  k_update  (the voxel's own miss, then alias misses),
// which is "all hits, then all misses" again; equal updates commute.  k_alias_refresh then
// recomputes the aggregates of the wrapped blocks from their leaves and clears the masks.
__device__ __forceinline__ void atomic_apply(const DeviceMap& M, float* addr, float u)
{
	uint32_t* p = reinterpret_cast<uint32_t*>(addr);
	uint32_t old = *reinterpret_cast<volatile uint32_t*>(p);
	while (true) {
		const uint32_t nv = __float_as_uint(apply_update(M, __uint_as_float(old), u));
		const uint32_t prev = atomicCAS(p, old, nv);
		if (prev == old) break;
		old = prev;
	}
}

// one thread per (touched alias brick, child block), grid-stride over the scan's touched list
__global__ void __launch_bounds__(256) k_alias_apply(DeviceMap M, float upd, int hits)
{
	if ((__ldg(&M.ctr->overflow) & ~4u) || !__ldg(&M.ctr->alias_marks)) return;
	const size_t n = (size_t)__ldg(&M.ctr->n_touched) * 64;
	for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
		const uint32_t brick = M.touched[e >> 6];
		const size_t b = (size_t)brick * 64 + (e & 63);
		uint32_t tx, ty, tz;
		if (!alias_source(M, brick, tx, ty, tz)) continue;
		unsigned long long m = (hits ? M.alias_hit : M.alias_miss)[b];
		if (!m) continue;
		const uint32_t dst = brick_find(M, pack_key(tx, ty, tz));
		if (dst == kNone) continue;
		float* leaf = M.leaf + ((size_t)dst * 64 + (b & 63)) * 64;
		while (m) {
			const uint32_t bit = __ffsll((long long)m) - 1;
			m &= m - 1;
			// mask bit order is linear (x + 4y + 16z), leaves are in Morton order
			atomic_apply(M, leaf + morton2(bit & 3u, (bit >> 2) & 3u, bit >> 4), upd);
		}
	}
}

// one thread per (touched alias brick, child block): recompute the wrapped block's aggregates
__global__ void __launch_bounds__(256) k_alias_refresh(DeviceMap M)
{
	if ((__ldg(&M.ctr->overflow) & ~4u) || !__ldg(&M.ctr->alias_marks)) return;
	const size_t n = (size_t)__ldg(&M.ctr->n_touched) * 64;
	for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
		const uint32_t brick = M.touched[e >> 6];
		const size_t b = (size_t)brick * 64 + (e & 63);
		uint32_t tx, ty, tz;
		if (!alias_source(M, brick, tx, ty, tz)) continue;
		if (!(M.alias_hit[b] | M.alias_miss[b])) continue;
		M.alias_hit[b] = 0ull;
		M.alias_miss[b] = 0ull;
		const uint32_t dst = brick_find(M, pack_key(tx, ty, tz));
		if (dst == kNone) continue;
		const size_t tb = (size_t)dst * 64 + (b & 63);
		const float* leaf = M.leaf + tb * 64;
		float om[8];
		uint32_t meta = 0;
		for (int o = 0; o < 8; ++o) {
			float omax = -3.402823466e+38f;
			uint32_t ofl = 0;
			for (int j = 0; j < 8; ++j) {
				const float v = *reinterpret_cast<const volatile float*>(&leaf[8 * o + j]);
				omax = fmaxf(omax, v);
				ofl |= leaf_flags(M, v);
			}
			om[o] = omax;
			meta |= ofl << (2 * o);
		}
		// every octet now holds real values; several sources refreshing one target write the same
		M.line_max[tb] = line_maxima(om);
		M.meta[tb] = meta | 0xff0000u | (M.scan_id << 24);
		if (M.color) {
			// the wrapped leaves' colours changed too (k_wrapped_colors): depth 1 and 2 colours
			const volatile uint32_t* lrgb = M.leaf_rgb + tb * 64;
			uint32_t oc[8];
			for (int o = 0; o < 8; ++o) {
				uint32_t c[8];
				for (int j = 0; j < 8; ++j) c[j] = lrgb[8 * o + j];
				oc[o] = rms_rgb(c, 8);
				M.sum1_rgb[tb * 8 + o] = oc[o];
			}
			M.rgb2[tb] = rms_rgb(oc, 8);
		}
	}
}

// ---------------------------------------------------------------------------
// K4: upper levels (depth >= 5)
// ---------------------------------------------------------------------------
// Push-up propagation.  A node that changed reports its aggregate into its parent's child slot
// and puts the parent on the next level's dirty list; a dirty node is recomputed from its eight
// child slots (one 64-byte read by eight lanes), never from hash lookups.  Parent slots are
// resolved through the hash once and cached (brick_parent / up_parent).
__device__ __forceinline__ void report_to_parent(const DeviceMap& M, uint32_t p, uint32_t ci, Agg a, uint32_t rgb,
                                                 uint32_t* out, uint32_t* out_count, uint32_t list_cap)
{
	*reinterpret_cast<volatile unsigned long long*>(&M.up_child[(size_t)p * 8 + ci]) =
	    (unsigned long long)__float_as_uint(a.occ) | ((unsigned long long)a.flags << 32);
	if (M.color) st_volatile_u32(&M.up_child_rgb[(size_t)p * 8 + ci], rgb);
	if (!((ld_volatile_u32(&M.up_valid[p]) >> ci) & 1u)) atomicOr(&M.up_valid[p], 1u << ci);
	if (atomicExch(&M.up_stamp[p], M.up_epoch) != M.up_epoch) {
		const uint32_t idx = atomicAdd(out_count, 1u);
		if (idx < list_cap) out[idx] = p;
	}
}

// Seeds the depth-5 dirty list from the bricks touched this scan.  Grid-stride over the touched
// list; the pass is identified by M.up_epoch (a pass repeated after the upper-node pool was
// regrown gets a fresh epoch, so every node is listed again).
__global__ void __launch_bounds__(256) k_upper_seed(DeviceMap M, uint32_t* list, uint32_t list_cap)
{
	if (__ldg(&M.ctr->overflow)) return;
	const uint32_t n = __ldg(&M.ctr->n_touched);
	for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
		const uint32_t b = M.touched[e];
		uint32_t x, y, z;
		unpack_key(M.brick_key[b], x, y, z);
		if ((x | y | z) & ~(M.g.key_mask >> 4)) continue;  // alias collector brick
		uint32_t p = M.brick_parent[b];
		if (p == kNone) {
			p = upper_find_or_create(M, upper_key(5, x >> 1, y >> 1, z >> 1));
			if (p == kNone) continue;
			M.brick_parent[b] = p;
		}
		report_to_parent(M, p, (x & 1u) | ((y & 1u) << 1) | ((z & 1u) << 2), M.brick_sum4[b], M.color ? M.brick_rgb4[b] : 0u, list,
		                 &M.ctr->list_count[5 % 3], list_cap);
	}
}

// Paired pass, after K4: the upper nodes above the bricks of one of its scans (`second`: touched_mi2),
// which is what K4 of that scan alone would have recomputed.  Each node is counted by the first
// thread that stamps it with `epoch`, an id no propagation pass uses; a thread stops at a node
// stamped before it, whose ancestors are counted already.
__global__ void __launch_bounds__(256) k_upper_count(DeviceMap M, uint32_t second, uint32_t epoch)
{
	if (__ldg(&M.ctr->overflow)) return;
	const uint32_t n = __ldg(&M.ctr->n_touched);
	unsigned long long cnt = 0;
	for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
		if ((second ? M.touched_mi2[e] : M.touched_mi[e]) == kMiAbsent) continue;
		for (uint32_t p = M.brick_parent[M.touched[e]]; p != kNone && atomicExch(&M.up_stamp[p], epoch) != epoch;
		     p = ld_volatile_u32(&M.up_parent[p]))
			++cnt;
	}
	cnt = __reduce_add_sync(0xffffffffu, (uint32_t)cnt);
	if ((threadIdx.x & 31) == 0 && cnt) atomicAdd(&M.ctr->upper_pair[second], cnt);
}

// Recomputes the nodes of `in` (all at depth d) from their child slots and reports them to their
// parents (-> `out`).  Eight lanes per node, one child each.  Counters rotate three ways:
// level d reads list_count[d % 3], appends to [(d + 1) % 3] and clears [(d + 2) % 3]
// (the next level's output), so no separate reset launches are needed.
__device__ __forceinline__ void upper_level_pass(const DeviceMap& M, uint32_t depth, const uint32_t* in,
                                                 uint32_t* out, uint32_t list_cap, uint32_t n,
                                                 uint32_t gid, uint32_t stride)
{
	const uint32_t lane8 = threadIdx.x & 7;
	uint32_t* out_count = &M.ctr->list_count[(depth + 1) % 3];
	// n is uniform, groups of 8 lanes stay together
	for (uint32_t i = gid; i < ((n + 3) & ~3u); i += stride) {
		bool valid = i < n;
		uint32_t s = valid ? ld_volatile_u32(&in[i]) : 0;
		float occ = 0.0f;
		uint32_t fl = M.default_flags, rgb = 0;
		unsigned long long nkey = 0;
		uint32_t npar = kNone;
		if (valid) {
			// everything this node needs is requested at once (one round trip per level, not four).
			// volatile: in k_upper_tail the slots were written by this same CTA a level earlier
			const uint32_t vmask = ld_volatile_u32(&M.up_valid[s]);
			const unsigned long long raw = ld_volatile_u64(reinterpret_cast<const unsigned long long*>(&M.up_child[(size_t)s * 8 + lane8]));
			const uint32_t crgb1 = M.color ? ld_volatile_u32(&M.up_child_rgb[(size_t)s * 8 + lane8]) : 0u;
			if (lane8 == 0) {
				nkey = ld_volatile_u64(&M.up_key[s]);
				npar = ld_volatile_u32(&M.up_parent[s]);
			}
			if ((vmask >> lane8) & 1u) {
				occ = __uint_as_float((uint32_t)raw);
				fl = (uint32_t)(raw >> 32);
				rgb = crgb1;
			}
		}
		uint32_t crgb[8];
		if (M.color) {
#pragma unroll
			for (int j = 0; j < 8; ++j) crgb[j] = __shfl_sync(0xffffffffu, rgb, (threadIdx.x & 24) + j);
		}
#pragma unroll
		for (int o = 1; o < 8; o <<= 1) {
			occ = fmaxf(occ, __shfl_xor_sync(0xffffffffu, occ, o));
			fl |= __shfl_xor_sync(0xffffffffu, fl, o);
		}
		if (valid && lane8 == 0) {
			const uint32_t my_rgb = M.color ? rms_rgb(crgb, 8) : 0u;
			M.up_agg[s] = {occ, fl};
			if (M.color) M.up_rgb[s] = my_rgb;
			atomicAdd(&M.ctr->upper_nodes, 1ull);
			if (depth < M.g.depth_levels) {
				uint32_t x, y, z;
				unpack_key(nkey, x, y, z);
				x &= 0xffffu;  // strip the depth tag
				uint32_t p = npar;
				if (p == kNone) {
					p = upper_find_or_create(M, upper_key(depth + 1, x >> 1, y >> 1, z >> 1));
					if (p != kNone) st_volatile_u32(&M.up_parent[s], p);
				}
				if (p != kNone) report_to_parent(M, p, (x & 1u) | ((y & 1u) << 1) | ((z & 1u) << 2), {occ, fl}, my_rgb, out, out_count, list_cap);
			}
		}
	}
}

__global__ void __launch_bounds__(256) k_upper_level(DeviceMap M, uint32_t depth, const uint32_t* in,
                                                     uint32_t* out, uint32_t list_cap)
{
	uint32_t n = ld_volatile_u32(&M.ctr->list_count[depth % 3]);
	if (n > list_cap) n = list_cap;
	if (blockIdx.x == 0 && threadIdx.x == 0) M.ctr->list_count[(depth + 2) % 3] = 0;
	upper_level_pass(M, depth, in, out, list_cap, n, (blockIdx.x * blockDim.x + threadIdx.x) >> 3,
	                 (gridDim.x * blockDim.x) >> 3);
}

// Levels first..L in ONE CTA: the dirty lists above depth ~7 hold a few hundred nodes,
// so a launch per level would be pure launch latency.
__global__ void __launch_bounds__(1024) k_upper_tail(DeviceMap M, uint32_t first, uint32_t* list0,
                                                     uint32_t* list1, uint32_t list_cap)
{
	for (uint32_t depth = first; depth <= M.g.depth_levels; ++depth) {
		uint32_t n = ld_volatile_u32(&M.ctr->list_count[depth % 3]);
		if (n > list_cap) n = list_cap;
		if (threadIdx.x == 0) M.ctr->list_count[(depth + 2) % 3] = 0;
		const uint32_t* in = (depth & 1) ? list0 : list1;
		uint32_t* out = (depth & 1) ? list1 : list0;
		upper_level_pass(M, depth, in, out, list_cap, n, threadIdx.x >> 3, blockDim.x >> 3);
		__threadfence();
		__syncthreads();
	}
}

// ---------------------------------------------------------------------------
// utility kernels
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_rebuild_brick_hash(DeviceMap M, uint32_t n_bricks)
{
	uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= n_bricks) return;
	unsigned long long key = M.brick_key[b];
	uint32_t i = hash_u64(key) & M.bh_mask & ~1u;
	while (true) {
		unsigned long long k = atomicCAS(&M.bh_tab[i].x, kEmptyKey, key);
		if (k == kEmptyKey) {
			M.bh_tab[i].y = b;
			return;
		}
		i = (i + 1) & M.bh_mask;
	}
}

__global__ void __launch_bounds__(256) k_rebuild_upper_hash(DeviceMap M, uint32_t n_upper)
{
	uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= n_upper) return;
	unsigned long long key = M.up_key[b];
	uint32_t i = hash_u64(key) & M.uh_mask;
	while (true) {
		unsigned long long k = atomicCAS(&M.uh_keys[i], kEmptyKey, key);
		if (k == kEmptyKey) {
			M.uh_vals[i] = b;
			return;
		}
		i = (i + 1) & M.uh_mask;
	}
}

// value-field export: one thread per voxel of every block of every brick
__global__ void __launch_bounds__(256) k_export(DeviceMap M, uint32_t n_bricks, unsigned long long* codes,
                                                float* occ, uint32_t* rgb, unsigned long long cap,
                                                unsigned long long* count)
{
	size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	const size_t blk = t >> 6;
	const uint32_t v = (uint32_t)(t & 63);
	bool emit = false;
	float o = 0.0f;
	uint32_t c = 0;
	if (blk < (size_t)n_bricks * 64 && (M.meta[blk] >> 16)) {
		o = M.leaf[blk * 64 + v];
		c = M.color ? M.leaf_rgb[blk * 64 + v] : 0u;
		emit = (o != 0.0f) || (c != 0u);
	}
	uint32_t ballot = __ballot_sync(0xffffffffu, emit);
	if (!ballot) return;
	unsigned long long base = 0;
	uint32_t lane = threadIdx.x & 31;
	if (lane == 0) base = atomicAdd(count, (unsigned long long)__popc(ballot));
	base = __shfl_sync(0xffffffffu, base, 0);
	if (!emit || !codes) return;
	unsigned long long idx = base + __popc(ballot & ((1u << lane) - 1u));
	if (idx >= cap) return;
	uint32_t bx, by, bz;
	unpack_key(M.brick_key[blk >> 6], bx, by, bz);
	// child and voxel indices are Morton: de-interleave 2 bits per axis
	const uint32_t ch = (uint32_t)(blk & 63);
	uint32_t cx = (ch & 1u) | ((ch >> 2) & 2u), cy = ((ch >> 1) & 1u) | ((ch >> 3) & 2u),
	         cz = ((ch >> 2) & 1u) | ((ch >> 4) & 2u);
	uint32_t vx = (v & 1u) | ((v >> 2) & 2u), vy = ((v >> 1) & 1u) | ((v >> 3) & 2u),
	         vz = ((v >> 2) & 1u) | ((v >> 4) & 2u);
	codes[idx] = key_to_code({(bx << 4) | (cx << 2) | vx, (by << 4) | (cy << 2) | vy, (bz << 4) | (cz << 2) | vz});
	occ[idx] = o;
	if (rgb) rgb[idx] = c;
}

// Change detection read-out: the codes, at `depth` (0..4), of the nodes that hold a voxel whose
// value changed since the last reset (the reference's changes_ set, occupancy_map_base.h:1070,
// :1094, :1106).  One thread per block; a node shared by several blocks of a warp is emitted by
// its first changed block.  Codes carry the centre bits a Code built from a depth-d Key has
// (octree.h:317-324).  Nodes of depth 4 can be emitted twice (one per half brick): the host
// removes duplicates.
__global__ void __launch_bounds__(256) k_changed(DeviceMap M, uint32_t n_bricks, uint32_t depth,
                                                 unsigned long long* codes, unsigned long long cap,
                                                 unsigned long long* count)
{
	const size_t blk = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t lane = threadIdx.x & 31;
	unsigned long long m = 0ull;
	if (blk < (size_t)n_bricks * 64) m = M.chg_mask[blk];
	// how many codes this thread emits
	uint32_t n = 0, t8 = 0;
	if (depth == 0) {
		n = __popcll(m);
	} else if (depth == 1) {
		for (uint32_t o = 0; o < 8; ++o) {
			const uint32_t base = ((o & 1u) << 1) | ((o & 2u) << 2) | ((o & 4u) << 3);
			t8 |= (((m >> base) & 0x330033ull) ? 1u : 0u) << o;
		}
		n = __popc(t8);
	} else if (depth == 2) {
		n = m ? 1u : 0u;
	} else {
		const uint32_t any = __ballot_sync(0xffffffffu, m != 0ull);
		const uint32_t grp = depth == 3 ? (0xffu << (lane & 24)) : 0xffffffffu;
		n = (m != 0ull && (any & grp & ((1u << lane) - 1u)) == 0u) ? 1u : 0u;
	}
	if (!n) return;
	const unsigned long long at = atomicAdd(count, (unsigned long long)n);
	if (!codes) return;
	uint32_t bx, by, bz;
	unpack_key(M.brick_key[blk >> 6], bx, by, bz);
	const uint32_t ch = (uint32_t)(blk & 63);
	const uint32_t cx = (ch & 1u) | ((ch >> 2) & 2u), cy = ((ch >> 1) & 1u) | ((ch >> 3) & 2u),
	               cz = ((ch >> 2) & 1u) | ((ch >> 4) & 2u);
	const uint32_t x0 = (bx << 4) | (cx << 2), y0 = (by << 4) | (cy << 2), z0 = (bz << 4) | (cz << 2);
	const uint32_t centre = depth ? (1u << (depth - 1)) : 0u, snap = ~((1u << depth) - 1u);
	unsigned long long k = at;
	if (depth == 0) {
		while (m) {
			const uint32_t bit = __ffsll((long long)m) - 1;
			m &= m - 1;
			if (k < cap) codes[k] = key_to_code({x0 | (bit & 3u), y0 | ((bit >> 2) & 3u), z0 | (bit >> 4)});
			++k;
		}
	} else if (depth == 1) {
		while (t8) {
			const uint32_t o = __ffs(t8) - 1;
			t8 &= t8 - 1;
			if (k < cap) codes[k] = key_to_code({x0 | ((o & 1u) << 1) | 1u, y0 | (o & 2u) | 1u, z0 | ((o & 4u) >> 1) | 1u});
			++k;
		}
	} else if (k < cap) {
		codes[k] = key_to_code({(x0 & snap) | centre, (y0 & snap) | centre, (z0 & snap) | centre});
	}
}

// value of node (key, depth) with the intended getNode semantics: the aggregate the map keeps
// for it, the default (0.0, unknown) where nothing was ever written
__device__ __forceinline__ void node_value(const DeviceMap& M, Key3 k, uint32_t d, float& o, uint32_t& f, uint32_t& c)
{
	k.x &= M.g.key_mask;
	k.y &= M.g.key_mask;
	k.z &= M.g.key_mask;
	o = 0.0f;
	f = M.default_flags;
	c = 0;
	if (d >= 5) {
		if (d <= M.g.depth_levels) {
			uint32_t s = upper_find(M, upper_key(d, k.x >> d, k.y >> d, k.z >> d));
			if (s != kNone) {
				o = M.up_agg[s].occ;
				f = M.up_agg[s].flags;
				if (M.color) c = M.up_rgb[s];
			}
		}
		return;
	}
	uint32_t brick = brick_find(M, pack_key(k.x >> 4, k.y >> 4, k.z >> 4));
	if (brick == kNone) return;
	if (d == 4) {
		o = M.brick_sum4[brick].occ;
		f = M.brick_sum4[brick].flags;
		if (M.color) c = M.brick_rgb4[brick];
	} else if (d == 3) {
		uint32_t j = ((k.x >> 3) & 1u) | (((k.y >> 3) & 1u) << 1) | (((k.z >> 3) & 1u) << 2);
		o = M.brick_sum3[(size_t)brick * 8 + j].occ;
		f = M.brick_sum3[(size_t)brick * 8 + j].flags;
		if (M.color) c = M.brick_rgb3[(size_t)brick * 8 + j];
	} else {
		const size_t slot = (size_t)brick * 64 + morton2(k.x >> 2, k.y >> 2, k.z >> 2);
		const uint32_t meta = M.meta[slot];
		if (!(meta >> 16)) return;
		if (d == 2) {
			o = block_occ(M.line_max[slot]);
			f = block_flags(M, meta);
			if (M.color) c = M.rgb2[slot];
		} else if (d == 1) {
			uint32_t j = ((k.x >> 1) & 1u) | (((k.y >> 1) & 1u) << 1) | (((k.z >> 1) & 1u) << 2);
			if ((meta >> (16 + j)) & 1u) {
				o = octet_occ(M.leaf + slot * 64 + 8 * j);
				f = (meta >> (2 * j)) & 3u;
				if (M.color) c = M.sum1_rgb[slot * 8 + j];
			}
		} else {
			uint32_t v = morton2(k.x, k.y, k.z);
			o = M.leaf[slot * 64 + v];
			f = leaf_flags(M, o);
			if (M.color) c = M.leaf_rgb[slot * 64 + v];
		}
	}
}

// node queries with the intended getNode semantics
__global__ void __launch_bounds__(256) k_query(DeviceMap M, const unsigned long long* codes,
                                               const uint32_t* depths, uint32_t n, float* occ,
                                               uint8_t* flags, uint32_t* rgb)
{
	uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	float o;
	uint32_t f, c;
	node_value(M, code_to_key(codes[i]), depths[i], o, f, c);
	occ[i] = o;
	flags[i] = (uint8_t)f;
	if (rgb) rgb[i] = c;
}

// castRay (occupancy_map_base.h:449-486, intended semantics -- DESIGN.md section 8 states them):
// one thread per ray, forward walk at `depth` from the origin's node; an occupied node is the
// hit, an unknown one stops the ray unless ignore_unknown.  rays: [n][6] = origin, direction.
__global__ void __launch_bounds__(128) k_cast_rays(DeviceMap M, const double* rays, uint32_t n, int ignore_unknown,
                                                   double max_range, uint32_t depth, unsigned long long* codes,
                                                   uint8_t* hit)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const double* r = rays + 6 * (size_t)i;
	Vec3 o = {r[0], r[1], r[2]}, d = {r[3], r[4], r[5]};
	if (0 > max_range) {
		const double hs = node_half(M.g, M.g.depth_levels), e = dop::add(hs, hs);
		max_range = vnorm({e, e, e});
	}
	d = vdiv(d, vnorm(d));
	Vec3 e = vadd(o, vscale(d, max_range));
	unsigned long long code = 0;
	uint8_t h = 0;
	if (move_line_inside(M.g, o, e)) {
		Walk w;
		walk_init(M.g, o, e, d, depth, w);
		while (true) {
			float occ;
			uint32_t f, c;
			node_value(M, w.cur, depth, occ, f, c);
			const bool last = w.same || w.cur == w.end || !(walk_tmin(w) <= max_range);
			if (M.occ_thr < (double)occ) {
				code = key_to_code({w.cur.x & 0x1fffffu, w.cur.y & 0x1fffffu, w.cur.z & 0x1fffffu});
				h = 1;
				break;
			}
			if (last) break;
			if (!ignore_unknown && M.free_thr <= (double)occ && M.occ_thr >= (double)occ) break;
			walk_step(w);
		}
	}
	codes[i] = code;
	hit[i] = h;
}

}  // namespace ufo_b200
