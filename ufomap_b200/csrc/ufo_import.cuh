// ufo_import.cuh -- Octree::readData (octree.h:733-770) / readNodes (occupancy_map_base.h:1379-1456)
// on the value field: a node stream (file body, or a UFOMap message as the ROS layer merges it,
// ufomap_msgs/conversions.h:122-134) is parsed on the host into LEAF RECORDS -- (node code, depth,
// payload): "every voxel below this node takes this value" (deleteChildren + readData + updateNode)
// -- and applied here.  Records of depth <= 2 are written by one thread each, whole bricks by one
// CTA each, default-payload nodes above the brick level wipe the existing bricks below them; the
// depth 1-4 aggregates of every touched brick are then rebuilt from its leaves and the usual
// propagation pass (k_upper_*) follows.
//
// On a routed map every rank takes the same stream and applies the records of the bricks it owns
// (brick_owned): a foreign record is skipped before its brick is found or created, and a wipe
// leaves the foreign bricks a rank holds alone, so the ranks keep disjoint bricks whose union is
// the single map that read the stream.
#pragma once

#include "ufo_kernels.cuh"

namespace ufo_b200
{
struct ImportRec {
	unsigned long long code;  // Morton code of the node's first voxel
	uint32_t depth;
	float occ;
	uint32_t rgb;
	uint32_t pad;
};

// key of the brick that holds a record's first voxel
UFO_HD uint64_t record_brick(unsigned long long code)
{
	const Key3 k = code_to_key(code);
	return pack_key(k.x >> 4, k.y >> 4, k.z >> 4);
}

// records of depth 0..2: one thread each
__global__ void __launch_bounds__(256) k_import_small(DeviceMap M, const ImportRec* recs, uint32_t n)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const ImportRec r = recs[i];
		const uint64_t key = record_brick(r.code);
		if (!brick_owned(M, key)) continue;
		const uint32_t brick = brick_find_or_create(M, key);
		if (brick == kNone) continue;
		const Key3 k = code_to_key(r.code);
		touch_brick(M, brick);
		const size_t b = (size_t)brick * 64 + morton2(k.x >> 2, k.y >> 2, k.z >> 2);
		float* leaf = M.leaf + b * 64;
		uint32_t* lrgb = M.color ? M.leaf_rgb + b * 64 : nullptr;
		if (r.depth == 0) {
			const uint32_t v = morton2(k.x, k.y, k.z);
			leaf[v] = r.occ;
			if (lrgb) lrgb[v] = r.rgb;
			atomicOr(&M.meta[b], 1u << (16 + (v >> 3)));
		} else if (r.depth == 1) {
			const uint32_t o = morton2(k.x, k.y, k.z) >> 3;
			for (uint32_t j = 0; j < 8; ++j) {
				leaf[8 * o + j] = r.occ;
				if (lrgb) lrgb[8 * o + j] = r.rgb;
			}
			atomicOr(&M.meta[b], 1u << (16 + o));
		} else {
			for (uint32_t j = 0; j < 64; ++j) {
				leaf[j] = r.occ;
				if (lrgb) lrgb[j] = r.rgb;
			}
			atomicOr(&M.meta[b], 0xff0000u);
		}
	}
}

// whole bricks (depth-4 records): one CTA of 64 threads per record, one block per thread
__global__ void __launch_bounds__(64) k_import_bricks(DeviceMap M, const ImportRec* recs, uint32_t n)
{
	__shared__ uint32_t s_brick;
	for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
		const ImportRec r = recs[i];
		if (threadIdx.x == 0) {
			const uint64_t key = record_brick(r.code);
			const uint32_t brick = brick_owned(M, key) ? brick_find_or_create(M, key) : kNone;
			if (brick != kNone) touch_brick(M, brick);
			s_brick = brick;
		}
		__syncthreads();
		const uint32_t brick = s_brick;
		if (brick != kNone) {
			const size_t b = (size_t)brick * 64 + threadIdx.x;
			float4* leaf = reinterpret_cast<float4*>(M.leaf + b * 64);
			const float4 v = make_float4(r.occ, r.occ, r.occ, r.occ);
			for (int j = 0; j < 16; ++j) leaf[j] = v;
			if (M.color) {
				uint4* c = reinterpret_cast<uint4*>(M.leaf_rgb + b * 64);
				const uint4 cv = make_uint4(r.rgb, r.rgb, r.rgb, r.rgb);
				for (int j = 0; j < 16; ++j) c[j] = cv;
			}
			M.meta[b] = M.meta[b] | 0xff0000u;
		}
		__syncthreads();
	}
}

// nodes above the brick level: every EXISTING brick below one of them takes the node's payload
// (for the default payload this is how a subtree is deleted).  One thread per (brick, block).  A
// routed rank may hold empty foreign bricks (gathered by its fused walk); they stay empty.
__global__ void __launch_bounds__(256) k_import_wipe(DeviceMap M, uint32_t n_bricks, const ImportRec* recs, uint32_t n)
{
	const size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= (size_t)n_bricks * 64) return;
	const uint32_t brick = (uint32_t)(b >> 6);
	const uint64_t key = M.brick_key[brick];
	uint32_t x, y, z;
	unpack_key(key, x, y, z);
	if (((x | y | z) & ~(M.g.key_mask >> 4)) || !brick_owned(M, key)) return;
	const unsigned long long code = key_to_code({x << 4, y << 4, z << 4});
	for (uint32_t i = 0; i < n; ++i) {
		const ImportRec r = recs[i];
		if ((code >> (3 * r.depth)) != (r.code >> (3 * r.depth))) continue;
		if ((b & 63) == 0) touch_brick(M, brick);
		float4* leaf = reinterpret_cast<float4*>(M.leaf + b * 64);
		const float4 v = make_float4(r.occ, r.occ, r.occ, r.occ);
		for (int j = 0; j < 16; ++j) leaf[j] = v;
		if (M.color) {
			uint4* c = reinterpret_cast<uint4*>(M.leaf_rgb + b * 64);
			const uint4 cv = make_uint4(r.rgb, r.rgb, r.rgb, r.rgb);
			for (int j = 0; j < 16; ++j) c[j] = cv;
		}
		M.meta[b] = M.meta[b] | 0xff0000u;
	}
}

// pair maxima, octet flags and depth-1 / depth-2 colours of every block of the touched bricks from
// the leaves (initialised octets only); one thread per (touched brick, block)
__global__ void __launch_bounds__(256) k_import_refresh(DeviceMap M)
{
	if (__ldg(&M.ctr->overflow) & ~4u) return;
	const size_t n = (size_t)__ldg(&M.ctr->n_touched) * 64;
	for (size_t e = (size_t)blockIdx.x * blockDim.x + threadIdx.x; e < n; e += (size_t)gridDim.x * blockDim.x) {
		const size_t b = (size_t)M.touched[e >> 6] * 64 + (e & 63);
		const uint32_t mt = M.meta[b];
		if (!(mt & 0xff0000u)) continue;
		const float* leaf = M.leaf + b * 64;
		float om[8];
		uint32_t fl16 = 0;
		uint32_t oc[8];
		for (uint32_t o = 0; o < 8; ++o) {
			om[o] = 0.0f;
			oc[o] = 0;
			if ((mt >> (16 + o)) & 1u) {
				om[o] = octet_occ(leaf + 8 * o);
				uint32_t ofl = 0;
				for (int j = 0; j < 8; ++j) ofl |= leaf_flags(M, leaf[8 * o + j]);
				fl16 |= ofl << (2 * o);
				if (M.color) {
					oc[o] = rms_rgb(M.leaf_rgb + b * 64 + 8 * o, 8);
					M.sum1_rgb[b * 8 + o] = oc[o];
				}
			}
		}
		M.pair_max[b] = make_float4(fmaxf(om[0], om[1]), fmaxf(om[2], om[3]), fmaxf(om[4], om[5]), fmaxf(om[6], om[7]));
		if (M.color) M.rgb2[b] = rms_rgb(oc, 8);
		M.meta[b] = (mt & 0xff0000u) | fl16 | (M.scan_id << 24);
	}
}

}  // namespace ufo_b200
