// ufo_import.cuh -- Octree::readData (octree.h:733-770) / readNodes (occupancy_map_base.h:1379-1456)
// on the value field: a node stream (file body, or a UFOMap message as the ROS layer merges it,
// ufomap_msgs/conversions.h:122-134) is applied here.  The host walks the levels above the bricks
// (ufo_map.cu, import_rec): a leaf there becomes a LEAF RECORD -- (node code, depth, payload):
// "every voxel below this node takes this value" (deleteChildren + readData + updateNode) -- and a
// depth-4 node with children becomes a SUB-STREAM, the node's bytes of the stream, located by
// reading only its children bytes.  Default-payload nodes above the brick level wipe the existing
// bricks below them, depth-4 leaves are written by one CTA each, and every sub-stream is parsed by
// one CTA (k_import_parse); the depth 1-4 aggregates of every touched brick are then rebuilt from
// its leaves and the usual propagation pass (k_upper_*) follows.
//
// On a routed map every rank takes the same stream and applies the records and sub-streams of the
// bricks it owns (brick_owned): a foreign one is skipped before its brick is found or created, and
// a wipe leaves the foreign bricks a rank holds alone, so the ranks keep disjoint bricks whose union
// is the single map that read the stream.
#pragma once

#include "ufo_kernels.cuh"
#include "ufo_export.cuh"

namespace ufo_b200
{
struct ImportRec {
	unsigned long long code;  // Morton code of the node's first voxel
	uint32_t depth;
	float occ;
	uint32_t rgb;
	uint32_t pad;
};

// the stream bytes of one depth-4 node with children, in a chunk of the stream on the device
struct ImportSub {
	unsigned long long code;  // Morton code of the brick's first voxel
	uint32_t off;             // first byte (the node's children byte) in the chunk's data
	uint32_t len;             // bytes, as the host walk counted them
};

// key of the brick that holds a record's first voxel
UFO_HD uint64_t record_brick(unsigned long long code)
{
	const Key3 k = code_to_key(code);
	return pack_key(k.x >> 4, k.y >> 4, k.z >> 4);
}

// a payload of the stream: float occupancy, then (colour maps) r, g, b; byte loads, any alignment
template <bool COLOR>
__device__ __forceinline__ void get_payload(const uint8_t* p, float& occ, uint32_t& rgb)
{
	occ = __uint_as_float((uint32_t)p[0] | ((uint32_t)p[1] << 8) | ((uint32_t)p[2] << 16) | ((uint32_t)p[3] << 24));
	rgb = COLOR ? ((uint32_t)p[4] | ((uint32_t)p[5] << 8) | ((uint32_t)p[6] << 16)) : 0u;
}

// n voxels from leaf / lrgb onward take one payload (n a multiple of 4, 16-byte aligned)
__device__ __forceinline__ void fill_leaves(float* leaf, uint32_t* lrgb, uint32_t n, float occ, uint32_t rgb)
{
	float4* l4 = reinterpret_cast<float4*>(leaf);
	const float4 v = make_float4(occ, occ, occ, occ);
	for (uint32_t j = 0; j < n / 4; ++j) l4[j] = v;
	if (lrgb) {
		uint4* c4 = reinterpret_cast<uint4*>(lrgb);
		const uint4 cv = make_uint4(rgb, rgb, rgb, rgb);
		for (uint32_t j = 0; j < n / 4; ++j) c4[j] = cv;
	}
}

constexpr uint32_t kSubAbsent = 0xffffffffu;  // node outside the volume: no bytes
constexpr uint32_t kSubInner = 1u << 31;      // node offset flag: a children byte, not a payload

// One CTA of 64 threads per sub-stream (one thread per 4^3 block, as k_brick_stream writes them).
// The sub-stream is copied into shared memory; which children the stream holds follows from the
// volume alone (readNodesRecurs skips a child whose cube misses it, the writer did not write it),
// which of them carry children from the children bytes.  One thread walks the at most 1 + 8 + 64
// children bytes in stream order -- a node's bytes depend on every node before it -- and records
// the offset of every depth-3 and depth-2 node, taking the size of a depth-2 node with children
// from its children byte and the per-octet voxel counts; each thread then takes the prefix sums of
// its block's octets and writes its 64 leaves: a leaf above depth 0 broadcasts its payload, a
// depth-1 node with children is its voxels' payloads in Morton order.  Octet "initialised" bits as
// a leaf record of the same node would set them.  A parsed length other than the host's sets
// overflow bit 512 (internal error: never expected).  G: the general volume test (ufo_volume.cuh).
template <bool COLOR, bool G>
__global__ void __launch_bounds__(64) k_import_parse(DeviceMap M, Volume vol, const ImportSub* subs, uint32_t n,
                                                     const uint8_t* data)
{
	__shared__ uint4 s_raw[(kBrickStreamMax + 15) / 16 + 1];  // the sub-stream from a 16-byte boundary on
	__shared__ uint32_t s_d3_off[8], s_blk_off[64];
	__shared__ uint8_t s_d3_hit[8], s_blk_hit[64], s_oct_hit[64], s_vox_n[64][8];
	__shared__ uint32_t s_brick, s_bad;
	__shared__ double s_center[3];
	constexpr uint32_t P = COLOR ? 7u : 4u;
	const uint32_t t = threadIdx.x, j3 = t >> 3, k3 = t & 7u;
	const bool filtered = vol.n != 0;
	for (uint32_t i = blockIdx.x; i < n; i += gridDim.x) {
		const ImportSub sub = subs[i];
		if (t == 0) {
			const Key3 k = code_to_key(sub.code);
			const uint64_t key = pack_key(k.x >> 4, k.y >> 4, k.z >> 4);
			const uint32_t brick = brick_owned(M, key) ? brick_find_or_create(M, key) : kNone;
			if (brick != kNone) touch_brick(M, brick);
			s_brick = brick;
			s_bad = sub.len > (uint32_t)kBrickStreamMax ? 1u : 0u;
			if (filtered) brick_center(M.g, k.x >> 4, k.y >> 4, k.z >> 4, s_center);
		}
		__syncthreads();
		const uint32_t brick = s_brick;
		if (brick != kNone && !s_bad) {
			const uint32_t lead = sub.off & 15u;
			const uint4* src = reinterpret_cast<const uint4*>(data + (sub.off - lead));
			for (uint32_t w = t; w < (lead + sub.len + 15) / 16; w += 64) s_raw[w] = src[w];
			// which cubes of this thread's block the volume keeps
			uint32_t oct_hit = 0xffu;
			bool d3_hit = true, blk_hit = true;
			if (filtered) {
				const double bc[3] = {s_center[0], s_center[1], s_center[2]};
				double d3c[3], blkc[3];
				child_center(bc, M.g.half_size[3], j3, d3c);
				child_center(d3c, M.g.half_size[2], k3, blkc);
				d3_hit = vol_hits_t<G>(vol, d3c, M.g.half_size[3]);
				blk_hit = d3_hit && vol_hits_t<G>(vol, blkc, M.g.half_size[2]);
				oct_hit = 0;
				for (uint32_t o = 0; o < 8; ++o) {
					double oc[3];
					child_center(blkc, M.g.half_size[1], o, oc);
					uint32_t nv = 0;
					if (blk_hit && vol_hits_t<G>(vol, oc, M.g.half_size[1])) {
						oct_hit |= 1u << o;
						for (uint32_t v = 0; v < 8; ++v) {
							double vc[3];
							child_center(oc, M.g.half_size[0], v, vc);
							nv += vol_hits_t<G>(vol, vc, M.g.half_size[0]) ? 1u : 0u;
						}
					}
					s_vox_n[t][o] = (uint8_t)nv;
				}
			} else {
				for (uint32_t o = 0; o < 8; ++o) s_vox_n[t][o] = 8;
			}
			if (k3 == 0) s_d3_hit[j3] = d3_hit ? 1 : 0;
			s_blk_hit[t] = blk_hit ? 1 : 0;
			s_oct_hit[t] = (uint8_t)oct_hit;
		}
		__syncthreads();
		const uint8_t* s = reinterpret_cast<const uint8_t*>(s_raw) + (sub.off & 15u);
		if (brick != kNone && !s_bad && t == 0) {
			// the children bytes in stream order
			uint32_t at = 0;
			bool bad = false;
			auto byte = [&](uint32_t p) -> uint32_t {
				if (p >= sub.len) bad = true;
				return bad ? 0u : s[p];
			};
			const uint32_t c4 = byte(at++);
			for (uint32_t j = 0; j < 8; ++j) {
				s_d3_off[j] = kSubAbsent;
				for (uint32_t k = 0; k < 8; ++k) s_blk_off[8 * j + k] = kSubAbsent;
				if (!s_d3_hit[j]) continue;
				if (!((c4 >> j) & 1u)) {
					s_d3_off[j] = at;
					at += P;
					continue;
				}
				s_d3_off[j] = kSubInner;
				const uint32_t c3 = byte(at++);
				for (uint32_t k = 0; k < 8; ++k) {
					const uint32_t blk = 8 * j + k;
					if (!s_blk_hit[blk]) continue;
					s_blk_off[blk] = at;
					if (!((c3 >> k) & 1u)) {
						at += P;
						continue;
					}
					s_blk_off[blk] |= kSubInner;
					const uint32_t c2 = byte(at++);
					for (uint32_t o = 0; o < 8; ++o)
						if ((s_oct_hit[blk] >> o) & 1u) at += ((c2 >> o) & 1u) ? P * s_vox_n[blk][o] : P;
				}
			}
			if (bad || at != sub.len) {
				s_bad = 1u;
				atomicOr(&M.ctr->overflow, 512u);
			}
		}
		__syncthreads();
		if (brick != kNone && !s_bad) {
			// this block: one payload at leaf_at for all of it, or a children byte at inner_at
			const uint32_t o3 = s_d3_off[j3], o2 = s_blk_off[t];
			uint32_t leaf_at = kSubAbsent, inner_at = kSubAbsent;
			if (o3 != kSubAbsent) {
				if (!(o3 & kSubInner)) leaf_at = o3;
				else if (o2 != kSubAbsent && (o2 & kSubInner)) inner_at = o2 & ~kSubInner;
				else if (o2 != kSubAbsent) leaf_at = o2;
			}
			const size_t b = (size_t)brick * 64 + t;
			float* leaf = M.leaf + b * 64;
			uint32_t* lrgb = COLOR ? M.leaf_rgb + b * 64 : nullptr;
			float occ;
			uint32_t rgb;
			uint32_t init = 0;  // octets written
			if (leaf_at != kSubAbsent) {
				get_payload<COLOR>(s + leaf_at, occ, rgb);
				fill_leaves(leaf, lrgb, 64, occ, rgb);
				init = 0xffu;
			} else if (inner_at != kSubAbsent) {
				const uint32_t c2 = s[inner_at];
				uint32_t at = inner_at + 1;
				for (uint32_t o = 0; o < 8; ++o) {
					if (!((s_oct_hit[t] >> o) & 1u)) continue;
					if (!((c2 >> o) & 1u)) {
						get_payload<COLOR>(s + at, occ, rgb);
						at += P;
						fill_leaves(leaf + 8 * o, COLOR ? lrgb + 8 * o : nullptr, 8, occ, rgb);
						init |= 1u << o;
						continue;
					}
					const uint32_t nv = s_vox_n[t][o];
					if (!nv) continue;
					double oc[3] = {0.0, 0.0, 0.0};
					if (nv != 8) {
						const double bc[3] = {s_center[0], s_center[1], s_center[2]};
						double d3c[3], blkc[3];
						child_center(bc, M.g.half_size[3], j3, d3c);
						child_center(d3c, M.g.half_size[2], k3, blkc);
						child_center(blkc, M.g.half_size[1], o, oc);
					}
					for (uint32_t v = 0; v < 8; ++v) {
						if (nv != 8) {
							double vc[3];
							child_center(oc, M.g.half_size[0], v, vc);
							if (!vol_hits_t<G>(vol, vc, M.g.half_size[0])) continue;
						}
						get_payload<COLOR>(s + at, occ, rgb);
						at += P;
						leaf[8 * o + v] = occ;
						if (COLOR) lrgb[8 * o + v] = rgb;
					}
					init |= 1u << o;
				}
			}
			if (init) M.meta[b] = M.meta[b] | (init << 16);
		}
		__syncthreads();
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

// line maxima, octet flags and depth-1 / depth-2 colours of every block of the touched bricks from
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
		M.line_max[b] = line_maxima(om);
		if (M.color) M.rgb2[b] = rms_rgb(oc, 8);
		M.meta[b] = (mt & 0xff0000u) | fl16 | (M.scan_id << 24);
	}
}

}  // namespace ufo_b200
