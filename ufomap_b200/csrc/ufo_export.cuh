// ufo_export.cuh -- the map in the reference's file/wire format (SURVEY.md 8(f) N2).
//
//   Octree::write / writeData     map/octree.h:833-917   (text header + node stream)
//   writeNodes / writeNodesRecurs map/occupancy_map_base.h:1457-1533
//   node payloads                 map/occupancy_map_node.h:71-75 (float), :106-110 (+3 colour bytes)
//
// The stream is a pre-order walk: one byte per inner node that has children (bit i = child i
// has children), then the children in order -- a recursive record for a child with children, a
// payload for a leaf child; the eight children of a depth-1 node are written as eight payloads
// with no mask byte.  Pre-order over an octree is Morton order, so the stream of a 16^3 brick
// (depth 4 downward) is self-contained: k_brick_stream builds it in shared memory, one CTA per
// brick, one thread per 4^3 block; the host strings the bricks together with the few bytes of
// the levels above (ufo_map.cu, export_image).
//
// Tree shape.  pruned != 0 (the default of the C ABI): the canonical minimal tree of the value
// field -- a node whose eight children are leaves with equal payload is a leaf; untouched space
// is a leaf with the default payload (0.0, no colour).  The reference collapses such nodes itself
// whenever an update passes through them (updateNode, occupancy_map_base.h:1210-1212; with
// automatic pruning off it still marks them is_leaf, octree.h:1060-1066), so its file is this one
// unless its update order left a collapsible node behind (updateParents stops at the first
// unchanged aggregate, :1126-1133).  pruned == 0: every octet that was ever touched ("initialised"
// bits of the block meta word) is written as eight voxels -- value-equivalent, larger.
#pragma once

#include <cuda/std/tuple>

#include "ufo_device.cuh"
#include "ufo_volume.cuh"

namespace ufo_b200
{
constexpr int kBrickStreamMax = 1 + 8 * (1 + 8 * (1 + 64 * 7));  // colour payloads: 28 745 bytes

// Partial / truncated export (Octree::writeData(stream, bounding_volume, false, min_depth),
// octree.h:885-917): children at min_depth are written as leaves carrying their aggregate
// payload; a child whose cube misses the volume is skipped.  The cube test is vol_hits
// (ufo_volume.cuh); node centres are accumulated top-down like getChildCenter
// (octree.h:625-633) so that the comparisons see the same doubles.
UFO_HD void child_center(const double c[3], double hs, uint32_t i, double out[3])
{
	out[0] = dop::add(c[0], (i & 1u) ? hs : -hs);
	out[1] = dop::add(c[1], (i & 2u) ? hs : -hs);
	out[2] = dop::add(c[2], (i & 4u) ? hs : -hs);
}

// The canonical-leaf rule, the one place that decides the tree shape of the file writer and of the
// iteration (k_brick_stream, k_brick_iter, build_upper): a node keeps its children unless none of
// them has children and all eight carry the same payload, colour included.  rgb == nullptr: no colour.
UFO_HD bool keeps_children(bool a_child_has_children, const float* occ, const uint32_t* rgb)
{
	if (a_child_has_children) return true;
	for (int i = 1; i < 8; ++i)
		if (occ[i] != occ[0] || (rgb && rgb[i] != rgb[0])) return true;
	return false;
}

// centre of the brick's cube, accumulated from the root like the reference's recursion
UFO_HD void brick_center(const Geometry& g, uint32_t kx, uint32_t ky, uint32_t kz, double c[3])
{
	c[0] = c[1] = c[2] = 0.0;
	for (uint32_t d = g.depth_levels; d > 4; --d) {
		const uint32_t bit = d - 5;  // brick-key bit that selects the child of the depth-d node
		const uint32_t i = ((kx >> bit) & 1u) | (((ky >> bit) & 1u) << 1) | (((kz >> bit) & 1u) << 2);
		double n[3];
		child_center(c, g.half_size[d - 1], i, n);
		c[0] = n[0];
		c[1] = n[1];
		c[2] = n[2];
	}
}

struct BrickInfo {
	uint32_t size;   // bytes the brick contributes to the stream (0: skipped by the box); k_brick_iter: records
	uint32_t flags;  // bit 0: has children (in the map); bit 1: not part of the map (alias collector);
	                 // bit 2: written as a record (size bytes at its offset), else as a payload
	float occ;       // payload when bit 2 is clear: the leaf value, or the depth-4 aggregate
	uint32_t rgb;
};

template <bool COLOR>
__device__ __forceinline__ void put_payload(uint8_t* p, float occ, uint32_t rgb)
{
	const uint32_t u = __float_as_uint(occ);
	p[0] = (uint8_t)u;
	p[1] = (uint8_t)(u >> 8);
	p[2] = (uint8_t)(u >> 16);
	p[3] = (uint8_t)(u >> 24);
	if (COLOR) {
		p[4] = (uint8_t)rgb;
		p[5] = (uint8_t)(rgb >> 8);
		p[6] = (uint8_t)(rgb >> 16);
	}
}

// One octet of block b: returns its bytes in the stream and writes them when dst != nullptr.
template <bool COLOR, bool G>
__device__ __forceinline__ uint32_t octet_record(const DeviceMap& M, size_t b, uint32_t o, bool has,
                                                 float leaf_occ, uint32_t leaf_rgb, uint32_t min_depth,
                                                 const Volume& bx, const double oc[3], uint8_t* dst)
{
	constexpr uint32_t P = COLOR ? 7u : 4u;
	if (!vol_hits_t<G>(bx, oc, M.g.half_size[1])) return 0;
	if (has && min_depth == 0) {
		uint32_t n = 0;
		for (uint32_t j = 0; j < 8; ++j) {
			double vc[3];
			child_center(oc, M.g.half_size[0], j, vc);
			if (!vol_hits_t<G>(bx, vc, M.g.half_size[0])) continue;
			if (dst) put_payload<COLOR>(dst + n, M.leaf[b * 64 + 8 * o + j], COLOR ? M.leaf_rgb[b * 64 + 8 * o + j] : 0u);
			n += P;
		}
		return n;
	}
	if (dst) {
		if (has) put_payload<COLOR>(dst, octet_occ(M.leaf + b * 64 + 8 * o), COLOR ? M.sum1_rgb[b * 8 + o] : 0u);
		else put_payload<COLOR>(dst, leaf_occ, leaf_rgb);
	}
	return P;
}

// offsets == nullptr: size pass (fills info); otherwise the record of every brick whose info has
// bit 2 set is written to out + offsets[brick].
template <bool COLOR, bool G>
__global__ void __launch_bounds__(64) k_brick_stream(DeviceMap M, uint32_t n_bricks, int pruned, uint32_t min_depth,
                                                     Volume bx, BrickInfo* info,
                                                     const unsigned long long* offsets, uint8_t* out)
{
	extern __shared__ uint8_t s_buf[];
	__shared__ uint32_t s_blk_size[64], s_blk_rgb[64], s_d3_size[8], s_d3_rgb[8], s_d3_off[8];
	__shared__ float s_blk_occ[64], s_d3_occ[8];
	__shared__ uint8_t s_blk_has[64], s_d3_has[8], s_d3_mask[8], s_d3_hit[8];
	__shared__ uint32_t s_brick_size, s_brick_record;
	__shared__ double s_center[3];
	constexpr uint32_t P = COLOR ? 7u : 4u;
	const uint32_t brick = blockIdx.x, t = threadIdx.x;
	if (brick >= n_bricks) return;
	uint32_t kx, ky, kz;
	unpack_key(M.brick_key[brick], kx, ky, kz);
	if ((kx | ky | kz) & ~(M.g.key_mask >> 4)) {  // collects out-of-tree marks, owns no voxels
		if (!offsets && t == 0) info[brick] = {0u, 2u, 0.0f, 0u};
		return;
	}
	if (t == 0) {
		double c[3];
		brick_center(M.g, kx, ky, kz, c);
		s_center[0] = c[0];
		s_center[1] = c[1];
		s_center[2] = c[2];
	}
	__syncthreads();
	const uint32_t j3 = t >> 3, k3 = t & 7u;
	double bc[3], d3c[3], blkc[3];
	bc[0] = s_center[0];
	bc[1] = s_center[1];
	bc[2] = s_center[2];
	child_center(bc, M.g.half_size[3], j3, d3c);
	child_center(d3c, M.g.half_size[2], k3, blkc);
	const bool brick_hit = vol_hits_t<G>(bx, bc, M.g.half_size[4]);
	const bool d3_hit = vol_hits_t<G>(bx, d3c, M.g.half_size[3]);
	const bool blk_hit = vol_hits_t<G>(bx, blkc, M.g.half_size[2]);

	const size_t b = (size_t)brick * 64 + t;
	const uint32_t init8 = (M.meta[b] >> 16) & 0xffu;
	// octets in the map: has children, or a leaf with one payload
	uint32_t oct_has = 0;
	float oocc[8];
	uint32_t orgb[8];
#pragma unroll
	for (uint32_t o = 0; o < 8; ++o) {
		oocc[o] = 0.0f;
		orgb[o] = 0u;
		if (!((init8 >> o) & 1u)) continue;
		if (!pruned) {
			oct_has |= 1u << o;
			continue;
		}
		const float* lp = M.leaf + b * 64 + 8 * o;
		const uint32_t* cp = COLOR ? M.leaf_rgb + b * 64 + 8 * o : nullptr;
		if (keeps_children(false, lp, cp)) {
			oct_has |= 1u << o;
		} else {
			oocc[o] = lp[0];
			orgb[o] = COLOR ? cp[0] : 0u;
		}
	}
	const bool blk_has = pruned ? keeps_children(oct_has != 0, oocc, orgb) : oct_has != 0;
	// the block's contribution to the stream
	uint32_t blk_size = 0;
	if (blk_hit && d3_hit && brick_hit) {
		if (blk_has && min_depth < 2) {
			blk_size = 1;
#pragma unroll
			for (uint32_t o = 0; o < 8; ++o) {
				double oc[3];
				child_center(blkc, M.g.half_size[1], o, oc);
				blk_size += octet_record<COLOR, G>(M, b, o, (oct_has >> o) & 1u, oocc[o], orgb[o], min_depth, bx, oc, nullptr);
			}
		} else {
			blk_size = P;
		}
	}
	s_blk_has[t] = blk_has ? 1 : 0;
	s_blk_size[t] = blk_size;
	// payload when the block is written as a leaf: its value, or its depth-2 aggregate
	s_blk_occ[t] = blk_has ? block_occ(M.line_max[b]) : oocc[0];
	s_blk_rgb[t] = blk_has ? (COLOR ? M.rgb2[b] : 0u) : orgb[0];
	__syncthreads();
	if (t < 8) {
		double c3[3];
		child_center(bc, M.g.half_size[3], t, c3);
		const bool hit = brick_hit && vol_hits_t<G>(bx, c3, M.g.half_size[3]);
		bool has = false;
		uint32_t size = 1, mask = 0;
		for (int k = 0; k < 8; ++k) {
			const int c = 8 * t + k;
			has = has || s_blk_has[c];
			if (min_depth < 2) mask |= (uint32_t)s_blk_has[c] << k;
			size += s_blk_size[c];
		}
		// leaf blocks only reach the payload test: s_blk_occ / s_blk_rgb hold their leaf payloads
		if (pruned) has = keeps_children(has, s_blk_occ + 8 * t, s_blk_rgb + 8 * t);
		s_d3_has[t] = has ? 1 : 0;
		s_d3_hit[t] = hit ? 1 : 0;
		s_d3_mask[t] = (uint8_t)mask;
		s_d3_size[t] = !hit ? 0u : ((has && min_depth < 3) ? size : P);
		s_d3_occ[t] = has ? M.brick_sum3[(size_t)brick * 8 + t].occ : s_blk_occ[8 * t];
		s_d3_rgb[t] = has ? (COLOR ? M.brick_rgb3[(size_t)brick * 8 + t] : 0u) : s_blk_rgb[8 * t];
	}
	__syncthreads();
	if (t == 0) {
		bool has = false;
		uint32_t size = 1;
		for (int j = 0; j < 8; ++j) {
			has = has || s_d3_has[j];
			s_d3_off[j] = size;
			size += s_d3_size[j];
		}
		if (pruned) has = keeps_children(has, s_d3_occ, s_d3_rgb);
		const bool record = has && min_depth < 4 && brick_hit;
		s_brick_record = record ? 1u : 0u;
		s_brick_size = !brick_hit ? 0u : (record ? size : P);
		if (!offsets) {
			const float occ = has ? M.brick_sum4[brick].occ : s_d3_occ[0];
			const uint32_t rgb = has ? (COLOR ? M.brick_rgb4[brick] : 0u) : s_d3_rgb[0];
			info[brick] = {s_brick_size, (has ? 1u : 0u) | (record ? 4u : 0u), occ, rgb};
		}
	}
	__syncthreads();
	if (!offsets || !s_brick_record) return;

	// ---- build the record in shared memory ----
	if (t == 0) {
		uint32_t mask4 = 0;
		if (min_depth < 3)
			for (int q = 0; q < 8; ++q) mask4 |= (uint32_t)s_d3_has[q] << q;
		s_buf[0] = (uint8_t)mask4;
	}
	if (s_d3_hit[j3]) {
		if (s_d3_has[j3] && min_depth < 3) {
			uint32_t at = s_d3_off[j3];
			if (k3 == 0) s_buf[at] = s_d3_mask[j3];
			at += 1;
			for (uint32_t q = 0; q < k3; ++q) at += s_blk_size[8 * j3 + q];
			if (blk_size) {
				if (blk_has && min_depth < 2) {
					s_buf[at++] = (uint8_t)(min_depth < 1 ? oct_has : 0u);
#pragma unroll
					for (uint32_t o = 0; o < 8; ++o) {
						double oc[3];
						child_center(blkc, M.g.half_size[1], o, oc);
						at += octet_record<COLOR, G>(M, b, o, (oct_has >> o) & 1u, oocc[o], orgb[o], min_depth, bx, oc, s_buf + at);
					}
				} else {
					put_payload<COLOR>(s_buf + at, s_blk_occ[t], s_blk_rgb[t]);
				}
			}
		} else if (k3 == 0) {
			put_payload<COLOR>(s_buf + s_d3_off[j3], s_d3_occ[j3], s_d3_rgb[j3]);
		}
	}
	__syncthreads();
	uint8_t* dst = out + offsets[brick];
	for (uint32_t i = t; i < s_brick_size; i += 64) dst[i] = s_buf[i];
}

// ---------------------------------------------------------------------------
// Iteration: beginTree / beginLeaves (occupancy_map_base.h:93-163) over the canonical tree of the
// file writer, in the reference's order -- pre-order, children 0..7 (iterator/octree.h:181-316) --
// with its filters (iterator/occupancy_map.h:168-208).  A node is visited when its parent is
// descended into and validNode holds: its cube passes the volume (centres accumulated like
// getChildCenter) and, when contains or depth != min_depth, one of the contains tests passes
// (containsOccupied: max > occupied threshold; containsFree / containsUnknown: the node's flags, its
// own state at depth 0), else one of the own-state tests.  A visited node is descended into when
// depth > min_depth and it is not a leaf.  It is returned when validReturnNode holds: leaves
// iterator -- depth == min_depth or a leaf, and the own state; tree iterator -- the contains tests
// when contains, else the own state.  Values are the file writer's: a leaf carries its payload, an
// inner node its aggregate; flags are those ufo_b200_query reports.
//
// k_brick_iter produces the records of one brick's subtree (depth 4 down) assuming its parent is
// descended into; the host walks the levels above and splices the bricks it reaches in Morton
// order (ufo_map.cu, iterate).  Size pass (offsets == nullptr): info[brick] = records, shape and
// payload of the brick node.  Emit pass: the records of every brick with offsets[brick] != ~0 go
// to out + offsets[brick].  One CTA per brick, one thread per 4^3 block; only the octets whose
// "initialised" bit is set are read below depth 2.
struct IterArgs {
	Volume vol;
	double occ_thr, free_thr;
	uint32_t min_depth;
	int leaves_only, occupied, free_, unknown, contains;
};

// One returned node.  meta: rgb in bits 0..23, depth in 24..28, bit 29 contains_free, bit 30
// contains_unknown, bit 31 leaf.
struct IterRec {
	unsigned long long code;
	float occ;
	uint32_t meta;
};

UFO_HD IterRec iter_rec(unsigned long long code, float v, uint32_t rgb, uint32_t d, uint32_t fl, bool leaf)
{
	return {code, v, (rgb & 0xffffffu) | (d << 24) | ((fl & 3u) << 29) | (leaf ? 1u << 31 : 0u)};
}

UFO_HD bool iter_own(const IterArgs& a, float v)
{
	const bool occ = a.occ_thr < (double)v, fre = a.free_thr > (double)v;
	return (a.occupied && occ) || (a.free_ && fre) || (a.unknown && !occ && !fre);
}

// flags: bit 0 contains_free, bit 1 contains_unknown (at depth 0: the node's own free / unknown state)
UFO_HD bool iter_contains(const IterArgs& a, float v, uint32_t fl)
{
	return (a.occupied && a.occ_thr < (double)v) || (a.unknown && (fl & 2u)) || (a.free_ && (fl & 1u));
}

// validNode without the cube test
UFO_HD bool iter_valid(const IterArgs& a, uint32_t d, float v, uint32_t fl)
{
	return (a.contains || d != a.min_depth) ? iter_contains(a, v, fl) : iter_own(a, v);
}

UFO_HD bool iter_returns(const IterArgs& a, uint32_t d, bool leaf, float v, uint32_t fl)
{
	if (a.leaves_only) return (d == a.min_depth || leaf) && iter_own(a, v);
	return a.contains ? iter_contains(a, v, fl) : iter_own(a, v);
}

// validNode of a node whose parent is descended into; *ret = validReturnNode
template <bool G>
__device__ __forceinline__ bool iter_visit(const IterArgs& a, const double c[3], double hs, uint32_t d, float v, uint32_t fl,
                                           bool leaf, bool* ret)
{
	*ret = false;
	if (!vol_hits_t<G>(a.vol, c, hs) || !iter_valid(a, d, v, fl)) return false;
	*ret = iter_returns(a, d, leaf, v, fl);
	return true;
}

// The records of one depth-2 node (block b) and its subtree, its parent being descended into.  oct_has / oocc / orgb: the block's octets as the canonical
// shape sees them.
// emit(n, record, centre, depth) receives the n-th record of the block.
template <bool COLOR, bool G, class Emit>
__device__ __forceinline__ uint32_t block_records(const DeviceMap& M, const IterArgs& a, size_t b, uint32_t meta,
                                                  uint32_t oct_has, const float oocc[8], const uint32_t orgb[8],
                                                  bool blk_has, float blk_v, uint32_t blk_rgb, const double blkc[3],
                                                  unsigned long long code, Emit&& emit)
{
	const uint32_t blk_fl = (meta >> 16) ? block_flags(M, meta) : M.default_flags;
	uint32_t n = 0;
	bool ret;
	if (!iter_visit<G>(a, blkc, M.g.half_size[2], 2, blk_v, blk_fl, !blk_has, &ret)) return 0;
	if (ret) {
		emit(n, iter_rec(code, blk_v, blk_rgb, 2, blk_fl, !blk_has), blkc, 2u);
		++n;
	}
	if (a.min_depth >= 2 || !blk_has) return n;
	for (uint32_t o = 0; o < 8; ++o) {
		const bool oi = (meta >> (16 + o)) & 1u, oh = (oct_has >> o) & 1u;
		const float ov = oh ? octet_occ(M.leaf + b * 64 + 8 * o) : oocc[o];
		const uint32_t orv = oh ? (COLOR ? M.sum1_rgb[b * 8 + o] : 0u) : orgb[o];
		const uint32_t ofl = oi ? (meta >> (2 * o)) & 3u : M.default_flags;
		const unsigned long long ocode = code | ((unsigned long long)o << 3);
		double oc[3];
		child_center(blkc, M.g.half_size[1], o, oc);
		if (!iter_visit<G>(a, oc, M.g.half_size[1], 1, ov, ofl, !oh, &ret)) continue;
		if (ret) {
			emit(n, iter_rec(ocode, ov, orv, 1, ofl, !oh), oc, 1u);
			++n;
		}
		if (a.min_depth >= 1 || !oh) continue;
		for (uint32_t j = 0; j < 8; ++j) {
			const float v = M.leaf[b * 64 + 8 * o + j];
			const uint32_t fl = leaf_flags(M, v);
			double vc[3];
			child_center(oc, M.g.half_size[0], j, vc);
			if (!iter_visit<G>(a, vc, M.g.half_size[0], 0, v, fl, true, &ret) || !ret) continue;
			emit(n, iter_rec(ocode | j, v, COLOR ? M.leaf_rgb[b * 64 + 8 * o + j] : 0u, 0, fl, true), vc, 0u);
			++n;
		}
	}
	return n;
}

// Shared memory of one brick's CTA in brick_descend: the canonical shape of the brick's subtree down to
// the blocks and the iterator's decisions on its depth-4 and depth-3 nodes.
struct BrickWalk {
	float blk_occ[64], d3_occ[8];
	uint32_t blk_rgb[64], d3_rgb[8];
	uint8_t blk_has[64], d3_has[8], desc3[8], ret3[8];
	IterRec rec4, rec3[8];
	uint8_t has4, desc4, ret4;
	double center[3];
};

// This thread's block (t = Morton index of the block in the brick) as the canonical shape sees it.
struct BlockShape {
	size_t b;
	uint32_t meta, oct_has;
	float oocc[8];
	uint32_t orgb[8];
	bool blk_has;
	float blk_v;
	uint32_t blk_rgb;
	double blkc[3];
};

// The descent k_brick_iter and k_brick_info share: one CTA of 64 threads per brick (an in-tree one), one
// thread per 4^3 block.  Fills S and B with the canonical shape (as k_brick_stream, pruned) and with
// validNode / validReturnNode of the brick node and its depth-3 nodes, assuming the brick's parent is
// descended into.  Ends with the CTA synchronised.
template <bool COLOR, bool G>
__device__ __forceinline__ void brick_descend(const DeviceMap& M, uint32_t brick, const IterArgs& a, BrickWalk& S, BlockShape& B)
{
	const uint32_t t = threadIdx.x;
	uint32_t kx, ky, kz;
	unpack_key(M.brick_key[brick], kx, ky, kz);
	const unsigned long long code4 = key_to_code({kx << 4, ky << 4, kz << 4});
	if (t == 0) brick_center(M.g, kx, ky, kz, S.center);
	const size_t b = (size_t)brick * 64 + t;
	B.b = b;
	const uint32_t meta = M.meta[b];
	B.meta = meta;
	uint32_t oct_has = 0;
#pragma unroll
	for (uint32_t o = 0; o < 8; ++o) {
		B.oocc[o] = 0.0f;
		B.orgb[o] = 0u;
		if (!((meta >> (16 + o)) & 1u)) continue;
		const float* lp = M.leaf + b * 64 + 8 * o;
		const uint32_t* cp = COLOR ? M.leaf_rgb + b * 64 + 8 * o : nullptr;
		if (keeps_children(false, lp, cp)) {
			oct_has |= 1u << o;
		} else {
			B.oocc[o] = lp[0];
			B.orgb[o] = COLOR ? cp[0] : 0u;
		}
	}
	B.oct_has = oct_has;
	B.blk_has = keeps_children(oct_has != 0, B.oocc, B.orgb);
	B.blk_v = B.blk_has ? block_occ(M.line_max[b]) : B.oocc[0];
	B.blk_rgb = B.blk_has ? (COLOR ? M.rgb2[b] : 0u) : B.orgb[0];
	S.blk_has[t] = B.blk_has ? 1 : 0;
	S.blk_occ[t] = B.blk_v;
	S.blk_rgb[t] = B.blk_rgb;
	__syncthreads();
	const uint32_t j3 = t >> 3, k3 = t & 7u;
	const double bc[3] = {S.center[0], S.center[1], S.center[2]};
	double d3c[3];
	child_center(bc, M.g.half_size[3], j3, d3c);
	child_center(d3c, M.g.half_size[2], k3, B.blkc);
	if (t < 8) {
		bool any = false;
		for (int k = 0; k < 8; ++k) any = any || S.blk_has[8 * t + k];
		const bool has = keeps_children(any, S.blk_occ + 8 * t, S.blk_rgb + 8 * t);
		S.d3_has[t] = has ? 1 : 0;
		S.d3_occ[t] = has ? M.brick_sum3[(size_t)brick * 8 + t].occ : S.blk_occ[8 * t];
		S.d3_rgb[t] = has ? (COLOR ? M.brick_rgb3[(size_t)brick * 8 + t] : 0u) : S.blk_rgb[8 * t];
	}
	__syncthreads();
	if (t == 0) {
		bool any = false;
		for (int j = 0; j < 8; ++j) any = any || S.d3_has[j];
		const bool has = keeps_children(any, S.d3_occ, S.d3_rgb);
		const float v = has ? M.brick_sum4[brick].occ : S.d3_occ[0];
		const uint32_t rgb = has ? (COLOR ? M.brick_rgb4[brick] : 0u) : S.d3_rgb[0];
		const uint32_t fl = M.brick_sum4[brick].flags;
		bool ret;
		const bool vis = a.min_depth <= 4 && iter_visit<G>(a, bc, M.g.half_size[4], 4, v, fl, !has, &ret);
		S.has4 = has ? 1 : 0;
		S.desc4 = (vis && a.min_depth < 4 && has) ? 1 : 0;
		S.ret4 = (vis && ret) ? 1 : 0;
		S.rec4 = iter_rec(code4, v, rgb, 4, fl, !has);
	}
	__syncthreads();
	if (t < 8) {
		const bool has = S.d3_has[t];
		const float v = S.d3_occ[t];
		const uint32_t fl = M.brick_sum3[(size_t)brick * 8 + t].flags;
		double c3[3];
		child_center(bc, M.g.half_size[3], t, c3);
		bool ret = false;
		const bool vis = S.desc4 && iter_visit<G>(a, c3, M.g.half_size[3], 3, v, fl, !has, &ret);
		S.desc3[t] = (vis && a.min_depth < 3 && has) ? 1 : 0;
		S.ret3[t] = (vis && ret) ? 1 : 0;
		S.rec3[t] = iter_rec(code4 | ((unsigned long long)t << 9), v, S.d3_rgb[t], 3, fl, !has);
	}
	__syncthreads();
}

// the records of this thread's block and its subtree (block_records) when its depth-3 node is descended into
template <bool COLOR, bool G, class Emit>
__device__ __forceinline__ uint32_t block_walk(const DeviceMap& M, const IterArgs& a, const BrickWalk& S, const BlockShape& B,
                                               unsigned long long blk_code, Emit&& emit)
{
	if (!S.desc3[threadIdx.x >> 3]) return 0;
	return block_records<COLOR, G>(M, a, B.b, B.meta, B.oct_has, B.oocc, B.orgb, B.blk_has, B.blk_v, B.blk_rgb, B.blkc, blk_code,
	                               emit);
}

template <bool COLOR, bool G>
__global__ void __launch_bounds__(64) k_brick_iter(DeviceMap M, uint32_t n_bricks, IterArgs a, BrickInfo* info,
                                                   const unsigned long long* offsets, IterRec* out)
{
	__shared__ BrickWalk S;
	__shared__ uint32_t s_warp[2];
	const uint32_t brick = blockIdx.x, t = threadIdx.x;
	if (brick >= n_bricks) return;
	if (offsets && offsets[brick] == ~0ull) return;  // not reached by the walk above the bricks
	uint32_t kx, ky, kz;
	unpack_key(M.brick_key[brick], kx, ky, kz);
	if ((kx | ky | kz) & ~(M.g.key_mask >> 4)) {  // collects out-of-tree marks, owns no voxels
		if (!offsets && t == 0) info[brick] = {0u, 2u, 0.0f, 0u};
		return;
	}
	BlockShape B;
	brick_descend<COLOR, G>(M, brick, a, S, B);
	if (!offsets && t == 0) info[brick] = {0u, S.has4, S.rec4.occ, S.rec4.meta & 0xffffffu};  // size: below
	// this thread's records, in pre-order: the brick node (t == 0), the depth-3 node (k3 == 0), the block
	const uint32_t j3 = t >> 3, k3 = t & 7u;
	const unsigned long long blk_code = S.rec4.code | ((unsigned long long)t << 6);
	const uint32_t head = (t == 0 ? S.ret4 : 0u) + (k3 == 0 ? S.ret3[j3] : 0u);
	const uint32_t mine = head + block_walk<COLOR, G>(M, a, S, B, blk_code, [](uint32_t, const IterRec&, const double*, uint32_t) {});
	const uint32_t lane = t & 31u, warp = t >> 5;
	uint32_t incl = mine;
#pragma unroll
	for (uint32_t off = 1; off < 32; off <<= 1) {
		const uint32_t y = __shfl_up_sync(0xffffffffu, incl, off);
		if (lane >= off) incl += y;
	}
	if (lane == 31) s_warp[warp] = incl;
	__syncthreads();
	if (!offsets) {
		if (t == 0) info[brick].size = s_warp[0] + s_warp[1];
		return;
	}
	IterRec* dst = out + offsets[brick] + (incl - mine) + (warp ? s_warp[0] : 0u);
	if (t == 0 && S.ret4) *dst++ = S.rec4;
	if (k3 == 0 && S.ret3[j3]) *dst++ = S.rec3[j3];
	if (mine > head)
		block_walk<COLOR, G>(M, a, S, B, blk_code, [dst](uint32_t n, const IterRec& r, const double*, uint32_t) { dst[n] = r; });
}

// Tree size of the live bricks (ufo_b200_tree_info): per brick the size-pass info of k_brick_iter, with
// size = 1 when the brick node is itself a returned leaf (the host places it, as it is reached or not);
// into out, the nodes with children at depth 1..4 and the known box of the leaves below the brick nodes
// that have children, which the walk above always reaches.  `a` is beginLeaves(occupied, free, !unknown).
struct TreeTotals {
	unsigned long long with_children[4];  // [d - 1]
	unsigned long long box[6];            // encode_ordered: min xyz (atomicMin), max xyz (atomicMax)
};

template <bool COLOR>
__global__ void __launch_bounds__(64) k_brick_info(DeviceMap M, uint32_t n_bricks, IterArgs a, BrickInfo* info, TreeTotals* out)
{
	__shared__ BrickWalk S;
	__shared__ unsigned long long s_part[2][10];
	const uint32_t brick = blockIdx.x, t = threadIdx.x;
	if (brick >= n_bricks) return;
	uint32_t kx, ky, kz;
	unpack_key(M.brick_key[brick], kx, ky, kz);
	if ((kx | ky | kz) & ~(M.g.key_mask >> 4)) {  // collects out-of-tree marks, owns no voxels
		if (t == 0) info[brick] = {0u, 2u, 0.0f, 0u};
		return;
	}
	BlockShape B;
	brick_descend<COLOR, false>(M, brick, a, S, B);
	if (t == 0) info[brick] = {S.ret4 && !S.has4 ? 1u : 0u, S.has4, S.rec4.occ, S.rec4.meta & 0xffffffu};
	if (!S.has4) return;
	double lo[3] = {DBL_MAX, DBL_MAX, DBL_MAX}, hi[3] = {-DBL_MAX, -DBL_MAX, -DBL_MAX};
	auto grow = [&](const double c[3], double hs) {
		for (int i = 0; i < 3; ++i) {
			lo[i] = fmin(lo[i], dop::sub(c[i], hs));
			hi[i] = fmax(hi[i], dop::add(c[i], hs));
		}
	};
	const uint32_t j3 = t >> 3;
	if ((t & 7u) == 0 && S.ret3[j3]) {
		double c3[3];
		const double bc[3] = {S.center[0], S.center[1], S.center[2]};
		child_center(bc, M.g.half_size[3], j3, c3);
		grow(c3, M.g.half_size[3]);
	}
	block_walk<COLOR, false>(M, a, S, B, 0ull, [&](uint32_t, const IterRec&, const double* c, uint32_t d) { grow(c, M.g.half_size[d]); });
	// per warp, then the two warps, then one atomic per value and brick
	unsigned long long v[10];
	v[0] = __popc(B.oct_has);
	v[1] = B.blk_has ? 1u : 0u;
	v[2] = t < 8 ? S.d3_has[t] : 0u;
	v[3] = t == 0 ? 1u : 0u;
	for (int i = 0; i < 3; ++i) {
		v[4 + i] = lo[i] <= hi[i] ? encode_ordered(lo[i]) : ~0ull;
		v[7 + i] = lo[i] <= hi[i] ? encode_ordered(hi[i]) : 0ull;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1)
#pragma unroll
		for (int i = 0; i < 10; ++i) {
			const unsigned long long y = __shfl_xor_sync(0xffffffffu, v[i], o);
			v[i] = i < 4 ? v[i] + y : (i < 7 ? (y < v[i] ? y : v[i]) : (y > v[i] ? y : v[i]));
		}
	if ((t & 31u) == 0)
		for (int i = 0; i < 10; ++i) s_part[t >> 5][i] = v[i];
	__syncthreads();
	if (t < 10) {
		const unsigned long long x = s_part[0][t], y = s_part[1][t];
		if (t < 4) {
			if (x + y) atomicAdd(&out->with_children[t], x + y);
		} else if (t < 7) {
			const unsigned long long m = y < x ? y : x;
			if (m != ~0ull) atomicMin(&out->box[t - 4], m);
		} else {
			const unsigned long long m = y > x ? y : x;
			if (m) atomicMax(&out->box[t - 4], m);
		}
	}
}

// ---------------------------------------------------------------------------
// Nearest-first iteration (beginNNTree / beginNNLeaves, occupancy_map_base.h:169-245): the nodes of
// beginTree / beginLeaves in non-decreasing squared distance from a point, delivered in shells
// lo <= d2 < hi.  The distance is the reference's squaredDistance (iterator/octree_nearest.h:198-202):
// the point minus the point clamped (std::clamp) to [centre - hs, centre + hs], then (x*x + y*y) + z*z,
// all in doubles without contraction.  A child's cube lies inside its parent's, so no node is nearer
// than its parent: a brick whose cube is at hi or beyond holds no node of the shell.
UFO_HD double node_d2(const double p[3], const double c[3], double hs)
{
	double s[3];
	for (int i = 0; i < 3; ++i) {
		const double lo = dop::sub(c[i], hs), hi = dop::add(c[i], hs);
		const double q = p[i] < lo ? lo : (hi < p[i] ? hi : p[i]);
		s[i] = dop::sub(p[i], q);
	}
	return vsqnorm(Vec3{s[0], s[1], s[2]});
}

struct NearShell {
	double p[3];
	double lo, hi;
};

// Sort key of a shell record: d2 (non-negative, so its bits order as the value), then the order of
// beginTree / beginLeaves -- code ascending, depth descending (codes are aligned to their depth).
struct NearKey {
	unsigned long long d2;
	unsigned long long code;
	uint8_t neg_depth;  // ~depth
};

struct NearKeyParts {
	__host__ __device__ cuda::std::tuple<unsigned long long&, unsigned long long&, uint8_t&> operator()(NearKey& k) const
	{
		return {k.d2, k.code, k.neg_depth};
	}
};

// The shell's records of the candidate bricks bricks[0, n): one CTA of 64 threads per brick runs the
// descent of k_brick_iter (brick_descend / block_records, the brick's parent being descended into) and
// keeps the records with lo <= d2 < hi.  They are appended at *count (one atomic per CTA), in no
// particular order; records past cap are counted, not written, and the host repeats with room.
template <bool COLOR, bool G>
__global__ void __launch_bounds__(64) k_brick_nearest(DeviceMap M, const uint32_t* bricks, uint32_t n, IterArgs a, NearShell q,
                                                      NearKey* keys, IterRec* recs, unsigned long long* count,
                                                      unsigned long long cap)
{
	__shared__ BrickWalk S;
	__shared__ uint32_t s_warp[2];
	__shared__ unsigned long long s_base;
	if (blockIdx.x >= n) return;
	const uint32_t brick = bricks[blockIdx.x], t = threadIdx.x;
	BlockShape B;
	brick_descend<COLOR, G>(M, brick, a, S, B);
	const uint32_t j3 = t >> 3, k3 = t & 7u;
	const double bc[3] = {S.center[0], S.center[1], S.center[2]};
	double c3[3];
	child_center(bc, M.g.half_size[3], j3, c3);
	const double d2_4 = t == 0 && S.ret4 ? node_d2(q.p, bc, M.g.half_size[4]) : 0.0;
	const double d2_3 = k3 == 0 && S.ret3[j3] ? node_d2(q.p, c3, M.g.half_size[3]) : 0.0;
	const bool keep4 = t == 0 && S.ret4 && q.lo <= d2_4 && d2_4 < q.hi;
	const bool keep3 = k3 == 0 && S.ret3[j3] && q.lo <= d2_3 && d2_3 < q.hi;
	const unsigned long long blk_code = S.rec4.code | ((unsigned long long)t << 6);
	uint32_t mine = (keep4 ? 1u : 0u) + (keep3 ? 1u : 0u);
	block_walk<COLOR, G>(M, a, S, B, blk_code, [&](uint32_t, const IterRec&, const double* c, uint32_t d) {
		const double d2 = node_d2(q.p, c, M.g.half_size[d]);
		if (q.lo <= d2 && d2 < q.hi) ++mine;
	});
	const uint32_t lane = t & 31u, warp = t >> 5;
	uint32_t incl = mine;
#pragma unroll
	for (uint32_t off = 1; off < 32; off <<= 1) {
		const uint32_t y = __shfl_up_sync(0xffffffffu, incl, off);
		if (lane >= off) incl += y;
	}
	if (lane == 31) s_warp[warp] = incl;
	__syncthreads();
	if (t == 0) {
		const uint32_t total = s_warp[0] + s_warp[1];
		s_base = total ? atomicAdd(count, (unsigned long long)total) : 0ull;
	}
	__syncthreads();
	if (!mine) return;
	unsigned long long at = s_base + (incl - mine) + (warp ? s_warp[0] : 0u);
	auto put = [&](const IterRec& r, double d2) {
		if (at < cap) {
			keys[at] = NearKey{(unsigned long long)__double_as_longlong(d2), r.code, (uint8_t)~((r.meta >> 24) & 31u)};
			recs[at] = r;
		}
		++at;
	};
	if (keep4) put(S.rec4, d2_4);
	if (keep3) put(S.rec3[j3], d2_3);
	block_walk<COLOR, G>(M, a, S, B, blk_code, [&](uint32_t, const IterRec& r, const double* c, uint32_t d) {
		const double d2 = node_d2(q.p, c, M.g.half_size[d]);
		if (q.lo <= d2 && d2 < q.hi) put(r, d2);
	});
}

// ---------------------------------------------------------------------------
// Filtered node read-out (SURVEY.md 8(f) N3): the leaf iteration of the reference with state and
// bounding-volume filters (beginLeaves(occupied, free, unknown, contains = false, min_depth),
// occupancy_map_base.h:130-216; validity rule iterator/occupancy_map.h:168-207), on the value
// field: every node of depth `depth` inside the known space (existing bricks / upper nodes) whose
// own state -- occupied: value > occupied threshold, free: value < free threshold, unknown: in
// between, the value of an inner node being the maximum of its subtree -- passes the filter and
// whose cube passes the volume filter.  The reference returns a collapsed leaf above `depth` as
// one node; here it appears as its depth-`depth` cells (same space, same state).
// Volume filter (CHAIN, a template parameter of the kernels): chain == 0 tests the node's own cube
// (centre from toCoord) -- ufo_b200_export_nodes;
// chain != 0 tests every cube on the node's path from the root down, centres accumulated like
// getChildCenter, as the reference's iterator does (validNode, iterator/octree.h:213-245) --
// ufo_b200_export_nodes_bv.  The chain above depth 4 comes from k_brick_chain (brick_ok, brick_c).
// One thread per (brick, block) for depth 0..4; k_export_upper for depth >= 5.
struct NodeFilter {
	uint32_t depth;
	int occupied, free_, unknown;
	Volume vol;
	int chain;
	const uint8_t* brick_ok;
	const double* brick_c;
};

__device__ __forceinline__ bool node_passes(const DeviceMap& M, const NodeFilter& f, float v)
{
	const bool occ = M.occ_thr < (double)v, fre = M.free_thr > (double)v;
	return (f.occupied && occ) || (f.free_ && fre) || (f.unknown && !occ && !fre);
}

// inside: the chain test of the caller (chain mode)
template <bool CHAIN>
__device__ __forceinline__ void node_emit(const DeviceMap& M, const NodeFilter& f, uint32_t x, uint32_t y, uint32_t z,
                                          float v, uint32_t rgb, unsigned long long* codes, float* occ, uint32_t* rgbs,
                                          unsigned long long cap, unsigned long long* count, bool inside = true)
{
	if (!inside || !node_passes(M, f, v)) return;
	const uint32_t d = f.depth;
	const uint32_t centre = d ? (1u << (d - 1)) : 0u, snap = ~((1u << d) - 1u);
	const Key3 k = {(x & snap) | centre, (y & snap) | centre, (z & snap) | centre};
	if (!CHAIN && f.vol.n) {
		const Vec3 c = key_to_coord(M.g, k, d);
		const double cc[3] = {c.x, c.y, c.z};
		if (!vol_hits_t<false>(f.vol, cc, M.g.half_size[d])) return;
	}
	const unsigned long long at = atomicAdd(count, 1ull);
	if (codes && at < cap) {
		codes[at] = key_to_code(k);
		occ[at] = v;
		if (rgbs) rgbs[at] = rgb;
	}
}

// The chain test of one brick: c receives the centre of its cube accumulated from the root; true iff
// every cube from the root's children down to the brick itself passes the volume (the root is tested
// on the host).
__device__ __forceinline__ bool brick_chain(const DeviceMap& M, unsigned long long brick_key, const Volume& vol, double c[3])
{
	uint32_t kx, ky, kz;
	unpack_key(brick_key, kx, ky, kz);
	c[0] = c[1] = c[2] = 0.0;
	bool ok = !((kx | ky | kz) & ~(M.g.key_mask >> 4));  // alias collector bricks own no voxels
	for (uint32_t d = M.g.depth_levels; d > 4 && ok; --d) {
		const uint32_t bit = d - 5;
		const uint32_t i = ((kx >> bit) & 1u) | (((ky >> bit) & 1u) << 1) | (((kz >> bit) & 1u) << 2);
		double n[3];
		child_center(c, M.g.half_size[d - 1], i, n);
		c[0] = n[0];
		c[1] = n[1];
		c[2] = n[2];
		ok = vol_hits(vol, c, M.g.half_size[d - 1]);
	}
	return ok;
}

__global__ void __launch_bounds__(256) k_brick_chain(DeviceMap M, uint32_t n_bricks, Volume vol, uint8_t* ok_out, double* c_out)
{
	const uint32_t brick = blockIdx.x * blockDim.x + threadIdx.x;
	if (brick >= n_bricks) return;
	double c[3];
	const bool ok = brick_chain(M, M.brick_key[brick], vol, c);
	ok_out[brick] = ok ? 1 : 0;
	c_out[3 * (size_t)brick] = c[0];
	c_out[3 * (size_t)brick + 1] = c[1];
	c_out[3 * (size_t)brick + 2] = c[2];
}

template <bool CHAIN>
__global__ void __launch_bounds__(256) k_export_nodes(DeviceMap M, uint32_t n_bricks, NodeFilter f, unsigned long long* codes,
                                                      float* occ, uint32_t* rgbs, unsigned long long cap,
                                                      unsigned long long* count)
{
	const size_t blk = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (blk >= (size_t)n_bricks * 64) return;
	const uint32_t brick = (uint32_t)(blk >> 6), ch = (uint32_t)(blk & 63);
	uint32_t bx, by, bz;
	unpack_key(M.brick_key[brick], bx, by, bz);
	if ((bx | by | bz) & ~(M.g.key_mask >> 4)) return;  // alias collector brick
	const uint32_t cx = (ch & 1u) | ((ch >> 2) & 2u), cy = ((ch >> 1) & 1u) | ((ch >> 3) & 2u),
	               cz = ((ch >> 2) & 1u) | ((ch >> 4) & 2u);
	const uint32_t x0 = (bx << 4) | (cx << 2), y0 = (by << 4) | (cy << 2), z0 = (bz << 4) | (cz << 2);
	const uint32_t d = f.depth;
	// chain mode: the cubes of the brick's depth-3 node and of this block, below the brick's chain
	double blkc[3] = {0.0, 0.0, 0.0};
	bool in3 = true, in2 = true;
	if (CHAIN) {
		if (!f.brick_ok[brick]) return;
		if (d <= 3) {
			const double bc[3] = {f.brick_c[3 * (size_t)brick], f.brick_c[3 * (size_t)brick + 1], f.brick_c[3 * (size_t)brick + 2]};
			double d3c[3];
			child_center(bc, M.g.half_size[3], ch >> 3, d3c);
			in3 = vol_hits_t<true>(f.vol, d3c, M.g.half_size[3]);
			if (d <= 2 && in3) {
				child_center(d3c, M.g.half_size[2], ch & 7u, blkc);
				in2 = vol_hits_t<true>(f.vol, blkc, M.g.half_size[2]);
			}
			if (!in3 || !in2) return;
		}
	}
	if (d == 4) {
		if (ch == 0) node_emit<CHAIN>(M, f, x0, y0, z0, M.brick_sum4[brick].occ, M.color ? M.brick_rgb4[brick] : 0u, codes, occ, rgbs, cap, count);
		return;
	}
	if (d == 3) {
		if ((ch & 7u) == 0) {
			const uint32_t j = ch >> 3;
			node_emit<CHAIN>(M, f, x0, y0, z0, M.brick_sum3[(size_t)brick * 8 + j].occ, M.color ? M.brick_rgb3[(size_t)brick * 8 + j] : 0u, codes,
			          occ, rgbs, cap, count);
		}
		return;
	}
	const uint32_t meta = M.meta[blk];
	const bool init = (meta >> 16) != 0;
	if (d == 2) {
		node_emit<CHAIN>(M, f, x0, y0, z0, init ? block_occ(M.line_max[blk]) : 0.0f, (init && M.color) ? M.rgb2[blk] : 0u, codes, occ, rgbs, cap, count);
		return;
	}
	for (uint32_t o = 0; o < 8; ++o) {
		const bool oi = init && ((meta >> (16 + o)) & 1u);
		const uint32_t ox = x0 | ((o & 1u) << 1), oy = y0 | (o & 2u), oz = z0 | ((o & 4u) >> 1);
		double oc[3] = {0.0, 0.0, 0.0};
		if (CHAIN) {
			child_center(blkc, M.g.half_size[1], o, oc);
			if (!vol_hits_t<true>(f.vol, oc, M.g.half_size[1])) continue;
		}
		if (d == 1) {
			node_emit<CHAIN>(M, f, ox, oy, oz, oi ? octet_occ(M.leaf + blk * 64 + 8 * o) : 0.0f, (oi && M.color) ? M.sum1_rgb[blk * 8 + o] : 0u, codes, occ, rgbs,
			          cap, count);
			continue;
		}
		for (uint32_t j = 0; j < 8; ++j) {
			const float v = oi ? M.leaf[blk * 64 + 8 * o + j] : 0.0f;
			const uint32_t c = (oi && M.color) ? M.leaf_rgb[blk * 64 + 8 * o + j] : 0u;
			bool in0 = true;
			if (CHAIN) {
				double vc[3];
				child_center(oc, M.g.half_size[0], j, vc);
				in0 = vol_hits_t<true>(f.vol, vc, M.g.half_size[0]);
			}
			node_emit<CHAIN>(M, f, ox | (j & 1u), oy | ((j >> 1) & 1u), oz | (j >> 2), v, c, codes, occ, rgbs, cap, count, in0);
		}
	}
}

template <bool CHAIN>
__global__ void __launch_bounds__(256) k_export_upper(DeviceMap M, uint32_t n_upper, NodeFilter f, unsigned long long* codes,
                                                      float* occ, uint32_t* rgbs, unsigned long long cap,
                                                      unsigned long long* count)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_upper) return;
	uint32_t x, y, z;
	const unsigned long long key = M.up_key[i];
	unpack_key(key, x, y, z);
	const uint32_t d = x >> 16;  // depth tag (upper_key)
	if (d != f.depth) return;
	x &= 0xffffu;
	const uint32_t X = x << d, Y = y << d, Z = z << d;
	bool inside = true;
	if (CHAIN) {
		// every cube from the root's children down to the node (the root is tested on the host)
		double c[3] = {0.0, 0.0, 0.0};
		for (uint32_t D = M.g.depth_levels; D > d && inside; --D) {
			const uint32_t bit = D - 1;
			const uint32_t ci = ((X >> bit) & 1u) | (((Y >> bit) & 1u) << 1) | (((Z >> bit) & 1u) << 2);
			double n[3];
			child_center(c, M.g.half_size[D - 1], ci, n);
			c[0] = n[0];
			c[1] = n[1];
			c[2] = n[2];
			inside = vol_hits_t<true>(f.vol, c, M.g.half_size[D - 1]);
		}
	}
	node_emit<CHAIN>(M, f, X, Y, Z, M.up_agg[i].occ, M.color ? M.up_rgb[i] : 0u, codes, occ, rgbs, cap, count, inside);
}

// ---------------------------------------------------------------------------
// setValueVolume(AABB, value, min_depth)   occupancy_map_base.h:492-518, :986-1031
// ---------------------------------------------------------------------------
// The reference descends from the root and, at every level down to min_depth, keeps the children
// whose cube intersects the box; the nodes reached at min_depth are collapsed and set.  On the
// value field: a voxel is set iff every ancestor cube from depth L-1 down to min_depth (itself at
// min_depth 0) intersects the box.  k_volume_mark evaluates exactly that chain -- centres
// accumulated top-down like getChildCenter -- for one candidate brick per CTA, one 4^3 block per
// thread, and leaves the result as a bit mask in the block's miss mask; the set itself is the K3
// update kernel in SET mode, followed by the usual aggregate passes.
struct VolumeArgs {
	Volume vol;
	uint32_t min_depth;       // 0..4
	uint32_t bx0, by0, bz0;   // first candidate brick (brick coordinates)
	uint32_t nx, ny, nz;      // candidate bricks per axis
	const unsigned long long* cand;  // != nullptr: the candidates are these packed brick keys (nx of them)
	int general;                     // the volume holds a shape other than an AABB (k_volume_mark<true>)
};

template <bool G>
__global__ void __launch_bounds__(64) k_volume_mark(DeviceMap M, VolumeArgs v)
{
	__shared__ double s_center[3];
	__shared__ uint32_t s_slot;
	const uint32_t t = threadIdx.x;
	uint32_t kx, ky, kz;
	if (v.cand) {
		unpack_key(v.cand[blockIdx.x], kx, ky, kz);
	} else {
		kx = v.bx0 + blockIdx.x % v.nx;
		ky = v.by0 + (blockIdx.x / v.nx) % v.ny;
		kz = v.bz0 + blockIdx.x / (v.nx * v.ny);
	}
	if (t == 0) {
		double c[3] = {0.0, 0.0, 0.0};
		bool ok = true;
		for (uint32_t d = M.g.depth_levels; d > 4; --d) {
			const uint32_t bit = d - 5;
			const uint32_t i = ((kx >> bit) & 1u) | (((ky >> bit) & 1u) << 1) | (((kz >> bit) & 1u) << 2);
			double n[3];
			child_center(c, M.g.half_size[d - 1], i, n);
			c[0] = n[0];
			c[1] = n[1];
			c[2] = n[2];
			ok = ok && vol_hits_t<G>(v.vol, c, M.g.half_size[d - 1]);  // cube of the depth d-1 ancestor
		}
		uint32_t slot = kNone;
		if (ok && brick_owned(M, pack_key(kx, ky, kz))) {
			slot = brick_find_or_create(M, pack_key(kx, ky, kz));
			if (slot != kNone) touch_brick(M, slot);
		}
		s_slot = slot;
		s_center[0] = c[0];
		s_center[1] = c[1];
		s_center[2] = c[2];
	}
	__syncthreads();
	const uint32_t slot = s_slot;
	if (slot == kNone) return;
	unsigned long long mask = 0ull;
	if (v.min_depth >= 4) {
		mask = ~0ull;
	} else {
		double bc[3] = {s_center[0], s_center[1], s_center[2]}, d3c[3], blkc[3];
		child_center(bc, M.g.half_size[3], t >> 3, d3c);
		child_center(d3c, M.g.half_size[2], t & 7u, blkc);
		if (vol_hits_t<G>(v.vol, d3c, M.g.half_size[3])) {
			if (v.min_depth == 3) {
				mask = ~0ull;
			} else if (vol_hits_t<G>(v.vol, blkc, M.g.half_size[2])) {
				if (v.min_depth == 2) {
					mask = ~0ull;
				} else {
					for (uint32_t o = 0; o < 8; ++o) {
						double oc[3];
						child_center(blkc, M.g.half_size[1], o, oc);
						if (!vol_hits_t<G>(v.vol, oc, M.g.half_size[1])) continue;
						const uint32_t x0 = (o & 1u) << 1, y0 = o & 2u, z0 = (o & 4u) >> 1;
						if (v.min_depth == 1) {
							mask |= octet_mask_of(x0, y0, z0);
							continue;
						}
						for (uint32_t j = 0; j < 8; ++j) {
							double vc[3];
							child_center(oc, M.g.half_size[0], j, vc);
							if (vol_hits_t<G>(v.vol, vc, M.g.half_size[0]))
								mask |= 1ull << linear2(x0 + (j & 1u), y0 + ((j >> 1) & 1u), z0 + (j >> 2));
						}
					}
				}
			}
		}
	}
	// the masks of a block belong to one thread here, and no scan is in flight
	if (mask) M.miss_mask[(size_t)slot * 64 + t] |= mask;
}

// One level of the device descent of setValueVolume for a general volume: one thread per (frontier
// node, child); the children whose cube passes go to the next frontier (keys in units of the child
// depth, centres accumulated like getChildCenter).  *out_n counts every passing child, also those
// beyond cap, so that the host can tell an overflow.
__global__ void __launch_bounds__(256) k_volume_descend(Volume vol, const unsigned long long* in_key, const double* in_c, uint32_t n_in,
                                                        double chs, unsigned long long* out_key, double* out_c, uint32_t cap,
                                                        unsigned int* out_n)
{
	const size_t t = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (t >= (size_t)n_in * 8) return;
	const uint32_t node = (uint32_t)(t >> 3), i = (uint32_t)(t & 7);
	const double pc[3] = {in_c[3 * (size_t)node], in_c[3 * (size_t)node + 1], in_c[3 * (size_t)node + 2]};
	double c[3];
	child_center(pc, chs, i, c);
	if (!vol_hits(vol, c, chs)) return;
	const uint32_t at = atomicAdd(out_n, 1u);
	if (at >= cap) return;
	uint32_t x, y, z;
	unpack_key(in_key[node], x, y, z);
	out_key[at] = pack_key((x << 1) | (i & 1u), (y << 1) | ((i >> 1) & 1u), (z << 1) | (i >> 2));
	out_c[3 * (size_t)at] = c[0];
	out_c[3 * (size_t)at + 1] = c[1];
	out_c[3 * (size_t)at + 2] = c[2];
}
}  // namespace ufo_b200
