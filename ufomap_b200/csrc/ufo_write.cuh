// ufo_write.cuh -- ordered per-node writes on the value field: updateValue / integrateHit /
// integrateMiss / updateOccupancy / setOccupancy (occupancy_map_base.h:524-593, :1037-1120) and
// insertMissOnRay / insertRay (:251-268) as batches.
//
// Unlike a scan, a batch may update one voxel any number of times and clamps after every update,
// so the order of the updates matters.  A batch is applied in three phases:
//   1. k_write_expand: one thread per entry (or ray) finds or creates the bricks it covers and
//      writes WRITE RECORDS -- (brick slot, sequence number) -> which blocks / voxels, ADD or SET,
//      value -- into a region the host reserved for it.  No leaf is written here, so the phase can
//      be repeated after a pool growth.  On a routed map every rank expands the whole batch --
//      ray walks included -- and keeps the records of the bricks it owns (brick_owned); the
//      others become padding.
//   2. a stable radix sort of the record keys (brick slot << 32 | sequence number), then
//      k_write_segments finds each brick's run of records.
//   3. k_write_apply: one CTA of 64 threads per brick, thread = 4^3 block; the brick's records
//      stream through shared memory in sequence order and every thread applies the ones that cover
//      its block to its voxels.
// The depth 1-4 aggregates are then rebuilt from the leaves (k_import_refresh, k_brick_agg) and the
// usual propagation pass runs.
//
// Colour maps add two depth-0 ops (ufo_b200_update_nodes_color): ADD_COLOR, the colour map's
// updateValue(code, value, Color) (occupancy_map_color.h:269-287), and SET_COLOR, setColor(code,
// Color) (occupancy_map_color.cpp:74-81).  Their colour rides in the record's op word, and only a
// batch holding one runs the colour variant of phase 3.
#pragma once

#include "ufo_import.cuh"

namespace ufo_b200
{
constexpr uint32_t kWriteAdd = 0, kWriteSet = 1, kWriteAddColor = 2, kWriteSetColor = 3;
constexpr unsigned long long kWritePad = ~0ull;  // key of an unused record slot (sorts last)

// what one record does inside its brick: every voxel of vmask (Morton order, bit j = leaf[j]) in
// every block of bmask (Morton child index of the block) takes the update.  op: bits 0-7 the op,
// bits 8-31 the colour of a colour op (r | g << 8 | b << 16, the leaf_rgb layout)
struct WriteRec {
	unsigned long long bmask, vmask;
	float value;
	uint32_t op;
};
static_assert(sizeof(WriteRec) == 24, "write records stay 24 bytes");

struct WriteArgs {
	uint32_t n;       // entries or rays
	uint32_t rays;    // 0: node entries, 1: rays
	// node entries
	const unsigned long long* codes;
	const uint32_t* depths;
	const uint8_t* ops;
	const float* values;
	const uint8_t* rgb;  // [n][3]; set only when the batch holds a colour op
	// rays: origins / ends [n][3]
	const double* origins;
	const double* ends;
	double max_range;
	uint32_t depth;
	uint32_t hit_end;
	float miss, hit;
	// output: region [offs[i], offs[i+1]) of entry / ray i
	const unsigned long long* offs;
	unsigned long long* keys;
	uint32_t* idx;
	WriteRec* recs;
	// segments of the sorted keys
	uint32_t* seg_begin;  // [brick_cap]
	uint32_t* seg_end;    // [brick_cap]
	uint32_t* seg_list;   // [brick_cap] bricks with at least one record
	unsigned long long n_rec;
};

// blocks / voxels of one brick covered by the node (key k, depth d <= 4); k is the node's first voxel
__device__ __forceinline__ void node_cover(Key3 k, uint32_t d, unsigned long long& bmask, unsigned long long& vmask)
{
	const uint32_t blk = morton2(k.x >> 2, k.y >> 2, k.z >> 2);
	const uint32_t vox = morton2(k.x, k.y, k.z);
	if (d == 0) {
		bmask = 1ull << blk;
		vmask = 1ull << vox;
	} else if (d == 1) {
		bmask = 1ull << blk;
		vmask = 0xffull << (vox & ~7u);
	} else if (d == 2) {
		bmask = 1ull << blk;
		vmask = ~0ull;
	} else if (d == 3) {
		bmask = 0xffull << (blk & ~7u);
		vmask = ~0ull;
	} else {
		bmask = ~0ull;
		vmask = ~0ull;
	}
}

__device__ __forceinline__ void put_record(const DeviceMap& M, const WriteArgs& a, unsigned long long at, uint32_t seq,
                                           uint32_t bx, uint32_t by, uint32_t bz, unsigned long long bmask,
                                           unsigned long long vmask, float value, uint32_t op)
{
	const unsigned long long key = pack_key(bx, by, bz);
	if (!brick_owned(M, key)) {
		// another rank of a routed map applies it: the slot stays padding
		a.keys[at] = kWritePad;
		a.idx[at] = (uint32_t)at;
		return;
	}
	const uint32_t slot = brick_find_or_create(M, key);  // kNone: a pool overflowed
	a.keys[at] = ((unsigned long long)slot << 32) | seq;
	a.idx[at] = (uint32_t)at;
	a.recs[at] = WriteRec{bmask, vmask, value, op};
}

// every record of the node (first voxel k, depth d): one per brick it covers
__device__ __forceinline__ unsigned long long put_node(const DeviceMap& M, const WriteArgs& a, unsigned long long at,
                                                       uint32_t seq, Key3 k, uint32_t d, float value, uint32_t op)
{
	if (d <= 4) {
		unsigned long long bm, vm;
		node_cover(k, d, bm, vm);
		put_record(M, a, at, seq, k.x >> 4, k.y >> 4, k.z >> 4, bm, vm, value, op);
		return at + 1;
	}
	const uint32_t side = 1u << (d - 4);
	for (uint32_t i = 0; i < side * side * side; ++i) {
		const uint32_t x = i % side, y = (i / side) % side, z = i / (side * side);
		put_record(M, a, at++, seq, (k.x >> 4) + x, (k.y >> 4) + y, (k.z >> 4) + z, ~0ull, ~0ull, value, op);
	}
	return at;
}

__device__ __forceinline__ bool key_in_tree(const DeviceMap& M, Key3 k)
{
	return !((k.x | k.y | k.z) & ~M.g.key_mask);
}

// Phase 1.  Records of entry / ray i go to [offs[i], offs[i+1]); unused slots get kWritePad.
__global__ void __launch_bounds__(128) k_write_expand(DeviceMap M, WriteArgs a)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n) return;
	unsigned long long at = a.offs[i];
	const unsigned long long stop = a.offs[i + 1];
	if (!a.rays) {
		const uint32_t d = a.depths[i];
		const Key3 c = code_to_key(a.codes[i]);
		const Key3 k = {(c.x >> d) << d, (c.y >> d) << d, (c.z >> d) << d};
		uint32_t op = a.ops[i];
		if (a.rgb && op >= kWriteAddColor) {
			const uint8_t* c3 = a.rgb + 3 * (size_t)i;
			op |= ((uint32_t)c3[0] | ((uint32_t)c3[1] << 8) | ((uint32_t)c3[2] << 16)) << 8;
		}
		at = put_node(M, a, at, i, k, d, a.values[i], op);
	} else {
		// the walk of ufo_b200_compute_ray (Octree::computeRay, octree.h:449-496)
		const uint32_t d = a.depth;
		const double* po = a.origins + 3 * (size_t)i;
		const double* pe = a.ends + 3 * (size_t)i;
		const Vec3 o = {po[0], po[1], po[2]};
		const Vec3 end = {pe[0], pe[1], pe[2]};
		Vec3 e = end, dir = vsub(e, o);
		double dist = vnorm(dir);
		dir = vdiv(dir, dist);
		if (0 <= a.max_range && dist > a.max_range) {
			e = vadd(o, vscale(dir, a.max_range));
			dist = a.max_range;
		}
		Walk w;
		walk_init(M.g, o, e, dir, d, w);
		// depth <= 2: consecutive nodes of one block are merged into one record
		uint32_t cb[3] = {0, 0, 0};
		unsigned long long cbm = 0, cvm = 0;
		if (!w.same) {
			while (w.cur != w.end && walk_tmin(w) <= dist) {
				const Key3 k = d ? Key3{(w.cur.x >> d) << d, (w.cur.y >> d) << d, (w.cur.z >> d) << d} : w.cur;
				if (key_in_tree(M, k)) {
					if (d <= 2) {
						unsigned long long bm, vm;
						node_cover(k, d, bm, vm);
						const uint32_t b[3] = {k.x >> 2, k.y >> 2, k.z >> 2};
						if (cvm && (b[0] != cb[0] || b[1] != cb[1] || b[2] != cb[2])) {
							if (at >= stop) {
								atomicOr(&M.ctr->overflow, 16u);
								return;
							}
							put_record(M, a, at++, i, cb[0] >> 2, cb[1] >> 2, cb[2] >> 2, cbm, cvm, a.miss, kWriteAdd);
							cvm = 0;
						}
						cb[0] = b[0];
						cb[1] = b[1];
						cb[2] = b[2];
						cbm = bm;
						cvm |= vm;
					} else {
						const uint32_t need = d <= 4 ? 1u : 1u << (3 * (d - 4));
						if (at + need > stop) {
							atomicOr(&M.ctr->overflow, 16u);
							return;
						}
						at = put_node(M, a, at, i, k, d, a.miss, kWriteAdd);
					}
				}
				walk_step(w);
			}
		}
		if (cvm) {
			if (at >= stop) {
				atomicOr(&M.ctr->overflow, 16u);
				return;
			}
			put_record(M, a, at++, i, cb[0] >> 2, cb[1] >> 2, cb[2] >> 2, cbm, cvm, a.miss, kWriteAdd);
		}
		if (a.hit_end) {
			// integrateHit(end) on the end point as given (insertRay, occupancy_map_base.h:260-268)
			if (at >= stop) {
				atomicOr(&M.ctr->overflow, 16u);
				return;
			}
			at = put_node(M, a, at, i, point_to_key(M.g, end, 0), 0, a.hit, kWriteAdd);
		}
	}
	for (; at < stop; ++at) {
		a.keys[at] = kWritePad;
		a.idx[at] = (uint32_t)at;
	}
}

// Phase 2b: first / one-past-last record of every brick in the sorted keys
__global__ void __launch_bounds__(256) k_write_segments(DeviceMap M, WriteArgs a)
{
	if (__ldg(&M.ctr->overflow) & ~4u) return;
	for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < a.n_rec;
	     i += (unsigned long long)gridDim.x * blockDim.x) {
		const unsigned long long s = a.keys[i] >> 32;
		if (s >= M.brick_cap) continue;  // padding
		if (i == 0 || (a.keys[i - 1] >> 32) != s) {
			a.seg_begin[s] = (uint32_t)i;
			a.seg_list[atomicAdd(&M.ctr->n_dirty, 1u)] = (uint32_t)s;
		}
		if (i + 1 == a.n_rec || (a.keys[i + 1] >> 32) != s) a.seg_end[s] = (uint32_t)(i + 1);
	}
}

constexpr uint32_t kWriteChunk = 64;

// Phase 3: one CTA per brick, thread = block.  A thread loads its block's 64 voxels into shared
// memory the first time a record covers it, applies every covering record in sequence order
// (float add + clamp, or clamp of the set value, one clamp per update), and writes back the block,
// its octet "initialised" bits and the voxels whose value changed at some update.
// COLOR (batches with a colour op): the block's 64 leaf colours are loaded into shared memory too,
// at the first colour record that covers it, and written back at the end.  ADD_COLOR blends with
// the log-odds the earlier records left, before its own add; SET_COLOR replaces the colour.  Both
// initialise the voxel's octet; only a log-odds change enters the change mask.
template <bool COLOR>
__global__ void __launch_bounds__(64) k_write_apply(DeviceMap M, WriteArgs a)
{
	__shared__ float s_v[64][68];
	__shared__ __align__(16) uint32_t s_c[COLOR ? 64 : 1][68];
	__shared__ unsigned long long s_bm[kWriteChunk], s_vm[kWriteChunk];
	__shared__ float s_val[kWriteChunk];
	__shared__ uint32_t s_op[kWriteChunk];
	if (__ldg(&M.ctr->overflow) & ~4u) return;
	const uint32_t t = threadIdx.x;
	const uint32_t n_seg = __ldg(&M.ctr->n_dirty);
	unsigned int s_vox = 0, s_blk = 0, s_new = 0;
	for (uint32_t s = blockIdx.x; s < n_seg; s += gridDim.x) {
		const uint32_t brick = a.seg_list[s];
		const uint32_t begin = a.seg_begin[brick], end = a.seg_end[brick];
		if (t == 0) touch_brick(M, brick);
		const size_t b = (size_t)brick * 64 + t;
		float* leaf = M.leaf + b * 64;
		float* v = s_v[t];
		uint32_t* col = s_c[COLOR ? t : 0];
		bool col_loaded = false;
		unsigned long long written = 0, changed = 0;
		for (uint32_t c0 = begin; c0 < end; c0 += kWriteChunk) {
			__syncthreads();
			if (c0 + t < end) {
				const WriteRec r = a.recs[a.idx[c0 + t]];
				s_bm[t] = r.bmask;
				s_vm[t] = r.vmask;
				s_val[t] = r.value;
				s_op[t] = r.op;
			}
			__syncthreads();
			const uint32_t cn = min(kWriteChunk, end - c0);
			for (uint32_t r = 0; r < cn; ++r) {
				if (!((s_bm[r] >> t) & 1ull)) continue;
				if (!written) {
					const float4* lp = reinterpret_cast<const float4*>(leaf);
#pragma unroll
					for (int q = 0; q < 16; ++q) reinterpret_cast<float4*>(v)[q] = lp[q];
				}
				unsigned long long vm = s_vm[r];
				const float u = s_val[r];
				if (COLOR && (s_op[r] & 0xffu) >= kWriteAddColor) {
					if (!col_loaded) {
						const uint4* cp = reinterpret_cast<const uint4*>(M.leaf_rgb + b * 64);
#pragma unroll
						for (int q = 0; q < 16; ++q) reinterpret_cast<uint4*>(col)[q] = cp[q];
						col_loaded = true;
					}
					const uint32_t rgb = s_op[r] >> 8;
					const bool add = (s_op[r] & 0xffu) == kWriteAddColor;
					const double prob = add ? to_prob(u) : 0.0;
					written |= vm;
					while (vm) {
						const uint32_t j = __ffsll((long long)vm) - 1;
						vm &= vm - 1;
						if (!add) {
							col[j] = rgb;
							continue;
						}
						const float old = v[j];
						col[j] = blended_color(col[j], rgb, prob, old);
						const float nv = apply_update(M, old, u);
						changed |= (unsigned long long)(__float_as_uint(nv) != __float_as_uint(old)) << j;
						v[j] = nv;
					}
					continue;
				}
				const bool set = s_op[r] == kWriteSet;
				written |= vm;
				while (vm) {
					const uint32_t j = __ffsll((long long)vm) - 1;
					vm &= vm - 1;
					const float old = v[j];
					const float nv = set ? fminf(fmaxf(u, M.clamp_min), M.clamp_max) : apply_update(M, old, u);
					changed |= (unsigned long long)(__float_as_uint(nv) != __float_as_uint(old)) << j;
					v[j] = nv;
				}
			}
		}
		if (written) {
			float4* lp = reinterpret_cast<float4*>(leaf);
#pragma unroll
			for (int q = 0; q < 16; ++q) lp[q] = reinterpret_cast<const float4*>(v)[q];
			if (COLOR && col_loaded) {
				uint4* cp = reinterpret_cast<uint4*>(M.leaf_rgb + b * 64);
#pragma unroll
				for (int q = 0; q < 16; ++q) cp[q] = reinterpret_cast<const uint4*>(col)[q];
			}
			uint32_t init = 0;
#pragma unroll
			for (uint32_t o = 0; o < 8; ++o) init |= ((written >> (8 * o)) & 0xffull) ? (1u << (16 + o)) : 0u;
			const uint32_t mt = M.meta[b];
			M.meta[b] = mt | init;
			if (M.chg_mask && changed) {
				unsigned long long lin = 0;
#pragma unroll
				for (uint32_t o = 0; o < 8; ++o) lin |= octet_unbits8((uint32_t)(changed >> (8 * o)) & 0xffu, o);
				M.chg_mask[b] |= lin;
			}
			s_vox += __popcll(written);
			s_blk += 1;
			s_new += (mt & 0xff0000u) ? 0u : 1u;
		}
	}
	unsigned long long* slot = M.ctr->stat[(blockIdx.x * 64 + t) % kStatSlots];
	if (s_vox) atomicAdd(&slot[0], (unsigned long long)s_vox);
	if (s_blk) atomicAdd(&slot[3], (unsigned long long)s_blk);
	if (s_new) atomicAdd(&slot[4], (unsigned long long)s_new);
}

}  // namespace ufo_b200
