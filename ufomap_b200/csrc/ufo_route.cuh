// ufo_route.cuh -- routed multi-GPU mode (SURVEY.md 8(e) variant 2; BASELINE config #4 "octant
// shard" and config #5 "one GPU per sensor with boundary merge").
//
// State is owned by space: rank = brick_owner(brick key).  Marking is parallel over rays: every
// rank walks ITS rays (a slice of one scan, or its own sensor's scan) into its own map with the
// ordinary fused kernels.  What crosses GPUs is the per-scan SET UNION only:
//   k_outbox   one warp per touched brick: the 64 miss masks of a brick another rank owns are
//              written, behind the brick key, straight into that rank's inbox (peer memory over
//              NVLink -- plain coalesced stores on a mapped peer pointer; no staging, no NCCL on
//              the data path) and cleared locally;  hit voxels were forwarded by K1 (mark_hit)
//   k_outbox_publish   record counts -> the owners' inbox headers
//   [barrier across the ranks: the one collective, a stream-ordered NCCL all-reduce of 4 bytes]
//   k_inbox    one warp per received brick record: find-or-create the brick, OR the 64 masks in;
//              one thread per received hit voxel
// followed by the ordinary K3 / K4 over the touched list.  With route_self the rank's own marks
// take the same way, so that the owner can apply the sensors ONE AFTER THE OTHER in sensor order
// (clamping makes the order matter): k_inbox(source s) + K3 for s = 0..G-1.
//
// Every marking path of a single-GPU insert works here (fused, record, fixed-step; discrete; insert
// depth 0-6); the record paths mark through the brick hash, which k_outbox reads like the fused
// walk's non-dense marks.  Two kinds of hit-region record come on top of the voxel keys:
//   whole bricks   insert depth 5/6: k_expand_nodes does not create the bricks another rank owns
//                  below a free-space node; it sends the brick key | kFullBrick, and k_inbox sets
//                  all 64 masks on the owner (a node collected by several ranks arrives several
//                  times: OR is idempotent)
//   colour hits    only the point with the lowest GLOBAL cloud index of a hit voxel blends its
//                  colour (occupancy_map_color.h:269-287), and that point may sit on any rank.
//                  k_route_hits sends each rank's own winner (the scan table's minimum) with its
//                  global index and rgb -- own voxels included, since the owner cannot blend before
//                  it has seen the other ranks' candidates.  k_inbox takes the minimum index per
//                  voxel over the sources of the apply call (apply table, atomicMin) and
//                  k_inbox_color lets the winner blend and set the hit bit, before K3 of those
//                  sources.  Applied per source (merge mode), this is the single map inserting the
//                  sensors' clouds one after the other.
// Inbox regions are double-buffered by scan parity; the barrier of scan k+1 orders the reads of
// scan k before the writes of scan k+2.
//
// The pools grow during a pass as they do on one GPU.  route_mark waits for the marking kernels
// and, if a pool ran full, grows it and marks again before anything reaches an inbox header
// (k_outbox_publish).  An apply call whose k_inbox runs into a full pool backs off with every later
// call of the pass; the host replays them at its next synchronising call, from the regions the
// peers published, which stay valid until the peers' mark of pass k+2.
#pragma once

#include "ufo_kernels.cuh"

namespace ufo_b200
{
__global__ void __launch_bounds__(256) k_outbox(DeviceMap M)
{
	const uint32_t lane = threadIdx.x & 31;
	constexpr uint32_t FULL = 0xffffffffu;
	RouteTable* R = M.route;
	if (__ldg(&M.ctr->overflow) & ~4u) return;
	const uint32_t n = __ldg(&M.ctr->n_touched);
	for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < n; e += (gridDim.x * blockDim.x) >> 5) {
		const uint32_t brick = M.touched[e];
		const unsigned long long key = M.brick_key[brick];
		const uint32_t owner = brick_owner(key, M.route_world);
		unsigned long long* mp = M.mask_base + (size_t)(M.touched_mi[e] & ~kMiNoHits) * 64 + 2 * lane;
		const ulonglong2 mk = *reinterpret_cast<const ulonglong2*>(mp);
		if (owner == M.route_rank && !M.route_self) {
			// own brick, marks stay: it opens the touched list of the apply phase (scan id + 1),
			// which reads every mask from miss_mask -- masks marked into the scan volume move there
			if (M.dense) {
				*reinterpret_cast<ulonglong2*>(M.miss_mask + (size_t)brick * 64 + 2 * lane) = mk;
				*reinterpret_cast<ulonglong2*>(mp) = make_ulonglong2(0ull, 0ull);
			}
			if (lane == 0) {
				M.brick_stamp[brick] = M.scan_id + 1u;
				const uint32_t i = atomicAdd(&M.ctr->n_touched_alt, 1u);
				M.touched_alt[i] = brick;
				M.touched_alt_mi[i] = brick;
			}
			continue;
		}
		if (!__any_sync(FULL, (mk.x | mk.y) != 0ull)) continue;
		uint32_t slot = 0;
		if (lane == 0) slot = atomicAdd(&R->out_miss[owner], 1u);
		slot = __shfl_sync(FULL, slot, 0);
		if (slot >= R->cap_m) {
			if (lane == 0) atomicOr(&R->overflow, 2u);
			continue;
		}
		unsigned long long* dst = R->out[owner].miss + (size_t)slot * kMissRecWords;
		if (lane == 0) dst[0] = key;
		dst[1 + 2 * lane] = mk.x;
		dst[2 + 2 * lane] = mk.y;
		*reinterpret_cast<ulonglong2*>(mp) = make_ulonglong2(0ull, 0ull);
	}
}

__global__ void k_outbox_publish(DeviceMap M)
{
	RouteTable* R = M.route;
	const uint32_t d = threadIdx.x;
	uint32_t nm = 0, nh = 0;
	if (d < M.route_world) {
		nm = min(R->out_miss[d], R->cap_m);
		nh = min(R->out_hit[d], R->cap_h);
		R->out[d].hdr[0] = nm;
		R->out[d].hdr[1] = nh;
		R->out_miss[d] = 0;
		R->out_hit[d] = 0;
	}
	nm = __reduce_add_sync(0xffffffffu, nm);
	nh = __reduce_add_sync(0xffffffffu, nh);
	if (d == 0) {
		R->sent[0] = nm;
		R->sent[1] = R->out_full;
		R->sent[2] = nh - R->out_full;
		R->out_full = 0;
		// the apply phase starts from the own bricks that kept local marks
		M.ctr->n_touched = M.ctr->n_touched_alt;
		M.ctr->n_touched_alt = 0;
	}
	__threadfence_system();
}

// K1b of a routed colour pass: every hit voxel's winner on this rank (lowest local index, as k_hits)
// goes to the voxel's owner with its global cloud index index_base + i * index_stride and its rgb
__global__ void __launch_bounds__(256) k_route_hits(DeviceMap M, ScanArgs a, unsigned long long index_base,
                                                     uint32_t index_stride)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n) return;
	const uint32_t t = a.hit_tab[i];
	if (t == kNone || a.tab_min[t] != i) return;
	const Key3 k = code_to_key(a.tab_keys[t]);
	if ((k.x | k.y | k.z) & ~M.g.key_mask) {
		atomicOr(&M.ctr->overflow, 32u);  // out-of-tree key: routed maps do not take them
		return;
	}
	Vec3 p;
	uint32_t rgb;
	load_point(a, i, p, rgb);
	const uint32_t owner = brick_owner(pack_key(k.x >> 4, k.y >> 4, k.z >> 4), M.route_world);
	route_hit(M, owner, pack_key(k.x, k.y, k.z), (uint32_t)(index_base + (unsigned long long)i * index_stride), rgb);
}

// An apply call after the first one starts from an empty touched list -- unless a call before it
// backed off: that call's list stays, for its replay after the pool growth (finalize_scan).
__global__ void k_route_next_apply(Counters* c)
{
	if (!(c->overflow & ~4u)) c->n_touched = 0;
}

// applies the records of sources [first, first + count), apply call `call` of the pass.  Colour maps:
// hit records only enter the apply table t (minimum global index per voxel); k_inbox_color applies
// them.  A brick pool that runs full leaves the records it could not place unapplied and flags the
// map; K3, the upper seed and every later call of the pass then back off, and the host grows the pool
// and replays the calls from this one on (finalize_scan).  route_call tells it which call that is.
__global__ void __launch_bounds__(256) k_inbox(DeviceMap M, uint32_t first, uint32_t count, ScanArgs t, uint32_t call)
{
	if (__ldg(&M.ctr->overflow) & ~4u) return;  // an earlier call of the pass backed off: replayed as a whole
	if (blockIdx.x == 0 && threadIdx.x == 0) M.ctr->route_call = call;
	const uint32_t lane = threadIdx.x & 31;
	constexpr uint32_t FULL = 0xffffffffu;
	const RouteTable* R = M.route;
	const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, warps = (gridDim.x * blockDim.x) >> 5;
	const uint32_t hw = M.color ? 2u : 1u;  // words per hit record
	for (uint32_t s = first; s < first + count; ++s) {
		const RouteBox box = R->in[s];
		const uint32_t nm = ld_volatile_u32(&box.hdr[0]), nh = ld_volatile_u32(&box.hdr[1]);
		for (uint32_t i = warp; i < nm; i += warps) {
			const unsigned long long* src = box.miss + (size_t)i * kMissRecWords;
			uint32_t slot = kNone;
			if (lane == 0) {
				slot = brick_find_or_create(M, src[0]);
				if (slot != kNone) touch_brick(M, slot);
			}
			slot = __shfl_sync(FULL, slot, 0);
			if (slot == kNone) continue;
			const unsigned long long m0 = src[1 + 2 * lane], m1 = src[2 + 2 * lane];
			unsigned long long* mp = M.miss_mask + (size_t)slot * 64 + 2 * lane;
			if (m0) atomicOr(mp, m0);
			if (m1) atomicOr(mp + 1, m1);
		}
		for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nh; i += gridDim.x * blockDim.x) {
			const unsigned long long rec = box.hit[(size_t)i * hw];
			if (rec & kFullBrick) {
				const uint32_t brick = brick_find_or_create(M, rec & ~kFullBrick);
				if (brick == kNone) continue;
				touch_brick(M, brick);
				ulonglong2* mm = reinterpret_cast<ulonglong2*>(M.miss_mask + (size_t)brick * 64);
				for (int c = 0; c < 32; ++c) mm[c] = make_ulonglong2(~0ull, ~0ull);
				continue;
			}
			uint32_t x, y, z;
			unpack_key(rec, x, y, z);
			const uint32_t brick = brick_find_or_create(M, pack_key(x >> 4, y >> 4, z >> 4));
			if (brick == kNone) continue;
			touch_brick(M, brick);
			if (M.color) {
				bool fresh;
				const uint32_t ts = table_insert(t, rec, &fresh);
				atomicMin(&t.tab_min[ts], (uint32_t)box.hit[2 * (size_t)i + 1]);
				continue;
			}
			atomicOr(&M.hit_mask[(size_t)brick * 64 + morton2(x >> 2, y >> 2, z >> 2)], 1ull << linear2(x, y, z));
			M.hit_stamp[brick] = M.scan_id;
		}
	}
}

// The bricks a routed pass touched -- stamped by its apply calls, scan ids first .. first + n - 1 --
// become the touched list again, so that the upper levels of a replayed pass are seeded from them.
// (Scan ids skip 0, the stamp of a brick no scan touched.)
__global__ void __launch_bounds__(256) k_touch_pass(DeviceMap M, uint32_t n_bricks, uint32_t first, uint32_t n)
{
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t stride = gridDim.x * blockDim.x;
	for (uint32_t b0 = blockIdx.x * blockDim.x; b0 < n_bricks; b0 += stride) {
		const uint32_t b = b0 + threadIdx.x, st = b < n_bricks ? M.brick_stamp[b] : 0u;
		const bool in = st != 0u && st - first < n;
		const uint32_t bal = __ballot_sync(0xffffffffu, in);
		if (!bal) continue;
		uint32_t base = 0;
		if (lane == 0) base = atomicAdd(&M.ctr->n_touched, (uint32_t)__popc(bal));
		base = __shfl_sync(0xffffffffu, base, 0);
		if (in) M.touched[base + __popc(bal & ((1u << lane) - 1u))] = b;
	}
}

// colour maps, after k_inbox: the record that holds its voxel's minimum global index sets the hit
// bit and blends its colour, as k_hits does on one GPU (same guard against blending twice)
__global__ void __launch_bounds__(256) k_inbox_color(DeviceMap M, uint32_t first, uint32_t count, ScanArgs t)
{
	if (__ldg(&M.ctr->overflow) & ~4u) return;  // k_inbox could not place every record: the call is replayed
	const RouteTable* R = M.route;
	for (uint32_t s = first; s < first + count; ++s) {
		const RouteBox box = R->in[s];
		const uint32_t nh = ld_volatile_u32(&box.hdr[1]);
		for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < nh; i += gridDim.x * blockDim.x) {
			const ulonglong2 r = reinterpret_cast<const ulonglong2*>(box.hit)[i];
			if (r.x & kFullBrick) continue;
			const uint32_t index = (uint32_t)r.y;
			bool fresh;
			const uint32_t ts = table_insert(t, r.x, &fresh);
			if (t.tab_min[ts] != index) continue;
			uint32_t x, y, z;
			unpack_key(r.x, x, y, z);
			const uint32_t brick = brick_find(M, pack_key(x >> 4, y >> 4, z >> 4));
			if (brick == kNone) continue;
			const size_t slot = (size_t)brick * 64 + morton2(x >> 2, y >> 2, z >> 2);
			const unsigned long long hbit = 1ull << linear2(x, y, z);
			const unsigned long long old = atomicOr(&M.hit_mask[slot], hbit);
			M.hit_stamp[brick] = M.scan_id;
			if ((old & hbit) || index == kNone) continue;  // already blended, or a point without colour
			blend_color(M, slot * 64 + morton2(x, y, z), (uint32_t)(r.y >> 32));
		}
	}
}

}  // namespace ufo_b200
