// ufo_device.cuh -- device-side data layout of one map and the lock-free
// find-or-create primitives the integration kernels share.
//
// Layout (DESIGN.md "Data layout in HBM"):
//   voxel  = depth-0 leaf            float log-odds (+ packed rgb for colour maps)
//   block  = 4^3 voxels  (depth 2)   64 floats = 256 B, Morton order inside the block, so
//                                    one 2^3 octet (depth-1 node) = 8 consecutive floats = one
//                                    32 B sector; per-scan miss/hit bit masks are one u64 each
//   brick  = 4^3 blocks  (depth 4)   hashed by packed (kx>>4, ky>>4, kz>>4).  A brick owns 64
//                                    CONSECUTIVE block slots (slot = brick*64 + Morton child), so
//                                    everything one warp of the update kernel touches is
//                                    contiguous (16 KB of leaves, 512 B of masks, ...), there is
//                                    no per-block allocation and no child-pointer indirection
//   upper  = depth >= 5 nodes        hashed by (depth, key>>depth); aggregates only
// This replaces the reference's pointer octree (octree_node.h:52-111,
// occupancy_map_node.h:55-185) with flat SoA pools addressed by slot index.
#pragma once

#include <cuda_runtime.h>

#include <cstdint>
#include <cstring>

#include "ufo_index.cuh"

namespace ufo_b200
{
constexpr uint64_t kEmptyKey = ~0ull;
constexpr uint32_t kPending = 0xffffffffu;  // hash value not published yet
constexpr uint32_t kFailed = 0xfffffffeu;   // allocation behind this key overflowed
constexpr uint32_t kNone = 0xffffffffu;     // "no such brick / node"
// touched_mi flag, set by k_gather for a brick without a hit this scan: k_update_brick does not
// stage its hit masks.  Lists built elsewhere leave it clear, so their bricks stage them.
constexpr uint32_t kMiNoHits = 1u << 31;
// touched_mi / touched_mi2 of a paired pass: the brick was not marked by that scan
constexpr uint32_t kMiAbsent = kNone;

// aggregate of an inner node: max log-odds of the subtree + contains_* flags
// (occupancy_map_base.h:1179-1224).  flags: bit0 contains_free, bit1 contains_unknown.
struct Agg {
	float occ;
	uint32_t flags;
};

struct Counters {
	uint32_t n_blocks;   // blocks that ever received an update (statistics only)
	uint32_t n_bricks;   // next free brick slot
	uint32_t n_upper;    // next free upper-node slot
	uint32_t overflow;   // bit1 bricks/brick hash, bit2 upper nodes, bit3 ray-record buffer, bit4 ray bound violated (bug), bit5 alias arrays needed, bit8 early-stopping buffers
	uint32_t n_touched;    // bricks stamped by this scan = length of DeviceMap::touched
	uint32_t item_cursor;  // next work unit of the fused walk (k_walk_mark)
	uint32_t k3_cursor;    // touched entries claimed by k_update_brick's warps beyond their first (zeroed before each launch)
	uint32_t max_span;     // longest ray of the scan in dominant-axis steps (sets the shell thickness)
	uint32_t n_touched_alt;  // routed mode: length of DeviceMap::touched_alt
	uint32_t route_call;     // routed mode: the last apply call of the pass whose k_inbox ran (did not back off)
	uint32_t n_dirty;        // dense mode: length of DeviceMap::vol_list (also: node list of insert depth 5/6, bricks of a write batch)
	uint32_t list_count[3];  // dirty-list lengths of the upper-level pass (rotating by depth % 3)
	uint32_t n_rays;
	uint32_t ray_batch;  // next batch of 32 rays for the persistent ray-walk warps
	uint32_t n_chunks;   // longest ray-record region of the scan, in kChunk slices
	uint32_t alias_marks;  // out-of-range keys marked this scan (0 almost always)
	unsigned long long seg_total;  // ray-walk records reserved by K1
	unsigned long long visits;
	unsigned long long touched_voxels;
	unsigned long long hit_voxels;
	unsigned long long touched_octets;
	unsigned long long touched_blocks;
	unsigned long long touched_d3;
	unsigned long long touched_bricks;
	unsigned long long upper_nodes;
	unsigned long long upper_pair[2];  // paired pass: upper nodes above the bricks of its first / second scan
	unsigned long long bbox[6];  // order-preserving encoding of min xyz / max xyz of this scan
	// dense fused walk, profiling level 2 only (k_walk_mark<COUNT = true>): block records pushed,
	// global mask reductions issued, of those the ones that found the word empty, dirty-bit reductions
	unsigned long long walk_records, walk_mask_reds, walk_words, walk_dirty_reds;
	// early stopping (ufo_early.cuh): visits and distinct nodes of the walks, nodes in the free set,
	// rounds run, 1 when the rounds reached their fixed point; the lowest ray whose prefix changed
	// (two slots, alternating by round)
	unsigned long long e_visits, e_nodes, e_free;
	uint32_t e_rounds, e_converged, e_low[2];
	// k_update statistics spread over slots: [slot][0 voxels, 1 hit voxels, 2 octets, 3 blocks,
	// 4 first-touched blocks, 5 bricks, 6 depth-3 nodes, 7 128 B leaf lines read]; a paired pass counts
	// its first scan in slots 0..31 and its second in 32..63
	unsigned long long stat[64][8];
};

// k_update_brick at profiling level 2 only, in an allocation of its own (not part of the per-scan
// copies of Counters), same slots as Counters::stat: [slot][0 touched octets of saturated pairs,
// 1 leaf lines not read because of them, 2 leaf sectors not written back]
struct K3Stats {
	unsigned long long slot[64][3];
};

// Routed multi-GPU mode (SURVEY.md 8(e) variant 2): every rank walks ITS rays into its own map,
// then the per-brick miss masks and the hit voxels of bricks another rank owns are written
// straight into that rank's inbox over NVLink peer memory (ufo_route.cuh).
constexpr uint32_t kMaxRanks = 16;
constexpr uint32_t kMissRecWords = 65;  // brick key + 64 block masks
// Hit-region record flag: the record is a brick key whose 64 blocks are all free space (insert
// depth 5/6: a brick below a free-space node), not a voxel key.  Packed keys use bits 0..62.
constexpr unsigned long long kFullBrick = 1ull << 63;
struct RouteBox {                       // one (source -> destination) region of one parity, in the destination's memory
	unsigned long long* miss;             // [cap_m][kMissRecWords]
	// [cap_h] hit records.  Mono maps: one word, the packed voxel key.  Colour maps: two words,
	// {packed voxel key, global cloud index | rgb << 32}; index kNone = a point without colour.
	unsigned long long* hit;
	uint32_t* hdr;                        // [0] records, [1] hit keys: published by the source when its pass is complete
};
struct RouteTable {
	RouteBox out[kMaxRanks];  // where this rank's records for rank d go (peer memory)
	RouteBox in[kMaxRanks];   // where the records of rank s arrive (own memory)
	uint32_t out_miss[kMaxRanks], out_hit[kMaxRanks];  // cursors of the current pass
	uint32_t out_full;  // whole-brick records of the current pass (statistics)
	uint32_t cap_m, cap_h;
	uint32_t overflow;  // a region was too small
	uint32_t sent[3];   // last pass, all destinations: mask records, whole-brick records, hit records (read with overflow)
};

struct DeviceMap {
	Geometry g;
	// sensor model (occupancy_map_base.h:1537-1542): thresholds compared in double,
	// updates applied in float
	double occ_thr, free_thr;
	float hit, clamp_min, clamp_max;
	float free_ceil, occ_floor;  // float thresholds equivalent to the double compares (see leaf_flags)
	double prob_hit;         // toProb(float(hit)) used by the colour blend
	uint32_t default_flags;  // flags of a never-touched voxel / subtree (value 0.0)
	// no leaf value of the map lies below clamp_min, and clamp_min is nonzero and <= clamp_max: a scan
	// may leave saturated pairs alone (see apply_update)
	uint32_t sat_skip;
	K3Stats* k3_stat;  // profiling level 2: k_update_brick counts into it (nullptr: not counted)
	uint32_t color;
	uint32_t scan_id;
	// spatial sharding over several GPUs: this map only keeps the bricks it owns
	uint32_t shard_rank, shard_world;  // world <= 1: owns everything
	// routed mode: ownership as above, but foreign marks are forwarded instead of dropped
	uint32_t route_rank, route_world, route_self;  // route_self: own marks go through the inbox too (ordered merge of several sensors)
	RouteTable* route;

	// brick hash (open addressing, linear probing): 16-byte entries {key, slot} so one
	// 128-bit load resolves a probe
	ulonglong2* bh_tab;
	uint32_t bh_mask;
	// brick pool
	unsigned long long* brick_key;
	uint32_t* brick_stamp;  // scan id of the last scan that touched the brick
	uint32_t* touched;      // [brick_cap] bricks stamped by the current scan, in stamping order (touch_brick)
	uint32_t* touched_mi;   // [brick_cap] where the free-space masks of touched[i] are: mask_base + (mi & ~kMiNoHits) * 64
	uint32_t* hit_stamp;    // [brick_cap] scan id of the last scan that set a hit bit of the brick
	unsigned long long* mask_base;  // per scan: miss_mask (mi = brick slot) or the dense scan volume (mi = volume brick)
	// Paired pass (two consecutive scans, one leaf update): the second scan marks into a second dense
	// volume (mask_base2) and a second hit-mask array; touched_mi2[i] locates its masks of touched[i]
	// (kMiAbsent: not marked by it, and likewise touched_mi for the first scan).  touch_idx[brick] is the
	// brick's entry in the touched list of the last dense gather, pair_id the first scan's id while the
	// second one gathers (0 otherwise)
	unsigned long long* mask_base2;
	unsigned long long* hit_mask2;
	uint32_t* touched_mi2;
	uint32_t* touch_idx;
	uint32_t pair_id;
	// Dense scan volume (ufo_walk.cuh): block masks of the cube of bricks around the sensor that a
	// range-limited scan can reach, brick-major ([volume brick][64 blocks in Morton order]), so that
	// the ray walk marks with a computed address and no lookup.  vol_dirty: one bit per volume brick.
	unsigned long long* vol;
	unsigned long long* vol_dirty;
	uint32_t* vol_list;                  // [words of vol_dirty] non-empty words of the dirty bitmap (k_gather_scan)
	uint32_t vol_db;                     // bricks per axis
	uint32_t vol_g0x, vol_g0y, vol_g0z;  // brick coordinates (key >> 4) of the volume's origin
	uint32_t dense;                      // this scan marks into the volume
	uint32_t* touched_alt;  // routed mode: own bricks that keep local marks after the outbox pass (next touched list)
	uint32_t* touched_alt_mi;
	Agg* brick_sum3;        // [brick][8]
	Agg* brick_sum4;        // [brick]
	uint32_t* brick_rgb3;   // colour maps: [brick][8] packed rgb of depth-3 nodes
	uint32_t* brick_rgb4;
	uint32_t brick_cap;
	// block arrays, index b = brick * 64 + Morton child index (brick-contiguous)
	float* leaf;                    // [b][64] log-odds, Morton order inside the block
	uint32_t* leaf_rgb;             // colour maps: [b][64] packed r | g<<8 | b<<16
	unsigned long long* miss_mask;  // [b] per-scan free-set bits, linear order x + 4y + 16z
	unsigned long long* hit_mask;   // [b] per-scan hit bits
	unsigned long long* chg_mask;   // [b] voxels changed since the last reset (allocated by enableChangeDetection)
	uint32_t* meta;                 // [b] bits 0..15: flags of the 8 octets, bits 16..23: octet initialised
	// [b] line maxima: component h = max of the depth-1 nodes (octets) 4h..4h+3, the octets of the
	// block's 128 B leaf line h, an uninitialised octet counting as 0.0.  The depth-2 value is their
	// max (block_occ), the depth-2 flags follow from meta (block_flags), a depth-1 value is the max of
	// the octet's 32 B leaf sector (octet_occ).
	float2* line_max;
	uint32_t* rgb2;                 // colour maps: [b]
	uint32_t* sum1_rgb;             // colour maps: [b][8]
	// Keys outside [0, 2^L) (a coordinate exactly on the + face of the map, or a walk that
	// overshoots the - face): the reference's per-scan sets keep them as distinct voxels
	// (code.h keeps 21 bits per axis) while its tree only consumes L bits, so the wrapped
	// voxel is updated once more.  Such marks are collected under their UNWRAPPED brick key
	// in these two arrays (allocated on first use) and applied by k_alias_* (see there).
	unsigned long long* alias_miss;  // [b]
	unsigned long long* alias_hit;   // [b]
	// upper nodes
	unsigned long long* uh_keys;
	uint32_t* uh_vals;
	uint32_t uh_mask;
	unsigned long long* up_key;
	Agg* up_agg;
	uint32_t* up_rgb;
	uint32_t* up_stamp;
	// Push-up propagation (k_upper_*): every node keeps the aggregates of its eight children
	// (written by the children when they change) and the slot of its parent, so that a level of
	// the propagation pass is one 64-byte read per dirty node and no hash probe.
	Agg* up_child;           // [up_cap][8]
	uint32_t* up_child_rgb;  // colour maps: [up_cap][8]
	uint32_t* up_valid;      // [up_cap] bit c: child c has reported (others count as never-touched space)
	uint32_t* up_parent;     // [up_cap] slot of the parent node (kNone: not resolved yet)
	uint32_t* brick_parent;  // [brick_cap] slot of the brick's depth-5 parent (kNone: not resolved yet)
	uint32_t up_cap;
	uint32_t up_epoch;  // id of the current upper-level pass (a pass repeated after a pool growth gets a new one)

	Counters* ctr;
};

// ---------------------------------------------------------------------------
__device__ __forceinline__ uint32_t ld_volatile_u32(const uint32_t* p)
{
	return *reinterpret_cast<const volatile uint32_t*>(p);
}
__device__ __forceinline__ unsigned long long ld_volatile_u64(const unsigned long long* p)
{
	return *reinterpret_cast<const volatile unsigned long long*>(p);
}
__device__ __forceinline__ void st_volatile_u32(uint32_t* p, uint32_t v)
{
	*reinterpret_cast<volatile uint32_t*>(p) = v;
}

UFO_HD uint32_t hash_u64(uint64_t k)
{
	k ^= k >> 33;
	k *= 0xff51afd7ed558ccdull;
	k ^= k >> 33;
	k *= 0xc4ceb9fe1a85ec53ull;
	k ^= k >> 33;
	return (uint32_t)k;
}

// Owner rank of a brick when a map is sharded over several GPUs: a hash of the brick key, so
// that every rank gets an equal share of the touched space wherever the sensor is.
UFO_HD uint32_t brick_owner(uint64_t brick_key, uint32_t world)
{
	return (uint32_t)((hash_u64(brick_key ^ 0x9e3779b97f4a7c15ull) >> 7) % world);
}

// Whether a write batch or setValueVolume applies to the brick on this map: every rank of a routed
// map takes the same call and only the owner creates and writes the brick, so that the ranks keep
// disjoint bricks whose union is the single map.
UFO_HD bool brick_owned(const DeviceMap& M, uint64_t brick_key)
{
	return M.route_world <= 1 || brick_owner(brick_key, M.route_world) == M.route_rank;
}

// 21 bits per axis
UFO_HD uint64_t pack_key(uint32_t x, uint32_t y, uint32_t z)
{
	return (uint64_t)x | ((uint64_t)y << 21) | ((uint64_t)z << 42);
}
UFO_HD void unpack_key(uint64_t k, uint32_t& x, uint32_t& y, uint32_t& z)
{
	x = (uint32_t)(k & 0x1fffffu);
	y = (uint32_t)((k >> 21) & 0x1fffffu);
	z = (uint32_t)((k >> 42) & 0x1fffffu);
}
// key of an upper node: depth tag in bits 63.. is not available (3*21 = 63 bits
// used), but an upper node at depth d >= 5 only uses 16 bits per axis, so the tag
// sits in the unused high bits of the x field.
UFO_HD uint64_t upper_key(uint32_t depth, uint32_t x, uint32_t y, uint32_t z)
{
	return pack_key(x, y, z) | ((uint64_t)depth << 16);
}

// ---------------------------------------------------------------------------
// brick hash
// ---------------------------------------------------------------------------
__device__ __forceinline__ ulonglong2 ld_volatile_entry(const ulonglong2* p)
{
	ulonglong2 v;
	asm volatile("ld.volatile.global.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
	return v;
}

// L1-cached read of an entry, for optimistic first probes: a stale line can only show an entry
// as still empty / pending or with an old stamp (keys never change inside a kernel), and every
// caller falls back to the volatile / atomic path in those cases.
__device__ __forceinline__ ulonglong2 ld_cached_entry(const ulonglong2* p)
{
	ulonglong2 v;
	asm volatile("ld.global.ca.v2.u64 {%0, %1}, [%2];" : "=l"(v.x), "=l"(v.y) : "l"(p));
	return v;
}

// value field of an entry: low 32 bits = brick slot / kPending / kFailed
__device__ __forceinline__ uint32_t brick_find(const DeviceMap& M, uint64_t key)
{
	uint32_t i = hash_u64(key) & M.bh_mask & ~1u;  // buckets of two entries (one 32 B sector)
	for (uint32_t probes = 0; probes <= M.bh_mask; ++probes) {
		ulonglong2 e = ld_volatile_entry(&M.bh_tab[i]);
		if (e.x == key) {
			uint32_t v = (uint32_t)e.y;
			return (v == kPending || v == kFailed) ? kNone : v;
		}
		if (e.x == kEmptyKey) return kNone;
		i = (i + 1) & M.bh_mask;
	}
	return kNone;
}

// First mark of a brick in a scan: stamp it and append it to the scan's touched list, which is
// what the update and propagation kernels iterate over (cost of a scan = O(touched), not O(map)).
__device__ __forceinline__ void touch_brick(const DeviceMap& M, uint32_t slot)
{
	if (ld_volatile_u32(&M.brick_stamp[slot]) == M.scan_id) return;
	if (atomicExch(&M.brick_stamp[slot], M.scan_id) != M.scan_id) {
		const uint32_t i = atomicAdd(&M.ctr->n_touched, 1u);
		M.touched[i] = slot;
		M.touched_mi[i] = slot;
	}
}

// dense mode: index of the volume brick that holds brick coordinates (bx, by, bz) = key >> 4, or
// kNone outside the volume
__device__ __forceinline__ uint32_t vol_brick(const DeviceMap& M, uint32_t bx, uint32_t by, uint32_t bz)
{
	const uint32_t rx = bx - M.vol_g0x, ry = by - M.vol_g0y, rz = bz - M.vol_g0z;
	if (rx >= M.vol_db || ry >= M.vol_db || rz >= M.vol_db) return kNone;
	return (rz * M.vol_db + ry) * M.vol_db + rx;
}
// a volume brick received a mark: one fire-and-forget reduction on the dirty bitmap (a returning
// atomic here costs the walk measurably); k_gather_scan / k_gather turn
// the bitmap into the touched list
__device__ __forceinline__ void vol_touch(const DeviceMap& M, uint32_t vb)
{
	atomicOr(&M.vol_dirty[vb >> 6], 1ull << (vb & 63u));
}

// continues a probe sequence at table index i (entry e already loaded or not)
__device__ __forceinline__ uint32_t brick_find_or_create_from(const DeviceMap& M, uint64_t key, uint32_t i)
{
	for (uint32_t probes = 0; probes <= M.bh_mask; ++probes) {
		unsigned long long* kp = &M.bh_tab[i].x;
		uint32_t* vp = reinterpret_cast<uint32_t*>(&M.bh_tab[i].y);
		unsigned long long k = ld_volatile_u64(kp);
		if (k == kEmptyKey) {
			if (ld_volatile_u32(&M.ctr->overflow) & 2u) return kNone;
			k = atomicCAS(kp, kEmptyKey, (unsigned long long)key);
			if (k == kEmptyKey) {
				uint32_t s = atomicAdd(&M.ctr->n_bricks, 1u);
				if (s >= M.brick_cap) {
					atomicOr(&M.ctr->overflow, 2u);
					st_volatile_u32(vp, kFailed);
					return kNone;
				}
				// brick_key / block_key are only read by later kernels (export, rebuild), so
				// publishing the slot needs no fence
				M.brick_key[s] = key;
				vp[1] = 0;  // cached scan stamp (see k_scatter)
				st_volatile_u32(vp, s);
				return s;
			}
		}
		if (k == key) {
			// The key is in the table but its slot may not be published yet (value == kPending).
			// Forward progress of this wait: the thread that won the CAS publishes with straight-line
			// code -- one atomicAdd, two stores, no wait of its own -- so it finishes as soon as it is
			// scheduled.  (a) Winner in another warp: it is a resident thread (it executed the CAS), and
			// resident warps keep being scheduled.  (b) Winner in THIS warp: it diverged from the waiting
			// lanes at `k == kEmptyKey` above; sm_70+ schedules the diverged paths of a warp
			// independently, and there is no convergence barrier (__syncwarp, *_sync shuffle or vote)
			// between the CAS and the publishing store, so the winner's path runs while these lanes
			// poll.  The volatile load keeps the loop an actual re-read.  Callers must not invoke this
			// function from inside a region that some lanes leave through a warp-synchronous primitive.
			uint32_t v;
			while ((v = ld_volatile_u32(vp)) == kPending) {
			}
			return v == kFailed ? kNone : v;
		}
		i = (i + 1) & M.bh_mask;
	}
	atomicOr(&M.ctr->overflow, 2u);
	return kNone;
}

__device__ __forceinline__ uint32_t brick_find_or_create(const DeviceMap& M, uint64_t key)
{
	return brick_find_or_create_from(M, key, hash_u64(key) & M.bh_mask & ~1u);
}

__device__ __forceinline__ uint32_t upper_find(const DeviceMap& M, uint64_t key)
{
	uint32_t i = hash_u64(key) & M.uh_mask;
	for (uint32_t probes = 0; probes <= M.uh_mask; ++probes) {
		unsigned long long k = ld_volatile_u64(&M.uh_keys[i]);
		if (k == key) {
			uint32_t v = ld_volatile_u32(&M.uh_vals[i]);
			return (v == kPending || v == kFailed) ? kNone : v;
		}
		if (k == kEmptyKey) return kNone;
		i = (i + 1) & M.uh_mask;
	}
	return kNone;
}

__device__ __forceinline__ uint32_t upper_find_or_create(const DeviceMap& M, uint64_t key)
{
	uint32_t i = hash_u64(key) & M.uh_mask;
	for (uint32_t probes = 0; probes <= M.uh_mask; ++probes) {
		unsigned long long k = ld_volatile_u64(&M.uh_keys[i]);
		if (k == kEmptyKey) {
			if (ld_volatile_u32(&M.ctr->overflow) & 4u) return kNone;
			k = atomicCAS(&M.uh_keys[i], kEmptyKey, (unsigned long long)key);
			if (k == kEmptyKey) {
				uint32_t s = atomicAdd(&M.ctr->n_upper, 1u);
				if (s >= M.up_cap) {
					atomicOr(&M.ctr->overflow, 4u);
					st_volatile_u32(&M.uh_vals[i], kFailed);
					return kNone;
				}
				M.up_key[s] = key;
				__threadfence();
				st_volatile_u32(&M.uh_vals[i], s);
				return s;
			}
		}
		if (k == key) {
			uint32_t v;
			// same wait as in brick_find_or_create_from (see the forward-progress argument there)
			while ((v = ld_volatile_u32(&M.uh_vals[i])) == kPending) {
			}
			return v == kFailed ? kNone : v;
		}
		i = (i + 1) & M.uh_mask;
	}
	atomicOr(&M.ctr->overflow, 4u);
	return kNone;
}

// ---------------------------------------------------------------------------
// order-preserving double <-> u64 for atomicMin/atomicMax on the change bbox
// ---------------------------------------------------------------------------
UFO_HD unsigned long long encode_ordered(double d)
{
	unsigned long long u;
#if defined(__CUDA_ARCH__)
	u = (unsigned long long)__double_as_longlong(d);
#else
	memcpy(&u, &d, sizeof(u));
#endif
	return (u & 0x8000000000000000ull) ? ~u : (u | 0x8000000000000000ull);
}

UFO_HD double decode_ordered(unsigned long long u)
{
	u = (u & 0x8000000000000000ull) ? (u & 0x7fffffffffffffffull) : ~u;
#if defined(__CUDA_ARCH__)
	return __longlong_as_double((long long)u);
#else
	double d;
	memcpy(&d, &u, sizeof(d));
	return d;
#endif
}

// sensor-model predicates (occupancy_map_base.h:926-940).  The reference compares the
// float value against DOUBLE thresholds; for a float v and a double T,
//   T > v  <=>  v < ceil_f32(T)      T <= v  <=>  v >= ceil_f32(T)      T >= v  <=>  v <= floor_f32(T)
// (no float lies strictly between floor_f32(T) and ceil_f32(T)), so two float compares
// against host-computed free_ceil / occ_floor are exactly equivalent.
__device__ __forceinline__ uint32_t leaf_flags(const DeviceMap& M, float v)
{
	uint32_t f = (v < M.free_ceil) ? 1u : 0u;
	if (v >= M.free_ceil && v <= M.occ_floor) f |= 2u;
	return f;
}

// depth-1 value of an initialised octet: the max of its eight leaves (one 32 B sector)
__device__ __forceinline__ float octet_occ(const float* lp)
{
	const float4 a = reinterpret_cast<const float4*>(lp)[0], c = reinterpret_cast<const float4*>(lp)[1];
	return fmaxf(fmaxf(fmaxf(a.x, a.y), fmaxf(a.z, a.w)), fmaxf(fmaxf(c.x, c.y), fmaxf(c.z, c.w)));
}
// depth-2 value of a block from its line maxima
__device__ __forceinline__ float block_occ(float2 q) { return fmaxf(q.x, q.y); }
// line maxima of a block from the maxima of its 8 octets
__device__ __forceinline__ float2 line_maxima(const float (&om)[8])
{
	return make_float2(fmaxf(fmaxf(om[0], om[1]), fmaxf(om[2], om[3])), fmaxf(fmaxf(om[4], om[5]), fmaxf(om[6], om[7])));
}
// depth-2 flags of a block from its meta word: an uninitialised octet is unknown space
__device__ __forceinline__ uint32_t block_flags(const DeviceMap& M, uint32_t mt)
{
	uint32_t f = 0;
#pragma unroll
	for (uint32_t o = 0; o < 8; ++o) f |= ((mt >> (16 + o)) & 1u) ? (mt >> (2 * o)) & 3u : M.default_flags;
	return f;
}

// float add + float clamp (occupancy_map_base.h:1139-1145).
// Saturated lines.  Let c = clamp_min be nonzero with c <= clamp_max, and let no leaf of the map lie
// below c (DeviceMap::sat_skip; the voxels of an initialised octet that no update has reached hold
// 0.0, so this needs c < 0).  If all four octets of a leaf line are initialised and the line maximum
// is c bit for bit, every one of its 32 leaves is >= c and <= c, so it equals c, and being nonzero it
// has c's bits.  For a miss u <= 0 (and not NaN), v + u <= c, so fmaxf(v + u, c) = c and fminf(c,
// clamp_max) = c: every marked voxel keeps its bits, the reference's updateOccupancy reports no
// change, and leaves, octet flags, line maximum, colours, change mask and every aggregate above stay
// as they are.  c = 0 is left out because -0.0 and +0.0 compare equal but differ in their bits.  Hits
// are applied before misses and can raise a voxel, so a line with a hit bit is updated as usual.
__device__ __forceinline__ float apply_update(const DeviceMap& M, float v, float u)
{
	return fminf(fmaxf(__fadd_rn(v, u), M.clamp_min), M.clamp_max);
}

// toProb(float) (occupancy_map_base.h:911): 1/(1+expf(-x)); expf evaluated via the
// double exp and rounded to float, which matches a correctly rounded expf.
__device__ __forceinline__ double to_prob(float logit)
{
	float e = (float)exp((double)(-logit));
	return 1.0 / (1.0 + (double)e);
}

}  // namespace ufo_b200
