// ufo_page.cuh -- a map in bounded memory: release the bricks outside a bounding volume
// (ufo_b200_retain_bv), write them into a page blob first (ufo_b200_page_out_bv) and put a blob's
// bricks back (ufo_b200_page_in).  The reference has no counterpart: its pruneNode /
// deleteNodeChildren do not compile (SURVEY.md G5) and its stream format overwrites every node it
// reads, so a stream of the evicted part would wipe the retained part.
//
// One rule decides which bricks a volume keeps: a brick (depth-4 node) is kept iff every cube on its
// path from the root down to its own cube passes the volume (brick_chain, ufo_export.cuh).  Whole
// bricks only.  Retain compacts every per-brick array into a new, smaller allocation: classify,
// exclusive prefix sum of the keep flags (stable: survivors keep their order), one gather per array.
// A page holds what cannot be derived -- brick keys, leaves, octet-initialised bits, leaf colours --
// so it stays valid when the thresholds change before it comes back; page-in recomputes the rest
// with the import path's kernels (ufo_import.cuh).
#pragma once

#include "ufo_export.cuh"

namespace ufo_b200
{
constexpr unsigned long long kPageMagic = 0x31454741504f4655ull;  // "UFOPAGE1"
constexpr uint32_t kPageVersion = 1;

// Blob: this header, then whole sections: brick keys [n] u64 (ascending), leaves [n][4096] f32,
// octet-initialised bits [n][64] u8 (bits 16..23 of DeviceMap::meta), colour maps: leaf colours
// [n][4096] u32.  Blocks in Morton order inside a brick, voxels in Morton order inside a block, as
// in DeviceMap::leaf.
struct PageHeader {
	unsigned long long magic;
	uint32_t version;
	uint32_t color;
	unsigned long long resolution_bits;  // the map's resolution, the double's bits
	uint32_t depth_levels;
	uint32_t reserved;
	unsigned long long n_bricks;
	unsigned long long pad[3];
};
static_assert(sizeof(PageHeader) == 64, "the page header is 64 bytes");

constexpr size_t kPageLeafBytes = 4096 * sizeof(float);  // leaves (and leaf colours) of one brick
constexpr size_t kPageBitsBytes = 64;

UFO_HD size_t page_bytes(unsigned long long n_bricks, bool color)
{
	return sizeof(PageHeader) + (size_t)n_bricks * (8 + kPageLeafBytes + kPageBitsBytes + (color ? kPageLeafBytes : 0));
}

// One thread per live brick.  keep[b] = 1 iff the volume keeps brick b (`none`: the root misses the
// volume, nothing is kept).  For a page-out (skey != nullptr) the bricks to write get their packed key
// as sort key and every other brick ~0, so that a sort by key puts them first in ascending order;
// *n_out counts them.  Bricks that only collect out-of-tree marks own no voxels: never kept, never
// written.
__global__ void __launch_bounds__(256) k_page_classify(DeviceMap M, uint32_t n_bricks, Volume vol, int none, uint32_t* keep,
                                                       unsigned long long* skey, uint32_t* slot, uint32_t* n_out)
{
	const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b >= n_bricks) return;
	const unsigned long long key = M.brick_key[b];
	double c[3];
	const bool ok = !none && brick_chain(M, key, vol, c);
	if (keep) keep[b] = ok ? 1u : 0u;
	if (skey) {
		uint32_t x, y, z;
		unpack_key(key, x, y, z);
		const bool out = !ok && !((x | y | z) & ~(M.g.key_mask >> 4));
		skey[b] = out ? key : ~0ull;
		slot[b] = b;
		if (out) atomicAdd(n_out, 1u);
	}
}

// new slot -> old slot of the kept bricks, from the exclusive prefix sum of the keep flags
__global__ void __launch_bounds__(256) k_page_sources(uint32_t n_bricks, const uint32_t* keep, const uint32_t* new_slot, uint32_t* src)
{
	const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
	if (b < n_bricks && keep[b]) src[new_slot[b]] = b;
}

// Moves whole bricks of one array: 2^log2_per units of V per brick, brick-contiguous, so a warp
// reads and writes consecutive 128-bit words.  Gather: dst brick i <- src brick slot[i] (compaction,
// page-out staging).  Scatter: dst brick slot[i] <- src brick i (page-in).
template <class V, bool SCATTER>
__global__ void __launch_bounds__(256) k_page_move(V* __restrict__ dst, const V* __restrict__ src, const uint32_t* __restrict__ slot,
                                                   size_t n_units, uint32_t log2_per)
{
	const size_t low = ((size_t)1 << log2_per) - 1;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_units; i += (size_t)gridDim.x * blockDim.x) {
		const size_t j = ((size_t)__ldg(&slot[i >> log2_per]) << log2_per) | (i & low);
		if (SCATTER) dst[j] = src[i];
		else dst[i] = src[j];
	}
}

// octet-initialised bits of the blocks of bricks slot[0..n): meta -> bytes (page-out) ...
__global__ void __launch_bounds__(256) k_page_bits_out(const uint32_t* __restrict__ meta, const uint32_t* __restrict__ slot, size_t n_blocks,
                                                       uint8_t* __restrict__ out)
{
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_blocks; i += (size_t)gridDim.x * blockDim.x)
		out[i] = (uint8_t)(meta[(size_t)slot[i >> 6] * 64 + (i & 63)] >> 16);
}
// ... and bytes -> meta of bricks that were just created (page-in; k_import_refresh adds the flags)
__global__ void __launch_bounds__(256) k_page_bits_in(uint32_t* __restrict__ meta, const uint32_t* __restrict__ slot, size_t n_blocks,
                                                      const uint8_t* __restrict__ in)
{
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_blocks; i += (size_t)gridDim.x * blockDim.x)
		meta[(size_t)slot[i >> 6] * 64 + (i & 63)] = (uint32_t)in[i] << 16;
}

// Page-in, before anything is created: counts[0] = keys of the blob that exist in the map,
// counts[1] = keys no writer produces (outside the tree, or not in strictly ascending order)
__global__ void __launch_bounds__(256) k_page_lookup(DeviceMap M, const unsigned long long* keys, uint32_t n, uint32_t* counts)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const unsigned long long key = keys[i];
	uint32_t x, y, z;
	unpack_key(key, x, y, z);
	if ((key >> 63) || ((x | y | z) & ~(M.g.key_mask >> 4)) || (i && keys[i - 1] >= key)) atomicAdd(&counts[1], 1u);
	else if (brick_find(M, key) != kNone) atomicAdd(&counts[0], 1u);
}

// Page-in: slot of every key of the blob.  Idempotent, so a pass that ran into a full pool is
// repeated as a whole after the pool has grown (slot kNone: ctr->overflow is set).
__global__ void __launch_bounds__(256) k_page_create(DeviceMap M, const unsigned long long* keys, uint32_t n, uint32_t* slot)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) slot[i] = brick_find_or_create(M, keys[i]);
}

// The touched list of a pass over bricks slot[0..n) (nullptr: bricks 0..n) without stamping them:
// k_import_refresh, k_brick_agg and the upper-level pass read the list, the scan stamps stay as
// they are.
__global__ void __launch_bounds__(256) k_page_touch(DeviceMap M, const uint32_t* slot, uint32_t n)
{
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) M.touched[i] = slot ? slot[i] : i;
	if (blockIdx.x == 0 && threadIdx.x == 0) M.ctr->n_touched = n;
}

// blocks of bricks 0..n_bricks that hold a written octet (the host's block count after a retain)
__global__ void __launch_bounds__(256) k_page_count_blocks(const uint32_t* __restrict__ meta, size_t n_blocks, unsigned long long* count)
{
	uint32_t c = 0;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_blocks; i += (size_t)gridDim.x * blockDim.x)
		c += (meta[i] & 0xff0000u) ? 1u : 0u;
	c = __reduce_add_sync(0xffffffffu, c);
	if ((threadIdx.x & 31) == 0 && c) atomicAdd(count, (unsigned long long)c);
}

}  // namespace ufo_b200
