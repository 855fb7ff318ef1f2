// ufo_early.cuh -- early stopping (insertPointCloud[Discrete] with early_stopping = E > 0) on the
// device, equal to the reference's sequential walk (freeSpaceNormal / freeSpaceSimple,
// occupancy_map_base.h:1261-1339).  DESIGN.md section 7a states the contract and the proofs.
//
//   E1 [discrete: k_early_rank, k_early_place] k_early_count -> exclusive scan -> k_early_check -> k_early_fill: every ray's visit sequence
//      (the walk k_rays / k_rays_simple perform) as slots of a scan-local node table, in CSR form
//   E2 k_early_rounds: Jacobi rounds over the rays' prefix lengths, one cooperative kernel with
//      grid-wide barriers, until no prefix changes
//   E3 k_early_mark: every node some prefix holds gets the miss, through the marking helpers of the
//      record path (shard filter and out-of-tree keys included); the table is emptied for the next scan
//
// The map after a scan depends only on the union of the prefixes (one miss per node of the free
// set, hits independent of it), so K1, K1b, K3 and K4 run unchanged around E1-E3.
#pragma once

#include <cooperative_groups.h>

#include "ufo_kernels.cuh"

namespace ufo_b200
{
constexpr uint32_t kEarlyThreads = 256;

struct EarlyArgs {
	uint32_t stop;              // E: the walk ends at the visit that makes E present nodes in a row
	int simple;                 // fixed-step samples instead of the DDA
	unsigned long long* keys;   // [tab_mask + 1] node key (unwrapped, >> depth, packed), kEmptyKey = free slot
	uint32_t* first;            // [tab_mask + 1] lowest ray whose prefix holds the node, kNone = none
	uint32_t tab_mask;
	unsigned long long* cnt;    // [n + 1] visits per ray (cnt[n] = 0)
	unsigned long long* off;    // [n + 1] exclusive sum of cnt: the ray's first visit; off[n] = all visits
	uint32_t* ids;              // [id_cap] table slot of every visit, ray after ray
	unsigned long long id_cap;
	uint32_t* plen;             // [n] prefix length of the last round
	uint32_t* pnext;            // [n] prefix length computed by the current round
};

// The visit sequence of ray i, in walk order (end point -> sensor), as keys at the insert depth:
// the backward DDA of k_rays (walk_init / walk_step, loop condition of occupancy_map_base.h:1300),
// the single node when both ends share it (:1281-1284), or the fixed-step samples of k_rays_simple.
template <class F>
__device__ __forceinline__ void early_walk(const DeviceMap& M, const ScanArgs& a, int simple, uint32_t i, F&& visit)
{
	const double* r = a.ray_end + 3 * (size_t)i;
	Vec3 to = {r[0], r[1], r[2]};
	if (to.x != to.x) return;
	Vec3 from = a.origin;
	if (!move_line_inside(M.g, from, to)) return;
	Vec3 dir = vsub(from, to);
	const double dist = vnorm(dir);
	dir = vdiv(dir, dist);
	if (simple) {
		const double size = node_size(M.g, a.depth);
		const int num_steps = (int)dop::div(dist, size);
		const Vec3 step = vscale(dir, size);
		Vec3 cur = to;
		for (int s = 0; s <= num_steps; ++s) {
			visit(point_to_key(M.g, cur, a.depth));
			cur = vadd(cur, step);
		}
		return;
	}
	Walk w;
	walk_init(M.g, to, from, dir, a.depth, w);
	if (w.same) {
		visit(w.cur);
		return;
	}
	while (true) {
		visit(w.cur);
		walk_step(w);
		if (w.cur == w.end || !(w.tx <= dist || w.ty <= dist || w.tz <= dist)) break;
	}
}

// A Code keeps 21 bits per axis (code.h:336-347), so a key outside the tree is its own node, as in
// the reference's CodeMap; the bits below the insert depth are the same for every key of a node.
__device__ __forceinline__ unsigned long long early_node(Key3 k, uint32_t depth)
{
	return pack_key((k.x & 0x1fffffu) >> depth, (k.y & 0x1fffffu) >> depth, (k.z & 0x1fffffu) >> depth);
}

// Discrete scans: K1 keeps one ray per end node (and per hit voxel), whichever thread wins the
// table insert, while the reference keeps the first point of the group in cloud order
// (occupancy_map_base.h:354-399).  The rays of a group are identical and a later copy adds nothing
// to the free set, but the kept ray's position in the order matters.  The end node of point i is
// found as K1 finds it (same branches), for the points K1 drops as duplicates too.
__device__ __forceinline__ bool early_end_node(const DeviceMap& M, const ScanArgs& a, uint32_t i, Key3& ek)
{
	const Geometry& g = M.g;
	Vec3 end;
	uint32_t rgb;
	if (!load_point(a, i, end, rgb)) return false;
	const double sq_max = dop::mul(a.max_range, a.max_range);
	if (!(0 > a.max_range || vsqnorm(vsub(end, a.origin)) < sq_max)) {
		Vec3 dir = vsub(key_to_coord(g, point_to_key(g, end, a.depth), a.depth), a.origin);
		if (a.use_color) {
			const double sq = vsqnorm(dir);
			if (0 <= a.max_range && sq > sq_max) {
				dir = vdiv(dir, dop::sqrt(sq));
				end = vadd(a.origin, vscale(dir, a.max_range));
			}
		} else {
			const double nrm = vnorm(dir);
			dir = vdiv(dir, nrm);
			if (0 <= a.max_range && nrm > a.max_range) end = vadd(a.origin, vscale(dir, a.max_range));
		}
	}
	Vec3 cur = a.origin;
	if (!move_line_inside(g, cur, end)) return false;
	ek = point_to_key(g, end, a.depth);
	return true;
}

constexpr unsigned long long kRankTag = 1ull << 63;  // table entries of end nodes (node keys use 63 bits)

// slot of `key` in the scan-local table (find or insert); *fresh is set when this call inserted it
__device__ __forceinline__ uint32_t early_slot(const EarlyArgs& e, unsigned long long key, bool* fresh = nullptr)
{
	uint32_t s = hash_u64(key) & e.tab_mask;
	while (true) {
		unsigned long long cur = ld_volatile_u64(&e.keys[s]);
		if (cur == kEmptyKey) {
			cur = atomicCAS(&e.keys[s], kEmptyKey, key);
			if (cur == kEmptyKey) {
				if (fresh) *fresh = true;
				return s;
			}
		}
		if (cur == key) return s;
		s = (s + 1) & e.tab_mask;
	}
}

// lowest cloud index per end node
__global__ void __launch_bounds__(kEarlyThreads) k_early_rank(DeviceMap M, ScanArgs a, EarlyArgs e)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	Key3 ek;
	if (i >= a.n || !early_end_node(M, a, i, ek)) return;
	atomicMin(&e.first[early_slot(e, early_node(ek, a.depth) | kRankTag)], i);
}

// the kept ray of every group moves to the group's lowest cloud index (that point cast no ray in K1)
__global__ void __launch_bounds__(kEarlyThreads) k_early_place(DeviceMap M, ScanArgs a, EarlyArgs e)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n) return;
	double* r = a.ray_end + 3 * (size_t)i;
	Key3 ek;
	if (r[0] != r[0] || !early_end_node(M, a, i, ek)) return;
	const uint32_t m = e.first[early_slot(e, early_node(ek, a.depth) | kRankTag)];
	if (m >= i) return;
	double* t = a.ray_end + 3 * (size_t)m;
	t[0] = r[0];
	t[1] = r[1];
	t[2] = r[2];
	r[0] = __longlong_as_double(0x7ff8000000000000ll);
}

__global__ void __launch_bounds__(kEarlyThreads) k_early_count(DeviceMap M, ScanArgs a, EarlyArgs e)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i > a.n) return;
	unsigned long long c = 0;
	if (i < a.n) early_walk(M, a, e.simple, i, [&](Key3) { ++c; });
	e.cnt[i] = c;
}

// After the scan of the counts: the id buffer must hold every visit and the table stay below 80 %
// load (distinct nodes <= visits, end nodes of a discrete scan <= n), otherwise the host grows both
// and repeats the scan (bit 256).
__global__ void k_early_check(DeviceMap M, EarlyArgs e, uint32_t n)
{
	const unsigned long long total = e.off[n];
	M.ctr->e_visits = total;
	M.ctr->e_low[0] = M.ctr->e_low[1] = kNone;
	if (total > e.id_cap || total + total / 4 + n + 1 > (unsigned long long)e.tab_mask + 1) atomicOr(&M.ctr->overflow, 256u);
}

__global__ void __launch_bounds__(kEarlyThreads) k_early_fill(DeviceMap M, ScanArgs a, EarlyArgs e)
{
	if (ld_volatile_u32(&M.ctr->overflow) & 256u) return;
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= a.n) return;
	uint32_t* out = e.ids + e.off[i];
	uint32_t k = 0, fresh = 0;
	early_walk(M, a, e.simple, i, [&](Key3 key) {
		bool inserted = false;
		const uint32_t s = early_slot(e, early_node(key, a.depth), &inserted);
		fresh += inserted ? 1u : 0u;
		out[k++] = s;
		atomicMin(&e.first[s], i);  // round 0: every prefix is the whole walk
	});
	e.plen[i] = k;
	if (fresh) atomicAdd(&M.ctr->e_nodes, (unsigned long long)fresh);
}

// E2.  Round r computes every prefix at or above the frontier F from `first` of round r - 1:
// visit k of ray j is "present" when an earlier ray's prefix holds the node (first < j) or the same
// ray visited it just before (the samples of one node are consecutive: every axis key is monotone
// along a ray).  f = the lowest ray whose prefix changed.  Rays below f are final, and so is f
// itself (it depends on rays below f only), so `first` is repaired for rays >= f alone: their old
// contributions are removed (a node whose first is >= f is held by no ray below f) and the new
// prefixes added.  The next round starts at f + 1; a round without a change ends the loop.
// Loads of data other threads wrote in earlier phases bypass L1 (__ldcg).
__global__ void __launch_bounds__(kEarlyThreads) k_early_rounds(DeviceMap M, EarlyArgs e, uint32_t n)
{
	namespace cg = cooperative_groups;
	cg::grid_group grid = cg::this_grid();
	Counters* c = M.ctr;
	if (ld_volatile_u32(&c->overflow) & 256u) return;  // uniform: every block returns
	const uint32_t tid = blockIdx.x * blockDim.x + threadIdx.x, nth = gridDim.x * blockDim.x;
	uint32_t F = 0, round = 0;
	while (true) {
		uint32_t* low = &c->e_low[round & 1];
		for (uint32_t j = F + tid; j < n; j += nth) {
			const unsigned long long b = e.off[j];
			const uint32_t L = (uint32_t)(e.off[j + 1] - b);
			uint32_t P = L, run = 0, prev = kNone;
			for (uint32_t k = 0; k < L; ++k) {
				const uint32_t v = __ldg(&e.ids[b + k]);
				const bool present = v == prev || __ldcg(&e.first[v]) < j;
				prev = v;
				if (!present) {
					run = 0;
				} else if (++run >= e.stop) {
					P = k + 1;
					break;
				}
			}
			__stcg(&e.pnext[j], P);
			if (P != __ldcg(&e.plen[j])) atomicMin(low, j);
		}
		// the other slot was last read in round - 1, before this round's first barrier
		if (tid == 0) c->e_low[(round + 1) & 1] = kNone;
		grid.sync();
		const uint32_t f = ld_volatile_u32(low);
		++round;
		if (f == kNone) break;
		for (uint32_t j = f + tid; j < n; j += nth) {
			const unsigned long long b = e.off[j];
			const uint32_t P = __ldcg(&e.plen[j]);
			for (uint32_t k = 0; k < P; ++k) {
				const uint32_t v = __ldg(&e.ids[b + k]);
				if (__ldcg(&e.first[v]) >= f) __stcg(&e.first[v], kNone);
			}
		}
		grid.sync();
		for (uint32_t j = f + tid; j < n; j += nth) {
			const unsigned long long b = e.off[j];
			const uint32_t P = __ldcg(&e.pnext[j]);
			for (uint32_t k = 0; k < P; ++k) atomicMin(&e.first[__ldg(&e.ids[b + k])], j);
			__stcg(&e.plen[j], P);
		}
		grid.sync();
		F = f + 1;
	}
	if (tid == 0) {
		c->e_rounds = round;
		c->e_converged = 1;
	}
}

// E3.  One thread per table slot: a node with first < kNone is in the free set and is marked as the
// record path marks it (k_scatter / k_rays_simple): a block mask at depth 0-2, whole blocks at 3-4,
// the scan's node set + k_expand_nodes at 5-6.  Every slot is emptied for the next scan.
template <int DEPTH>
__global__ void __launch_bounds__(kEarlyThreads) k_early_mark(DeviceMap M, ScanArgs a, EarlyArgs e)
{
	const bool skip = ld_volatile_u32(&M.ctr->overflow) & 256u;
	const size_t slots = (size_t)e.tab_mask + 1;
	uint32_t marked = 0;
	for (size_t s = (size_t)blockIdx.x * blockDim.x + threadIdx.x; s < slots; s += (size_t)gridDim.x * blockDim.x) {
		const unsigned long long node = e.keys[s];
		if (node == kEmptyKey) continue;
		const uint32_t f = e.first[s];
		e.keys[s] = kEmptyKey;
		e.first[s] = kNone;
		if (f == kNone || skip || (node & kRankTag)) continue;
		++marked;
		uint32_t x, y, z;
		unpack_key(node, x, y, z);
		x <<= a.depth;
		y <<= a.depth;
		z <<= a.depth;
		if (DEPTH <= 2) {
			BrickCache bc = {0, 0, 0, kNone};
			flush_block(M, bc, x, y, z, voxel_bits<DEPTH>(Key3{x, y, z}));
		} else if (DEPTH <= 4) {
			mark_node_miss(M, x, y, z, a.depth);
		} else {
			collect_node(M, a, x, y, z, a.depth);
		}
	}
	if (marked) atomicAdd(&M.ctr->e_free, (unsigned long long)marked);
}
}  // namespace ufo_b200
