// ufo_walk.cuh -- K2 of the common case: the fused free-space walk.
//
//   k_split      per ray: cuts the exact voxel walk into segments at fixed distances from the
//                sensor ("shells") WITHOUT changing a single visited voxel, and stores each
//                segment's start state
//   k_walk_mark  one thread per segment, warp in lock-step: the exact FP64 voxel walk of
//                freeSpaceNormal (occupancy_map_base.h:1261-1301, octree.h:1192-1233); the visited
//                voxels of a 4^3 block are OR-ed into a register and, when the lane leaves the
//                block, merged into the block's per-scan miss mask with one fire-and-forget
//                64-bit reduction (set semantics of CodeMap::try_emplace, code.h:675-694)
//
// Why segments.  (1) Load balance: rays differ 10x in length, and one thread per ray leaves the
// machine a quarter full while the long rays finish.  Segments of at most `S` dominant-axis steps
// are handed to persistent warps through an atomic cursor.  (2) Locality of the mark atomics:
// 64-bit reductions are several times faster while the touched masks fit in the L2 than at the
// ~125 MB a whole 30 m scan touches, which is more than the H100's 50 MB L2 (tools/atomic_ceiling.cu
// measures both).  Segments are grouped by their distance from the sensor and the shells are
// processed one after the other by the whole GPU, so at any time the live masks are one shell's
// (10-30 MB).
//
// Why this is exact.  The reference accumulates t_max by REPEATED ADDITION and picks the axis with
// the smallest t_max (ties x, then y, then z), so no closed form may be used -- but the values
// t_max[A] takes depend on axis A alone:  T_A(1) = t_max0[A], T_A(i+1) = T_A(i) + t_delta[A], and the
// walk is the merge of the three sequences ordered by (value, axis).  The state just before the
// (a+1)-th step along axis A is therefore
//     count_A = a, t_max[A] = T_A(a+1);   count_B = #{ j : (T_B(j), B) < (T_A(a+1), A) }, t_max[B] = T_B(count_B+1)
// -- three independent chains of additions and compares.  A segment is the ordinary walk from such
// a state with the next state's voxel as its end key; it exists iff the state still satisfies the
// loop condition (min t_max never decreases).  Proven voxel-for-voxel on the CPU
// (experiments/ray_split_poc.py, tests/test_ray_split_poc.py) and by every GPU parity test.
#pragma once

#include "ufo_kernels.cuh"

namespace ufo_b200
{
// dominant-axis steps per shell: the longest ray of the scan spans at most kShells shells
__device__ __forceinline__ uint32_t shell_steps(uint32_t max_span)
{
	const uint32_t s = (max_span + kShells - 1) / kShells;
	return s < 64u ? 64u : s;
}

// Dense mode: OR `bits` into the block of voxel key (x, y, z) (21 bits per axis) in the scan
// volume -- a computed address, no lookup -- and flag the brick in the dirty bitmap.
__device__ __forceinline__ void mark_dense(const DeviceMap& M, uint32_t x, uint32_t y, uint32_t z, unsigned long long bits)
{
	if ((x | y | z) & ~M.g.key_mask) {
		atomicOr(&M.ctr->overflow, 32u);  // out-of-tree key: repeated through the generic record path
		return;
	}
	const uint32_t vb = vol_brick(M, x >> 4, y >> 4, z >> 4);
	if (vb == kNone) {
		atomicOr(&M.ctr->overflow, 64u);
		return;
	}
	atomicOr(&M.vol[(size_t)vb * 64 + morton2(x >> 2, y >> 2, z >> 2)], bits);
	vol_touch(M, vb);
}

// Dense mode, after the walk: the dirty bitmap becomes the scan's touched list in two steps.
// k_gather_scan: all threads read the bitmap (coalesced) and append the non-empty words to a list;
// k_gather: one warp per non-empty word, lane l takes bits l and l + 32: find-or-create the brick
// through the brick hash and append (brick slot, volume brick holding its masks).  SHARD: bricks of
// another GPU are dropped (their masks zeroed) instead.
__global__ void __launch_bounds__(256) k_gather_scan(DeviceMap M)
{
	if (ld_volatile_u32(&M.ctr->overflow) & ~4u) return;
	constexpr uint32_t FULL = 0xffffffffu;
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t db = M.vol_db;
	const uint32_t n_words = (db * db * db + 63u) / 64u;
	const uint32_t n_round = (n_words + 31u) & ~31u;
	for (uint32_t wi = blockIdx.x * blockDim.x + threadIdx.x; wi < n_round; wi += gridDim.x * blockDim.x) {
		const bool any = wi < n_words && M.vol_dirty[wi] != 0ull;
		const uint32_t bal = __ballot_sync(FULL, any);
		if (!bal) continue;
		uint32_t base = 0;
		if (lane == 0) base = atomicAdd(&M.ctr->n_dirty, (uint32_t)__popc(bal));
		base = __shfl_sync(FULL, base, 0);
		if (any) M.vol_list[base + __popc(bal & ((1u << lane) - 1u))] = wi;
	}
}

template <bool SHARD>
__global__ void __launch_bounds__(256) k_gather(DeviceMap M)
{
	if (ld_volatile_u32(&M.ctr->overflow) & ~4u) return;
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t db = M.vol_db;
	const uint32_t n = ld_volatile_u32(&M.ctr->n_dirty);
	const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, n_warps = (gridDim.x * blockDim.x) >> 5;
	for (uint32_t e = warp; e < n; e += n_warps) {
		const uint32_t wi = M.vol_list[e];
		const unsigned long long w = M.vol_dirty[wi];
		__syncwarp();
		if (lane == 0) M.vol_dirty[wi] = 0ull;
#pragma unroll
		for (uint32_t h = 0; h < 2; ++h) {
			const uint32_t bit = lane + 32u * h;
			if (!((w >> bit) & 1ull)) continue;
			const uint32_t vb = wi * 64u + bit;
			const uint32_t rx = vb % db, ry = (vb / db) % db, rz = vb / (db * db);
			const unsigned long long key = pack_key(M.vol_g0x + rx, M.vol_g0y + ry, M.vol_g0z + rz);
			if (SHARD && brick_owner(key, M.shard_world) != M.shard_rank) {
				unsigned long long* v = M.vol + (size_t)vb * 64;
				for (int c = 0; c < 64; ++c) v[c] = 0ull;
				continue;
			}
			const uint32_t slot = brick_find_or_create(M, key);
			if (slot == kNone) continue;  // pool exhausted: flagged, the scan is repeated
			const uint32_t mi = vb | (M.hit_stamp[slot] == M.scan_id ? 0u : kMiNoHits);
			if (M.pair_id && M.brick_stamp[slot] == M.pair_id) {
				// second scan of a pair, brick already listed by the first: one entry, both mask slabs
				M.touched_mi2[M.touch_idx[slot]] = mi;
				continue;
			}
			M.brick_stamp[slot] = M.scan_id;
			// one list-cursor atomic per group of lanes, not per brick (same-address atomics serialise)
			const uint32_t peers = __activemask();
			const uint32_t leader = __ffs(peers) - 1;
			uint32_t base = 0;
			if (lane == leader) base = atomicAdd(&M.ctr->n_touched, (uint32_t)__popc(peers));
			base = __shfl_sync(peers, base, leader);
			const uint32_t i = base + __popc(peers & ((1u << lane) - 1u));
			M.touched[i] = slot;
			M.touched_mi[i] = M.pair_id ? kMiAbsent : mi;
			M.touched_mi2[i] = M.pair_id ? mi : kMiAbsent;
			M.touch_idx[slot] = i;
		}
	}
}

// component i (0, 1, 2) of (x, y, z)
template <class T>
__device__ __forceinline__ T pick3(T x, T y, T z, int i)
{
	return i == 0 ? x : (i == 1 ? y : z);
}

template <int DEPTH, bool COUNT>
__global__ void __launch_bounds__(128) k_split(DeviceMap M, ScanArgs a)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t n_batches = (a.n + 31) / 32;
	constexpr uint32_t FULL = 0xffffffffu;
	Walk w;
	w.tx = w.ty = w.tz = 0.0;
	w.dx = w.dy = w.dz = 0.0;
	w.sx = w.sy = w.sz = 0;
	w.cur = {0, 0, 0};
	w.end = {0, 0, 0};
	double dist = 0.0;
	bool live = false;
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
			walk_init(M.g, to, from, dir, a.depth, w);
			if (w.same) {
				// both ends in one voxel: that voxel alone (occupancy_map_base.h:1281-1284)
				if (M.dense) {
					mark_dense(M, w.cur.x & 0x1fffffu, w.cur.y & 0x1fffffu, w.cur.z & 0x1fffffu, voxel_bits<DEPTH>(w.cur));
				} else {
					BrickCache bc = {0, 0, 0, kNone};
					flush_block(M, bc, w.cur.x, w.cur.y, w.cur.z, voxel_bits<DEPTH>(w.cur));
				}
				if (COUNT) atomicAdd(&M.ctr->visits, 1ull);
			} else {
				live = true;
			}
		}
	}
	// dominant axis and number of segments
	const uint32_t S = shell_steps(ld_volatile_u32(&M.ctr->max_span));
	uint32_t nA = 0, J = 0;
	int A = 0;
	if (live) {
		const uint32_t nx = (uint32_t)abs((int)(w.end.x - w.cur.x)) >> a.depth;
		const uint32_t ny = (uint32_t)abs((int)(w.end.y - w.cur.y)) >> a.depth;
		const uint32_t nz = (uint32_t)abs((int)(w.end.z - w.cur.z)) >> a.depth;
		nA = nx;
		if (ny > nA) {
			nA = ny;
			A = 1;
		}
		if (nz > nA) {
			nA = nz;
			A = 2;
		}
		J = (nA + S - 1) / S;
		if (J > kShells) J = kShells;  // cannot happen (S covers max_span); keeps the arrays safe
		a.rc[i] = RayConst{w.dx, w.dy, w.dz, dist};
	}
	// which lanes of this batch own a segment in shell j (all lanes take part in the ballots)
	for (uint32_t j = 0; j < kShells; ++j) {
		const uint32_t vm = __ballot_sync(FULL, j < J);
		if (lane == 0 && (i >> 5) < n_batches) a.vmask[(size_t)j * n_batches + (i >> 5)] = vm;
	}
	if (!live) return;

	const uint32_t sgn = (w.sx > 0 ? 1u : (w.sx < 0 ? 2u : 0u)) | ((w.sy > 0 ? 1u : (w.sy < 0 ? 2u : 0u)) << 2) |
	                     ((w.sz > 0 ? 1u : (w.sz < 0 ? 2u : 0u)) << 4);
	Item* const out = a.items + i;
	const size_t stride = a.item_stride;
	// segment m = 0 is the outermost one (it starts at the ray's end point) and lies in shell J-1
	// per-axis values are picked with selects: an array indexed by A, B, C would live in local memory
	const int B = (A == 0) ? 1 : 0, C = (A == 2) ? 1 : 2;  // the other two axes, B < C
	const double dA = pick3(w.dx, w.dy, w.dz, A), dB = pick3(w.dx, w.dy, w.dz, B), dC = pick3(w.dx, w.dy, w.dz, C);
	const int sA = pick3(w.sx, w.sy, w.sz, A), sB = pick3(w.sx, w.sy, w.sz, B), sC = pick3(w.sx, w.sy, w.sz, C);
	double TA = pick3(w.tx, w.ty, w.tz, A), tB = pick3(w.tx, w.ty, w.tz, B), tC = pick3(w.tx, w.ty, w.tz, C);
	uint32_t a_done = 0, cntB = 0, cntC = 0;
	Key3 seg_cur = w.cur;
	Vec3 seg_t = {w.tx, w.ty, w.tz};
	uint32_t m = 0;
	uint32_t a_k = nA - (J - 1) * S;  // dominant-axis steps before the first cut, in 1..S
	for (; m + 1 < J; ++m, a_k += S) {
		// T_A(a_k + 1).  The j-th step along A only happens while T_A(j) <= dist (loop condition of
		// the walk), so the chain stops there: no later segment exists, and degenerate rays (NaN /
		// infinite geometry, keys that wrapped) cannot spin here.
		bool dead = false;
		for (; a_done < a_k; ++a_done) {
			if (!(TA <= dist)) {
				dead = true;
				break;
			}
			TA = dop::add(TA, dA);
		}
		if (dead) break;
		if (sB != 0)
			while (tB < TA || (tB == TA && B < A)) {
				tB = dop::add(tB, dB);
				++cntB;
			}
		if (sC != 0)
			while (tC < TA || (tC == TA && C < A)) {
				tC = dop::add(tC, dC);
				++cntC;
			}
		// axis i moved by a_k (A), cntB (B) or cntC (C) steps; {A, B, C} = {0, 1, 2}
		const uint32_t mA = a_k * (uint32_t)sA, mB = cntB * (uint32_t)sB, mC = cntC * (uint32_t)sC;
		const Key3 cut = {w.cur.x + (A == 0 ? mA : (B == 0 ? mB : mC)), w.cur.y + (A == 1 ? mA : (B == 1 ? mB : mC)),
		                  w.cur.z + (A == 2 ? mA : (B == 2 ? mB : mC))};
		const Vec3 tcut = {A == 0 ? TA : (B == 0 ? tB : tC), A == 1 ? TA : (B == 1 ? tB : tC),
		                   A == 2 ? TA : (B == 2 ? tB : tC)};
		// the next segment exists iff the walk gets here: loop condition of freeSpaceNormal
		const bool exists = cut != w.end && (tcut.x <= dist || tcut.y <= dist || tcut.z <= dist);
		if (!exists) break;
		out[(size_t)(J - 1 - m) * stride] =
		    Item{seg_t.x, seg_t.y, seg_t.z, seg_cur.x, seg_cur.y, seg_cur.z, cut.x, cut.y, cut.z, sgn, 0u};
		seg_cur = cut;
		seg_t = tcut;
	}
	// the last existing segment runs to the walk's own end
	out[(size_t)(J - 1 - m) * stride] =
	    Item{seg_t.x, seg_t.y, seg_t.z, seg_cur.x, seg_cur.y, seg_cur.z, w.end.x, w.end.y, w.end.z, sgn, 0u};
	for (++m; m < J; ++m) out[(size_t)(J - 1 - m) * stride].sgn = 0xffffffffu;  // announced by vmask, but empty
}

// One lock-step iteration of the walk for the whole warp (see walk_iteration in ufo_kernels.cuh;
// same arithmetic, same predicates).  Instead of appending a record, a lane that leaves its 4^3
// block or finishes reports push = 1 with the voxel key of the block it left (21 bits per axis)
// and the mask accumulated there.
__device__ __forceinline__ bool walk_iteration_fused(double& tx, double& ty, double& tz, const double dx,
                                                     const double dy, const double dz, const double dist,
                                                     uint32_t& kx, uint32_t& ky, uint32_t& kz, const int sx,
                                                     const int sy, const int sz, const uint32_t ex,
                                                     const uint32_t ey, const uint32_t ez,
                                                     unsigned long long& acc, const unsigned long long bits,
                                                     uint32_t& active, uint32_t& push, uint32_t& ox, uint32_t& oy,
                                                     uint32_t& oz, unsigned long long& pacc)
{
	uint32_t any;
	asm volatile(
	    "{\n\t"
	    ".reg .pred pa, px, py, pz, pt, pm, pn, pl, pp;\n\t"
	    ".reg .u32 vx, vy, vz;\n\t"
	    "setp.ne.u32 pa, %8, 0;\n\t"
	    "@pa or.b64 %7, %7, %24;\n\t"
	    "mov.u32 %10, %3;\n\t"
	    "mov.u32 %11, %4;\n\t"
	    "mov.u32 %12, %5;\n\t"
	    // axis selection (octree.h:1227-1233, vector3.h:244-251)
	    "setp.le.f64 px, %0, %1;\n\t"
	    "setp.le.and.f64 px, %0, %2, px;\n\t"
	    "setp.gt.f64 py, %0, %1;\n\t"
	    "setp.le.and.f64 py, %1, %2, py;\n\t"
	    "or.pred pt, px, py;\n\t"
	    "not.pred pz, pt;\n\t"
	    "and.pred px, px, pa;\n\t"
	    "and.pred py, py, pa;\n\t"
	    "and.pred pz, pz, pa;\n\t"
	    "@px add.rn.f64 %0, %0, %14;\n\t"
	    "@py add.rn.f64 %1, %1, %15;\n\t"
	    "@pz add.rn.f64 %2, %2, %16;\n\t"
	    "@px add.u32 %3, %3, %18;\n\t"
	    "@py add.u32 %4, %4, %19;\n\t"
	    "@pz add.u32 %5, %5, %20;\n\t"
	    // more = (cur != end) && (tx <= dist || ty <= dist || tz <= dist)   (occupancy_map_base.h:1300)
	    "setp.le.f64 pm, %0, %17;\n\t"
	    "setp.le.or.f64 pm, %1, %17, pm;\n\t"
	    "setp.le.or.f64 pm, %2, %17, pm;\n\t"
	    "setp.ne.u32 pn, %3, %21;\n\t"
	    "setp.ne.or.u32 pn, %4, %22, pn;\n\t"
	    "setp.ne.or.u32 pn, %5, %23, pn;\n\t"
	    "and.pred pm, pm, pn;\n\t"
	    // left = ((cur ^ old) >> 2) != 0 on any axis
	    "xor.b32 vx, %10, %3;\n\t"
	    "xor.b32 vy, %11, %4;\n\t"
	    "xor.b32 vz, %12, %5;\n\t"
	    "or.b32 vx, vx, vy;\n\t"
	    "or.b32 vx, vx, vz;\n\t"
	    "setp.gt.u32 pl, vx, 3;\n\t"
	    // push = active && (!more || left);  active' = active && more
	    "not.pred pt, pm;\n\t"
	    "or.pred pp, pt, pl;\n\t"
	    "and.pred pp, pp, pa;\n\t"
	    "and.pred pa, pa, pm;\n\t"
	    "selp.u32 %8, 1, 0, pa;\n\t"
	    "selp.u32 %9, 1, 0, pp;\n\t"
	    "and.b32 %10, %10, 0x1fffff;\n\t"
	    "and.b32 %11, %11, 0x1fffff;\n\t"
	    "and.b32 %12, %12, 0x1fffff;\n\t"
	    "mov.u64 %13, %7;\n\t"
	    "@pp mov.u64 %7, 0;\n\t"
	    "vote.sync.any.pred pt, pa, 0xffffffff;\n\t"
	    "selp.u32 %6, 1, 0, pt;\n\t"
	    "}"
	    : "+d"(tx), "+d"(ty), "+d"(tz), "+r"(kx), "+r"(ky), "+r"(kz), "=r"(any), "+l"(acc), "+r"(active),
	      "=r"(push), "=r"(ox), "=r"(oy), "=r"(oz), "=l"(pacc)
	    : "d"(dx), "d"(dy), "d"(dz), "d"(dist), "r"(sx), "r"(sy), "r"(sz), "r"(ex), "r"(ey), "r"(ez), "l"(bits)
	    : "memory");
	return any != 0;
}

// Dense mode.  Same lock-step iteration, but a lane that leaves its 4^3 block (or finishes) appends
// {mask, packed voxel key of the block it left} to the WARP's ring in shared memory, ballot-compacted
// and fully predicated -- no branch, no address arithmetic at 7 active lanes out of 32.  The ring is
// drained 32 records at a time by the whole warp (drain_marks): address computation and the
// reductions run with every lane busy.
constexpr uint32_t kRing = 64;  // records per warp (a power of two, >= 63)
__device__ __forceinline__ bool walk_iteration_ring(double& tx, double& ty, double& tz, const double dx,
                                                    const double dy, const double dz, const double dist,
                                                    uint32_t& kx, uint32_t& ky, uint32_t& kz, const int sx,
                                                    const int sy, const int sz, const uint32_t ex,
                                                    const uint32_t ey, const uint32_t ez,
                                                    unsigned long long& acc, const unsigned long long bits,
                                                    uint32_t& active, uint32_t& tail, const uint32_t ring_base,
                                                    const uint32_t lt_mask)
{
	uint32_t any;
	asm volatile(
	    "{\n\t"
	    ".reg .pred pa, px, py, pz, pt, pm, pn, pl, pp;\n\t"
	    ".reg .u32 ox, oy, oz, vx, vy, vz, bal, rank, idx, cnt, klo, khi, t, saddr;\n\t"
	    ".reg .u64 key;\n\t"
	    "setp.ne.u32 pa, %8, 0;\n\t"
	    "@pa or.b64 %7, %7, %22;\n\t"
	    "mov.u32 ox, %3;\n\t"
	    "mov.u32 oy, %4;\n\t"
	    "mov.u32 oz, %5;\n\t"
	    // axis selection (octree.h:1227-1233, vector3.h:244-251)
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
	    // more = (cur != end) && (tx <= dist || ty <= dist || tz <= dist)   (occupancy_map_base.h:1300)
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
	    // ballot-compacted append of {acc, voxel key of the block just left} to the warp's ring
	    "vote.sync.ballot.b32 bal, pp, 0xffffffff;\n\t"
	    "and.b32 rank, bal, %21;\n\t"
	    "popc.b32 rank, rank;\n\t"
	    "add.u32 idx, %9, rank;\n\t"
	    "and.b32 idx, idx, 63;\n\t"
	    "and.b32 ox, ox, 0x1fffff;\n\t"
	    "and.b32 oy, oy, 0x1fffff;\n\t"
	    "and.b32 oz, oz, 0x1fffff;\n\t"
	    "mad.lo.u32 klo, oy, 0x200000, ox;\n\t"
	    "shr.u32 t, oy, 11;\n\t"
	    "mad.lo.u32 khi, oz, 1024, t;\n\t"
	    "mov.b64 key, {klo, khi};\n\t"
	    "mad.lo.u32 saddr, idx, 16, %20;\n\t"
	    "@pp st.shared.v2.u64 [saddr], {%7, key};\n\t"
	    "@pp mov.u64 %7, 0;\n\t"
	    "popc.b32 cnt, bal;\n\t"
	    "add.u32 %9, %9, cnt;\n\t"
	    "vote.sync.any.pred pt, pa, 0xffffffff;\n\t"
	    "selp.u32 %6, 1, 0, pt;\n\t"
	    "}"
	    : "+d"(tx), "+d"(ty), "+d"(tz), "+r"(kx), "+r"(ky), "+r"(kz), "=r"(any), "+l"(acc), "+r"(active),
	      "+r"(tail)
	    : "d"(dx), "d"(dy), "d"(dz), "d"(dist), "r"(sx), "r"(sy), "r"(sz), "r"(ex), "r"(ey), "r"(ez),
	      "r"(ring_base), "r"(lt_mask), "l"(bits)
	    : "memory");
	return any != 0;
}

// What the dense walk sent, per lane (profiling level 2 only; see Counters::walk_*).
struct WalkCounts {
	uint32_t records, mask_reds, words, dirty_reds;
};

// Drains up to 32 records of the warp's ring, starting at `head`: lane l takes record head + l.
// Records that mark the same word of the scan volume (rays of a batch crossing the same 4^3 block;
// near the sensor, all of them) are merged first: the group's non-leaders OR their mask into the
// leader's ring slot, and the leader issues the one global reduction.  OR is idempotent and
// commutative, so no merge order can change a mask.  The brick's dirty bit is set by one lane per
// distinct brick, and not at all when a lane of the group already set it earlier in this kernel
// (`last_vb`: the brick of the lane's last drained record; the bitmap is only cleared by k_gather,
// after the walk).
template <bool COUNT>
__device__ __forceinline__ void drain_marks(const DeviceMap& M, ulonglong2* ring, uint32_t head, uint32_t n,
                                            uint32_t lane, uint32_t& last_vb, WalkCounts& wc)
{
	constexpr uint32_t FULL = 0xffffffffu;
	uint32_t vb = kNone, word = kNone;  // word = vb * 64 + block < 325^3 * 64 < 2^32 (volume_bricks)
	unsigned long long mask = 0;
	if (lane < n) {
		const ulonglong2 e = ring[(head + lane) & (kRing - 1)];
		uint32_t x, y, z;
		unpack_key(e.y, x, y, z);
		vb = vol_brick(M, x >> 4, y >> 4, z >> 4);
		if (((x | y | z) & ~M.g.key_mask) || vb == kNone) {
			// a key outside the tree (no alias path here) or outside the volume: the host repeats the
			// scan through the generic record path / without the volume
			atomicOr(&M.ctr->overflow, ((x | y | z) & ~M.g.key_mask) ? 32u : 64u);
			vb = kNone;
		} else {
			word = vb * 64u + morton2(x >> 2, y >> 2, z >> 2);
			mask = e.x;
		}
		if (COUNT) ++wc.records;
	}
	const uint32_t grp = __match_any_sync(FULL, word);
	const uint32_t leader = __ffs(grp) - 1;
	const bool alone = grp == (1u << lane);
	if (word != kNone && lane != leader) {
		// two 32-bit ORs: native shared-memory atomics (a 64-bit one is a compare-and-swap loop)
		uint32_t* const lm = reinterpret_cast<uint32_t*>(&ring[(head + leader) & (kRing - 1)].x);
		atomicOr(lm, (uint32_t)mask);
		atomicOr(lm + 1, (uint32_t)(mask >> 32));
	}
	__syncwarp();
	if (word != kNone && lane == leader) {
		if (!alone) mask = ring[(head + lane) & (kRing - 1)].x;
#ifdef UFO_WALK_NO_RED
		// timing-only build: every address is computed but no reduction is issued (a pushed mask is
		// never 0); the map comes out wrong
		if (mask == 0ull)
#endif
		if (COUNT) {
			wc.words += atomicOr(&M.vol[word], mask) == 0ull;
			++wc.mask_reds;
		} else {
			atomicOr(&M.vol[word], mask);
		}
	}
	const uint32_t bgrp = __match_any_sync(FULL, vb);
	const bool seen = (__ballot_sync(FULL, last_vb == vb) & bgrp) != 0u;
	if (vb != kNone) {
		if (!seen && lane == (uint32_t)(__ffs(bgrp) - 1)) {
#ifdef UFO_WALK_NO_RED
			if (vb == 0xfffffffeu)
#endif
			vol_touch(M, vb);
			if (COUNT) ++wc.dirty_reds;
		}
		last_vb = vb;
	}
}

// brick slot of `bkey` for marking: one probe of the two-entry bucket (L1-cached: neighbouring
// rays resolve the same few bricks at the same time), find-or-create on a miss; stamps the brick
// into the scan's touched list on its first mark.  SHARD: bricks of another GPU give kNone.
template <bool SHARD>
__device__ __forceinline__ uint32_t resolve_brick(const DeviceMap& M, unsigned long long bkey)
{
	if (SHARD && brick_owner(bkey, M.shard_world) != M.shard_rank) return kNone;
	const uint32_t hidx = hash_u64(bkey) & M.bh_mask & ~1u;
	ulonglong2 ent = ld_cached_entry(&M.bh_tab[hidx]);
	uint32_t hpos = hidx;
	bool hit = ent.x == bkey;
	if (!hit) {
		ent = ld_cached_entry(&M.bh_tab[hidx + 1]);
		hit = ent.x == bkey;
		hpos = hidx + 1;
	}
	uint32_t brick = (uint32_t)ent.y;
	if (hit && brick != kPending && brick != kFailed) {
		if ((uint32_t)(ent.y >> 32) != M.scan_id) {
			touch_brick(M, brick);
			reinterpret_cast<uint32_t*>(&M.bh_tab[hpos].y)[1] = M.scan_id;  // cached stamp: later probes skip the touch
		}
		return brick;
	}
	brick = brick_find_or_create_from(M, bkey, hidx);
	if (brick != kNone) touch_brick(M, brick);
	return brick;
}

#ifndef UFO_WALK_MINBLOCKS
#define UFO_WALK_MINBLOCKS 7
#endif
constexpr int kWalkThreads = 128;
#ifndef UFO_UNITS_PER_GRAB
#define UFO_UNITS_PER_GRAB 1
#endif
constexpr uint32_t kUnitsPerGrab = UFO_UNITS_PER_GRAB;

// Work unit = (shell, batch of 32 consecutive rays); units are numbered shell by shell and handed
// out through an atomic cursor, kUnitsPerGrab at a time.
// DENSE: marks go to the scan volume (computed address + dirty bit, nothing is loaded in the
// loop); otherwise to the bricks' miss masks through the brick hash, one probe per brick change.
template <int DEPTH, bool SHARD, bool COUNT, bool DENSE>
__global__ void __launch_bounds__(kWalkThreads, UFO_WALK_MINBLOCKS) k_walk_mark(DeviceMap M, ScanArgs a)
{
	const uint32_t lane = threadIdx.x & 31;
	constexpr uint32_t FULL = 0xffffffffu;
	const uint32_t n_batches = (a.n + 31) / 32;
	const uint32_t units = kShells * n_batches;
	if (ld_volatile_u32(&M.ctr->overflow) & ~4u) return;  // the scan will be repeated after a pool growth
	unsigned int visits = 0;
	unsigned long long ckey = ~0ull;  // brick of the lane's last mark and its slot
	uint32_t cslot = kNone;
#ifndef UFO_WALK_BRANCH
	__shared__ ulonglong2 s_ring[DENSE ? kWalkThreads / 32 : 1][DENSE ? kRing : 1];
	ulonglong2* ring = s_ring[DENSE ? (threadIdx.x >> 5) : 0];
	const uint32_t ring_base = (uint32_t)__cvta_generic_to_shared(ring);
	const uint32_t lt_mask = (1u << lane) - 1u;
	uint32_t q_head = 0, q_tail = 0;  // warp-uniform running counters
	uint32_t last_vb = kNone;         // drain_marks: brick whose dirty bit this lane's group last set
	WalkCounts wc = {0, 0, 0, 0};
#endif
	while (true) {
		uint32_t u0 = 0;
		if (lane == 0) u0 = atomicAdd(&M.ctr->item_cursor, kUnitsPerGrab);
		u0 = __shfl_sync(FULL, u0, 0);
		if (u0 >= units) break;
		const uint32_t u1 = min(u0 + kUnitsPerGrab, units);
		for (uint32_t u = u0; u < u1; ++u) {
			const uint32_t rs = u / n_batches, batch = u - rs * n_batches;
#ifdef UFO_SHELL_OUTER_FIRST
			const uint32_t shell = kShells - 1 - rs;
#else
			// innermost shell first: the sparse outer shells (few, partial segments) come last, which
			// keeps the end-of-kernel tail short
			const uint32_t shell = rs;
#endif
			const uint32_t vm = __ldg(&a.vmask[(size_t)shell * n_batches + batch]);
			if (!vm) continue;
			const uint32_t i = batch * 32 + lane;
			uint32_t active = (vm >> lane) & 1u;
			double tx = 0.0, ty = 0.0, tz = 0.0, dx = 0.0, dy = 0.0, dz = 0.0, dist = 0.0;
			uint32_t kx = 0, ky = 0, kz = 0, ex = 0, ey = 0, ez = 0;
			int sx = 0, sy = 0, sz = 0;
			if (active) {
				const Item* ip = a.items + (size_t)shell * a.item_stride + i;
				const uint4 q0 = reinterpret_cast<const uint4*>(ip)[0];
				const uint4 q1 = reinterpret_cast<const uint4*>(ip)[1];
				const uint4 q2 = reinterpret_cast<const uint4*>(ip)[2];
				const uint2 q3 = reinterpret_cast<const uint2*>(ip)[6];
				const uint32_t sgn = q3.x;
				if (sgn == 0xffffffffu) {
					active = 0;
				} else {
					tx = __hiloint2double((int)q0.y, (int)q0.x);
					ty = __hiloint2double((int)q0.w, (int)q0.z);
					tz = __hiloint2double((int)q1.y, (int)q1.x);
					kx = q1.z;
					ky = q1.w;
					kz = q2.x;
					ex = q2.y;
					ey = q2.z;
					ez = q2.w;
					const int step = 1 << a.depth;
					sx = (sgn & 1u) ? step : ((sgn & 2u) ? -step : 0);
					sy = (sgn & 4u) ? step : ((sgn & 8u) ? -step : 0);
					sz = (sgn & 16u) ? step : ((sgn & 32u) ? -step : 0);
					const double4 rc = *reinterpret_cast<const double4*>(a.rc + i);
					dx = rc.x;
					dy = rc.y;
					dz = rc.z;
					dist = rc.w;
				}
			}
			unsigned long long acc = 0;
			bool any = __any_sync(FULL, active != 0u);
			while (any) {
				if (COUNT) visits += active;
				uint32_t push, ox, oy, oz;
				unsigned long long pacc;
#ifndef UFO_WALK_BRANCH
				if (DENSE) {
					any = walk_iteration_ring(tx, ty, tz, dx, dy, dz, dist, kx, ky, kz, sx, sy, sz, ex, ey, ez, acc,
					                          voxel_bits<DEPTH>(Key3{kx, ky, kz}), active, q_tail, ring_base, lt_mask);
					if (q_tail - q_head >= 32u) {
						__syncwarp();
						drain_marks<COUNT>(M, ring, q_head, 32u, lane, last_vb, wc);
						__syncwarp();
						q_head += 32u;
					}
					continue;
				}
#endif
				any = walk_iteration_fused(tx, ty, tz, dx, dy, dz, dist, kx, ky, kz, sx, sy, sz, ex, ey, ez, acc,
				                           voxel_bits<DEPTH>(Key3{kx, ky, kz}), active, push, ox, oy, oz, pacc);
				if (DENSE) {
					if (push) {
						const uint32_t vb = vol_brick(M, ox >> 4, oy >> 4, oz >> 4);
						if (((ox | oy | oz) & ~M.g.key_mask) || vb == kNone) {
							// a key outside the tree (no alias path here) or outside the volume: the host
							// repeats the scan through the generic record path / without the volume
							atomicOr(&M.ctr->overflow, ((ox | oy | oz) & ~M.g.key_mask) ? 32u : 64u);
						} else {
							atomicOr(&M.vol[(size_t)vb * 64 + morton2(ox >> 2, oy >> 2, oz >> 2)], pacc);
							if (vb != cslot) {
								cslot = vb;
								vol_touch(M, vb);
							}
						}
					}
				} else if (push) {
					if ((ox | oy | oz) & ~M.g.key_mask) {
						// a key outside the tree: this lean kernel has no alias path; the host allocates the
						// alias arrays and repeats the scan through the generic record path
						atomicOr(&M.ctr->overflow, 32u);
					} else {
						const unsigned long long bkey = pack_key(ox >> 4, oy >> 4, oz >> 4);
						if (bkey != ckey) {
							ckey = bkey;
							cslot = resolve_brick<SHARD>(M, bkey);
						}
						if (cslot != kNone) atomicOr(&M.miss_mask[(size_t)cslot * 64 + morton2(ox >> 2, oy >> 2, oz >> 2)], pacc);
					}
				}
			}
		}
	}
#ifndef UFO_WALK_BRANCH
	if (DENSE && q_tail != q_head) {
		__syncwarp();
		drain_marks<COUNT>(M, ring, q_head, q_tail - q_head, lane, last_vb, wc);
	}
	if (COUNT && DENSE) {
		if (wc.records) atomicAdd(&M.ctr->walk_records, (unsigned long long)wc.records);
		if (wc.mask_reds) atomicAdd(&M.ctr->walk_mask_reds, (unsigned long long)wc.mask_reds);
		if (wc.words) atomicAdd(&M.ctr->walk_words, (unsigned long long)wc.words);
		if (wc.dirty_reds) atomicAdd(&M.ctr->walk_dirty_reds, (unsigned long long)wc.dirty_reds);
	}
#endif
	if (COUNT && visits) atomicAdd(&M.ctr->visits, (unsigned long long)visits);
}

}  // namespace ufo_b200
