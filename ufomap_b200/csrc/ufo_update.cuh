// ufo_update.cuh -- K3: hit-then-miss float log-odds update of the marked voxels
// (updateOccupancy, occupancy_map_base.h:1139-1145) and the depth 1-4 aggregates
// (updateNode, :1179-1224), over the bricks the scan touched.
#pragma once

#include "ufo_device.cuh"

namespace ufo_b200
{
constexpr int kStatSlots = 64;  // per-scan counters are spread over slots to avoid same-address atomics

__device__ __forceinline__ uint32_t rms_rgb(const uint32_t* c, int n)
{
	// getAverageColor (occupancy_map_color.cpp:200-222) over the set colours
	double s[3] = {0, 0, 0};
	int cnt = 0;
	for (int i = 0; i < n; ++i) {
		if (!c[i]) continue;
		for (int k = 0; k < 3; ++k) {
			double v = (double)((c[i] >> (8 * k)) & 0xffu);
			s[k] = dop::add(s[k], dop::mul(v, v));
		}
		++cnt;
	}
	if (!cnt) return 0;
	uint32_t out = 0;
	for (int k = 0; k < 3; ++k)
		out |= ((uint32_t)(int)dop::sqrt(dop::div(s[k], (double)cnt)) & 0xffu) << (8 * k);
	return out;
}

// SET = true: the marked voxels are set to `miss` (already clamped) instead of updated --
// setValueVolume, occupancy_map_base.h:492-518, :1151-1157.
// Change detection (enableChangeDetection, occupancy_map_base.h:779-790): when M.chg_mask is
// allocated, the voxels whose value actually changed (updateOccupancy returned true, :1139-1145)
// are OR-ed into the block's change mask (linear bit order, like the miss / hit masks).
__device__ __forceinline__ unsigned long long octet_unbits8(uint32_t c8, uint32_t o)
{
	const uint32_t base = ((o & 1u) << 1) | ((o & 2u) << 2) | ((o & 4u) << 3);
	const unsigned long long s = (c8 & 3u) | ((c8 & 0xcu) << 2) | ((c8 & 0x30u) << 12) | ((c8 & 0xc0u) << 14);
	return s << base;
}

// CLEAN: a scan update writes the octet's 32 B sector back only when one of its voxels changed (bit
// for bit), so that an unchanged sector leaves no dirty line in the L2; an uninitialised octet
// (`init` false, its leaves read as 0.0 without a load) is always written.  Returns true when the
// store was skipped.  SET always writes, and so do colour maps (K3 leaves their colour path as it was).
// PAIR: a second scan's hits h8b and misses m8b follow, in the order two passes would apply them.
template <bool SET = false, bool CLEAN = false, bool PAIR = false>
__device__ __forceinline__ bool update_octet(const DeviceMap& M, float miss, float* lp, uint32_t m8,
                                             uint32_t h8, float4 a0, float4 a1, float& omax,
                                             uint32_t& oflags, size_t blk = 0, uint32_t oct = 0,
                                             bool init = false, uint32_t m8b = 0, uint32_t h8b = 0)
{
	float v[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
	const float v0[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
	omax = -3.402823466e+38f;
	float omin = 3.402823466e+38f;
	bool unk = false;
	// all hits of a scan are applied before its misses (occupancy_map_base.h:1351-1365);
	// hits are rare (one voxel per ray), so their arithmetic is skipped for octets without one
	if (!SET && h8) {
#pragma unroll
		for (int j = 0; j < 8; ++j) {
			float hv = apply_update(M, v[j], M.hit);
			v[j] = ((h8 >> j) & 1u) ? hv : v[j];
		}
	}
	if (PAIR) {
#pragma unroll
		for (int j = 0; j < 8; ++j) {
			float mv = apply_update(M, v[j], miss);
			v[j] = ((m8 >> j) & 1u) ? mv : v[j];
		}
		if (h8b) {
#pragma unroll
			for (int j = 0; j < 8; ++j) {
				float hv = apply_update(M, v[j], M.hit);
				v[j] = ((h8b >> j) & 1u) ? hv : v[j];
			}
		}
		m8 = m8b;
	}
#pragma unroll
	for (int j = 0; j < 8; ++j) {
		float mv = SET ? miss : apply_update(M, v[j], miss);
		v[j] = ((m8 >> j) & 1u) ? mv : v[j];
		omax = fmaxf(omax, v[j]);
		omin = fminf(omin, v[j]);
		unk = unk || (v[j] >= M.free_ceil && v[j] <= M.occ_floor);
	}
	// contains_free = any voxel below the free threshold, contains_unknown = any in between
	oflags = (omin < M.free_ceil ? 1u : 0u) | (unk ? 2u : 0u);
	if (!SET && (CLEAN || M.chg_mask)) {
		uint32_t c8 = 0;
#pragma unroll
		for (int j = 0; j < 8; ++j) c8 |= (__float_as_uint(v[j]) != __float_as_uint(v0[j]) ? 1u : 0u) << j;
		if (c8 && M.chg_mask) atomicOr(&M.chg_mask[blk], octet_unbits8(c8, oct));
		if (CLEAN && !c8 && init) return true;
	}
	reinterpret_cast<float4*>(lp)[0] = make_float4(v[0], v[1], v[2], v[3]);
	reinterpret_cast<float4*>(lp)[1] = make_float4(v[4], v[5], v[6], v[7]);
	return false;
}

// ---- mbarrier + 1-D bulk copy (TMA engine, cp.async.bulk) -------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(unsigned long long* bar, uint32_t count)
{
	asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long* bar, uint32_t bytes)
{
	asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, uint32_t parity)
{
	asm volatile(
	    "{\n\t"
	    ".reg .pred p;\n\t"
	    "UFO_MBAR_WAIT_%=:\n\t"
	    "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
	    "@p bra UFO_MBAR_DONE_%=;\n\t"
	    "bra UFO_MBAR_WAIT_%=;\n\t"
	    "UFO_MBAR_DONE_%=:\n\t"
	    "}" ::"r"(smem_u32(bar)),
	    "r"(parity)
	    : "memory");
}
// global -> shared, `bytes` a multiple of 16, both addresses 16-byte aligned; completion is
// signalled on `bar` as transaction bytes
__device__ __forceinline__ void bulk_load(void* smem_dst, const void* gmem_src, uint32_t bytes, unsigned long long* bar)
{
	asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(
	                 smem_u32(smem_dst)),
	             "l"(gmem_src), "r"(bytes), "r"(smem_u32(bar))
	             : "memory");
}
// the octets of every leaf line (octets 4h..4h+3) that holds an octet of o8
__device__ __forceinline__ uint32_t line_octets(uint32_t o8) { return ((o8 & 0x0fu) ? 0x0fu : 0u) | ((o8 & 0xf0u) ? 0xf0u : 0u); }
__device__ __forceinline__ void fence_proxy_async()
{
	asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

// A brick whose key lies outside the tree only collects out-of-tree marks (see k_alias_*):
// returns true for such a brick and the wrapped brick coordinates its marks land in.
__device__ __forceinline__ bool alias_source(const DeviceMap& M, uint32_t brick, uint32_t& tx, uint32_t& ty,
                                             uint32_t& tz)
{
	uint32_t x, y, z;
	unpack_key(M.brick_key[brick], x, y, z);
	const uint32_t km = M.g.key_mask >> 4;
	tx = x & km;
	ty = y & km;
	tz = z & km;
	return ((x | y | z) & ~km) != 0;
}

// A paired pass stages the second scan's miss masks in `hm` and reads the hit masks of both scans from
// global memory (most bricks have none): the slab, and so the kernel's shared memory, keeps its size.
struct __align__(128) WarpSlab {
	unsigned long long mm[64];
	unsigned long long hm[64];
	uint32_t meta[64];
	float2 q[64];  // line maxima
};
// list entry of a loaded octet: (block << 3) | octet, plus
constexpr uint32_t kEntInit = 1u << 9;      // the octet is initialised (its leaves are loaded; otherwise 0.0)
constexpr uint32_t kEntTouched = 1u << 10;  // the scan marked a voxel of it (otherwise only its max is needed)
constexpr uint32_t kEntHitA = 1u << 11;     // paired pass: the block has a hit of the first scan
constexpr uint32_t kEntHitB = 1u << 12;     // paired pass: the block has a hit of the second scan

// octets of a block holding a bit of the linear-order voxel mask u
__device__ __forceinline__ uint32_t mask_octets(unsigned long long u)
{
	uint32_t t = 0;
#pragma unroll
	for (uint32_t o = 0; o < 8; ++o) {
		const uint32_t base = ((o & 1u) << 1) | ((o & 2u) << 2) | ((o & 4u) << 3);
		t |= (((u >> base) & 0x330033ull) ? 1u : 0u) << o;
	}
	return t;
}
// depth-3 nodes (groups of eight block lanes) with a lane set in ballot b
__device__ __forceinline__ uint32_t ballot_groups(uint32_t b)
{
	return ((b & 0xffu) ? 1u : 0u) + ((b & 0xff00u) ? 1u : 0u) + ((b & 0xff0000u) ? 1u : 0u) + ((b & 0xff000000u) ? 1u : 0u);
}

// K3: one WARP per brick of the scan's TOUCHED LIST (the cost of a scan does not depend on the size
// of the map), no CTA-wide barrier at all: a warp waiting for its leaf sectors never holds others at
// a __syncthreads (a CTA-cooperative version spent a large share of its stall samples there).
//  * warps claim their bricks from a work cursor (the cost of a brick varies by more than 10x);
//  * lane 0 stages the header slab of the warp's NEXT brick -- miss masks 512 B, hit masks 512 B
//    (only for a brick with a hit this scan: most bricks are crossed by free space only), meta
//    256 B, line maxima 512 B -- with bulk copies (cp.async.bulk) on a per-warp mbarrier, two stages;
//  * lane = block (twice: 64 blocks): masks from shared memory, list of the octets to load of the
//    WHOLE brick by warp prefix sums: the touched octets and the initialised untouched octets of
//    every leaf line with a touched octet (a line, octets 4h..4h+3, is one 128 B-aligned piece of
//    the block that HBM delivers whole, so its other sectors come with the same DRAM access, and
//    the block keeps one maximum per line instead of one per octet); built one brick EARLY, right after the previous brick's leaf
//    loop, so that the brick's leaf sectors can be pulled into the L2 (prefetch.global.L2, no
//    registers) while the previous brick's aggregates are still being written;
//  * colour maps: the old depth-1 / depth-2 colours the block lanes need at the end travel by
//    cp.async into shared memory behind the leaf loop (no registers held across it);
//  * lanes then own list entries = 32 B leaf sectors, UFO_UB_INFLIGHT requested per lane before the
//    first is used (an uninitialised octet is not loaded: its leaves are 0.0): v = clamp(v + hit),
//    then v = clamp(v + miss) (float, order fixed), written back in place; an untouched octet is only read;
//    octet maxima / flags return through warp-private shared memory (__syncwarp only);
//  * block lanes write the line maxima and the meta word, clear the masks; depth-3 / depth-4
//    aggregates by shuffles.
// Alternatives that were slower on the bench workload: a list per half brick (latency exposed twice
// per brick); 2 sectors in flight at 6 CTAs of 80 registers; no L2 prefetch; more shared memory per
// SM (less L1 left for the sectors in flight); a cp.async leaf pipeline through shared memory (fewer
// warps, more instructions).
__device__ __forceinline__ void cp_async16(void* smem_dst, const void* g)
{
	asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem_dst)), "l"(g) : "memory");
}
__device__ __forceinline__ void cp_async4(void* smem_dst, const void* g)
{
	asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem_dst)), "l"(g) : "memory");
}
__device__ __forceinline__ void prefetch_l2(const void* g) { asm volatile("prefetch.global.L2 [%0];" ::"l"(g)); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

#ifndef UFO_UB_MINBLOCKS
#define UFO_UB_MINBLOCKS 5
#endif
#ifndef UFO_UB_PREFETCH
#define UFO_UB_PREFETCH 1  // pull the next brick's leaf sectors into the L2 one brick early
#endif
#ifndef UFO_UB_INFLIGHT_COLOR
#define UFO_UB_INFLIGHT_COLOR 1  // colour maps (each entry is two sectors: log-odds + colour): more in flight is slower on config #3
#endif
#ifndef UFO_UB_INFLIGHT
#define UFO_UB_INFLIGHT 3  // leaf sectors requested per lane before the first is used
#endif
#ifndef UFO_UB_MINBLOCKS_COLOR
#define UFO_UB_MINBLOCKS_COLOR 7
#endif
// One warp's shared memory.  Kept small on purpose: 5 CTAs per SM (30.5 KB each + 1 KB reserved) fit
// the 196 KB carve-out of the SM's 256 KB of L1 + shared memory; one step more (228 KB) leaves 28 KB
// of L1, too little for the leaf sectors the warps keep in flight.
template <bool COLOR>
struct __align__(128) BrickWork {
	WarpSlab slab[2];
	// colour maps: old depth-1 colours of a marked block; for an unmarked block the first word of
	// c1lo holds its old depth-2 colour instead
	uint4 c1lo[COLOR ? 64 : 1], c1hi[COLOR ? 64 : 1];
	float omax[512];
	uint32_t orgb[COLOR ? 512 : 2];
	// touched octets of a brick: (block << 3) | octet; after use the slot carries the octet's flags.
	// [it & 1]: the brick being processed, the other one: the warp's next brick (built one brick early)
	uint16_t list[2][512];
	unsigned long long bar[2];
};
template <bool COLOR>
struct UbShape {
	static constexpr int kWarps = COLOR ? 2 : 4;
	static constexpr int kMinBlocks = COLOR ? UFO_UB_MINBLOCKS_COLOR : UFO_UB_MINBLOCKS;
};

// PAIR: one pass over the touched list of two consecutive scans (DESIGN.md section 4, "Paired
// scans"): entry i holds the first scan's masks at touched_mi[i] and the second's at touched_mi2[i],
// and every voxel gets hit, miss of the first scan, then hit, miss of the second, as two passes
// would apply them.  Each scan's counters go to its own half of the statistics slots.
template <bool COLOR, bool SET = false, bool PAIR = false>
__global__ void __launch_bounds__(UbShape<COLOR>::kWarps * 32, UbShape<COLOR>::kMinBlocks) k_update_brick(DeviceMap M, float miss)
{
	constexpr int WARPS = UbShape<COLOR>::kWarps;
	__shared__ BrickWork<COLOR> s_work[WARPS];
	constexpr uint32_t FULL = 0xffffffffu;
	const uint32_t lane = threadIdx.x & 31, w = threadIdx.x >> 5;
	BrickWork<COLOR>& S = s_work[w];
	if (__ldg(&M.ctr->overflow) & ~4u) return;  // a pool overflowed while marking: the host grows it and repeats the scan
	const uint32_t n_touched = __ldg(&M.ctr->n_touched);
	const uint32_t gw = blockIdx.x * WARPS + w, n_warps = gridDim.x * WARPS;
	if (gw >= n_touched) return;
	const bool fold = M.alias_miss == nullptr;

	// lane 0: (brick, touched_mi) of the two stages.  A brick flagged kMiNoHits has no hit bit: its
	// hit masks are not staged, the lanes zero the slab's copy instead (zero_hits)
	uint32_t st_brick0 = kNone, st_brick1 = kNone, st_mi0 = 0, st_mi1 = 0, st_mj0 = 0, st_mj1 = 0;
	auto issue = [&](uint32_t stage, uint32_t e) {
		const uint32_t brick = M.touched[e], mi = M.touched_mi[e], mj = PAIR ? M.touched_mi2[e] : 0u;
		if (stage == 0) {
			st_brick0 = brick;
			st_mi0 = mi;
			st_mj0 = mj;
		} else {
			st_brick1 = brick;
			st_mi1 = mi;
			st_mj1 = mj;
		}
		fence_proxy_async();
		if (PAIR) {
			const bool a = mi != kMiAbsent, b = mj != kMiAbsent;
			mbar_expect_tx(&S.bar[stage], (a ? 512u : 0u) + (b ? 512u : 0u) + 256u + 512u);
			if (a) bulk_load(S.slab[stage].mm, M.mask_base + (size_t)(mi & ~kMiNoHits) * 64, 512u, &S.bar[stage]);
			if (b) bulk_load(S.slab[stage].hm, M.mask_base2 + (size_t)(mj & ~kMiNoHits) * 64, 512u, &S.bar[stage]);
		} else {
			const bool hits = !(mi & kMiNoHits);
			mbar_expect_tx(&S.bar[stage], 512u + (hits ? 512u : 0u) + 256u + 512u);
			bulk_load(S.slab[stage].mm, M.mask_base + (size_t)(mi & ~kMiNoHits) * 64, 512u, &S.bar[stage]);
			if (hits) bulk_load(S.slab[stage].hm, M.hit_mask + (size_t)brick * 64, 512u, &S.bar[stage]);
		}
		bulk_load(S.slab[stage].meta, M.meta + (size_t)brick * 64, 256u, &S.bar[stage]);
		bulk_load(S.slab[stage].q, M.line_max + (size_t)brick * 64, 512u, &S.bar[stage]);
	};
	// all lanes, before the stage's list is built (a __syncwarp in between)
	auto zero_hits = [&](uint32_t stage) {
		const uint32_t mi = __shfl_sync(FULL, stage == 0 ? st_mi0 : st_mi1, 0);
		if (PAIR) {  // a scan that did not mark the brick: its miss masks are zero
			const uint32_t mj = __shfl_sync(FULL, stage == 0 ? st_mj0 : st_mj1, 0);
			if (mi == kMiAbsent) reinterpret_cast<ulonglong2*>(S.slab[stage].mm)[lane] = make_ulonglong2(0ull, 0ull);
			if (mj == kMiAbsent) reinterpret_cast<ulonglong2*>(S.slab[stage].hm)[lane] = make_ulonglong2(0ull, 0ull);
		} else if (mi & kMiNoHits) {
			reinterpret_cast<ulonglong2*>(S.slab[stage].hm)[lane] = make_ulonglong2(0ull, 0ull);
		}
	};
	// Bricks are claimed, not dealt: a warp starts with touched entry gw and then takes the next
	// unclaimed entry (k3_cursor counts the claims beyond the first n_warps entries).  A brick next
	// to the sensor costs an order of magnitude more than one at the end of the range, so a fixed
	// deal ends with a few warps that drew heavy bricks and too few sectors in flight to keep the
	// DRAM busy.  Lane 0 claims one brick ahead, so the atomic's latency is hidden behind a brick.
	uint32_t claim = 0;
	if (lane == 0) {
		mbar_init(&S.bar[0], 1);
		mbar_init(&S.bar[1], 1);
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
		issue(0, gw);
		claim = n_warps + atomicAdd(&M.ctr->k3_cursor, 1u);
	}
	zero_hits(0);
	__syncwarp();

	unsigned int s_vox = 0, s_hit = 0, s_oct = 0, s_blk = 0, s_new = 0, s_lin = 0;
	unsigned int s_vox2 = 0, s_hit2 = 0, s_oct2 = 0, s_blk2 = 0, s_new2 = 0;  // PAIR: the second scan's
	// saturated lines (see apply_update): a miss-only leaf line whose 32 voxels all sit at clamp_min is
	// left as it is, so it is neither loaded nor written.  Exact only when the map holds no value below
	// clamp_min (M.sat_skip, kept by the host) and the marks land in the tree (fold).  Mono maps only:
	// on colour maps (config #3) the skip's extra code cost more K3 time than the lines it saved, so
	// the colour kernel still reads every touched line
	const bool sat = !COLOR && !SET && fold && M.sat_skip && miss <= 0.0f;

	// lane = block lane of either half: touched octets of the brick in `slab` and the octets to load
	// (touched, and the initialised octets of their lines), list by warp prefix sums.  t8 = the touched
	// octets that are loaded | the touched octets of saturated lines << 8 (not loaded)
	// PAIR: brick, mi, mj of the slab (their hit masks are read here)
	auto build_list = [&](const WarpSlab& slab, uint16_t* list, uint32_t (&t8)[2], uint32_t (&excl)[2], uint32_t& total,
	                      uint32_t brick, uint32_t mi, uint32_t mj) {
		total = 0;
#pragma unroll
		for (uint32_t h = 0; h < 2; ++h) {
			const uint32_t blk = h * 32 + lane;
			unsigned long long hm = slab.hm[blk], u = slab.mm[blk] | hm, ha = 0, hb = 0;
			if (PAIR) {
				const size_t b = (size_t)brick * 64 + blk;
				ha = (mi & kMiNoHits) ? 0ull : M.hit_mask[b];
				hb = (mj & kMiNoHits) ? 0ull : M.hit_mask2[b];
				hm = ha | hb;
				u = slab.mm[blk] | slab.hm[blk] | hm;
			}
			uint32_t t = 0, ld = 0, init = 0, sk = 0, eh = 0;
			if (u) {
				if (PAIR) {
					const unsigned long long ua = slab.mm[blk] | ha, ub = slab.hm[blk] | hb;
					const uint32_t ta = mask_octets(ua), tb = mask_octets(ub);
					t = ta | tb;
					s_vox += __popcll(ua);
					s_hit += __popcll(ha);
					s_oct += __popc(ta);
					s_vox2 += __popcll(ub);
					s_hit2 += __popcll(hb);
					s_oct2 += __popc(tb);
					eh = (ha ? kEntHitA : 0u) | (hb ? kEntHitB : 0u);
				} else {
					t = mask_octets(u);
				}
				if (!COLOR && !PAIR) {  // colour maps skip nothing and count in the leaf loop
					s_vox += __popcll(u);
					s_hit += __popcll(hm);
					s_oct += __popc(t);
				}
				init = (slab.meta[blk] >> 16) & 0xffu;
				if (sat) {
					const float2 q = slab.q[blk];
					const float qh[2] = {q.x, q.y};
#pragma unroll
					for (uint32_t k = 0; k < 2; ++k) {
						// line k = octets 4k..4k+3 = voxels with z in {2k, 2k+1}: bits 32k..32k+31 (linear mask order)
						const bool s = ((init >> (4 * k)) & 15u) == 15u && !((hm >> (32 * k)) & 0xffffffffull) &&
						               __float_as_uint(qh[k]) == __float_as_uint(M.clamp_min);
						sk |= s ? t & (15u << (4 * k)) : 0u;
					}
					t &= ~sk;
				}
				ld = t | (line_octets(t) & init);
				// out-of-tree hits (k_alias_apply, before this kernel) may have written an octet whose
				// initialised bit is still clear: touched octets are then loaded all the same
				if (!fold) init |= t;
			}
			uint32_t incl = __popc(ld);
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				const uint32_t v = __shfl_up_sync(FULL, incl, o);
				if (lane >= (uint32_t)o) incl += v;
			}
			excl[h] = total + incl - __popc(ld);
			t8[h] = t | (sk << 8);
			{
				uint32_t bits = ld, at = excl[h];
				while (bits) {
					const uint32_t o = __ffs(bits) - 1;
					bits &= bits - 1;
					list[at++] = (uint16_t)((blk << 3) | o | (((init >> o) & 1u) ? kEntInit : 0u) | (((t >> o) & 1u) ? kEntTouched | eh : 0u));
				}
			}
			total += __shfl_sync(FULL, incl, 31);
		}
	};

	uint32_t t8[2], excl[2], total = 0;     // the brick being processed
	uint32_t t8n[2], excln[2], totaln = 0;  // the warp's next brick (its list is built one brick early)
	mbar_wait(&S.bar[0], 0u);
	build_list(S.slab[0], S.list[0], t8, excl, total, __shfl_sync(FULL, st_brick0, 0), __shfl_sync(FULL, st_mi0, 0),
	           __shfl_sync(FULL, st_mj0, 0));
	__syncwarp();
	for (uint32_t it = 0;; ++it) {
		const uint32_t st = it & 1u;
		const uint32_t e_next = __shfl_sync(FULL, claim, 0);
		const bool has_next = e_next < n_touched;
		if (lane == 0 && has_next) {
			issue(st ^ 1u, e_next);  // stage st^1 was released by the __syncwarp at the end of the loop
			claim = n_warps + atomicAdd(&M.ctr->k3_cursor, 1u);
		}
		const uint32_t brick = __shfl_sync(FULL, st == 0 ? st_brick0 : st_brick1, 0);
		const uint32_t mi_raw = __shfl_sync(FULL, st == 0 ? st_mi0 : st_mi1, 0), mi = mi_raw & ~kMiNoHits;
		const uint32_t mj_raw = PAIR ? __shfl_sync(FULL, st == 0 ? st_mj0 : st_mj1, 0) : 0u, mj = mj_raw & ~kMiNoHits;
		const WarpSlab& slab = S.slab[st];
		const uint16_t* list = S.list[st];
		const size_t b0 = (size_t)brick * 64;

		// colours the block lanes need after the leaf loop: requested now, into shared memory
		if (COLOR) {
#pragma unroll
			for (uint32_t h = 0; h < 2; ++h) {
				const uint32_t blk = h * 32 + lane;
				if (t8[h]) {  // a marked block; its octets that are not loaded keep their old colour
					if ((t8[h] & 0xffu) != 0xffu) {
						cp_async16(&S.c1lo[COLOR ? blk : 0], M.sum1_rgb + (b0 + blk) * 8);
						cp_async16(&S.c1hi[COLOR ? blk : 0], M.sum1_rgb + (b0 + blk) * 8 + 4);
					}
				} else if (fold && (slab.meta[blk] & 0xff0000u)) {
					cp_async4(&S.c1lo[COLOR ? blk : 0], &M.rgb2[b0 + blk]);
				}
			}
			cp_async_commit();
		}
		__syncwarp();
		// lanes own list entries = 32 B leaf sectors (+ the colour sector of the same octet), NF of them
		// requested per lane before the first is used
		constexpr int NF = COLOR ? UFO_UB_INFLIGHT_COLOR : UFO_UB_INFLIGHT;
		for (uint32_t i = lane; i < total; i += 32 * NF) {
			float4 a0[NF], a1[NF];
			uint4 x0[COLOR ? NF : 1], x1[COLOR ? NF : 1];
			uint32_t en[NF];
#pragma unroll
			for (int f = 0; f < NF; ++f) {
				const uint32_t idx = i + 32 * f;
				en[f] = idx < total ? (uint32_t)list[idx] : 0xffffffffu;
				if (en[f] != 0xffffffffu) {
					const size_t off = (b0 + ((en[f] >> 3) & 63u)) * 64 + 8 * (en[f] & 7u);
					a0[f] = a1[f] = make_float4(0.f, 0.f, 0.f, 0.f);
					if (en[f] & kEntInit) {
						const float4* lp = reinterpret_cast<const float4*>(M.leaf + off);
						a0[f] = lp[0];
						a1[f] = lp[1];
					}
					if (COLOR && (en[f] & kEntTouched)) {
						const uint4* cp = reinterpret_cast<const uint4*>(M.leaf_rgb + off);
						x0[COLOR ? f : 0] = cp[0];
						x1[COLOR ? f : 0] = cp[1];
					}
				}
			}
#pragma unroll
			for (int f = 0; f < NF; ++f) {
				if (en[f] == 0xffffffffu) continue;
				const uint32_t idx = i + 32 * f, t = (en[f] >> 3) & 63u, o = en[f] & 7u;
				if (!(en[f] & kEntTouched)) {  // line-mate of a touched octet: its max only
					const float4 p = a0[f], q = a1[f];
					S.omax[idx] = fmaxf(fmaxf(fmaxf(p.x, p.y), fmaxf(p.z, p.w)), fmaxf(fmaxf(q.x, q.y), fmaxf(q.z, q.w)));
					continue;
				}
				const uint32_t m8 = octet_bits8(slab.mm[t], o);
				uint32_t h8, m8b = 0, h8b = 0;
				if (PAIR) {
					h8 = (en[f] & kEntHitA) ? octet_bits8(M.hit_mask[b0 + t], o) : 0u;
					m8b = octet_bits8(slab.hm[t], o);
					h8b = (en[f] & kEntHitB) ? octet_bits8(M.hit_mask2[b0 + t], o) : 0u;
				} else {
					h8 = octet_bits8(slab.hm[t], o);
				}
				float omax;
				uint32_t ofl;
				const bool clean = update_octet<SET, !COLOR, PAIR>(M, miss, M.leaf + (b0 + t) * 64 + 8 * o, m8, h8, a0[f], a1[f], omax,
				                                               ofl, b0 + t, o, (en[f] & kEntInit) != 0u, m8b, h8b);
				S.omax[idx] = omax;
				// the entry has been consumed: the slot carries the flags back (bit 2: not written back)
				S.list[st][idx] = (uint16_t)(ofl | (clean ? 4u : 0u));
				if (COLOR) {
					const uint4 c0 = x0[COLOR ? f : 0], c1 = x1[COLOR ? f : 0];
					const uint32_t cc[8] = {c0.x, c0.y, c0.z, c0.w, c1.x, c1.y, c1.z, c1.w};
					S.orgb[COLOR ? idx : 0] = rms_rgb(cc, 8);
					s_vox += __popc(m8 | h8);
					s_hit += __popc(h8);
					s_oct += 1;
				}
			}
		}
		if (has_next) {
			// the next brick of this warp: its slab was requested at the top of this iteration; build its
			// list now and pull its leaf sectors into the L2 while this brick's aggregates are written
			zero_hits(st ^ 1u);
			__syncwarp();
			mbar_wait(&S.bar[st ^ 1u], ((it + 1u) >> 1) & 1u);
			const uint32_t brick_n = __shfl_sync(FULL, st == 0 ? st_brick1 : st_brick0, 0);
			build_list(S.slab[st ^ 1u], S.list[st ^ 1u], t8n, excln, totaln, brick_n, __shfl_sync(FULL, st == 0 ? st_mi1 : st_mi0, 0),
			           __shfl_sync(FULL, st == 0 ? st_mj1 : st_mj0, 0));
#if UFO_UB_PREFETCH
			__syncwarp();
			const float* leaf_n = M.leaf + (size_t)brick_n * 64 * 64;
			for (uint32_t i = lane; i < totaln; i += 32) {
				const uint32_t en = S.list[st ^ 1u][i], off = ((en >> 3) & 63u) * 64 + 8 * (en & 7u);
				if (en & kEntInit) prefetch_l2(leaf_n + off);
				if (COLOR && (en & kEntTouched)) prefetch_l2(M.leaf_rgb + (size_t)brick_n * 64 * 64 + off);
			}
#endif
		}
		if (COLOR) cp_async_wait_all();
		__syncwarp();
		// block lanes: line maxima, meta, mask clearing
		float agg_occ[2];
		uint32_t agg_fl[2], agg_rgb[2];
		uint32_t n_clean = 0;  // profiling level 2: this lane's sectors that were not written back
		uint32_t mk[2] = {0u, 0u};  // PAIR: bit 0 the first scan marked the block, bit 1 the second
#pragma unroll
		for (uint32_t h = 0; h < 2; ++h) {
			const uint32_t blk = h * 32 + lane;
			const size_t b = b0 + blk;
			unsigned long long hm = slab.hm[blk], ha = 0, hb = 0;
			if (PAIR) {
				ha = (mi_raw & kMiNoHits) ? 0ull : M.hit_mask[b];
				hb = (mj_raw & kMiNoHits) ? 0ull : M.hit_mask2[b];
				mk[h] = ((slab.mm[blk] | ha) ? 1u : 0u) | ((slab.hm[blk] | hb) ? 2u : 0u);
				hm = ha | hb;
			}
			const uint32_t mt = slab.meta[blk];
			const bool marked = PAIR ? mk[h] != 0u : (slab.mm[blk] | hm) != 0ull;
			float my_occ = 0.0f;
			uint32_t my_fl = M.default_flags, my_rgb = 0;
			if (marked) {
				// t: the touched octets that were loaded.  An octet of a saturated line (t8 bits 8..15) is
				// treated like an untouched initialised one: flags from meta, old colour, old line max
				const uint32_t t = t8[h] & 0xffu, init = (mt >> 16) & 0xffu;
				uint4 q0 = make_uint4(0u, 0u, 0u, 0u), q1 = q0;
				if (COLOR && t != 0xffu) {
					q0 = S.c1lo[COLOR ? blk : 0];
					q1 = S.c1hi[COLOR ? blk : 0];
				}
				const uint32_t oldc[8] = {q0.x, q0.y, q0.z, q0.w, q1.x, q1.y, q1.z, q1.w};
				const float2 oq = slab.q[blk];
				const uint32_t ld = t | (line_octets(t) & init);
				float om[8];
				uint32_t newc[8];
				uint32_t bfl = 0, newmeta = 0, at = excl[h];
#pragma unroll
				for (uint32_t o = 0; o < 8; ++o) {
					uint32_t fl = M.default_flags, oc = 0;
					om[o] = 0.0f;  // an uninitialised octet (only used in a loaded line)
					if ((ld >> o) & 1u) {
						om[o] = S.omax[at];
						if ((t >> o) & 1u) {
							fl = S.list[st][at];
							if (!COLOR) {  // colour maps write every sector back
								n_clean += fl >> 2;
								fl &= 3u;
							}
							if (COLOR) oc = S.orgb[COLOR ? at : 0];
						}
						++at;
					}
					if (!((t >> o) & 1u) && ((init >> o) & 1u)) {
						fl = (mt >> (2 * o)) & 3u;
						if (COLOR) oc = oldc[o];
					}
					newc[o] = oc;
					bfl |= fl;
					newmeta |= (fl << (2 * o)) | (((t >> o) & 1u) << (16 + o));
				}
				// a line without a loaded touched octet keeps its maximum
				const float2 nq = line_maxima(om), q = make_float2((t & 0x0fu) ? nq.x : oq.x, (t & 0xf0u) ? nq.y : oq.y);
				const float bmax = block_occ(q);
				M.line_max[b] = q;
				if (COLOR) {
					uint4* cp = reinterpret_cast<uint4*>(M.sum1_rgb + b * 8);
					cp[0] = make_uint4(newc[0], newc[1], newc[2], newc[3]);
					cp[1] = make_uint4(newc[4], newc[5], newc[6], newc[7]);
					my_rgb = rms_rgb(newc, 8);
					M.rgb2[b] = my_rgb;
				}
				if (PAIR) {
					// the block carries the id of the last scan that marked it, as after two passes
					M.meta[b] = (newmeta & 0xffffffu) | (mt & 0xff0000u) | (((mk[h] & 2u) ? M.scan_id : M.pair_id) << 24);
					if (slab.mm[blk]) M.mask_base[(size_t)mi * 64 + blk] = 0ull;
					if (slab.hm[blk]) M.mask_base2[(size_t)mj * 64 + blk] = 0ull;
					if (ha) M.hit_mask[b] = 0ull;
					if (hb) M.hit_mask2[b] = 0ull;
					s_blk += mk[h] & 1u;
					s_blk2 += mk[h] >> 1;
					// a first-touched block counts for the first scan that marked it
					if (!(mt & 0xff0000u)) {
						s_new += mk[h] & 1u;
						s_new2 += mk[h] == 2u ? 1u : 0u;
					}
				} else {
					M.meta[b] = (newmeta & 0xffffffu) | (mt & 0xff0000u) | (M.scan_id << 24);
					M.mask_base[(size_t)mi * 64 + blk] = 0ull;  // masks cleared for the next scan
					if (hm) M.hit_mask[b] = 0ull;
					s_blk += 1;
					s_new += (mt & 0xff0000u) ? 0u : 1u;
				}
				s_lin += ((t & 0x0fu) ? 1u : 0u) + ((t & 0xf0u) ? 1u : 0u);  // leaf lines read
				my_occ = bmax;
				my_fl = bfl | 0x100u;
			} else if (fold && (mt & 0xff0000u)) {
				my_occ = block_occ(slab.q[blk]);
				my_fl = block_flags(M, mt);
				if (COLOR) my_rgb = S.c1lo[COLOR ? blk : 0].x;
			}
			agg_occ[h] = my_occ;
			agg_fl[h] = my_fl;
			agg_rgb[h] = my_rgb;
		}
		// depth-3 / depth-4 aggregates: half h holds depth-3 nodes 4h..4h+3, eight lanes each
		if (fold) {
			float m3[2], m4 = -3.402823466e+38f;
			uint32_t f3[2], u3[2], f4 = 0, rgb3[2] = {0, 0};
#pragma unroll
			for (int h = 0; h < 2; ++h) {
				m3[h] = agg_occ[h];
				f3[h] = agg_fl[h] & 3u;
				u3[h] = (agg_fl[h] >> 8) & 1u;
#pragma unroll
				for (int o = 1; o < 8; o <<= 1) {
					m3[h] = fmaxf(m3[h], __shfl_xor_sync(FULL, m3[h], o));
					f3[h] |= __shfl_xor_sync(FULL, f3[h], o);
					u3[h] |= __shfl_xor_sync(FULL, u3[h], o);
				}
				if (COLOR) {
					uint32_t cc[8];
#pragma unroll
					for (int q = 0; q < 8; ++q) cc[q] = __shfl_sync(FULL, agg_rgb[h], (lane & 24) + q);
					rgb3[h] = rms_rgb(cc, 8);
				}
				float t = m3[h];
				uint32_t tf = f3[h];
#pragma unroll
				for (int o = 8; o < 32; o <<= 1) {
					t = fmaxf(t, __shfl_xor_sync(FULL, t, o));
					tf |= __shfl_xor_sync(FULL, tf, o);
				}
				m4 = fmaxf(m4, t);
				f4 |= tf;
			}
			uint32_t rgb4 = 0;
			if (COLOR) {
				uint32_t cc[8];
#pragma unroll
				for (int q = 0; q < 4; ++q) {
					cc[q] = __shfl_sync(FULL, rgb3[0], 8 * q);
					cc[4 + q] = __shfl_sync(FULL, rgb3[1], 8 * q);
				}
				rgb4 = rms_rgb(cc, 8);
			}
			const uint32_t ub0 = __ballot_sync(FULL, u3[0] != 0 && (lane & 7) == 0), ub1 = __ballot_sync(FULL, u3[1] != 0 && (lane & 7) == 0);
			uint32_t d3a = 0, d3b = 0;  // PAIR: depth-3 nodes marked by each scan
			if (PAIR) {
				d3a = ballot_groups(__ballot_sync(FULL, mk[0] & 1u)) + ballot_groups(__ballot_sync(FULL, mk[1] & 1u));
				d3b = ballot_groups(__ballot_sync(FULL, mk[0] & 2u)) + ballot_groups(__ballot_sync(FULL, mk[1] & 2u));
			}
			if ((lane & 7) == 0) {
#pragma unroll
				for (int h = 0; h < 2; ++h) {
					M.brick_sum3[(size_t)brick * 8 + 4 * h + (lane >> 3)] = {m3[h], f3[h]};
					if (COLOR) M.brick_rgb3[(size_t)brick * 8 + 4 * h + (lane >> 3)] = rgb3[h];
				}
			}
			if (lane == 0) {
				M.brick_sum4[brick] = {m4, f4};
				if (COLOR) M.brick_rgb4[brick] = rgb4;
				if (PAIR) {
					unsigned long long* sa = M.ctr->stat[brick % (kStatSlots / 2)];
					unsigned long long* sb = M.ctr->stat[kStatSlots / 2 + brick % (kStatSlots / 2)];
					if (mi_raw != kMiAbsent) {
						atomicAdd(&sa[5], 1ull);
						atomicAdd(&sa[6], (unsigned long long)d3a);
					}
					if (mj_raw != kMiAbsent) {
						atomicAdd(&sb[5], 1ull);
						atomicAdd(&sb[6], (unsigned long long)d3b);
					}
				} else {
					unsigned long long* slot = M.ctr->stat[brick % kStatSlots];
					atomicAdd(&slot[5], 1ull);
					atomicAdd(&slot[6], (unsigned long long)(__popc(ub0) + __popc(ub1)));
				}
			}
		}
		if (!COLOR && M.k3_stat) {
			// profiling level 2: touched octets of saturated lines, leaf lines that were not read because
			// of them, sectors not written back
			uint32_t n_sat = 0, n_lin = 0;
#pragma unroll
			for (uint32_t h = 0; h < 2; ++h) {
				const uint32_t t = t8[h] & 0xffu, sk = t8[h] >> 8;
				n_sat += __popc(sk);
				n_lin += ((sk & 0x0fu) && !(t & 0x0fu) ? 1u : 0u) + ((sk & 0xf0u) && !(t & 0xf0u) ? 1u : 0u);
			}
			n_sat = __reduce_add_sync(FULL, n_sat);
			n_lin = __reduce_add_sync(FULL, n_lin);
			n_clean = __reduce_add_sync(FULL, n_clean);
			if (lane == 0) {
				unsigned long long* slot = M.k3_stat->slot[brick % kStatSlots];
				if (n_sat) atomicAdd(&slot[0], (unsigned long long)n_sat);
				if (n_lin) atomicAdd(&slot[1], (unsigned long long)n_lin);
				if (n_clean) atomicAdd(&slot[2], (unsigned long long)n_clean);
			}
		}
		if (!has_next) break;
		t8[0] = t8n[0];
		t8[1] = t8n[1];
		excl[0] = excln[0];
		excl[1] = excln[1];
		total = totaln;
		__syncwarp();  // the slab stage, the list and the result arrays are reused
	}
	for (int o = 16; o > 0; o >>= 1) {
		s_vox += __shfl_xor_sync(FULL, s_vox, o);
		s_hit += __shfl_xor_sync(FULL, s_hit, o);
		s_oct += __shfl_xor_sync(FULL, s_oct, o);
		s_blk += __shfl_xor_sync(FULL, s_blk, o);
		s_new += __shfl_xor_sync(FULL, s_new, o);
		s_lin += __shfl_xor_sync(FULL, s_lin, o);
		if (PAIR) {
			s_vox2 += __shfl_xor_sync(FULL, s_vox2, o);
			s_hit2 += __shfl_xor_sync(FULL, s_hit2, o);
			s_oct2 += __shfl_xor_sync(FULL, s_oct2, o);
			s_blk2 += __shfl_xor_sync(FULL, s_blk2, o);
			s_new2 += __shfl_xor_sync(FULL, s_new2, o);
		}
	}
	if (PAIR && lane == 0) {
		// the leaf lines read are the pass's: they count for its last scan
		unsigned long long* slot = M.ctr->stat[kStatSlots / 2 + gw % (kStatSlots / 2)];
		if (s_vox2) atomicAdd(&slot[0], (unsigned long long)s_vox2);
		if (s_hit2) atomicAdd(&slot[1], (unsigned long long)s_hit2);
		if (s_oct2) atomicAdd(&slot[2], (unsigned long long)s_oct2);
		if (s_blk2) atomicAdd(&slot[3], (unsigned long long)s_blk2);
		if (s_new2) atomicAdd(&slot[4], (unsigned long long)s_new2);
		if (s_lin) atomicAdd(&slot[7], (unsigned long long)s_lin);
		s_lin = 0;
	}
	if (lane == 0) {
		unsigned long long* slot = M.ctr->stat[gw % (PAIR ? kStatSlots / 2 : kStatSlots)];
		if (s_vox) atomicAdd(&slot[0], (unsigned long long)s_vox);
		if (s_hit) atomicAdd(&slot[1], (unsigned long long)s_hit);
		if (s_oct) atomicAdd(&slot[2], (unsigned long long)s_oct);
		if (s_blk) atomicAdd(&slot[3], (unsigned long long)s_blk);
		if (s_new) atomicAdd(&slot[4], (unsigned long long)s_new);
		if (s_lin) atomicAdd(&slot[7], (unsigned long long)s_lin);
	}
}

// Stand-alone depth-3 / depth-4 pass over the touched list: only used when out-of-tree marks
// exist (they are applied after k_update_brick, which then skips its folded reduction).
// One warp per brick, lane owns children 2*lane and 2*lane+1 (both under depth-3 node lane/4).
template <bool COLOR>
__global__ void __launch_bounds__(256) k_brick_agg(DeviceMap M)
{
	const uint32_t lane = threadIdx.x & 31;
	const uint32_t n_touched = __ldg(&M.ctr->n_touched);
	if (__ldg(&M.ctr->overflow) & ~4u) return;
	constexpr uint32_t FULL = 0xffffffffu;
	for (uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; e < n_touched; e += (gridDim.x * blockDim.x) >> 5) {
		const uint32_t brick = M.touched[e];
		if (M.alias_miss) {  // bricks that only collect out-of-tree marks own no voxels
			uint32_t ax, ay, az;
			if (alias_source(M, brick, ax, ay, az)) continue;
		}
		const size_t b = (size_t)brick * 64 + 2 * lane;
		const uint2 mt = *reinterpret_cast<const uint2*>(&M.meta[b]);
		Agg c0 = {block_occ(M.line_max[b]), block_flags(M, mt.x)}, c1 = {block_occ(M.line_max[b + 1]), block_flags(M, mt.y)};
		if (!(mt.x & 0xff0000u)) c0 = {0.0f, M.default_flags};  // never written: unknown space
		if (!(mt.y & 0xff0000u)) c1 = {0.0f, M.default_flags};
		const uint32_t tag = M.scan_id & 0xffu;
		const bool upd = ((mt.x & 0xff0000u) && (mt.x >> 24) == tag) || ((mt.y & 0xff0000u) && (mt.y >> 24) == tag);
		float m3 = fmaxf(c0.occ, c1.occ);
		uint32_t f3 = (c0.flags | c1.flags) & 3u;
#pragma unroll
		for (int o = 1; o < 4; o <<= 1) {
			m3 = fmaxf(m3, __shfl_xor_sync(FULL, m3, o));
			f3 |= __shfl_xor_sync(FULL, f3, o);
		}
		float m4 = m3;
		uint32_t f4 = f3;
#pragma unroll
		for (int o = 4; o < 32; o <<= 1) {
			m4 = fmaxf(m4, __shfl_xor_sync(FULL, m4, o));
			f4 |= __shfl_xor_sync(FULL, f4, o);
		}
		if ((lane & 3) == 0) M.brick_sum3[(size_t)brick * 8 + (lane >> 2)] = {m3, f3};
		if (lane == 0) M.brick_sum4[brick] = {m4, f4};
		if (COLOR) {
			const uint2 cr = *reinterpret_cast<const uint2*>(&M.rgb2[b]);
			const uint32_t r0 = (mt.x & 0xff0000u) ? cr.x : 0u, r1 = (mt.y & 0xff0000u) ? cr.y : 0u;
			uint32_t cc[8];
#pragma unroll
			for (int j = 0; j < 4; ++j) {
				cc[2 * j] = __shfl_sync(FULL, r0, (lane & 28) + j);
				cc[2 * j + 1] = __shfl_sync(FULL, r1, (lane & 28) + j);
			}
			const uint32_t rgb3 = rms_rgb(cc, 8);
#pragma unroll
			for (int j = 0; j < 8; ++j) cc[j] = __shfl_sync(FULL, rgb3, 4 * j);
			const uint32_t rgb4 = rms_rgb(cc, 8);
			if ((lane & 3) == 0) M.brick_rgb3[(size_t)brick * 8 + (lane >> 2)] = rgb3;
			if (lane == 0) M.brick_rgb4[brick] = rgb4;
		}
		const uint32_t ub = __ballot_sync(FULL, upd);
		if (lane == 0) {
			uint32_t d3 = 0;
			for (int k = 0; k < 8; ++k) d3 += ((ub >> (4 * k)) & 0xfu) ? 1u : 0u;
			unsigned long long* slot = M.ctr->stat[brick % kStatSlots];
			atomicAdd(&slot[5], 1ull);
			atomicAdd(&slot[6], (unsigned long long)d3);
		}
	}
}

}  // namespace ufo_b200
