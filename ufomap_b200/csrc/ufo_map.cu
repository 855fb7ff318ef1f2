// ufo_map.cu -- host side of libufomap_b200.so: device pools, scan orchestration
// and the C ABI declared in include/ufomap_b200.h.
//
// One map = one CUDA device + one stream (+ a copy stream for the points).  An insert enqueues
//   H2D(points) -> K1 k_points [-> K1b k_hits] -> k_split -> k_walk_mark -> k_gather_scan ->
//   k_gather -> K3 k_update_brick -> K4 k_upper_* -> D2H(counters)
// and returns; the next call that looks at the map reads the counters, grows a pool and repeats
// the scan if an allocation overflowed (finalize_scan).  Insert depth >= 3, maps that have seen
// out-of-tree keys and the fixed-step walk use k_rays -> k_scatter instead of the fused walk,
// which mirrors insertPointCloud + insertPointCloudHelper
// (/root/reference/ufomap/include/ufo/map/occupancy_map_base.h:270-327, :1345-1373).
// early_stopping on a map that opted in replaces the walk by E1-E3 (ufo_early.cuh).
// There is no CPU fallback anywhere in this file.

#include <cuda_runtime.h>
#include <dlfcn.h>

#include <algorithm>
#include <chrono>
#include <functional>
#include <numeric>
#include <optional>
#include <queue>
#include <climits>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <new>
#include <string>
#include <utility>
#include <vector>

#include "../../include/ufomap_b200.h"
#include "ufo_kernels.cuh"
#include "ufo_export.cuh"
#include "ufo_walk.cuh"
#include "ufo_route.cuh"
#include "ufo_import.cuh"
#include "ufo_write.cuh"
#include "ufo_early.cuh"
#include "ufo_page.cuh"

#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>

using namespace ufo_b200;

namespace
{
constexpr uint32_t kMinHash = 1u << 16;

uint32_t next_pow2(uint64_t v)
{
	uint64_t p = 1;
	while (p < v) p <<= 1;
	return (uint32_t)std::min<uint64_t>(p, 1ull << 31);
}

struct CudaError {
	cudaError_t e;
	const char* what;
	int line;
};

#define CK(call)                                         \
	do {                                                   \
		cudaError_t e__ = (call);                            \
		if (e__ != cudaSuccess) throw CudaError{e__, #call, __LINE__}; \
	} while (0)

// Device memory for the duration of one call, freed on every way out of it.
struct DevBuf {
	void* p = nullptr;
	DevBuf() = default;
	DevBuf(const DevBuf&) = delete;
	DevBuf& operator=(const DevBuf&) = delete;
	~DevBuf() { release(); }
	// n elements of T (at least one), uninitialised, in place of what the buffer held
	template <class T>
	T* alloc(size_t n)
	{
		release();
		CK(cudaMalloc(&p, std::max<size_t>(n, 1) * sizeof(T)));
		return static_cast<T*>(p);
	}
	void release()
	{
		if (p) cudaFree(p);
		p = nullptr;
	}
};

// the events of one call
struct Events {
	cudaEvent_t e[4] = {};
	Events()
	{
		for (auto& x : e) CK(cudaEventCreate(&x));
	}
	Events(const Events&) = delete;
	Events& operator=(const Events&) = delete;
	~Events()
	{
		for (auto& x : e)
			if (x) cudaEventDestroy(x);
	}
};

double to_logit(double p) { return std::log(p / (1.0 - p)); }
}  // namespace

struct MapError {
	int code;
};

// everything needed to enqueue a scan again after a pool growth
struct PendingScan {
	bool valid = false;
	ScanArgs a{};
	bool use_color = false, need_table = false, simple = false, has_vol = false;
	bool routed = false;  // routed multi-GPU pass (ufo_route.cuh)
	bool applying = false;  // routed pass: the first apply call has run
	// routed pass: the apply calls enqueued so far (sources, scan id), replayed in their order from the
	// first one that backed off after a pool growth
	struct RouteCall {
		uint32_t first, count, scan_id;
	};
	std::vector<RouteCall> calls;
	bool dense = false;   // marks go to the dense scan volume
	// marked, leaf update (K3, K4) not enqueued yet: the next insert may share it (a paired pass), any
	// other call enqueues it alone (finalize_scan)
	bool defer = false;
	bool flushed = false;  // a deferred scan whose leaf update was enqueued alone
	VolumeArgs vol{};
	float set_value = 0.0f;
	uint32_t early = 0;  // early_stopping of a scan on a map that opted in (ufo_early.cuh); 0: off
	uint32_t regrows = 0;
	// write batch (ufo_write.cuh): ordered node updates or rays instead of a scan
	bool write = false;
	WriteArgs w{};
};

// Device memory a map holds across calls, and its size.  Every such allocation, these and the pool
// arrays of kPool, is made and freed by map_realloc, so device_bytes is the sum of the live ones.
template <class T>
struct DevMem {
	T* p = nullptr;
	size_t bytes = 0;
	DevMem() = default;
	DevMem(const DevMem&) = delete;
	DevMem& operator=(const DevMem&) = delete;
	~DevMem()
	{
		if (p) cudaFree(p);  // the map goes with it: nothing left to account for
	}
	// at least n bytes; a new allocation is filled with the byte `fill` (< 0: left uninitialised)
	void ensure(ufo_b200_map* m, size_t n, int fill);
	void release(ufo_b200_map* m);
};

struct ufo_b200_map {
	ufo_b200_params params{};
	DeviceMap M{};
	int device = 0;
	cudaStream_t own_stream = nullptr, stream = nullptr, copy_stream = nullptr;
	cudaEvent_t ev_copy0 = nullptr, ev_copied = nullptr;
	// sensor model as the reference stores it (double log-odds)
	double occ_thr_log = 0, free_thr_log = 0, hit_log = 0, miss_log = 0, cmin_log = 0, cmax_log = 0;
	// host mirror of the counters (pinned)
	Counters* h_ctr = nullptr;
	// owners of the device memory DeviceMap sees outside the pool arrays: counters, the hashes of the
	// two pools and the dense scan volume (setup_volume)
	DevMem<Counters> ctr;
	DevMem<K3Stats> k3_stat;  // profiling level 2, allocated on first use
	bool k3_counted = false;  // this scan's k_update_brick counts into k3_stat
	DevMem<ulonglong2> bh_tab;
	DevMem<unsigned long long> uh_keys;
	DevMem<uint32_t> uh_vals;
	DevMem<unsigned long long> vol, vol_dirty;
	DevMem<uint32_t> vol_list;
	// the second scan's dense volume of a paired pass, allocated by the first pair; no_pair once that
	// failed (the map then runs one scan per pass)
	DevMem<unsigned long long> vol2, vol2_dirty;
	DevMem<uint32_t> vol2_list;
	uint32_t vol2_db_cap = 0;
	bool no_pair = false;
	// change masks (a pool array): kept while detection is switched off, M.chg_mask only while recording
	unsigned long long* chg_mask = nullptr;
	bool chg_recording = false;
	// scan staging: two point buffers, so that the H2D copy of scan k+1 overlaps scan k
	DevMem<void> d_points[2];
	uint32_t stage = 0;
	DevMem<double> d_ray_end;
	DevMem<uint32_t> d_hit_tab;
	size_t ray_cap = 0;
	DevMem<unsigned long long> d_tab_keys;
	DevMem<uint32_t> d_tab_min;
	uint32_t tab_size = 0;
	uint32_t* d_list[2] = {nullptr, nullptr};
	// generic marking path: ray-walk records
	DevMem<QEntry> d_seg;
	unsigned long long seg_cap = 0;
	DevMem<uint32_t> d_seg_base, d_seg_count, d_order;
	DevMem<unsigned long long> d_nodes;  // insert depth 5/6: free-space nodes of the scan
	// fused walk: segments, validity masks, per-ray constants
	DevMem<Item> d_items;
	DevMem<uint32_t> d_vmask;
	DevMem<RayConst> d_rc;
	size_t item_cap = 0;
	// write batches: inputs + record regions, records (two key / index buffers for the sort), the
	// brick segments of the sorted keys, sort scratch
	DevMem<unsigned char> d_w_in;
	DevMem<unsigned long long> d_w_keys[2];
	DevMem<uint32_t> d_w_idx[2];
	DevMem<WriteRec> d_w_recs;
	size_t w_rec_cap = 0;
	DevMem<uint32_t> d_w_seg;
	DevMem<void> d_w_tmp;
	bool write_pass = false;  // the last pass was a write batch (its stats carry ms_update)
	// early stopping (ufo_early.cuh), allocated on the first such scan: node table, per-ray visit
	// counts / offsets / prefix lengths, visit ids, scan scratch
	int early_exact = 0;  // ufo_b200_set_early_stopping: early_stopping != 0 is computed, not rejected
	bool early_pass = false;  // the last pass was such a scan
	DevMem<unsigned long long> d_e_keys;
	DevMem<uint32_t> d_e_first;
	size_t e_tab_cap = 0;
	DevMem<unsigned long long> d_e_cnt, d_e_off;
	DevMem<uint32_t> d_e_plen, d_e_pnext;
	size_t e_ray_cap = 0;
	DevMem<uint32_t> d_e_ids;
	unsigned long long e_id_cap = 0;
	DevMem<void> d_e_tmp;
	int early_blocks_per_sm = 1;
	ufo_b200_early_stats early_stats{};
	// bookkeeping
	uint32_t n_blocks = 0, n_bricks = 0, n_upper = 0;  // host view after the last completed scan
	size_t device_bytes = 0;
	int profiling = 0;
	int force_records = 0;  // UFO_B200_MARK=records: always use the record path (A/B runs)
	int k3_blocks = 0;      // UFO_B200_K3_BLOCKS: resident K3 CTAs per SM (0: the kernel's launch bound)
	int no_dense = 0;       // UFO_B200_MARK=probe, or a scan left the volume: fused walk through the brick hash
	uint32_t vol_db_cap = 0;  // bricks per axis the allocated scan volume can hold
	uint64_t launches = 0;
	cudaEvent_t ev[10]{};  // [8]: start of the leaf update, [9]: end of a deferred scan's marking
	bool ev_valid = false, ev7_valid = false, h2d_valid = false;
	ufo_b200_scan_stats stats{};       // scan in flight / last scan
	ufo_b200_scan_stats done_stats{};  // last scan whose counters are folded into the host view
	ufo_b200_walk_stats walk_stats{};  // last scan, profiling level 2
	ufo_b200_update_stats update_stats{};  // last scan, profiling level 2
	// a lower bound of every leaf value the map holds: 0.0 (the voxels of an initialised octet that no
	// update has reached yet) and the lowest clamp_min any update could have clamped to; -inf once
	// values came in unclamped (readData, page_in).  Sets DeviceMap::sat_skip
	float value_floor = 0.0f;
	bool stats_pending = false;
	PendingScan pending;
	// Paired pass: `pending` is its second scan; the first one's scan id, touched entries and counters
	// up to its marking are kept here.  held_stats: the second scan's counters, which
	// completed_scan_stats reports one insert after the first scan's
	bool paired = false;
	uint32_t first_id = 0, first_touched = 0;
	ufo_b200_scan_stats first_stats{}, held_stats{};
	bool held = false;
	bool poisoned = false;
	// routed multi-GPU mode
	DevMem<unsigned char> route_inbox;  // this rank's inbox: [2 parities][world sources] regions
	DevMem<RouteTable> route_table;     // M.route
	size_t route_region = 0, route_miss_off = 0, route_hit_off = 0;
	void* route_peer[kMaxRanks] = {};
	RouteTable* h_route = nullptr;  // pinned mirror, pushed before every mark pass
	uint32_t* h_route_flag = nullptr;  // pinned: RouteTable::overflow, then ::sent[3] of the last mark pass
	// colour maps: apply table (minimum global cloud index per hit voxel of one apply call)
	DevMem<unsigned long long> d_route_tab_keys;
	DevMem<uint32_t> d_route_tab_min;
	uint32_t route_tab_size = 0;
	uint32_t route_parity = 0, route_cap_m = 0, route_cap_h = 0;
	int route_stage = 0;  // 0 idle, 1 marked (waiting for the apply calls), 2 applied
	double min_change[3], max_change[3];
	// nearest-first iteration: every call that writes the pools or the thresholds bumps the revision;
	// the tree shape above the bricks (TreeShape) is kept with the revision it was built at
	uint64_t revision = 1;
	std::shared_ptr<struct TreeShape> shape;
	ufo_b200_nearest_stats nearest_stats{};
	std::string err;
	int sm_count = 132;
	int ray_blocks_per_sm = 4, walk_blocks_per_sm = 4;

	void set_error(const char* fmt, ...)
	{
		char buf[512];
		va_list ap;
		va_start(ap, fmt);
		vsnprintf(buf, sizeof(buf), fmt, ap);
		va_end(ap);
		err = buf;
	}
};

namespace
{
using Map = ufo_b200_map;

// Scans may skip saturated leaf lines (apply_update) while no leaf lies below clamp_min: the floor only
// falls (a lowered clamp_min, unclamped values), so once clamp_min is raised above it the skip stays
// off until the map is cleared.  The floor is at most 0.0, so a positive clamp_min never skips.
void set_value_floor(Map* m, float floor)
{
	DeviceMap& M = m->M;
	m->value_floor = floor;
	M.sat_skip = (floor >= M.clamp_min && M.clamp_min != 0.0f && M.clamp_min <= M.clamp_max) ? 1u : 0u;
}

void refresh_model(Map* m)
{
	DeviceMap& M = m->M;
	M.occ_thr = m->occ_thr_log;
	M.free_thr = m->free_thr_log;
	M.hit = (float)m->hit_log;
	M.clamp_min = (float)m->cmin_log;
	M.clamp_max = (float)m->cmax_log;
	// toProb(float) with expf, as the reference evaluates it on the host
	M.prob_hit = 1.0 / (1.0 + (double)expf(-M.hit));
	// float thresholds exactly equivalent to the reference's double-vs-float compares
	{
		float fc = (float)m->free_thr_log;
		if ((double)fc < m->free_thr_log) fc = nextafterf(fc, INFINITY);
		float of = (float)m->occ_thr_log;
		if ((double)of > m->occ_thr_log) of = nextafterf(of, -INFINITY);
		M.free_ceil = fc;
		M.occ_floor = of;
	}
	uint32_t f = (m->free_thr_log > 0.0) ? 1u : 0u;
	if (m->free_thr_log <= 0.0 && m->occ_thr_log >= 0.0) f |= 2u;
	M.default_flags = f;
	set_value_floor(m, fminf(m->value_floor, M.clamp_min));
}

void reset_bbox(Map* m)
{
	double h = node_half(m->M.g, m->M.g.depth_levels);
	for (int i = 0; i < 3; ++i) {
		m->min_change[i] = h;
		m->max_change[i] = -h;
	}
}

// capacities of a new map: the params' hint, or the default
void initial_caps(const ufo_b200_params& p, uint32_t& bricks, uint32_t& upper)
{
	// a brick owns 64 block slots; the block hint is honoured through its brick equivalent
	// (a touched brick of a lidar scan holds ~32 touched blocks)
	const uint64_t bricks64 = p.initial_bricks ? p.initial_bricks : (p.initial_blocks ? p.initial_blocks / 32 : (1ull << 15));
	bricks = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(bricks64, 16), 0x3ffffffull);
	upper = std::max(bricks / 2, 4096u);
}

// The one place a map's device memory is allocated and freed (DevMem and the pool arrays): frees
// `old` (`old_bytes` long) and returns n new bytes, uninitialised (nullptr for none).
void* map_realloc(Map* m, void* old, size_t old_bytes, size_t n)
{
	if (old) {
		cudaFree(old);  // a failure here is a broken context, which the next checked call reports
		m->device_bytes -= old_bytes;
	}
	void* q = nullptr;
	if (n) {
		CK(cudaMalloc(&q, n));
		m->device_bytes += n;
	}
	return q;
}
}  // namespace

template <class T>
void DevMem<T>::ensure(Map* m, size_t n, int fill)
{
	if (p && n <= bytes) return;
	release(m);
	p = static_cast<T*>(map_realloc(m, nullptr, 0, n));
	bytes = n;
	if (fill >= 0 && n) CK(cudaMemsetAsync(p, fill, n, m->stream));
}

template <class T>
void DevMem<T>::release(Map* m)
{
	void* old = p;
	p = nullptr;
	map_realloc(m, old, bytes, 0);
	bytes = 0;
}

namespace
{
// at least `bytes` (uninitialised), with an eighth to spare so that a slowly growing need does not
// reallocate on every call
template <class T>
void ensure_spare(Map* m, DevMem<T>& b, size_t bytes, size_t min_bytes)
{
	if (!b.p || bytes > b.bytes) b.ensure(m, std::max(bytes + bytes / 8, min_bytes), -1);
}

// moves `n` whole bricks of `brick_bytes` each (k_page_move) with the widest word that divides a brick
template <bool SCATTER>
void launch_page_move(Map* m, void* dst, const void* src, const uint32_t* slot, size_t n, size_t brick_bytes)
{
	if (!n) return;
	auto run = [&](auto* d, size_t word) {
		using V = std::remove_pointer_t<decltype(d)>;
		const size_t per = brick_bytes / word;
		uint32_t lg = 0;
		while (((size_t)1 << lg) < per) ++lg;
		const size_t units = n * per;
		const uint32_t grid = (uint32_t)std::min<size_t>((units + 255) / 256, (size_t)m->sm_count * 32);
		k_page_move<V, SCATTER><<<grid, 256, 0, m->stream>>>(d, static_cast<const V*>(src), slot, units, lg);
	};
	if (brick_bytes % 16 == 0) run(static_cast<uint4*>(dst), 16);
	else if (brick_bytes % 8 == 0) run(static_cast<uint2*>(dst), 8);
	else run(static_cast<uint32_t*>(dst), 4);
	++m->launches;
}

// ---- the two pools: every per-brick and per-upper-node array, described once ----
enum class Pool : uint8_t { Brick, Upper };
// when an array exists: always, on colour maps, from the first out-of-tree key a scan meets, or from
// the first ufo_b200_enable_change_detection on
enum class Have : uint8_t { Always, Color, Aliases, Changes };
// what retain does with it: gather the surviving bricks, or start again from the fill
enum class Retain : uint8_t { Compact, Renew };

struct PoolArray {
	void** (*owner)(Map*);  // where the owning pointer lives
	size_t elem;            // bytes per element
	uint32_t per;           // elements per brick / per upper node
	int fill;               // byte of a slot nothing has written yet
	Pool pool;
	Have have;
	Retain retain;
};

#define UFO_POOL_ARRAY(ptr) [](Map* m) { return reinterpret_cast<void**>(&m->ptr); }, sizeof(*std::declval<Map&>().ptr)
// In the order a new map allocates them (the driver's sub-allocator packs the small arrays by it,
// which shows in the time of the scans right after a growth).
const PoolArray kPool[] = {
	{UFO_POOL_ARRAY(M.brick_key), 1, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.brick_stamp), 1, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.hit_stamp), 1, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.touched), 1, 0, Pool::Brick, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.touched_alt), 1, 0, Pool::Brick, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.touched_mi), 1, 0, Pool::Brick, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.touched_alt_mi), 1, 0, Pool::Brick, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.brick_sum3), 8, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.brick_sum4), 1, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.leaf), 64 * 64, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.miss_mask), 64, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.hit_mask), 64, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.hit_mask2), 64, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.touched_mi2), 1, 0, Pool::Brick, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.touch_idx), 1, 0, Pool::Brick, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.meta), 64, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.line_max), 64, 0, Pool::Brick, Have::Always, Retain::Compact},
	{UFO_POOL_ARRAY(M.brick_parent), 1, 0xff, Pool::Brick, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(chg_mask), 64, 0, Pool::Brick, Have::Changes, Retain::Compact},
	{UFO_POOL_ARRAY(M.alias_miss), 64, 0, Pool::Brick, Have::Aliases, Retain::Compact},
	{UFO_POOL_ARRAY(M.alias_hit), 64, 0, Pool::Brick, Have::Aliases, Retain::Compact},
	{UFO_POOL_ARRAY(M.brick_rgb3), 8, 0, Pool::Brick, Have::Color, Retain::Compact},
	{UFO_POOL_ARRAY(M.brick_rgb4), 1, 0, Pool::Brick, Have::Color, Retain::Compact},
	{UFO_POOL_ARRAY(M.leaf_rgb), 64 * 64, 0, Pool::Brick, Have::Color, Retain::Compact},
	{UFO_POOL_ARRAY(M.sum1_rgb), 64 * 8, 0, Pool::Brick, Have::Color, Retain::Compact},
	{UFO_POOL_ARRAY(M.rgb2), 64, 0, Pool::Brick, Have::Color, Retain::Compact},
	{UFO_POOL_ARRAY(M.up_key), 1, 0, Pool::Upper, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.up_agg), 1, 0, Pool::Upper, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.up_stamp), 1, 0, Pool::Upper, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.up_child), 8, 0, Pool::Upper, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.up_valid), 1, 0, Pool::Upper, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.up_parent), 1, 0xff, Pool::Upper, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(d_list[0]), 1, 0, Pool::Upper, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(d_list[1]), 1, 0, Pool::Upper, Have::Always, Retain::Renew},
	{UFO_POOL_ARRAY(M.up_rgb), 1, 0, Pool::Upper, Have::Color, Retain::Renew},
	{UFO_POOL_ARRAY(M.up_child_rgb), 8, 0, Pool::Upper, Have::Color, Retain::Renew},
};
#undef UFO_POOL_ARRAY

uint32_t pool_cap(const Map* m, Pool pool) { return pool == Pool::Brick ? m->M.brick_cap : m->M.up_cap; }

// Replaces pool array `a` of old_cap bricks / nodes by one of new_cap (0: frees it).  The first
// `kept` entries come from the old array, entries 0..kept or, with `src`, entries src[0..kept); the
// others get the array's fill.  With `from` they come from that map's array instead (a copy on the
// same device).  With nothing to keep from the old array it goes first.
void reshape(Map* m, const PoolArray& a, uint32_t old_cap, uint32_t new_cap, uint32_t kept, const uint32_t* src,
             Map* from = nullptr)
{
	cudaStream_t s = m->stream;
	void*& p = *a.owner(m);
	const size_t per = a.per * a.elem;
	void* old = p;
	if (!kept || from) {
		p = nullptr;
		map_realloc(m, old, (size_t)old_cap * per, 0);
		old = nullptr;
	}
	const void* in = from ? *a.owner(from) : old;
	void* q = map_realloc(m, nullptr, 0, (size_t)new_cap * per);
	if (kept && src) launch_page_move<false>(m, q, in, src, kept, per);
	else if (kept) CK(cudaMemcpyAsync(q, in, (size_t)kept * per, cudaMemcpyDeviceToDevice, s));
	if (q) CK(cudaMemsetAsync(static_cast<uint8_t*>(q) + (size_t)kept * per, a.fill, (size_t)(new_cap - kept) * per, s));
	if (old) {
		CK(cudaStreamSynchronize(s));
		p = nullptr;
		map_realloc(m, old, (size_t)old_cap * per, 0);
	}
	p = q;
	m->M.chg_mask = m->chg_recording ? m->chg_mask : nullptr;  // K3 records through the view of its owner
}

// the missing arrays of `pool` that exist from `have` on, at the pool's capacity
void alloc_arrays(Map* m, Pool pool, Have have)
{
	for (const PoolArray& a : kPool)
		if (a.pool == pool && a.have == have && !*a.owner(m)) reshape(m, a, 0, pool_cap(m, pool), 0, nullptr);
}

// The existing arrays of `pool`: the per-block ones first, and of those the leaves, so that when a
// growth or a retain cannot hold one more leaf array it fails before anything has changed.  Every
// later array is smaller than what has been freed.
template <class F>
void each_array(Map* m, Pool pool, F&& f)
{
	for (const bool blocks : {true, false})
		for (const PoolArray& a : kPool)
			if (a.pool == pool && (a.per >= 64) == blocks && *a.owner(m)) f(a);
}

// The brick hash, sized for the pool's capacity and rebuilt from its first `live` bricks (which
// drops the kFailed entries a full pool leaves behind).
void brick_hash(Map* m, uint32_t live)
{
	DeviceMap& M = m->M;
	const uint32_t n = std::max(kMinHash, next_pow2(2ull * M.brick_cap));
	m->bh_tab.release(m);
	m->bh_tab.ensure(m, (size_t)n * sizeof(ulonglong2), 0xff);
	M.bh_tab = m->bh_tab.p;
	M.bh_mask = n - 1;
	if (live) k_rebuild_brick_hash<<<(live + 255) / 256, 256, 0, m->stream>>>(M, live);
}

// the upper-node hash, as brick_hash
void upper_hash(Map* m, uint32_t live)
{
	DeviceMap& M = m->M;
	const uint32_t n = std::max(kMinHash, next_pow2(2ull * M.up_cap));
	m->uh_keys.release(m);
	m->uh_vals.release(m);
	m->uh_keys.ensure(m, (size_t)n * sizeof(unsigned long long), 0xff);
	m->uh_vals.ensure(m, (size_t)n * sizeof(uint32_t), 0xff);
	M.uh_keys = m->uh_keys.p;
	M.uh_vals = m->uh_vals.p;
	M.uh_mask = n - 1;
	if (live) k_rebuild_upper_hash<<<(live + 255) / 256, 256, 0, m->stream>>>(M, live);
}

void alloc_pools(Map* m, uint32_t brick_cap, uint32_t up_cap)
{
	m->M.brick_cap = brick_cap;
	m->M.up_cap = up_cap;
	brick_hash(m, 0);
	alloc_arrays(m, Pool::Brick, Have::Always);
	upper_hash(m, 0);
	alloc_arrays(m, Pool::Upper, Have::Always);
	if (m->M.color) {
		alloc_arrays(m, Pool::Upper, Have::Color);
		alloc_arrays(m, Pool::Brick, Have::Color);
	}
	m->ctr.ensure(m, sizeof(Counters), 0);
	m->M.ctr = m->ctr.p;
}

// the pool arrays; the map's DevMems go with the map
void free_pools(Map* m)
{
	for (const PoolArray& a : kPool)
		if (*a.owner(m)) reshape(m, a, pool_cap(m, a.pool), 0, 0, nullptr);
}

// `touched`: entries of the touched list to keep (the first scan's, when the second of a pair marks)
void push_counters(Map* m, uint32_t touched = 0)
{
	// host view -> device allocation counters, clears the per-scan part
	Counters c{};
	c.n_touched = touched;
	c.n_blocks = m->n_blocks;
	c.n_bricks = m->n_bricks;
	c.n_upper = m->n_upper;
	for (int i = 0; i < 3; ++i) {
		c.bbox[i] = ~0ull;
		c.bbox[3 + i] = 0ull;
	}
	*m->h_ctr = c;
	CK(cudaMemcpyAsync(m->M.ctr, m->h_ctr, sizeof(Counters), cudaMemcpyHostToDevice, m->stream));
	m->k3_counted = false;
}

// grow whichever pool overflowed; `want_*` are the allocation counters the failed
// run reached (an over-estimate of the need)
void grow_pools(Map* m, uint32_t overflow, uint32_t want_bricks, uint32_t want_upper)
{
	DeviceMap& M = m->M;
	CK(cudaStreamSynchronize(m->stream));
	auto grow = [&](Pool pool, uint32_t oc, uint32_t nc) {
		each_array(m, pool, [&](const PoolArray& a) { reshape(m, a, oc, nc, oc, nullptr); });
	};
	if (overflow & 2u) {
		uint32_t oc = M.brick_cap;
		// marking stops creating bricks once the pool is exhausted, so `want` is barely above the old
		// capacity: small pools grow by 4x, large ones by 2x
		uint32_t nc = (uint32_t)std::max<uint64_t>((oc < (1u << 18) ? 4ull : 2ull) * oc, (uint64_t)want_bricks + want_bricks / 4);
		if ((uint64_t)nc * 64 > 0xfffffff0ull) throw std::bad_alloc();
		grow(Pool::Brick, oc, nc);
		M.brick_cap = nc;
		brick_hash(m, std::min(m->h_ctr->n_bricks, oc));
		if (M.up_cap < nc / 2) overflow |= 4u;  // keep the upper-node pool in proportion
	}
	if (overflow & 4u) {
		uint32_t oc = M.up_cap;
		uint32_t nc = (uint32_t)std::max<uint64_t>(std::max<uint64_t>(2ull * oc, M.brick_cap / 2), (uint64_t)want_upper + want_upper / 4);
		grow(Pool::Upper, oc, nc);
		M.up_cap = nc;
		upper_hash(m, std::min(m->h_ctr->n_upper, oc));
	}
	// a pass that continues after the growth (the routed mark and apply phases) reads its masks
	// through mask_base, which points into the old miss_mask unless the pass marks into the volume
	M.mask_base = M.dense ? M.vol : M.miss_mask;
	CK(cudaGetLastError());
}

// The host takes the device's brick and upper-node counts, also after a pass that a full pool cut
// short: grow_pools rebuilds the hashes from these slots, so a repeated attempt must not hand them
// out again.
void keep_created(Map* m)
{
	m->n_bricks = std::min(m->h_ctr->n_bricks, m->M.brick_cap);
	m->n_upper = std::min(m->h_ctr->n_upper, m->M.up_cap);
}

// A new scan id (brick stamps) and a new upper-node epoch (up_stamp).  Neither is ever 0: the
// stamps are cleared to 0, and an id of 0 would make every brick or node look already listed.
void new_scan_id(Map* m) { if (++m->M.scan_id == 0) m->M.scan_id = 1; }
void new_up_epoch(Map* m) { if (++m->M.up_epoch == 0) m->M.up_epoch = 1; }
// Every call that writes the pools or the thresholds: a tree shape kept for the nearest search is stale
// from here on.
void bump_revision(Map* m) { ++m->revision; }

// depth 3 / 4 of the touched bricks from their blocks
void launch_brick_agg(Map* m)
{
	if (m->M.color) k_brick_agg<true><<<m->sm_count * 4, 256, 0, m->stream>>>(m->M);
	else k_brick_agg<false><<<m->sm_count * 4, 256, 0, m->stream>>>(m->M);
}

// every derived value of the touched bricks (depth 1 to 4) from their leaves
void launch_leaf_refresh(Map* m)
{
	k_import_refresh<<<m->sm_count * 8, 256, 0, m->stream>>>(m->M);
	launch_brick_agg(m);
}

// Runs a pass whose kernels find or create bricks and upper nodes, growing the pools until it
// completes; `attempt` enqueues the pass's kernels.  Creation is idempotent, so a pass that ran
// into a full pool is repeated as a whole, keeping what the failed attempt created.  Leaves the
// final counts in m->n_bricks and m->n_upper.
template <class F>
int run_growing(Map* m, const char* what, F&& attempt)
{
	for (int k = 0;; ++k) {
		push_counters(m);
		attempt();
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(m->h_ctr, m->M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, m->stream));
		CK(cudaStreamSynchronize(m->stream));
		keep_created(m);
		const uint32_t ov = m->h_ctr->overflow;
		if (!ov) return UFO_B200_OK;
		if (ov & ~6u) {
			m->set_error("%s: internal error (overflow flags %u)", what, ov);
			return UFO_B200_E_NOMEM;
		}
		if (k > 16) {
			m->set_error("%s: device pools keep overflowing", what);
			return UFO_B200_E_NOMEM;
		}
		grow_pools(m, ov, m->h_ctr->n_bricks, m->h_ctr->n_upper);
	}
}

size_t layout_stride(int layout)
{
	switch (layout) {
		case UFO_B200_XYZ_F64: return 24;
		case UFO_B200_XYZ_F32: return 12;
		case UFO_B200_XYZRGB_F64: return 32;
		case UFO_B200_XYZRGB_F32: return 16;
		default: return 0;
	}
}

// called with the stream idle
void ensure_scan_buffers(Map* m, size_t n, bool need_table, bool records, bool fused)
{
	DevMem<uint32_t>* batch_bufs[] = {&m->d_seg_base, &m->d_seg_count, &m->d_order};
	if (n > m->ray_cap) {
		const size_t cap = std::max<size_t>(n, 1024);
		m->d_ray_end.ensure(m, cap * 3 * sizeof(double), 0);
		m->d_hit_tab.ensure(m, cap * sizeof(uint32_t), 0xff);
		for (auto* b : batch_bufs) b->release(m);
		m->ray_cap = cap;
	}
	if (records)
		for (auto* b : batch_bufs) b->ensure(m, (m->ray_cap / 32 + 1) * sizeof(uint32_t), 0);
	if (fused && m->item_cap < m->ray_cap) {
		const size_t cap = m->ray_cap;
		m->d_items.ensure(m, cap * kShells * sizeof(Item), -1);  // written before read
		m->d_vmask.ensure(m, (cap / 32 + 1) * kShells * sizeof(uint32_t), 0);
		m->d_rc.ensure(m, cap * sizeof(RayConst), 0);
		m->item_cap = cap;
	}
	if (need_table) {
		uint32_t want = std::max(1u << 12, next_pow2(4ull * n));
		if (want > m->tab_size) {
			m->d_tab_keys.ensure(m, (size_t)want * sizeof(unsigned long long), 0xff);
			m->d_tab_min.ensure(m, (size_t)want * sizeof(uint32_t), 0xff);
			m->tab_size = want;
		}
	}
}

// K3's counters of one scan: statistics slots [lo, hi) (a paired pass counts its scans apart)
void update_counts(Map* m, ufo_b200_scan_stats& st, const Counters& c, int lo, int hi, unsigned long long upper)
{
	unsigned long long sum[8] = {0, 0, 0, 0, 0, 0, 0, 0};
	for (int sl = lo; sl < hi; ++sl)
		for (int k = 0; k < 8; ++k) sum[k] += c.stat[sl][k];
	st.touched_voxels = sum[0];
	st.hit_voxels = sum[1];
	st.touched_octets = sum[2];
	st.touched_blocks = sum[3];
	st.touched_d3 = sum[6];
	st.touched_bricks = sum[5];
	st.touched_lines = sum[7];
	st.upper_nodes = upper;
	m->n_blocks += (uint32_t)sum[4];
	st.blocks_in_map = m->n_blocks;
}

// the change box of a scan whose counters are in c
void fold_bbox(Map* m, const Counters& c)
{
	for (int i = 0; i < 3; ++i) {
		if (c.bbox[i] != ~0ull) m->min_change[i] = std::min(m->min_change[i], decode_ordered(c.bbox[i]));
		if (c.bbox[3 + i] != 0ull) m->max_change[i] = std::max(m->max_change[i], decode_ordered(c.bbox[3 + i]));
	}
}

// event times of a scan's marking (profiling level 1 and up)
void marking_times(Map* m, ufo_b200_scan_stats& st)
{
	cudaEventElapsedTime(&st.ms_points, m->ev[0], m->ev[2]);
	if (m->ev7_valid) {
		cudaEventElapsedTime(&st.ms_rays, m->ev[2], m->ev[7]);
		cudaEventElapsedTime(&st.ms_scatter, m->ev[7], m->ev[3]);
	} else {
		cudaEventElapsedTime(&st.ms_rays, m->ev[2], m->ev[3]);
	}
}

void finish_stats(Map* m)
{
	// called after the stream is idle and h_ctr holds the end-of-scan counters
	if (!m->stats_pending) return;
	const Counters& c = *m->h_ctr;
	ufo_b200_scan_stats& st = m->stats;
	st.rays = c.n_rays;
	st.visits = c.visits;
	m->walk_stats = ufo_b200_walk_stats{c.walk_records, c.walk_mask_reds, c.walk_words, c.walk_dirty_reds};
	m->update_stats = ufo_b200_update_stats{};
	if (m->k3_counted) {
		K3Stats h;
		if (cudaMemcpy(&h, m->k3_stat.p, sizeof(h), cudaMemcpyDeviceToHost) == cudaSuccess) {
			unsigned long long k3[3] = {0, 0, 0};
			for (int sl = 0; sl < kStatSlots; ++sl)
				for (int k = 0; k < 3; ++k) k3[k] += h.slot[sl][k];
			m->update_stats = ufo_b200_update_stats{k3[0], k3[1], k3[2]};
		}
	}
	m->early_stats = ufo_b200_early_stats{};
	if (m->early_pass) {
		ufo_b200_early_stats& es = m->early_stats;
		es.rounds = c.e_rounds;
		es.converged = c.e_converged;
		es.visits = c.e_visits;
		es.nodes = c.e_nodes;
		es.free_nodes = c.e_free;
		es.table_bytes = m->d_e_keys.bytes + m->d_e_first.bytes;
		es.id_bytes = m->d_e_ids.bytes + m->d_e_cnt.bytes + m->d_e_off.bytes + m->d_e_plen.bytes + m->d_e_pnext.bytes;
		if (m->ev_valid && m->profiling) {
			cudaEventElapsedTime(&es.ms_walk, m->ev[2], m->ev[1]);
			cudaEventElapsedTime(&es.ms_rounds, m->ev[1], m->ev[4]);
			cudaEventElapsedTime(&es.ms_mark, m->ev[4], m->ev[3]);
		}
	}
	if (m->paired) {
		update_counts(m, m->first_stats, c, 0, kStatSlots / 2, c.upper_pair[0]);
		update_counts(m, st, c, kStatSlots / 2, kStatSlots, c.upper_pair[1]);
	} else {
		update_counts(m, st, c, 0, kStatSlots, c.upper_nodes);
	}
	m->n_bricks = std::min(c.n_bricks, m->M.brick_cap);
	m->n_upper = std::min(c.n_upper, m->M.up_cap);
	st.bricks_in_map = m->n_bricks;
	st.device_bytes = m->device_bytes;
	if (c.n_rays || st.touched_voxels) fold_bbox(m, c);
	if (m->ev_valid) {
		cudaEventElapsedTime(&st.ms_total, m->ev[0], m->ev[6]);
		if (m->pending.flushed) {
			// device time of a deferred scan: its marking and its leaf update, not the wait between
			float mark = 0.0f, update = 0.0f;
			cudaEventElapsedTime(&mark, m->ev[0], m->ev[9]);
			cudaEventElapsedTime(&update, m->ev[8], m->ev[6]);
			st.ms_total = mark + update;
		}
		if (m->h2d_valid) cudaEventElapsedTime(&st.ms_h2d, m->ev_copy0, m->ev_copied);
		if (m->write_pass) {
			cudaEventElapsedTime(&st.ms_update, m->ev[3], m->ev[5]);
			cudaEventElapsedTime(&st.ms_propagate, m->ev[5], m->ev[6]);
		} else if (m->profiling) {
			marking_times(m, st);
			cudaEventElapsedTime(&st.ms_update, m->ev[8], m->ev[5]);
			cudaEventElapsedTime(&st.ms_propagate, m->ev[5], m->ev[6]);
		}
	}
	m->stats_pending = false;
}

void ensure_seg(Map* m, unsigned long long want)
{
	if (want <= m->seg_cap) return;
	CK(cudaStreamSynchronize(m->stream));
	m->d_seg.ensure(m, want * sizeof(QEntry), -1);
	m->seg_cap = want;
}

// K3 over the scan's touched list: persistent warps, the list length is read on the device.
// pair: the touched list of a paired pass (mono maps, scans only)
void launch_update(Map* m, float miss, bool set_mode = false, bool pair = false)
{
	CK(cudaMemsetAsync(&m->M.ctr->k3_cursor, 0, sizeof(uint32_t), m->stream));
	m->M.k3_stat = nullptr;
	if (m->profiling >= 2) {
		m->k3_stat.ensure(m, sizeof(K3Stats), 0);
		if (!m->k3_counted) CK(cudaMemsetAsync(m->k3_stat.p, 0, sizeof(K3Stats), m->stream));
		m->k3_counted = true;
		m->M.k3_stat = m->k3_stat.p;
	}
	if (m->M.color) {
		const uint32_t per_sm = UbShape<true>::kMinBlocks, T = UbShape<true>::kWarps * 32;
		const uint32_t grid = (uint32_t)m->sm_count * (m->k3_blocks ? std::min<uint32_t>(per_sm, (uint32_t)m->k3_blocks) : per_sm);
		if (set_mode) k_update_brick<true, true><<<grid, T, 0, m->stream>>>(m->M, miss);
		else k_update_brick<true, false><<<grid, T, 0, m->stream>>>(m->M, miss);
	} else {
		const uint32_t per_sm = UbShape<false>::kMinBlocks, T = UbShape<false>::kWarps * 32;
		const uint32_t grid = (uint32_t)m->sm_count * (m->k3_blocks ? std::min<uint32_t>(per_sm, (uint32_t)m->k3_blocks) : per_sm);
		if (set_mode) k_update_brick<false, true><<<grid, T, 0, m->stream>>>(m->M, miss);
		else if (pair) k_update_brick<false, false, true><<<grid, T, 0, m->stream>>>(m->M, miss);
		else k_update_brick<false, false><<<grid, T, 0, m->stream>>>(m->M, miss);
	}
	++m->launches;
}

// generic marking path: walk -> (block, mask) records -> k_scatter.  Handles every insert depth,
// out-of-tree keys and the fixed-step variant.
void launch_rays_records(Map* m, const ScanArgs& a, int simple)
{
	if (simple) {
		k_rays_simple<<<(a.n + 127) / 128, 128, 0, m->stream>>>(m->M, a);
		++m->launches;
		if (a.depth >= 5) {
			k_expand_nodes<<<m->sm_count * 8, 256, 0, m->stream>>>(m->M, a);
			++m->launches;
		}
		return;
	}
	// one resident wave; batches are ordered by work and dealt round-robin over the CTAs
	uint32_t* counter = &m->M.ctr->ray_batch;
	uint32_t n_batches = (a.n + 31) / 32;
	k_order_batches<<<1, 1024, 0, m->stream>>>(a.seg_count, n_batches, a.order);
	++m->launches;
	uint32_t need = (a.n + kRayThreads - 1) / kRayThreads;
	uint32_t grid = std::min<uint32_t>(need, (uint32_t)m->sm_count * m->ray_blocks_per_sm);
	if (a.count_visits) {
		if (a.depth == 0) k_rays<0, true><<<grid, kRayThreads, 0, m->stream>>>(m->M, a, counter);
		else if (a.depth == 1) k_rays<1, true><<<grid, kRayThreads, 0, m->stream>>>(m->M, a, counter);
		else k_rays<2, true><<<grid, kRayThreads, 0, m->stream>>>(m->M, a, counter);
	} else {
		if (a.depth == 0) k_rays<0, false><<<grid, kRayThreads, 0, m->stream>>>(m->M, a, counter);
		else if (a.depth == 1) k_rays<1, false><<<grid, kRayThreads, 0, m->stream>>>(m->M, a, counter);
		else k_rays<2, false><<<grid, kRayThreads, 0, m->stream>>>(m->M, a, counter);
	}
	++m->launches;
	if (m->profiling) {
		CK(cudaEventRecord(m->ev[7], m->stream));
		m->ev7_valid = true;
	}
	{
		// all CTAs resident, looping over the work items (j, region) with stride = grid size.
		// The grid size is made coprime with the number of regions so that every CTA walks
		// through ALL regions: region length correlates with the region index (ring order of
		// the sensor), and a stride sharing a factor with it gives some CTAs only long regions.
		uint32_t sgrid = (uint32_t)m->sm_count * 8;
		const uint32_t n_regions = (a.n + 31) / 32;
		while (sgrid > 1 && std::gcd(sgrid, n_regions) != 1) --sgrid;
		const bool generic = a.depth >= 3 || m->M.alias_miss, shard = m->M.shard_world > 1;
		if (generic && shard) k_scatter<true, true><<<sgrid, kChunk, 0, m->stream>>>(m->M, a);
		else if (generic) k_scatter<true, false><<<sgrid, kChunk, 0, m->stream>>>(m->M, a);
		else if (shard) k_scatter<false, true><<<sgrid, kChunk, 0, m->stream>>>(m->M, a);
		else k_scatter<false, false><<<sgrid, kChunk, 0, m->stream>>>(m->M, a);
	}
	++m->launches;
	if (a.depth >= 5) {
		k_expand_nodes<<<m->sm_count * 8, 256, 0, m->stream>>>(m->M, a);
		++m->launches;
	}
}

template <int DEPTH, bool DENSE>
void launch_fused_depth(Map* m, const ScanArgs& a)
{
	cudaStream_t s = m->stream;
	const uint32_t n_batches = (a.n + 31) / 32;
	const uint32_t sgrid = (n_batches * 32 + 127) / 128;
	if (a.count_visits) k_split<DEPTH, true><<<sgrid, 128, 0, s>>>(m->M, a);
	else k_split<DEPTH, false><<<sgrid, 128, 0, s>>>(m->M, a);
	const uint32_t grid = (uint32_t)m->sm_count * m->walk_blocks_per_sm;
	const bool shard = m->M.shard_world > 1 && !DENSE;  // dense: ownership is applied by k_gather
	if (a.count_visits) {
		if (shard) k_walk_mark<DEPTH, true, true, DENSE><<<grid, kWalkThreads, 0, s>>>(m->M, a);
		else k_walk_mark<DEPTH, false, true, DENSE><<<grid, kWalkThreads, 0, s>>>(m->M, a);
	} else {
		if (shard) k_walk_mark<DEPTH, true, false, DENSE><<<grid, kWalkThreads, 0, s>>>(m->M, a);
		else k_walk_mark<DEPTH, false, false, DENSE><<<grid, kWalkThreads, 0, s>>>(m->M, a);
	}
	m->launches += 2;
	if (DENSE) {
		if (m->profiling) {
			CK(cudaEventRecord(m->ev[7], s));
			m->ev7_valid = true;
		}
		k_gather_scan<<<m->sm_count * 2, 256, 0, s>>>(m->M);
		if (m->M.shard_world > 1) k_gather<true><<<m->sm_count * 8, 256, 0, s>>>(m->M);
		else k_gather<false><<<m->sm_count * 8, 256, 0, s>>>(m->M);
		m->launches += 2;
	}
}

// fused path (ufo_walk.cuh): insert depth <= 2, no out-of-tree keys seen by this map
void launch_rays_fused(Map* m, const ScanArgs& a)
{
	if (m->M.dense) {
		if (a.depth == 0) launch_fused_depth<0, true>(m, a);
		else if (a.depth == 1) launch_fused_depth<1, true>(m, a);
		else launch_fused_depth<2, true>(m, a);
	} else {
		if (a.depth == 0) launch_fused_depth<0, false>(m, a);
		else if (a.depth == 1) launch_fused_depth<1, false>(m, a);
		else launch_fused_depth<2, false>(m, a);
	}
}

bool use_fused(const Map* m, const PendingScan& p)
{
	return !p.has_vol && !p.simple && !p.early && p.a.depth <= 2 && !m->M.alias_miss && !m->force_records;
}

// Dense scan volume: bricks per axis a scan of this range needs around the sensor (0: no volume)
uint32_t volume_bricks(const Map* m, const PendingScan& p)
{
	if (m->no_dense || !(p.a.max_range > 0)) return 0;
	const double vox = p.a.max_range * m->M.g.resolution_factor + 4.0;  // ray length in voxels + slack
	if (vox > 16.0 * 160) return 0;  // > 320 bricks per axis (16.8 GB of masks): use the hash path
	const uint32_t half = (uint32_t)(vox / 16.0) + 2;
	return 2 * half + 1;
}

// empties the dense scan volume: its masks and the dirty bitmap
void wipe_volume(Map* m)
{
	if (!m->vol.p) return;
	CK(cudaMemsetAsync(m->vol.p, 0, m->vol.bytes, m->stream));
	CK(cudaMemsetAsync(m->vol_dirty.p, 0, m->vol_dirty.bytes, m->stream));
}

// Second dense volume of a paired pass, for db bricks per axis; false (and no pairs from then on)
// when it cannot be allocated.  Called with the stream idle.
bool ensure_volume2(Map* m, uint32_t db)
{
	if (db <= m->vol2_db_cap) return true;
	const size_t nb = (size_t)db * db * db;
	try {
		m->vol2.ensure(m, nb * 64 * sizeof(unsigned long long), 0);
		m->vol2_dirty.ensure(m, (nb / 64 + 1) * sizeof(unsigned long long), 0);
		m->vol2_list.ensure(m, (nb / 64 + 1) * sizeof(uint32_t), 0);
	} catch (CudaError&) {
		cudaGetLastError();  // an allocation failure is not sticky
		m->vol2.release(m);
		m->vol2_dirty.release(m);
		m->vol2_list.release(m);
		m->vol2_db_cap = 0;
		m->no_pair = true;
		return false;
	}
	m->vol2_db_cap = db;
	return true;
}

// empties the second dense volume and the second hit masks
void wipe_volume2(Map* m)
{
	if (m->vol2.p) {
		CK(cudaMemsetAsync(m->vol2.p, 0, m->vol2.bytes, m->stream));
		CK(cudaMemsetAsync(m->vol2_dirty.p, 0, m->vol2_dirty.bytes, m->stream));
	}
	CK(cudaMemsetAsync(m->M.hit_mask2, 0, (size_t)m->M.brick_cap * 64 * sizeof(unsigned long long), m->stream));
}

// While the second scan of a pair marks, the marking kernels see its volume and hit masks in place of
// the first's; restored when the object goes.
struct SecondMarks {
	Map* m;
	unsigned long long *vol, *dirty;
	uint32_t* list;
	explicit SecondMarks(Map* m_) : m(m_), vol(m_->M.vol), dirty(m_->M.vol_dirty), list(m_->M.vol_list)
	{
		DeviceMap& M = m->M;
		M.vol = m->vol2.p;
		M.vol_dirty = m->vol2_dirty.p;
		M.vol_list = m->vol2_list.p;
		std::swap(M.hit_mask, M.hit_mask2);
		M.pair_id = m->first_id;
	}
	~SecondMarks()
	{
		DeviceMap& M = m->M;
		M.vol = vol;
		M.vol_dirty = dirty;
		M.vol_list = list;
		std::swap(M.hit_mask, M.hit_mask2);
		M.pair_id = 0;
	}
};

// called with the stream idle; binds the volume to this scan's sensor position (the second volume
// has been allocated by ensure_volume2)
void setup_volume(Map* m, PendingScan& p, uint32_t db, bool second = false)
{
	DeviceMap& M = m->M;
	if (!second && db > m->vol_db_cap) {
		const size_t nb = (size_t)db * db * db;
		m->vol.ensure(m, nb * 64 * sizeof(unsigned long long), 0);
		m->vol_dirty.ensure(m, (nb / 64 + 1) * sizeof(unsigned long long), 0);
		m->vol_list.ensure(m, (nb / 64 + 1) * sizeof(uint32_t), 0);
		M.vol = m->vol.p;
		M.vol_dirty = m->vol_dirty.p;
		M.vol_list = m->vol_list.p;
		m->vol_db_cap = db;
	}
	const Geometry& g = M.g;
	const uint32_t half = (db - 1) / 2;
	const Key3 ko = point_to_key(g, p.a.origin, 0);
	M.vol_db = db;
	M.vol_g0x = ((ko.x & 0x1fffffu) >> 4) - half;
	M.vol_g0y = ((ko.y & 0x1fffffu) >> 4) - half;
	M.vol_g0z = ((ko.z & 0x1fffffu) >> 4) - half;
}

// K4: upper levels, depth 5 .. L, from the touched list
void launch_upper_seed(Map* m)
{
	DeviceMap& M = m->M;
	if (M.g.depth_levels < 5) return;
	// list_count[] is zero when the first seed of a pass runs; level d reads list d&1 ? 0 : 1
	k_upper_seed<<<m->sm_count * 2, 256, 0, m->stream>>>(M, m->d_list[0], M.up_cap);
	++m->launches;
}

void launch_upper_levels(Map* m)
{
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	if (M.g.depth_levels < 5) return;
	const uint32_t L = M.g.depth_levels;
	for (uint32_t d = 5; d <= std::min(6u, L); ++d) {
		k_upper_level<<<m->sm_count, 256, 0, s>>>(M, d, m->d_list[(d & 1) ? 0 : 1], m->d_list[(d & 1) ? 1 : 0], M.up_cap);
		++m->launches;
	}
	if (L >= 7) {
		k_upper_tail<<<1, 1024, 0, s>>>(M, 7, m->d_list[0], m->d_list[1], M.up_cap);
		++m->launches;
	}
	CK(cudaGetLastError());
}

void launch_upper(Map* m)
{
	launch_upper_seed(m);
	launch_upper_levels(m);
}

__global__ void k_reset_upper_pass(Counters* c, uint32_t n_upper)
{
	c->overflow = 0;
	c->list_count[0] = c->list_count[1] = c->list_count[2] = 0;
	c->upper_nodes = 0;
	c->upper_pair[0] = c->upper_pair[1] = 0;
	c->n_upper = n_upper;
}

// Early-stopping buffers (ufo_early.cuh) for n rays and `visits` walk visits; called with the stream
// idle.  The node table stays below 80 % load (distinct nodes <= visits, plus one end node per ray of
// a discrete scan) and every scan leaves it empty (E3 clears the slots it reads), so it is only
// cleared when it is allocated.
void ensure_early(Map* m, size_t n, unsigned long long visits)
{
	if (n + 1 > m->e_ray_cap) {
		const size_t cap = std::max<size_t>(n + 1, 1024);
		m->d_e_cnt.ensure(m, cap * sizeof(unsigned long long), 0);
		m->d_e_off.ensure(m, cap * sizeof(unsigned long long), 0);
		m->d_e_plen.ensure(m, cap * sizeof(uint32_t), 0);
		m->d_e_pnext.ensure(m, cap * sizeof(uint32_t), 0);
		m->e_ray_cap = cap;
	}
	if (visits > m->e_id_cap) {
		m->d_e_ids.ensure(m, (visits + visits / 8) * sizeof(uint32_t), -1);  // written before read
		m->e_id_cap = visits + visits / 8;
	}
	const unsigned long long need = std::max<unsigned long long>(visits + visits / 4 + n + 1, 2ull * (n + 1));
	if (need > m->e_tab_cap) {
		if (need > (1ull << 31)) throw std::bad_alloc();
		const size_t cap = next_pow2(need);
		m->d_e_keys.ensure(m, cap * sizeof(unsigned long long), 0xff);
		m->d_e_first.ensure(m, cap * sizeof(uint32_t), 0xff);
		m->e_tab_cap = cap;
	}
	size_t tmp = 0;
	CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp, m->d_e_cnt.p, m->d_e_off.p, (int)(n + 1), m->stream));
	ensure_spare(m, m->d_e_tmp, tmp, 1 << 12);
}

// E1-E3 (ufo_early.cuh): the scan's free set under early stopping, marked like the record path
// marks it.  The rounds run in one cooperative kernel, so nothing here waits for the device.
void launch_early(Map* m, const PendingScan& p)
{
	const ScanArgs& a = p.a;
	cudaStream_t s = m->stream;
	EarlyArgs e{};
	e.stop = p.early;
	e.simple = p.simple ? 1 : 0;
	e.keys = m->d_e_keys.p;
	e.first = m->d_e_first.p;
	e.tab_mask = (uint32_t)(m->e_tab_cap - 1);
	e.cnt = m->d_e_cnt.p;
	e.off = m->d_e_off.p;
	e.ids = m->d_e_ids.p;
	e.id_cap = m->e_id_cap;
	e.plen = m->d_e_plen.p;
	e.pnext = m->d_e_pnext.p;
	uint32_t n = a.n;
	if (a.discrete) {
		k_early_rank<<<(n + kEarlyThreads - 1) / kEarlyThreads, kEarlyThreads, 0, s>>>(m->M, a, e);
		k_early_place<<<(n + kEarlyThreads - 1) / kEarlyThreads, kEarlyThreads, 0, s>>>(m->M, a, e);
		m->launches += 2;
	}
	k_early_count<<<(n + kEarlyThreads) / kEarlyThreads, kEarlyThreads, 0, s>>>(m->M, a, e);  // n + 1 threads
	size_t tmp = m->d_e_tmp.bytes;
	CK(cub::DeviceScan::ExclusiveSum(m->d_e_tmp.p, tmp, e.cnt, e.off, (int)(n + 1), s));
	k_early_check<<<1, 1, 0, s>>>(m->M, e, n);
	k_early_fill<<<(n + kEarlyThreads - 1) / kEarlyThreads, kEarlyThreads, 0, s>>>(m->M, a, e);
	if (m->profiling) CK(cudaEventRecord(m->ev[1], s));
	{
		DeviceMap M = m->M;
		void* args[] = {&M, &e, &n};
		CK(cudaLaunchCooperativeKernel((const void*)k_early_rounds, dim3((unsigned)(m->sm_count * m->early_blocks_per_sm)),
		                               dim3(kEarlyThreads), args, 0, s));
	}
	if (m->profiling) CK(cudaEventRecord(m->ev[4], s));
	const uint32_t grid = (uint32_t)m->sm_count * 8;
	if (a.depth == 0) k_early_mark<0><<<grid, kEarlyThreads, 0, s>>>(m->M, a, e);
	else if (a.depth == 1) k_early_mark<1><<<grid, kEarlyThreads, 0, s>>>(m->M, a, e);
	else if (a.depth == 2) k_early_mark<2><<<grid, kEarlyThreads, 0, s>>>(m->M, a, e);
	else if (a.depth <= 4) k_early_mark<3><<<grid, kEarlyThreads, 0, s>>>(m->M, a, e);
	else k_early_mark<5><<<grid, kEarlyThreads, 0, s>>>(m->M, a, e);
	m->launches += 5;  // the scan's own launches not counted
	if (a.depth >= 5) {
		k_expand_nodes<<<m->sm_count * 8, 256, 0, s>>>(m->M, a);
		++m->launches;
	}
}

// Enqueues one write batch (ufo_write.cuh): expand -> sort -> segments -> apply -> aggregates.
// Called with the stream idle.  If a pool overflows while expanding, every later kernel backs off
// and finalize_scan() grows the pool and enqueues the whole batch again: no leaf was written, and
// finding or creating a brick twice is harmless, so every update is applied exactly once.
void enqueue_write(Map* m, PendingScan& p)
{
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	WriteArgs a = p.w;
	new_scan_id(m);
	new_up_epoch(m);
	M.dense = 0;
	M.mask_base = M.miss_mask;
	ensure_spare(m, m->d_w_seg, (size_t)M.brick_cap * 3 * sizeof(uint32_t), 1 << 12);
	a.seg_begin = m->d_w_seg.p;
	a.seg_end = m->d_w_seg.p + M.brick_cap;
	a.seg_list = m->d_w_seg.p + 2 * (size_t)M.brick_cap;
	// keys: brick slot << 32 | sequence number; only the bits a slot below brick_cap can use are sorted
	int end_bit = 32;
	while (end_bit < 64 && (1ull << (end_bit - 32)) <= M.brick_cap) ++end_bit;
	size_t tmp_bytes = 0;
	CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, m->d_w_keys[0].p, m->d_w_keys[1].p, m->d_w_idx[0].p,
	                                   m->d_w_idx[1].p, (int)a.n_rec, 0, end_bit, s));
	ensure_spare(m, m->d_w_tmp, tmp_bytes, 1 << 12);
	push_counters(m);
	a.keys = m->d_w_keys[0].p;
	a.idx = m->d_w_idx[0].p;
	a.recs = m->d_w_recs.p;
	if (a.n) k_write_expand<<<(a.n + 127) / 128, 128, 0, s>>>(M, a);
	tmp_bytes = m->d_w_tmp.bytes;
	CK(cub::DeviceRadixSort::SortPairs(m->d_w_tmp.p, tmp_bytes, m->d_w_keys[0].p, m->d_w_keys[1].p, m->d_w_idx[0].p,
	                                   m->d_w_idx[1].p, (int)a.n_rec, 0, end_bit, s));
	a.keys = m->d_w_keys[1].p;
	a.idx = m->d_w_idx[1].p;
	k_write_segments<<<m->sm_count * 8, 256, 0, s>>>(M, a);
	CK(cudaEventRecord(m->ev[3], s));
	if (a.rgb) k_write_apply<true><<<m->sm_count * 16, 64, 0, s>>>(M, a);
	else k_write_apply<false><<<m->sm_count * 16, 64, 0, s>>>(M, a);
	CK(cudaEventRecord(m->ev[5], s));
	launch_leaf_refresh(m);
	m->launches += 6;  // the sort's own launches not counted
	launch_upper(m);
	CK(cudaGetLastError());
	CK(cudaEventRecord(m->ev[6], s));
	m->ev_valid = true;
	m->write_pass = true;
	CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
	m->stats_pending = true;
	p.valid = true;
}

// (re-)binds the scan buffers to the scan's arguments: they may have been regrown since the scan
// was first enqueued
void bind_scan_buffers(Map* m, PendingScan& p, bool fused)
{
	ScanArgs& a = p.a;
	a.ray_end = m->d_ray_end.p;
	a.tab_keys = m->d_tab_keys.p;
	a.tab_min = m->d_tab_min.p;
	a.tab_mask = m->tab_size ? m->tab_size - 1 : 0;
	a.hit_tab = p.use_color ? m->d_hit_tab.p : nullptr;
	a.seg = nullptr;
	a.seg_base = a.seg_count = a.order = nullptr;
	a.items = nullptr;
	if (fused) {
		a.items = m->d_items.p;
		a.item_stride = m->item_cap;
		a.vmask = m->d_vmask.p;
		a.rc = m->d_rc.p;
	} else if (!p.simple && !p.has_vol && !p.early) {
		a.seg = m->d_seg.p;
		a.seg_cap = m->seg_cap;
		a.seg_base = m->d_seg_base.p;
		a.seg_count = m->d_seg_count.p;
		a.order = m->d_order.p;
	}
	if (a.depth >= 5) {
		m->d_nodes.ensure(m, sizeof(unsigned long long) << 20, 0);
		a.nodes = m->d_nodes.p;
		a.nodes_cap = 1u << 20;
	}
}

// The upper levels of a pass and, for a paired pass, each scan's count of them (k_upper_count)
void launch_upper_pass(Map* m)
{
	launch_upper(m);
	if (!m->paired || m->M.g.depth_levels < 5) return;
	for (uint32_t k = 0; k < 2; ++k) {
		new_up_epoch(m);
		k_upper_count<<<m->sm_count * 2, 256, 0, m->stream>>>(m->M, k, m->M.up_epoch);
		++m->launches;
	}
}

// K3 and K4 of an enqueued scan (of both scans of a paired pass) and the read-back of the counters
void enqueue_update(Map* m, PendingScan& p)
{
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	const ScanArgs& a = p.a;
	CK(cudaEventRecord(m->ev[8], s));
	// K3 and K4 run off the device-side touched list; if a pool overflowed while marking they
	// back off by themselves and the scan is repeated by finalize_scan() after the growth.
	const bool aliases = M.alias_miss != nullptr;
	const uint32_t agrid = (uint32_t)m->sm_count * 4;
	if (aliases) {
		k_alias_apply<<<agrid, 256, 0, s>>>(M, M.hit, 1);
		++m->launches;
	}
	if (m->paired) {
		M.mask_base2 = m->vol2.p;
		M.pair_id = m->first_id;
	}
	launch_update(m, p.has_vol ? p.set_value : a.miss, p.has_vol, m->paired);
	M.pair_id = 0;
	if (aliases) {
		k_alias_apply<<<agrid, 256, 0, s>>>(M, a.miss, 0);
		k_alias_refresh<<<agrid, 256, 0, s>>>(M);
		launch_brick_agg(m);
		m->launches += 3;
	}
	if (m->profiling) CK(cudaEventRecord(m->ev[5], s));
	launch_upper_pass(m);
	CK(cudaEventRecord(m->ev[6], s));
	m->ev_valid = true;
	CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
	m->stats_pending = true;
	p.valid = true;
}

// Enqueues every kernel of one scan and the read-back of its counters; never waits.  A deferred scan
// (p.defer) stops after its marking; m->paired: the scan is the second of a pair and marks into the
// second volume, then the pass updates the leaves of both.
void enqueue_scan(Map* m, PendingScan& p)
{
	if (p.write) {
		enqueue_write(m, p);
		return;
	}
	m->write_pass = false;
	m->early_pass = p.early != 0;
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	ScanArgs& a = p.a;
	new_scan_id(m);
	new_up_epoch(m);
	const bool fused = use_fused(m, p);
	M.dense = (fused && p.dense) ? 1u : 0u;
	M.mask_base = M.dense ? M.vol : M.miss_mask;
	bind_scan_buffers(m, p, fused);
	m->ev7_valid = false;
	push_counters(m, m->paired ? m->first_touched : 0u);
	std::optional<SecondMarks> second;
	if (m->paired) second.emplace(m);
	if (p.need_table) {
		CK(cudaMemsetAsync(m->d_tab_keys.p, 0xff, (size_t)m->tab_size * sizeof(unsigned long long), s));
		CK(cudaMemsetAsync(m->d_tab_min.p, 0xff, (size_t)m->tab_size * sizeof(uint32_t), s));
	}
	if (p.has_vol) {
		// setValueVolume: the marks come from the box instead of a scan
		if (p.vol.general) k_volume_mark<true><<<p.vol.nx * p.vol.ny * p.vol.nz, 64, 0, s>>>(M, p.vol);
		else k_volume_mark<false><<<p.vol.nx * p.vol.ny * p.vol.nz, 64, 0, s>>>(M, p.vol);
		++m->launches;
		if (m->profiling) CK(cudaEventRecord(m->ev[2], s));
	} else if (a.n) {
		uint32_t grid = (uint32_t)((a.n + 255) / 256);
		k_points<<<grid, 256, 0, s>>>(M, a);
		++m->launches;
		if (p.use_color) {
			k_hits<<<grid, 256, 0, s>>>(M, a);
			++m->launches;
		}
		if (m->profiling) CK(cudaEventRecord(m->ev[2], s));
		if (fused) launch_rays_fused(m, a);
		else if (p.early) launch_early(m, p);
		else launch_rays_records(m, a, p.simple);
		if (p.use_color && M.alias_miss) {
			// only maps that have met out-of-tree keys; after marking, before the occupancy update
			k_wrapped_colors<<<grid, 256, 0, s>>>(M, a);
			++m->launches;
		}
	} else if (m->profiling) {
		CK(cudaEventRecord(m->ev[2], s));
	}
	if (m->profiling) CK(cudaEventRecord(m->ev[3], s));
	second.reset();
	CK(cudaGetLastError());
	if (p.defer) {
		CK(cudaEventRecord(m->ev[9], s));
		m->ev_valid = true;
		CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
		m->stats_pending = true;
		p.valid = true;
		return;
	}
	enqueue_update(m, p);
}

// k_inbox, its colour pass and K3 of apply call `call` of a routed pass (ufo_route.cuh)
void enqueue_route_call(Map* m, uint32_t call)
{
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	const PendingScan::RouteCall& c = m->pending.calls[call];
	ScanArgs t{};
	if (M.color) {
		// apply table for the hit records of these sources: at most count * cap_h keys, half full
		const uint32_t size = std::min(m->route_tab_size, std::max(1u << 12, next_pow2(2ull * c.count * m->route_cap_h)));
		CK(cudaMemsetAsync(m->d_route_tab_keys.p, 0xff, (size_t)size * sizeof(unsigned long long), s));
		CK(cudaMemsetAsync(m->d_route_tab_min.p, 0xff, (size_t)size * sizeof(uint32_t), s));
		t.tab_keys = m->d_route_tab_keys.p;
		t.tab_min = m->d_route_tab_min.p;
		t.tab_mask = size - 1;
	}
	k_inbox<<<m->sm_count * 4, 256, 0, s>>>(M, c.first, c.count, t, call);
	++m->launches;
	if (M.color) {
		k_inbox_color<<<m->sm_count * 4, 256, 0, s>>>(M, c.first, c.count, t);
		++m->launches;
	}
	launch_update(m, m->pending.a.miss, false);
}

// A routed pass whose apply calls ran into a full pool (overflow flags `ov`; keep_created has run).
// k_inbox of call route_call could not place every record, and from there on K3, the upper seeds
// and the later calls backed off.  Grows the pools and replays those calls in their order under
// their own scan ids: the failed call keeps the touched list it built (its bricks carry its scan id,
// so touching them again lists nothing twice) and ORs its masks in again.  The inbox regions they
// read stay valid until the peers' mark of pass k+2 (DESIGN.md section 6).  The upper levels are then
// propagated again, under a new epoch, from every brick the pass's calls touched: the seeds of the
// calls that backed off are lost, and the levels of the last call already ran over the seeds before
// them.  A full upper-node pool alone takes the same propagation.  Leaves the counters' read-back
// in flight.
void regrow_routed(Map* m, uint32_t ov)
{
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	PendingScan& p = m->pending;
	const uint32_t from = m->h_ctr->route_call;
	grow_pools(m, ov, m->h_ctr->n_bricks, m->h_ctr->n_upper);
	// allocation cursors back to the slots kept, flags cleared; the touched list and statistics stay
	static_assert(offsetof(Counters, overflow) == offsetof(Counters, n_bricks) + 2 * sizeof(uint32_t), "cursor layout");
	m->h_ctr->n_bricks = m->n_bricks;
	m->h_ctr->n_upper = m->n_upper;
	m->h_ctr->overflow = 0;
	CK(cudaMemcpyAsync(&M.ctr->n_bricks, &m->h_ctr->n_bricks, 3 * sizeof(uint32_t), cudaMemcpyHostToDevice, s));
	if (ov & 2u) {
		for (uint32_t k = from; k < p.calls.size(); ++k) {
			M.scan_id = p.calls[k].scan_id;
			if (k != from) k_route_next_apply<<<1, 1, 0, s>>>(M.ctr);
			enqueue_route_call(m, k);
		}
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		if (m->h_ctr->overflow) return;  // full again: the caller grows and replays once more
		keep_created(m);
	}
	new_up_epoch(m);
	k_reset_upper_pass<<<1, 1, 0, s>>>(M.ctr, m->n_upper);
	CK(cudaMemsetAsync(&M.ctr->n_touched, 0, sizeof(uint32_t), s));
	const uint32_t first = p.calls.front().scan_id;
	k_touch_pass<<<m->sm_count * 4, 256, 0, s>>>(M, m->n_bricks, first, p.calls.back().scan_id - first + 1u);
	launch_upper(m);
	m->launches += 2;
	CK(cudaEventRecord(m->ev[6], s));
	CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
}

// The second scan of a pair could not be marked completely (a full pool; K3 and K4 backed off): the
// first scan's leaf update runs alone, the second's marks are wiped, and the caller repeats it as a scan
// of its own.  Called with the stream idle, after keep_created.
void split_pair(Map* m, uint32_t ov)
{
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	PendingScan& p = m->pending;
	const uint32_t want_bricks = m->h_ctr->n_bricks;  // what the second scan's marking reached: the caller's growth
	const ufo_b200_scan_stats second = m->stats;
	m->paired = false;
	m->stats = m->first_stats;
	new_scan_id(m);
	new_up_epoch(m);
	M.mask_base = M.vol;
	push_counters(m, m->first_touched);
	PendingScan first = p;
	first.has_vol = false;
	enqueue_update(m, first);
	CK(cudaStreamSynchronize(s));
	while (m->h_ctr->overflow == 4u) {  // only the upper-node pool can overflow here
		keep_created(m);
		grow_pools(m, 4u, 0, m->h_ctr->n_upper);
		new_up_epoch(m);
		k_reset_upper_pass<<<1, 1, 0, s>>>(M.ctr, m->n_upper);
		launch_upper(m);
		CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
	}
	finish_stats(m);
	// what the first scan's marking counted stays; the pass added its leaf update
	ufo_b200_scan_stats& a = m->stats;
	const ufo_b200_scan_stats& f = m->first_stats;
	a.rays = f.rays;
	a.visits = f.visits;
	a.ms_total = f.ms_total;
	a.ms_points = f.ms_points;
	a.ms_rays = f.ms_rays;
	a.ms_scatter = f.ms_scatter;
	m->done_stats = a;
	m->held = false;
	wipe_volume2(m);
	keep_created(m);
	// grow_pools sizes the brick pool by what the second scan's marking reached, and rebuilds both
	// hashes from the live slots: the upper nodes include those the first scan's K4 just created
	m->h_ctr->n_bricks = std::max(want_bricks, m->n_bricks);
	m->h_ctr->n_upper = m->n_upper;
	m->stats = second;
	if (p.dense) setup_volume(m, p, volume_bricks(m, p));
}

// Waits for the scan in flight, repeats it if a device pool overflowed, and folds its counters
// into the host view.  A deferred scan gets its leaf update enqueued first.  Throws MapError if the
// scan cannot be completed.
void finalize_scan(Map* m)
{
	PendingScan& p = m->pending;
	if (p.valid && p.defer) {
		p.defer = false;
		p.flushed = true;
		enqueue_update(m, p);
	}
	CK(cudaStreamSynchronize(m->stream));
	if (!p.valid) {
		finish_stats(m);
		return;
	}
	DeviceMap& M = m->M;
	if (p.routed) {
		const uint32_t rf = m->h_route_flag ? *m->h_route_flag : 0u;
		if (rf || (m->route_stage == 1 && m->h_ctr->overflow)) {
			if (rf) m->set_error("routed mode: an inbox region is too small (flags %u); raise cap_bricks / cap_hits", rf);
			else m->set_error("routed mode: a device pool overflowed while marking (flags %u); create the map with a larger initial_bricks", m->h_ctr->overflow);
			p.valid = false;
			m->stats_pending = false;
			m->poisoned = true;
			m->route_stage = 0;
			throw MapError{UFO_B200_E_NOMEM};
		}
		if (m->route_stage == 1) return;  // marked, not applied yet: nothing to fold in
	}
	while (true) {
		const uint32_t ov = m->h_ctr->overflow;
		if (!ov) break;
		++p.regrows;
		if (p.regrows > 16 || (ov & (16u | 128u)) || (p.routed && (ov & ~6u))) {
			if (ov & 128u) m->set_error("insert depth >= 5 with rays that leave the map (out-of-tree nodes) is not supported");
			else if (ov & 16u) m->set_error("internal error: a ray walk exceeded its record bound");
			else if (p.routed && (ov & ~6u)) m->set_error("routed mode: an apply call failed (overflow flags %u)", ov);
			else m->set_error("device pools keep overflowing");
			p.valid = false;
			m->stats_pending = false;
			m->poisoned = true;  // marks of the failed scan are still in the masks
			throw MapError{(ov & 128u) ? UFO_B200_E_UNSUPPORTED : ((ov & 16u) ? UFO_B200_E_CUDA : UFO_B200_E_NOMEM)};
		}
		try {
			keep_created(m);
			if (p.routed) {
				regrow_routed(m, ov);
			} else if (ov == 4u) {
				// only the upper-node pool overflowed: the leaves are updated, repeat the propagation
				grow_pools(m, 4u, 0, m->h_ctr->n_upper);
				new_up_epoch(m);
				k_reset_upper_pass<<<1, 1, 0, m->stream>>>(M.ctr, m->n_upper);
				launch_upper_pass(m);
				CK(cudaEventRecord(m->ev[6], m->stream));
				CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, m->stream));
			} else {
				// an allocation failed while marking a scan or expanding a write batch: nothing was
				// consumed (every later kernel backed off).  Grow and run the whole pass again under a
				// new scan id (marking is idempotent: OR into masks, find-or-create of bricks).  Only
				// scans set the flags other than 2 and 4.
				if (m->paired) split_pair(m, ov);
				if (ov & 64u) {
					// a mark fell outside the scan volume (cannot happen for rays within max_range; kept
					// as a safety net): wipe the volume and repeat through the brick hash
					m->no_dense = 1;
					p.dense = false;
					wipe_volume(m);
				}
				if (ov & 32u) {
					// first out-of-tree key ever seen by this map: allocate the alias mask arrays;
					// from now on this map uses the generic record path
					alloc_arrays(m, Pool::Brick, Have::Aliases);
					if (p.dense) {
						// the marks the walk already left in the volume are not consumed by the record path
						wipe_volume(m);
						p.dense = false;
					}
				}
				const bool fused = use_fused(m, p);
				if (ov & 256u) ensure_early(m, p.a.n, m->h_ctr->e_visits);  // the walks need more ids / table slots
				if (!p.write && !fused && !p.simple && !p.has_vol && !p.early) {
					ensure_scan_buffers(m, p.a.n, false, true, false);
					unsigned long long want = std::max<unsigned long long>(m->h_ctr->seg_total + m->h_ctr->seg_total / 4 + 1024,
					                                                        std::max<unsigned long long>(p.a.n, 1024) * 48ull);
					ensure_seg(m, want);
				}
				if (ov & 6u) grow_pools(m, ov & 6u, m->h_ctr->n_bricks, m->h_ctr->n_upper);
				enqueue_scan(m, p);
			}
		} catch (std::bad_alloc&) {
			m->set_error("block pool cannot grow beyond 2^32 slots");
			p.valid = false;
			m->stats_pending = false;
			m->poisoned = true;
			throw MapError{UFO_B200_E_NOMEM};
		}
		CK(cudaStreamSynchronize(m->stream));
	}
	m->stats.regrows = p.regrows;
	m->stats.launches = m->launches;
	m->stats.result_bytes = sizeof(Counters) * (1 + p.regrows);
	p.valid = false;
	finish_stats(m);
	if (m->paired) {
		m->paired = false;
		m->done_stats = m->first_stats;
		m->held_stats = m->stats;
		m->held = true;
	} else {
		m->done_stats = m->stats;
		m->held = false;
	}
}

// The deferred scan's marking is complete (stream idle, no pool overflowed) and the next scan pairs
// with it: its counters so far become the first scan's, and the pass goes on with the second.
void hold_first(Map* m)
{
	const Counters& c = *m->h_ctr;
	ufo_b200_scan_stats& st = m->first_stats;
	st = m->stats;
	st.rays = c.n_rays;
	st.visits = c.visits;
	keep_created(m);
	st.bricks_in_map = m->n_bricks;
	st.device_bytes = m->device_bytes;
	if (c.n_rays) fold_bbox(m, c);
	if (m->ev_valid) {
		cudaEventElapsedTime(&st.ms_total, m->ev[0], m->ev[9]);
		if (m->h2d_valid) cudaEventElapsedTime(&st.ms_h2d, m->ev_copy0, m->ev_copied);
		if (m->profiling) marking_times(m, st);
	}
	st.regrows = m->pending.regrows;
	st.launches = m->launches;
	st.result_bytes = sizeof(Counters) * (1 + m->pending.regrows);
	m->first_id = m->M.scan_id;
	m->first_touched = c.n_touched;
	m->paired = true;
	m->stats_pending = false;
	m->pending.valid = false;
}

// completed_scan_stats: the pair's second scan once a later call has been made
void release_held(Map* m)
{
	if (!m->held) return;
	m->done_stats = m->held_stats;
	m->held = false;
}

// every brick of the map becomes the "touched list" (whole-map passes: threshold changes)
__global__ void k_touch_all(DeviceMap M, uint32_t n_bricks)
{
	for (uint32_t b = blockIdx.x * blockDim.x + threadIdx.x; b < n_bricks; b += gridDim.x * blockDim.x) {
		M.touched[b] = b;
		M.brick_stamp[b] = M.scan_id;
	}
	if (blockIdx.x == 0 && threadIdx.x == 0) M.ctr->n_touched = n_bricks;
}

// contains_free / contains_unknown of depth 1 and 2 from the leaves, under the current thresholds
__global__ void __launch_bounds__(256) k_reflag(DeviceMap M, uint32_t n_bricks)
{
	const size_t n = (size_t)n_bricks * 64;
	for (size_t b = (size_t)blockIdx.x * blockDim.x + threadIdx.x; b < n; b += (size_t)gridDim.x * blockDim.x) {
		const uint32_t mt = M.meta[b];
		if (!(mt & 0xff0000u)) continue;
		const float* leaf = M.leaf + b * 64;
		uint32_t fl16 = 0;
		for (uint32_t o = 0; o < 8; ++o) {
			if ((mt >> (16 + o)) & 1u) {
				uint32_t ofl = 0;
				for (int j = 0; j < 8; ++j) ofl |= leaf_flags(M, leaf[8 * o + j]);
				fl16 |= ofl << (2 * o);
			}
		}
		M.meta[b] = (mt & 0xffff0000u) | fl16;  // the depth-2 flags follow from it (block_flags)
	}
}

// The reference re-reads the whole tree when the occupied / free thresholds change
// (setOccupiedFreeThres, occupancy_map_base.h:748-761): the contains_free / contains_unknown
// flags of every inner node are functions of the thresholds.  Same effect here.
void rebuild_flags(Map* m)
{
	finalize_scan(m);
	if (!m->n_bricks) return;
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	new_scan_id(m);
	new_up_epoch(m);
	push_counters(m);
	k_touch_all<<<m->sm_count, 256, 0, s>>>(M, m->n_bricks);
	k_reflag<<<m->sm_count * 8, 256, 0, s>>>(M, m->n_bricks);
	launch_brick_agg(m);
	launch_upper(m);
	CK(cudaStreamSynchronize(s));
}

int sync_map(Map* m)
{
	release_held(m);
	finalize_scan(m);
	release_held(m);
	return UFO_B200_OK;
}

// copies a scan's points into staging buffer `stg` on the copy stream (see do_insert)
void stage_points(Map* m, uint32_t stg, const void* points, size_t bytes)
{
	ensure_spare(m, m->d_points[stg], bytes, 1 << 16);
	CK(cudaEventRecord(m->ev_copy0, m->copy_stream));
	CK(cudaMemcpyAsync(m->d_points[stg].p, points, bytes, cudaMemcpyHostToDevice, m->copy_stream));
	CK(cudaEventRecord(m->ev_copied, m->copy_stream));
}

int do_insert(Map* m, const double origin[3], const void* points, bool on_device, size_t n,
              const double* frame_pose,
              int layout, double max_range, uint32_t depth, int simple, uint32_t early_stopping,
              int discrete, int async, const ufo_b200_cloud2* pc2 = nullptr, const VolumeArgs* vol = nullptr,
              float set_value = 0.0f)
{
	if (!m || !origin || (!points && n)) return UFO_B200_E_INVALID;
	size_t stride = pc2 ? pc2->point_step : layout_stride(layout);
	if (!stride || n > 0x7fffffffull) {
		m->set_error("invalid layout %d or point count %zu", layout, n);
		return UFO_B200_E_INVALID;
	}
	bool pc2_rgb = false;
	if (pc2) {
		layout = 4;
		pc2_rgb = pc2->off_r >= 0 && pc2->off_g >= 0 && pc2->off_b >= 0;
		const uint32_t fx[3] = {pc2->off_x, pc2->off_y, pc2->off_z};
		bool ok = pc2->point_step % 4 == 0;
		for (uint32_t f : fx) ok = ok && f % 4 == 0 && (size_t)f + 4 <= pc2->point_step;
		const int32_t fc[3] = {pc2->off_r, pc2->off_g, pc2->off_b};
		for (int32_t c : fc) ok = ok && (c < 0 || (size_t)c < pc2->point_step);
		if (!ok) {
			m->set_error("PointCloud2 descriptor: x/y/z must be 4-byte aligned FLOAT32 fields inside point_step");
			return UFO_B200_E_INVALID;
		}
	}
	if (early_stopping != 0 && !m->early_exact) {
		m->set_error("early_stopping is order-dependent in the reference (occupancy_map_base.h:1289-1298) and is not supported "
		             "unless the map opted in with ufo_b200_set_early_stopping(map, 1)");
		return UFO_B200_E_UNSUPPORTED;
	}
	if (depth > 6) {
		m->set_error("insert depth %u > 6 is not supported (a free-space node of depth 7 covers 512 bricks of the dense value field)", depth);
		return UFO_B200_E_UNSUPPORTED;
	}
	if (m->poisoned) {
		m->set_error("an earlier scan failed half-way; ufo_b200_clear() the map before inserting again");
		return UFO_B200_E_INVALID;
	}
	CK(cudaSetDevice(m->device));

	// The points go to the device first, on the copy stream, into the staging buffer the scan in
	// flight is not using: the H2D copy of scan k+1 overlaps the kernels of scan k (the reference
	// overlaps its own front end with the previous scan's helper thread the same way, OMB:315).
	const size_t bytes = n * stride;
	const bool copied = !on_device && bytes;
	const uint32_t stg = m->stage ^ 1u;
	if (copied) stage_points(m, stg, points, bytes);
	// Consecutive asynchronous scans of the plain kind share one leaf update (DESIGN.md section 4,
	// "Paired scans"): the first is marked and deferred, the second marks into the second volume and
	// the pass updates the leaves of both.  A scan of any other kind runs on its own.
	PendingScan probe;
	probe.a.max_range = max_range;
	const uint32_t pair_db = volume_bricks(m, probe);
	const DeviceMap& Mc = m->M;
	const bool eligible = async && !vol && !Mc.color && depth == 0 && !discrete && !simple && !early_stopping && pair_db &&
	                      !Mc.alias_miss && !Mc.chg_mask && Mc.shard_world <= 1 && Mc.route_world <= 1 && !m->force_records &&
	                      m->profiling < 2 && !m->no_pair;
	release_held(m);
	bool pairing = false;
	if (eligible && m->pending.valid && m->pending.defer) {
		CK(cudaStreamSynchronize(m->stream));
		pairing = !m->h_ctr->overflow && ensure_volume2(m, pair_db);
	}
	// one integration in flight at most (insertPointCloudWait, occupancy_map_base.h:315)
	if (pairing) {
		// what can fail is allocated first: until hold_first the deferred scan stays what it was
		ensure_scan_buffers(m, n, false, false, true);
		hold_first(m);
	} else {
		finalize_scan(m);
	}

	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	const bool has_rgb = layout == UFO_B200_XYZRGB_F64 || layout == UFO_B200_XYZRGB_F32 || pc2_rgb;
	PendingScan& p = m->pending;
	p = PendingScan{};
	p.use_color = M.color && has_rgb;
	p.need_table = discrete || p.use_color || depth >= 5;  // depth 5/6: the scan's set of free-space nodes
	p.simple = simple != 0;
	p.has_vol = vol != nullptr;
	if (vol) p.vol = *vol;
	p.set_value = set_value;
	p.early = vol ? 0u : early_stopping;

	ScanArgs& a = p.a;
	a.origin = {origin[0], origin[1], origin[2]};
	a.max_range = max_range;
	a.n = (uint32_t)n;
	a.depth = depth;
	a.layout = layout;
	a.discrete = discrete;
	a.use_color = p.use_color;
	a.miss = (float)(m->miss_log / (double)((2.0 * depth) + 1));
	a.count_visits = m->profiling >= 2;
	if (pc2) {
		a.pc2_step = pc2->point_step;
		a.pc2_x = pc2->off_x;
		a.pc2_y = pc2->off_y;
		a.pc2_z = pc2->off_z;
		a.pc2_r = pc2_rgb ? pc2->off_r : -1;
		a.pc2_g = pc2_rgb ? pc2->off_g : -1;
		a.pc2_b = pc2_rgb ? pc2->off_b : -1;
	}
	if (frame_pose) {
		a.has_frame = 1;
		a.frame = Frame{frame_pose[3], frame_pose[4], frame_pose[5], frame_pose[6],
		                frame_pose[0], frame_pose[1], frame_pose[2]};
	}
	const bool fused = use_fused(m, p);
	const bool records = !fused && !p.simple && !p.has_vol && !p.early;
	ensure_scan_buffers(m, n, p.need_table, records, fused);
	// first guess for the walks: 64 visits per ray; grown to the exact count on demand
	if (p.early) ensure_early(m, n, m->e_id_cap ? 0ull : std::max<size_t>(n, 1024) * 64ull);
	if (fused) {
		const uint32_t db = volume_bricks(m, p);
		p.dense = db != 0;
		if (p.dense) setup_volume(m, p, db, pairing);
	}
	p.defer = eligible && !pairing && p.dense;
	if (records) {
		// first guess for the record buffer: 48 records per ray; grown on demand
		ensure_seg(m, std::max<unsigned long long>(m->seg_cap, std::max<unsigned long long>(n, 1024) * 48ull));
	}
	// an on-device cloud is read in place: it has to stay valid until the scan is done
	a.points = on_device ? points : m->d_points[stg].p;
	if (copied) m->stage = stg;

	m->stats = ufo_b200_scan_stats{};
	m->stats.points = n;
	m->launches = 0;
	m->h2d_valid = copied;
	CK(cudaEventRecord(m->ev[0], s));
	if (copied) CK(cudaStreamWaitEvent(s, m->ev_copied, 0));
	enqueue_scan(m, p);
	// the caller's buffer is free again when this returns (the reference takes the cloud by value)
	if (copied) CK(cudaEventSynchronize(m->ev_copied));
	if (!async) return sync_map(m);
	return UFO_B200_OK;
}

// ---- routed multi-GPU mode (ufo_route.cuh) -------------------------------------------------
// hit_words: 1 for mono maps (packed voxel key), 2 for colour maps (+ global cloud index and rgb)
size_t route_layout(uint32_t world, uint32_t cap_m, uint32_t cap_h, uint32_t hit_words, size_t* region, size_t* miss_off,
                    size_t* hit_off)
{
	const size_t mo = 256;
	const size_t ho = mo + (((size_t)cap_m * kMissRecWords * 8 + 255) & ~(size_t)255);
	const size_t reg = ho + (((size_t)cap_h * 8 * hit_words + 255) & ~(size_t)255);
	if (region) *region = reg;
	if (miss_off) *miss_off = mo;
	if (hit_off) *hit_off = ho;
	return reg * world * 2;
}

void route_fill_table(Map* m)
{
	RouteTable& T = *m->h_route;
	memset(&T, 0, sizeof(T));
	T.cap_m = m->route_cap_m;
	T.cap_h = m->route_cap_h;
	const uint32_t W = m->M.route_world, me = m->M.route_rank;
	for (uint32_t r = 0; r < W; ++r) {
		// my records for rank r land in r's inbox, region (parity, source = me)
		unsigned char* bo = static_cast<unsigned char*>(m->route_peer[r]) + ((size_t)m->route_parity * W + me) * m->route_region;
		T.out[r].hdr = reinterpret_cast<uint32_t*>(bo);
		T.out[r].miss = reinterpret_cast<unsigned long long*>(bo + m->route_miss_off);
		T.out[r].hit = reinterpret_cast<unsigned long long*>(bo + m->route_hit_off);
		unsigned char* bi = m->route_inbox.p + ((size_t)m->route_parity * W + r) * m->route_region;
		T.in[r].hdr = reinterpret_cast<uint32_t*>(bi);
		T.in[r].miss = reinterpret_cast<unsigned long long*>(bi + m->route_miss_off);
		T.in[r].hit = reinterpret_cast<unsigned long long*>(bi + m->route_hit_off);
	}
}

// The mark phase of a routed pass.  Takes every option of do_insert except early_stopping, frames and
// PointCloud2 records; `ex` = false is ufo_b200_route_mark (mono maps only).  Local point i has the
// global cloud index index_base + i * index_stride (colour maps: it picks the voxel's colour winner).
int do_route_mark(Map* m, const double origin[3], const void* points, bool on_device, size_t n, int layout,
                  double max_range, uint32_t depth, int simple, uint32_t early_stopping, int discrete,
                  uint64_t index_base, uint32_t index_stride, int self_too, bool ex)
{
	if (!m || !origin || (!points && n)) return UFO_B200_E_INVALID;
	const size_t stride = layout_stride(layout);
	if (!stride || n > 0x7fffffffull) return UFO_B200_E_INVALID;
	DeviceMap& M = m->M;
	if (M.route_world < 2 || !m->route_peer[0]) {
		m->set_error("routed mode is not set up (ufo_b200_route_setup + ufo_b200_route_connect)");
		return UFO_B200_E_INVALID;
	}
	if (early_stopping != 0) {
		m->set_error("early_stopping is order-dependent in the reference (occupancy_map_base.h:1289-1298) and is not supported");
		return UFO_B200_E_UNSUPPORTED;
	}
	if (depth > 6) {
		m->set_error("insert depth %u > 6 is not supported", depth);
		return UFO_B200_E_UNSUPPORTED;
	}
	if (index_stride == 0) {
		m->set_error("ufo_b200_route_mark_ex: index_stride must be at least 1");
		return UFO_B200_E_INVALID;
	}
	if ((!ex && M.color) || M.alias_miss || m->poisoned || m->route_stage == 1) {
		m->set_error(m->route_stage == 1 ? "ufo_b200_route_mark: the previous pass was not applied"
		             : (!ex && M.color) ? "ufo_b200_route_mark takes mono maps; colour maps use ufo_b200_route_mark_ex"
		                                : "routed mode needs a healthy map without out-of-tree keys");
		return UFO_B200_E_UNSUPPORTED;
	}
	const bool has_rgb = layout == UFO_B200_XYZRGB_F64 || layout == UFO_B200_XYZRGB_F32;
	const bool use_color = M.color && has_rgb;
	if (use_color && n && (index_base >= kNone || (uint64_t)(n - 1) > (kNone - 1 - index_base) / index_stride)) {
		m->set_error("ufo_b200_route_mark_ex: global cloud indices must stay below 2^32 - 1");
		return UFO_B200_E_INVALID;
	}
	CK(cudaSetDevice(m->device));
	const size_t bytes = n * stride;
	const bool copied = !on_device && bytes;
	const uint32_t stg = m->stage ^ 1u;
	if (copied) stage_points(m, stg, points, bytes);
	finalize_scan(m);
	cudaStream_t s = m->stream;
	PendingScan& p = m->pending;
	p = PendingScan{};
	p.routed = true;
	p.use_color = use_color;
	p.need_table = discrete || use_color || depth >= 5;  // as do_insert
	p.simple = simple != 0;
	ScanArgs& a = p.a;
	a.origin = {origin[0], origin[1], origin[2]};
	a.max_range = max_range;
	a.n = (uint32_t)n;
	a.depth = depth;
	a.layout = layout;
	a.discrete = discrete;
	a.use_color = use_color;
	a.miss = (float)(m->miss_log / (double)((2.0 * depth) + 1));
	a.count_visits = m->profiling >= 2;
	// the marking path is chosen as for a single-GPU insert
	const bool fused = use_fused(m, p);
	const bool records = !fused && !p.simple;
	ensure_scan_buffers(m, n, p.need_table, records, fused);
	if (fused) {
		const uint32_t db = volume_bricks(m, p);
		p.dense = db != 0;
		if (p.dense) setup_volume(m, p, db);
	}
	M.dense = p.dense ? 1u : 0u;
	M.mask_base = M.dense ? M.vol : M.miss_mask;
	a.points = on_device ? points : m->d_points[stg].p;
	if (copied) m->stage = stg;
	bind_scan_buffers(m, p, fused);
	m->stats = ufo_b200_scan_stats{};
	m->stats.points = n;
	m->launches = 0;
	m->h2d_valid = copied;
	m->ev7_valid = false;
	M.route_self = self_too ? 1u : 0u;
	m->route_parity ^= 1u;
	route_fill_table(m);
	m->h_route_flag[0] = 0;
	CK(cudaEventRecord(m->ev[0], s));
	if (copied) CK(cudaStreamWaitEvent(s, m->ev_copied, 0));
	// Marking creates bricks, own and foreign, and K1 and k_expand_nodes write hit records straight
	// into the peers' inboxes, which the peers read right after the barrier.  So the marking is waited
	// for here: if a pool ran full, it grows and the marking runs again under a new scan id (OR into
	// masks, find-or-create of bricks: idempotent) from fresh outbox cursors (the table push), and
	// only the complete pass is published.
	const auto fail = [&](const char* why) {
		m->set_error("%s", why);
		p.valid = false;
		m->poisoned = true;  // the marks of the failed attempt are still in the masks
		m->route_stage = 0;
		throw MapError{UFO_B200_E_NOMEM};
	};
	for (;;) {
		CK(cudaMemcpyAsync(M.route, m->h_route, sizeof(RouteTable), cudaMemcpyHostToDevice, s));
		new_scan_id(m);
		push_counters(m);
		if (p.need_table) {
			CK(cudaMemsetAsync(m->d_tab_keys.p, 0xff, (size_t)m->tab_size * sizeof(unsigned long long), s));
			CK(cudaMemsetAsync(m->d_tab_min.p, 0xff, (size_t)m->tab_size * sizeof(uint32_t), s));
		}
		if (n) {
			const uint32_t grid = (uint32_t)((n + 255) / 256);
			// K1 reserves the walk's records without a bound; the buffer is sized to the reservation
			if (records) a.seg_cap = ~0ull;
			k_points<<<grid, 256, 0, s>>>(M, a);
			++m->launches;
			if (use_color) {
				k_route_hits<<<grid, 256, 0, s>>>(M, a, (unsigned long long)index_base, index_stride);
				++m->launches;
			}
			if (m->profiling) CK(cudaEventRecord(m->ev[2], s));
			if (fused) {
				launch_rays_fused(m, a);
			} else {
				if (records) {
					CK(cudaMemcpyAsync(&m->h_ctr->seg_total, &M.ctr->seg_total, sizeof(unsigned long long), cudaMemcpyDeviceToHost, s));
					CK(cudaStreamSynchronize(s));
					ensure_seg(m, std::max<unsigned long long>(m->h_ctr->seg_total, 1024));
					a.seg = m->d_seg.p;
					a.seg_cap = m->seg_cap;
				}
				launch_rays_records(m, a, p.simple);
			}
		} else if (m->profiling) {
			CK(cudaEventRecord(m->ev[2], s));
		}
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(&m->h_ctr->n_bricks, &M.ctr->n_bricks, 3 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		const uint32_t ov = m->h_ctr->overflow;
		if (!(ov & 6u) || (ov & ~6u)) break;  // complete, or a flag no growth clears (the next finalize_scan reports it)
		if (++p.regrows > 16) fail("device pools keep overflowing");
		try {
			keep_created(m);
			grow_pools(m, ov, m->h_ctr->n_bricks, m->h_ctr->n_upper);
		} catch (std::bad_alloc&) {
			fail("block pool cannot grow beyond 2^32 slots");
		}
	}
	k_outbox<<<m->sm_count * 4, 256, 0, s>>>(M);
	k_outbox_publish<<<1, 32, 0, s>>>(M);
	m->launches += 2;
	if (m->profiling) CK(cudaEventRecord(m->ev[3], s));
	CK(cudaGetLastError());
	CK(cudaMemcpyAsync(m->h_route_flag, &M.route->overflow, 4 * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
	p.valid = true;
	m->route_stage = 1;
	if (copied) CK(cudaEventSynchronize(m->ev_copied));
	return UFO_B200_OK;
}

int do_route_apply(Map* m, uint32_t first, uint32_t count, int last)
{
	if (!m) return UFO_B200_E_INVALID;
	DeviceMap& M = m->M;
	if (m->route_stage != 1 || first + count > M.route_world) {
		m->set_error("ufo_b200_route_apply without a marked pass, or sources out of range");
		return UFO_B200_E_INVALID;
	}
	CK(cudaSetDevice(m->device));
	cudaStream_t s = m->stream;
	PendingScan& p = m->pending;
	// every apply call is a scan of its own as far as the touched list goes: the first one starts
	// from the own bricks that kept local marks (list built by k_outbox under scan id + 1), the
	// following ones from an empty list
	new_scan_id(m);
	if (!p.applying) {
		std::swap(M.touched, M.touched_alt);
		std::swap(M.touched_mi, M.touched_alt_mi);
		M.dense = 0;
		M.mask_base = M.miss_mask;
		new_up_epoch(m);
		p.applying = true;
	} else {
		k_route_next_apply<<<1, 1, 0, s>>>(M.ctr);
		++m->launches;
	}
	p.calls.push_back({first, count, M.scan_id});
	enqueue_route_call(m, (uint32_t)p.calls.size() - 1);
	launch_upper_seed(m);
	if (last) {
		if (m->profiling) CK(cudaEventRecord(m->ev[5], s));
		launch_upper_levels(m);
		CK(cudaEventRecord(m->ev[6], s));
		m->ev_valid = true;
		CK(cudaMemcpyAsync(m->h_ctr, M.ctr, sizeof(Counters), cudaMemcpyDeviceToHost, s));
		m->stats_pending = true;
		m->route_stage = 2;
	}
	CK(cudaGetLastError());
	return UFO_B200_OK;
}

template <class F>
int guarded(Map* m, F&& f)
{
	if (m && m->device == -2) {
		m->set_error("geometry-only handle: no CUDA device bound");
		return UFO_B200_E_CUDA;
	}
	try {
		return f();
	} catch (CudaError& e) {
		if (m) m->set_error("CUDA error %s (%d) at ufo_map.cu:%d: %s", cudaGetErrorName(e.e), (int)e.e, e.line, e.what);
		return UFO_B200_E_CUDA;
	} catch (MapError& e) {
		return e.code;
	} catch (std::bad_alloc&) {
		if (m) m->set_error("out of memory");
		return UFO_B200_E_NOMEM;
	}
}
}  // namespace

// ---------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------
extern "C" {

const char* ufo_b200_version(void) { return "ufomap_b200 0.1 (sm_90a)"; }

void ufo_b200_default_params(ufo_b200_params* p)
{
	if (!p) return;
	memset(p, 0, sizeof(*p));
	p->resolution = 0.1;
	p->depth_levels = 16;
	p->automatic_pruning = 1;
	p->occupied_thres = 0.5;
	p->free_thres = 0.5;
	p->prob_hit = 0.7;
	p->prob_miss = 0.4;
	p->clamping_thres_min = 0.1192;
	p->clamping_thres_max = 0.971;
	p->color = 0;
	p->device = -1;
}

}  // extern "C"

namespace
{
// Everything of a new map on a device but its pools: device, streams, events, the counters' pinned
// mirror, geometry and sensor model (ufo_b200_create, clone).
void init_map(Map* m, const ufo_b200_params* p)
{
	int dev = p->device;
	if (dev < 0) CK(cudaGetDevice(&dev));
	CK(cudaSetDevice(dev));
	m->device = dev;
	cudaDeviceProp prop;
	CK(cudaGetDeviceProperties(&prop, dev));
	m->sm_count = prop.multiProcessorCount;
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&m->ray_blocks_per_sm, k_rays<0, false>, kRayThreads, 0));
	if (m->ray_blocks_per_sm < 1) m->ray_blocks_per_sm = 1;
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&m->walk_blocks_per_sm, k_walk_mark<0, false, false, true>, kWalkThreads, 0));
	if (m->walk_blocks_per_sm < 1) m->walk_blocks_per_sm = 1;
	// the rounds kernel is cooperative: every CTA of its grid must be resident
	CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&m->early_blocks_per_sm, k_early_rounds, kEarlyThreads, 0));
	if (m->early_blocks_per_sm < 1) m->early_blocks_per_sm = 1;
	{
		const char* e = getenv("UFO_B200_MARK");
		m->force_records = e && !strcmp(e, "records");
		m->no_dense = e && !strcmp(e, "probe");
		// resident CTAs per SM of the two long kernels (tuning / co-residency experiments)
		const char* kb = getenv("UFO_B200_K3_BLOCKS");
		if (kb && atoi(kb) > 0) m->k3_blocks = atoi(kb);
		const char* wb = getenv("UFO_B200_WALK_BLOCKS");
		if (wb && atoi(wb) > 0) m->walk_blocks_per_sm = std::min(m->walk_blocks_per_sm, atoi(wb));
	}
	m->params = *p;
	CK(cudaStreamCreateWithFlags(&m->own_stream, cudaStreamNonBlocking));
	CK(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
	CK(cudaEventCreate(&m->ev_copy0));
	CK(cudaEventCreate(&m->ev_copied));
	m->stream = m->own_stream;
	for (auto& e : m->ev) CK(cudaEventCreate(&e));
	CK(cudaHostAlloc(reinterpret_cast<void**>(&m->h_ctr), sizeof(Counters), cudaHostAllocDefault));
	m->M.g = make_geometry(p->resolution, p->depth_levels);
	m->M.color = p->color ? 1u : 0u;
	m->M.shard_rank = 0;
	m->M.shard_world = 1;
	m->occ_thr_log = to_logit(p->occupied_thres);
	m->free_thr_log = to_logit(p->free_thres);
	m->hit_log = to_logit(p->prob_hit);
	m->miss_log = to_logit(p->prob_miss);
	m->cmin_log = to_logit(p->clamping_thres_min);
	m->cmax_log = to_logit(p->clamping_thres_max);
	refresh_model(m);
}
}  // namespace

extern "C" {

int ufo_b200_create(const ufo_b200_params* p, ufo_b200_map** out)
{
	if (!p || !out) return UFO_B200_E_INVALID;
	*out = nullptr;
	if (p->depth_levels < 2 || p->depth_levels > 21 || !(p->resolution > 0)) return UFO_B200_E_INVALID;
	Map* m = new (std::nothrow) Map;
	if (!m) return UFO_B200_E_NOMEM;
	if (p->device == -2) {
		// geometry-only handle: indexing / computeRay helpers run on the host and need no
		// device; every call that touches map state fails with UFO_B200_E_CUDA
		m->device = -2;
		m->params = *p;
		m->M.g = make_geometry(p->resolution, p->depth_levels);
		m->occ_thr_log = to_logit(p->occupied_thres);
		m->free_thr_log = to_logit(p->free_thres);
		m->hit_log = to_logit(p->prob_hit);
		m->miss_log = to_logit(p->prob_miss);
		m->cmin_log = to_logit(p->clamping_thres_min);
		m->cmax_log = to_logit(p->clamping_thres_max);
		*out = m;
		return UFO_B200_OK;
	}
	int rc = guarded(m, [&]() {
		init_map(m, p);
		uint32_t bricks, upper;
		initial_caps(*p, bricks, upper);
		alloc_pools(m, bricks, upper);
		m->n_blocks = 0;
		m->n_bricks = 0;
		m->n_upper = 0;
		reset_bbox(m);
		CK(cudaStreamSynchronize(m->stream));
		return (int)UFO_B200_OK;
	});
	if (rc != UFO_B200_OK) {
		fprintf(stderr, "ufo_b200_create failed: %s\n", m->err.c_str());
		free_pools(m);
		delete m;
		return rc;
	}
	*out = m;
	return UFO_B200_OK;
}

void ufo_b200_destroy(ufo_b200_map* m)
{
	if (!m) return;
	if (m->device == -2) {
		delete m;
		return;
	}
	cudaSetDevice(m->device);
	cudaStreamSynchronize(m->stream);
	free_pools(m);
	for (auto& e : m->ev)
		if (e) cudaEventDestroy(e);
	if (m->h_ctr) cudaFreeHost(m->h_ctr);
	if (m->h_route) cudaFreeHost(m->h_route);
	if (m->h_route_flag) cudaFreeHost(m->h_route_flag);
	if (m->own_stream) cudaStreamDestroy(m->own_stream);
	if (m->copy_stream) cudaStreamDestroy(m->copy_stream);
	if (m->ev_copy0) cudaEventDestroy(m->ev_copy0);
	if (m->ev_copied) cudaEventDestroy(m->ev_copied);
	delete m;
}

const char* ufo_b200_last_error(const ufo_b200_map* m) { return m ? m->err.c_str() : "null map"; }

int ufo_b200_set_stream(ufo_b200_map* m, void* cuda_stream)
{
	if (!m) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		sync_map(m);
		m->stream = cuda_stream ? static_cast<cudaStream_t>(cuda_stream) : m->own_stream;
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_insert_pointcloud(ufo_b200_map* m, const double origin[3], const void* points,
                               size_t n, int layout, double max_range, uint32_t depth,
                               int simple_ray_casting, uint32_t early_stopping, int discrete,
                               int async)
{
	return guarded(m, [&]() {
		bump_revision(m);
		return do_insert(m, origin, points, false, n, nullptr, layout, max_range, depth,
		                 simple_ray_casting, early_stopping, discrete, async);
	});
}

int ufo_b200_insert_device(ufo_b200_map* m, const double origin[3], const void* d_points,
                           size_t n, int layout, double max_range, uint32_t depth,
                           int simple_ray_casting, uint32_t early_stopping, int discrete,
                           int async)
{
	return guarded(m, [&]() {
		bump_revision(m);
		return do_insert(m, origin, d_points, true, n, nullptr, layout, max_range, depth,
		                 simple_ray_casting, early_stopping, discrete, async);
	});
}

int ufo_b200_insert_pointcloud_frame(ufo_b200_map* m, const double origin[3], const void* points,
                                     size_t n, int layout, const double frame_pose[7],
                                     double max_range, uint32_t depth, int simple_ray_casting,
                                     uint32_t early_stopping, int discrete, int async)
{
	if (m && !frame_pose) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		bump_revision(m);
		return do_insert(m, origin, points, false, n, frame_pose, layout, max_range, depth,
		                 simple_ray_casting, early_stopping, discrete, async);
	});
}

int ufo_b200_insert_pointcloud2(ufo_b200_map* m, const double origin[3], const ufo_b200_cloud2* cloud,
                                const double* frame_pose, double max_range, uint32_t depth,
                                int simple_ray_casting, uint32_t early_stopping, int discrete, int async)
{
	if (m && !cloud) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		bump_revision(m);
		return do_insert(m, origin, cloud->data, cloud->on_device != 0, cloud->n, frame_pose, 4, max_range,
		                 depth, simple_ray_casting, early_stopping, discrete, async, cloud);
	});
}

int ufo_b200_transform_points(const double frame_pose[7], const void* points, size_t n, int layout,
                              double* out_xyz)
{
	if (!frame_pose || (n && (!points || !out_xyz)) || layout < 0 || layout > 3)
		return UFO_B200_E_INVALID;
	const Frame f{frame_pose[3], frame_pose[4], frame_pose[5], frame_pose[6],
	              frame_pose[0], frame_pose[1], frame_pose[2]};
	const size_t stride = (layout == UFO_B200_XYZ_F64 || layout == UFO_B200_XYZ_F32) ? 3 : 4;
	const bool f64 = layout == UFO_B200_XYZ_F64 || layout == UFO_B200_XYZRGB_F64;
	for (size_t i = 0; i < n; ++i) {
		Vec3 p;
		if (f64) {
			const double* q = static_cast<const double*>(points) + stride * i;
			p = {q[0], q[1], q[2]};
		} else {
			const float* q = static_cast<const float*>(points) + stride * i;
			p = {(double)q[0], (double)q[1], (double)q[2]};
		}
		Vec3 r = frame_transform(f, p);
		out_xyz[3 * i + 0] = r.x;
		out_xyz[3 * i + 1] = r.y;
		out_xyz[3 * i + 2] = r.z;
	}
	return UFO_B200_OK;
}

int ufo_b200_pose_from_rpy(double x, double y, double z, double roll, double pitch, double yaw,
                           double frame_pose[7])
{
	if (!frame_pose) return UFO_B200_E_INVALID;
	// Quaternion(roll, pitch, yaw) of the reference goes through the ZYX rotation matrix and the
	// trace formulas (math/quaternion.h:69-93); restated with the same expression order.
	const double sr = sin(roll), sp = sin(pitch), sy = sin(yaw);
	const double cr = cos(roll), cp = cos(pitch), cy = cos(yaw);
	const double m00 = cy * cp, m01 = cy * sp * sr - sy * cr, m02 = cy * sp * cr + sy * sr;
	const double m10 = sy * cp, m11 = sy * sp * sr + cy * cr, m12 = sy * sp * cr - cy * sr;
	const double m20 = -sp, m21 = cp * sr, m22 = cp * cr;
	const double qw = sqrt(std::max(0.0, 1 + m00 + m11 + m22)) / 2.0;
	const double ax = sqrt(std::max(0.0, 1 + m00 - m11 - m22)) / 2.0;
	const double ay = sqrt(std::max(0.0, 1 - m00 + m11 - m22)) / 2.0;
	const double az = sqrt(std::max(0.0, 1 - m00 - m11 + m22)) / 2.0;
	frame_pose[0] = x;
	frame_pose[1] = y;
	frame_pose[2] = z;
	frame_pose[3] = qw;
	frame_pose[4] = (m21 - m12) >= 0 ? fabs(ax) : -fabs(ax);
	frame_pose[5] = (m02 - m20) >= 0 ? fabs(ay) : -fabs(ay);
	frame_pose[6] = (m10 - m01) >= 0 ? fabs(az) : -fabs(az);
	return UFO_B200_OK;
}

int ufo_b200_wait(ufo_b200_map* m)
{
	if (!m) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		CK(cudaSetDevice(m->device));
		return sync_map(m);
	});
}

int ufo_b200_done(ufo_b200_map* m, int* done)
{
	if (!m || !done) return UFO_B200_E_INVALID;
	if (m->device == -2) return UFO_B200_E_CUDA;
	cudaError_t e = cudaStreamQuery(m->stream);
	if (e == cudaSuccess) {
		// a deferred scan still waits for its leaf update: enqueued now, so that a caller polling this
		// function gets to "done"
		if (m->pending.valid && m->pending.defer) {
			const int rc = guarded(m, [&]() {
				CK(cudaSetDevice(m->device));
				m->pending.defer = false;
				m->pending.flushed = true;
				enqueue_update(m, m->pending);
				return (int)UFO_B200_OK;
			});
			*done = 0;
			return rc;
		}
		// the stream is idle; if the scan ran into a full pool it is not integrated yet: grow and repeat
		// it now, so that a caller polling this function always gets to "done"
		if (m->pending.valid && m->h_ctr->overflow) {
			const int rc = guarded(m, [&]() {
				CK(cudaSetDevice(m->device));
				return sync_map(m);
			});
			if (rc != UFO_B200_OK) return rc;
		}
		*done = 1;
		return UFO_B200_OK;
	}
	if (e == cudaErrorNotReady) {
		*done = 0;
		return UFO_B200_OK;
	}
	m->set_error("cudaStreamQuery: %s", cudaGetErrorString(e));
	return UFO_B200_E_CUDA;
}

int ufo_b200_compute_ray(const ufo_b200_map* m, const double origin[3], const double end_in[3],
                         double max_range, uint32_t depth, uint64_t* codes, size_t cap, size_t* n)
{
	if (!m || !origin || !end_in || !n) return UFO_B200_E_INVALID;
	const Geometry& g = m->M.g;
	Vec3 o = {origin[0], origin[1], origin[2]}, e = {end_in[0], end_in[1], end_in[2]};
	Vec3 dir = vsub(e, o);
	double dist = vnorm(dir);
	dir = vdiv(dir, dist);
	if (0 <= max_range && dist > max_range) {
		e = vadd(o, vscale(dir, max_range));
		dist = max_range;
	}
	Walk w;
	walk_init(g, o, e, dir, depth, w);
	size_t cnt = 0;
	if (!w.same) {
		while (w.cur != w.end && walk_tmin(w) <= dist) {
			if (codes && cnt < cap) codes[cnt] = key_to_code(w.cur);
			++cnt;
			walk_step(w);
		}
	}
	*n = cnt;
	return UFO_B200_OK;
}

int ufo_b200_to_key(const ufo_b200_map* m, const double xyz[3], uint32_t depth, uint32_t key[3])
{
	if (!m || !xyz || !key) return UFO_B200_E_INVALID;
	Key3 k = point_to_key(m->M.g, {xyz[0], xyz[1], xyz[2]}, depth);
	key[0] = k.x;
	key[1] = k.y;
	key[2] = k.z;
	return UFO_B200_OK;
}

int ufo_b200_to_code(const ufo_b200_map* m, const double xyz[3], uint32_t depth, uint64_t* code)
{
	if (!m || !xyz || !code) return UFO_B200_E_INVALID;
	*code = key_to_code(point_to_key(m->M.g, {xyz[0], xyz[1], xyz[2]}, depth));
	return UFO_B200_OK;
}

int ufo_b200_key_to_coord(const ufo_b200_map* m, const uint32_t key[3], uint32_t depth, double xyz[3])
{
	if (!m || !key || !xyz) return UFO_B200_E_INVALID;
	Vec3 p = key_to_coord(m->M.g, {key[0], key[1], key[2]}, depth);
	xyz[0] = p.x;
	xyz[1] = p.y;
	xyz[2] = p.z;
	return UFO_B200_OK;
}

uint64_t ufo_b200_key_to_code(const uint32_t key[3]) { return key_to_code({key[0], key[1], key[2]}); }

void ufo_b200_code_to_key(uint64_t code, uint32_t key[3])
{
	Key3 k = code_to_key(code);
	key[0] = k.x;
	key[1] = k.y;
	key[2] = k.z;
}

int ufo_b200_query(ufo_b200_map* m, const uint64_t* codes, const uint32_t* depths, size_t n,
                   float* logodds, uint8_t* flags, uint8_t* rgb)
{
	if (!m || (n && (!codes || !depths || !logodds || !flags))) return UFO_B200_E_INVALID;
	if (!n) return UFO_B200_OK;
	return guarded(m, [&]() {
		CK(cudaSetDevice(m->device));
		sync_map(m);
		cudaStream_t s = m->stream;
		DevBuf b_codes, b_depths, b_occ, b_flags, b_rgb;
		unsigned long long* d_codes = b_codes.alloc<unsigned long long>(n);
		uint32_t* d_depths = b_depths.alloc<uint32_t>(n);
		float* d_occ = b_occ.alloc<float>(n);
		uint8_t* d_flags = b_flags.alloc<uint8_t>(n);
		uint32_t* d_rgb = rgb ? b_rgb.alloc<uint32_t>(n) : nullptr;
		CK(cudaMemcpyAsync(d_codes, codes, n * 8, cudaMemcpyHostToDevice, s));
		CK(cudaMemcpyAsync(d_depths, depths, n * 4, cudaMemcpyHostToDevice, s));
		k_query<<<(uint32_t)((n + 255) / 256), 256, 0, s>>>(m->M, d_codes, d_depths, (uint32_t)n, d_occ, d_flags, d_rgb);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(logodds, d_occ, n * 4, cudaMemcpyDeviceToHost, s));
		CK(cudaMemcpyAsync(flags, d_flags, n, cudaMemcpyDeviceToHost, s));
		std::vector<uint32_t> h_rgb;
		if (rgb) {
			h_rgb.resize(n);
			CK(cudaMemcpyAsync(h_rgb.data(), d_rgb, n * 4, cudaMemcpyDeviceToHost, s));
		}
		CK(cudaStreamSynchronize(s));
		if (rgb)
			for (size_t i = 0; i < n; ++i) {
				rgb[3 * i] = h_rgb[i] & 0xff;
				rgb[3 * i + 1] = (h_rgb[i] >> 8) & 0xff;
				rgb[3 * i + 2] = (h_rgb[i] >> 16) & 0xff;
			}
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_export_leaves(ufo_b200_map* m, uint64_t* codes, float* logodds, uint8_t* rgb,
                           size_t cap, size_t* n)
{
	if (!m || !n) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		CK(cudaSetDevice(m->device));
		sync_map(m);
		cudaStream_t s = m->stream;
		DevBuf b_count, b_codes, b_occ, b_rgb;
		unsigned long long* d_count = b_count.alloc<unsigned long long>(1);
		CK(cudaMemsetAsync(d_count, 0, 8, s));
		unsigned long long* d_codes = nullptr;
		float* d_occ = nullptr;
		uint32_t* d_rgb = nullptr;
		bool fill = codes != nullptr && cap > 0;
		if (fill) {
			d_codes = b_codes.alloc<unsigned long long>(cap);
			d_occ = b_occ.alloc<float>(cap);
			if (rgb) d_rgb = b_rgb.alloc<uint32_t>(cap);
		}
		size_t threads = (size_t)m->n_bricks * 64 * 64;
		if (threads)
			k_export<<<(uint32_t)((threads + 255) / 256), 256, 0, s>>>(m->M, m->n_bricks, d_codes, d_occ, d_rgb, fill ? cap : 0, d_count);
		CK(cudaGetLastError());
		unsigned long long cnt = 0;
		CK(cudaMemcpyAsync(&cnt, d_count, 8, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		*n = (size_t)cnt;
		if (fill) {
			size_t k = std::min<size_t>(cnt, cap);
			CK(cudaMemcpy(codes, d_codes, k * 8, cudaMemcpyDeviceToHost));
			if (logodds) CK(cudaMemcpy(logodds, d_occ, k * 4, cudaMemcpyDeviceToHost));
			if (rgb) {
				std::vector<uint32_t> h(k);
				CK(cudaMemcpy(h.data(), d_rgb, k * 4, cudaMemcpyDeviceToHost));
				for (size_t i = 0; i < k; ++i) {
					rgb[3 * i] = h[i] & 0xff;
					rgb[3 * i + 1] = (h[i] >> 8) & 0xff;
					rgb[3 * i + 2] = (h[i] >> 16) & 0xff;
				}
			}
		}
		return (int)UFO_B200_OK;
	});
}

}  // extern "C"

namespace
{
static_assert(sizeof(VolRec) == sizeof(ufo_b200_volume) && offsetof(ufo_b200_volume, v) == offsetof(VolRec, v),
              "ufo_b200_volume and VolRec must share their layout");

const VolRec* as_records(const ufo_b200_volume* bv) { return reinterpret_cast<const VolRec*>(bv); }

// the AABB record of a box6 (centre xyz, half size xyz)
VolRec aabb_record(const double* box6)
{
	VolRec r{};
	r.type = kVolAABB;
	for (int k = 0; k < 6; ++k) r.v[k] = box6[k];
	return r;
}

// a volume handed in through the C ABI: NULL only when empty, known shape types only
bool volume_ok(Map* m, const ufo_b200_volume* bv, size_t n_bv)
{
	if (n_bv && !bv) return false;
	if (n_bv > 0xffffffffull) {
		if (m) m->set_error("a bounding volume of %zu shapes is not supported (at most 2^32 - 1)", n_bv);
		return false;
	}
	for (size_t i = 0; i < n_bv; ++i) {
		if (bv[i].type >= kVolTypes) {
			if (m) m->set_error("bounding volume record %zu has the unknown type %u", i, bv[i].type);
			return false;
		}
	}
	return true;
}

// the records of a volume in device memory for the duration of one call
struct DeviceVolume {
	DevBuf recs;
	Volume upload(const Volume& host, cudaStream_t s)
	{
		Volume out = host;  // lo / hi travel as they are
		out.rec = nullptr;
		if (!host.n) return out;
		VolRec* d = recs.alloc<VolRec>(host.n);
		CK(cudaMemcpyAsync(d, host.rec, sizeof(VolRec) * host.n, cudaMemcpyHostToDevice, s));
		out.rec = d;
		return out;
	}
};

// ---- file image (ufo_export.cuh): the levels above the bricks, on the host ----
struct UpNode {
	int32_t child[8];  // -1: absent; >= 0: index into nodes (depth > 5) or into the sorted brick list (depth 5)
	uint8_t mask;      // children written as records (they have children and lie above min_depth)
	uint8_t hit;       // children whose cube intersects the export box
	bool has;          // false: collapsed to a leaf (canonical export only)
	float occ;
	uint32_t rgb;
	unsigned long long size;  // bytes of the node's record
};

struct ExportPlan {
	std::vector<uint32_t> order;  // bricks in Morton (= stream) order, as indices into info
	const BrickInfo* info = nullptr;
	std::vector<UpNode> nodes;    // nodes[0] = root (if any brick exists)
	const unsigned long long* codes = nullptr;  // Morton code of brick order[i]
	uint32_t P = 4;
	uint32_t levels = 16;
	uint32_t min_depth = 0;
	bool pruned = false;
	Volume vol{nullptr, 0, {}, {}};  // host records
	const Geometry* g = nullptr;
};

unsigned long long spread3_host(unsigned long long v)
{
	unsigned long long r = 0;
	for (int i = 0; i < 21; ++i) r |= ((v >> i) & 1ull) << (3 * i);
	return r;
}

// builds the node of depth d (centre c) that covers order[lo, hi); returns its index in plan.nodes
int32_t build_upper(ExportPlan& plan, uint32_t d, size_t lo, size_t hi, const double c[3])
{
	const int32_t self = (int32_t)plan.nodes.size();
	plan.nodes.push_back(UpNode{});
	UpNode n{};
	n.has = true;
	n.size = 1;
	const uint32_t shift = 3 * (d - 5);  // child index of a depth-d node inside the brick code
	const double chs = plan.g->half_size[d - 1];
	float occ[8];
	uint32_t rgb[8];
	bool any_children = false;
	size_t pos = lo;
	for (uint32_t i = 0; i < 8; ++i) {
		size_t end = pos;
		while (end < hi && ((plan.codes[end] >> shift) & 7ull) == i) ++end;
		double cc[3];
		child_center(c, chs, i, cc);
		const bool hit = vol_hits(plan.vol, cc, chs);
		if (hit) n.hit |= (uint8_t)(1u << i);
		n.child[i] = -1;
		occ[i] = 0.0f;
		rgb[i] = 0;
		unsigned long long bytes = plan.P;  // absent child: one default payload
		if (end > pos) {
			if (d == 5) {
				const BrickInfo& bi = plan.info[plan.order[pos]];
				n.child[i] = (int32_t)pos;
				occ[i] = bi.occ;
				rgb[i] = bi.rgb;
				if (bi.flags & 1u) {
					any_children = true;
					if (plan.min_depth < 4) n.mask |= (uint8_t)(1u << i);
				}
				bytes = bi.size;  // 0 when the brick's cube misses the box (same test on the device)
			} else {
				const int32_t ci = build_upper(plan, d - 1, pos, end, cc);
				const UpNode& ch = plan.nodes[ci];
				n.child[i] = ci;
				occ[i] = ch.occ;
				rgb[i] = ch.rgb;
				if (ch.has) {
					any_children = true;
					n.mask |= (uint8_t)(1u << i);  // d - 1 >= 5 > min_depth
					bytes = ch.size;
				}
			}
		}
		if (hit) n.size += bytes;
		pos = end;
	}
	if (plan.pruned) n.has = keeps_children(any_children, occ, rgb);
	n.occ = occ[0];  // payload if collapsed
	n.rgb = rgb[0];
	plan.nodes[self] = n;
	return self;
}

template <class Sink>
void put_payload_host(Sink& sink, uint32_t P, float occ, uint32_t rgb)
{
	uint8_t b[7];
	std::memcpy(b, &occ, 4);
	b[4] = (uint8_t)rgb;
	b[5] = (uint8_t)(rgb >> 8);
	b[6] = (uint8_t)(rgb >> 16);
	sink(b, P);
}

// rec[i]: the stream bytes of brick info[i] when it is written as a record
template <class Sink>
void emit_upper(const ExportPlan& plan, const std::vector<const uint8_t*>& rec, int32_t idx, uint32_t d, Sink& sink)
{
	const UpNode& n = plan.nodes[idx];
	sink(&n.mask, 1);
	for (uint32_t i = 0; i < 8; ++i) {
		if (!((n.hit >> i) & 1u)) continue;
		const int32_t c = n.child[i];
		if (c < 0) {
			put_payload_host(sink, plan.P, 0.0f, 0u);
		} else if (d == 5) {
			const uint32_t slot = plan.order[c];
			const BrickInfo& bi = plan.info[slot];
			if (bi.size == 0) continue;
			if (bi.flags & 4u) sink(rec[slot], bi.size);
			else put_payload_host(sink, plan.P, bi.occ, bi.rgb);
		} else if (plan.nodes[c].has) {
			emit_upper(plan, rec, c, d - 1, sink);
		} else {
			put_payload_host(sink, plan.P, plan.nodes[c].occ, plan.nodes[c].rgb);
		}
	}
}

// octree.h:850-860; doubles print with the default ostream precision = %g
int image_header(char* head, size_t cap, bool color, double resolution, uint32_t levels, bool compressed,
                 unsigned long long data_size)
{
	return snprintf(head, cap,
	                "# UFOMap file\n# (feel free to add / change comments, but leave the first line as it "
	                "is!)\n#\nversion 1.0.0\nid %s\nresolution %g\ndepth_levels %u\ncompressed %d\n"
	                "uncompressed_data_size %d\ndata\n",
	                color ? "occupancy_map_color" : "occupancy_map", resolution, levels, compressed ? 1 : 0, (int)data_size);
}

// One map's share of a file image for (volume, min_depth, pruned): the bricks that are part of the
// tree, ascending by Morton code, with their BrickInfo (k_brick_stream) and the stream bytes of those
// written as records.  Everything above the bricks is a function of these alone (build_upper), so
// the image of a union of maps that hold disjoint bricks -- the ranks of a routed map -- is the
// image of the union of their parts.
struct ImagePart {
	uint32_t color = 0, depth_levels = 0, min_depth = 0, pruned = 1;
	double resolution = 0.0;
	std::vector<VolRec> vol;                // the volume records as given (reserved = 0)
	std::vector<unsigned long long> codes;  // brick codes (Morton code of the brick key), ascending
	std::vector<BrickInfo> info;
	const uint8_t* stream = nullptr;  // record bytes of the bricks with info.flags & 4, in order
	size_t stream_bytes = 0;
	std::vector<uint8_t> own;  // the stream of a part made from a map
};

// The map's part (the device work of the file writers: both passes of k_brick_stream).
int make_part(Map* m, int pruned, uint32_t min_depth, const Volume& vol, ImagePart& part)
{
	if (m->device == -2) return UFO_B200_E_CUDA;
	if (m->M.g.depth_levels < 5) {
		m->set_error("export needs depth_levels >= 5");
		return UFO_B200_E_UNSUPPORTED;
	}
	if (min_depth > 4) {
		m->set_error("export with min_depth %u > 4 is not supported", min_depth);
		return UFO_B200_E_UNSUPPORTED;
	}
	CK(cudaSetDevice(m->device));
	sync_map(m);
	cudaStream_t s = m->stream;
	const uint32_t nb = m->n_bricks;
	const bool color = m->M.color != 0;
	part.color = color ? 1u : 0u;
	part.depth_levels = m->M.g.depth_levels;
	part.min_depth = min_depth;
	part.pruned = pruned ? 1u : 0u;
	part.resolution = m->M.g.resolution;
	part.vol.assign(vol.rec, vol.rec + vol.n);
	for (VolRec& r : part.vol) r.reserved = 0;
	const double c0[3] = {0.0, 0.0, 0.0};
	// "No node intersects": the reference writes no node data at all (OMB:1462-1468)
	if (!vol_hits(vol, c0, m->M.g.half_size[part.depth_levels])) return UFO_B200_OK;
	std::vector<BrickInfo> info(nb);
	std::vector<unsigned long long> keys(nb);
	DevBuf b_info, b_offs, b_out;
	BrickInfo* d_info = nullptr;
	DeviceVolume dvol;
	// an empty or single-box volume takes the instantiation with the inline box test
	Volume hv = vol;
	const bool general = volume_is_general(hv);
	const Volume dv = dvol.upload(hv, s);
	auto brick_stream = [&](uint32_t n, size_t smem, const unsigned long long* offs, uint8_t* out) {
		if (color && general) k_brick_stream<true, true><<<n, 64, smem, s>>>(m->M, n, pruned, min_depth, dv, d_info, offs, out);
		else if (color) k_brick_stream<true, false><<<n, 64, smem, s>>>(m->M, n, pruned, min_depth, dv, d_info, offs, out);
		else if (general) k_brick_stream<false, true><<<n, 64, smem, s>>>(m->M, n, pruned, min_depth, dv, d_info, offs, out);
		else k_brick_stream<false, false><<<n, 64, smem, s>>>(m->M, n, pruned, min_depth, dv, d_info, offs, out);
	};
	if (nb) {
		d_info = b_info.alloc<BrickInfo>(nb);
		brick_stream(nb, 0, nullptr, nullptr);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(info.data(), d_info, sizeof(BrickInfo) * nb, cudaMemcpyDeviceToHost, s));
		CK(cudaMemcpyAsync(keys.data(), m->M.brick_key, 8ull * nb, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
	}
	// bricks that are part of the tree, in Morton order; a leaf brick with the default payload is
	// indistinguishable from untouched space (so are the empty foreign bricks a routed rank keeps)
	std::vector<std::pair<unsigned long long, uint32_t>> sorted;
	sorted.reserve(nb);
	for (uint32_t b = 0; b < nb; ++b) {
		const BrickInfo& bi = info[b];
		if (bi.flags & 2u) continue;
		if (!(bi.flags & 1u) && bi.occ == 0.0f && bi.rgb == 0u) continue;
		uint32_t x, y, z;
		unpack_key(keys[b], x, y, z);
		sorted.emplace_back(spread3_host(x) | (spread3_host(y) << 1) | (spread3_host(z) << 2), b);
	}
	std::sort(sorted.begin(), sorted.end());
	part.codes.resize(sorted.size());
	part.info.resize(sorted.size());
	std::vector<unsigned long long> offs(nb, ~0ull);
	unsigned long long packed_bytes = 0;
	for (size_t i = 0; i < sorted.size(); ++i) {
		part.codes[i] = sorted[i].first;
		const BrickInfo& bi = info[sorted[i].second];
		part.info[i] = bi;
		if (bi.flags & 4u) {
			offs[sorted[i].second] = packed_bytes;
			packed_bytes += bi.size;
		}
	}
	part.own.resize(packed_bytes);
	if (packed_bytes) {
		unsigned long long* d_offs = b_offs.alloc<unsigned long long>(nb);
		uint8_t* d_out = b_out.alloc<uint8_t>(packed_bytes);
		CK(cudaMemcpyAsync(d_offs, offs.data(), 8ull * nb, cudaMemcpyHostToDevice, s));
		brick_stream(nb, kBrickStreamMax, d_offs, d_out);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(part.own.data(), d_out, packed_bytes, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
	}
	part.stream = part.own.data();
	part.stream_bytes = packed_bytes;
	return UFO_B200_OK;
}

bool same_image(const ImagePart& a, const ImagePart& b)
{
	return a.color == b.color && a.depth_levels == b.depth_levels && a.min_depth == b.min_depth && a.pruned == b.pruned &&
	       std::memcmp(&a.resolution, &b.resolution, sizeof(double)) == 0 && a.vol.size() == b.vol.size() &&
	       (a.vol.empty() || std::memcmp(a.vol.data(), b.vol.data(), sizeof(VolRec) * a.vol.size()) == 0);
}

// The image of the union of the parts through sink(ptr, len) calls, in order: the file image when
// with_header, else the bare node stream.  The parts must agree on everything but their bricks, and
// no brick may be in two of them (UFO_B200_E_INVALID).  *total = bytes produced, *data = bytes of the
// node stream among them.
template <class Sink>
int assemble(const std::vector<const ImagePart*>& parts, bool with_header, Sink&& sink, unsigned long long* total,
             unsigned long long* data = nullptr)
{
	*total = 0;
	if (data) *data = 0;
	if (parts.empty()) return UFO_B200_E_INVALID;
	const ImagePart& h = *parts[0];
	for (const ImagePart* p : parts)
		if (!same_image(*p, h)) return UFO_B200_E_INVALID;
	const Geometry g = make_geometry(h.resolution, h.depth_levels);
	ExportPlan plan;
	plan.P = h.color ? 7 : 4;
	plan.levels = h.depth_levels;
	plan.min_depth = h.min_depth;
	plan.pruned = h.pruned != 0;
	plan.g = &g;
	plan.vol = Volume{h.vol.data(), (uint32_t)h.vol.size(), {}, {}};
	const double c0[3] = {0.0, 0.0, 0.0};
	if (!vol_hits(plan.vol, c0, g.half_size[plan.levels])) {
		if (with_header) {
			char head[512];
			const int hl = image_header(head, sizeof head, h.color, h.resolution, plan.levels, false, 0);
			sink(head, (size_t)hl);
			*total = (unsigned long long)hl;
		}
		return UFO_B200_OK;
	}
	// the bricks of all parts in Morton order; rec[i]: stream bytes of brick i
	std::vector<BrickInfo> merged;
	std::vector<unsigned long long> merged_codes;
	std::vector<const uint8_t*> rec;
	if (parts.size() == 1) {
		plan.info = h.info.data();
		plan.codes = h.codes.data();
		rec.resize(h.info.size());
		const uint8_t* at = h.stream;
		for (size_t i = 0; i < h.info.size(); ++i) {
			rec[i] = at;
			if (h.info[i].flags & 4u) at += h.info[i].size;
		}
	} else {
		std::vector<std::pair<unsigned long long, std::pair<const BrickInfo*, const uint8_t*>>> all;
		size_t n = 0;
		for (const ImagePart* p : parts) n += p->codes.size();
		all.reserve(n);
		for (const ImagePart* p : parts) {
			const uint8_t* at = p->stream;
			for (size_t i = 0; i < p->codes.size(); ++i) {
				all.push_back({p->codes[i], {&p->info[i], at}});
				if (p->info[i].flags & 4u) at += p->info[i].size;
			}
		}
		std::sort(all.begin(), all.end(), [](const auto& a, const auto& b) { return a.first < b.first; });
		for (size_t i = 1; i < all.size(); ++i)
			if (all[i].first == all[i - 1].first) return UFO_B200_E_INVALID;  // two histories of one brick
		merged_codes.resize(n);
		merged.resize(n);
		rec.resize(n);
		for (size_t i = 0; i < n; ++i) {
			merged_codes[i] = all[i].first;
			merged[i] = *all[i].second.first;
			rec[i] = all[i].second.second;
		}
		plan.info = merged.data();
		plan.codes = merged_codes.data();
	}
	const size_t nb = rec.size();
	plan.order.resize(nb);
	std::iota(plan.order.begin(), plan.order.end(), 0u);
	bool root_has = false;
	unsigned long long data_size = 1 + plan.P;  // children byte + root payload
	if (nb) {
		build_upper(plan, plan.levels, 0, nb, c0);
		root_has = plan.nodes[0].has;
		if (root_has) data_size = 1 + plan.nodes[0].size;
	}
	unsigned long long produced = 0;
	auto counted = [&](const void* p, size_t len) {
		sink(p, len);
		produced += len;
	};
	if (with_header) {
		char head[512];
		const int hl = image_header(head, sizeof head, h.color, h.resolution, plan.levels, false, data_size);
		counted(head, (size_t)hl);
	}
	const unsigned long long head_bytes = produced;
	const uint8_t children = root_has ? 0xff : 0x00;
	counted(&children, 1);
	if (root_has) {
		emit_upper(plan, rec, 0, plan.levels, counted);
	} else {
		const float occ = nb ? plan.nodes[0].occ : 0.0f;
		const uint32_t rgb = nb ? plan.nodes[0].rgb : 0u;
		put_payload_host(counted, plan.P, occ, rgb);
	}
	*total = produced;
	if (data) *data = produced - head_bytes;
	return UFO_B200_OK;
}

// the map's image through sink: its part, assembled alone
template <class Sink>
int export_image(Map* m, int pruned, uint32_t min_depth, const Volume& vol, bool with_header, Sink&& sink,
                 unsigned long long* total)
{
	*total = 0;
	ImagePart part;
	const int rc = make_part(m, pruned, min_depth, vol, part);
	if (rc != UFO_B200_OK) return rc;
	return assemble({&part}, with_header, sink, total);
}
}  // namespace

namespace
{
// LZ4 block API of the system's liblz4 (the reference links it: octree.h:1428-1486), loaded on
// first use so that the library does not depend on LZ4 development files.
struct Lz4 {
	int (*bound)(int) = nullptr;
	int (*fast)(const char*, char*, int, int, int) = nullptr;
	int (*hc)(const char*, char*, int, int, int) = nullptr;
	int (*decompress)(const char*, char*, int, int) = nullptr;
	bool ok = false;
};

const Lz4& lz4()
{
	static Lz4 api = []() {
		Lz4 a;
		void* h = dlopen("liblz4.so.1", RTLD_NOW | RTLD_LOCAL);
		if (!h) h = dlopen("liblz4.so", RTLD_NOW | RTLD_LOCAL);
		if (h) {
			a.bound = reinterpret_cast<int (*)(int)>(dlsym(h, "LZ4_compressBound"));
			a.fast = reinterpret_cast<int (*)(const char*, char*, int, int, int)>(dlsym(h, "LZ4_compress_fast"));
			a.hc = reinterpret_cast<int (*)(const char*, char*, int, int, int)>(dlsym(h, "LZ4_compress_HC"));
			a.decompress = reinterpret_cast<int (*)(const char*, char*, int, int)>(dlsym(h, "LZ4_decompress_safe"));
			a.ok = a.bound && a.fast && a.hc && a.decompress;
		}
		return a;
	}();
	return api;
}

// compressData (octree.h:1428-1456): the whole node stream as ONE LZ4 block
bool lz4_compress(const std::vector<uint8_t>& in, int acceleration, int level, std::vector<uint8_t>& out)
{
	const Lz4& z = lz4();
	if (!z.ok || in.size() > 0x7e000000u) return false;
	const int cap = z.bound((int)in.size());
	out.resize((size_t)std::max(cap, 1));
	const int n = level <= 0 ? z.fast(reinterpret_cast<const char*>(in.data()), reinterpret_cast<char*>(out.data()), (int)in.size(), cap, acceleration)
	                         : z.hc(reinterpret_cast<const char*>(in.data()), reinterpret_cast<char*>(out.data()), (int)in.size(), cap, level);
	if (n < 0) return false;
	out.resize((size_t)n);
	return true;
}

// The image of the parts into buf (*size = its bytes; copied only when it fits into cap): the file
// image (with_header) or the bare node stream; compress: the node stream as one LZ4 block, behind
// the header with "compressed 1" when with_header.  *uncompressed_size = bytes of the node stream.
int image_to_buffer(const std::vector<const ImagePart*>& parts, bool with_header, bool compress, int acceleration, int level,
                    void* buf, size_t cap, size_t* size, size_t* uncompressed_size, Map* m)
{
	std::vector<uint8_t> raw;
	unsigned long long total = 0, data = 0;
	const int rc = assemble(parts, with_header && !compress, [&](const void* p, size_t len) {
		const uint8_t* b = static_cast<const uint8_t*>(p);
		raw.insert(raw.end(), b, b + len);
	}, &total, &data);
	if (rc != UFO_B200_OK) return rc;
	std::vector<uint8_t> packed;
	std::string head;
	if (compress) {
		if (!lz4_compress(raw, acceleration, level, packed)) {
			if (m) m->set_error("LZ4 compression failed");
			return UFO_B200_E_INVALID;
		}
		if (with_header) {
			const ImagePart& p = *parts[0];
			char h[512];
			const int hl = image_header(h, sizeof h, p.color != 0, p.resolution, p.depth_levels, true, raw.size());
			head.assign(h, (size_t)hl);
		}
	}
	const std::vector<uint8_t>& body = compress ? packed : raw;
	const size_t need = head.size() + body.size();
	*size = need;
	if (uncompressed_size) *uncompressed_size = (size_t)data;
	if (buf && cap >= need) {
		std::memcpy(buf, head.data(), head.size());
		std::memcpy(static_cast<uint8_t*>(buf) + head.size(), body.data(), body.size());
	}
	return UFO_B200_OK;
}

// ---- a part as bytes (ufo_b200_image_part_bv): header, volume records, {code, BrickInfo} per brick
// ascending, then the record bytes.  Little-endian, as the devices that make it.
constexpr uint32_t kPartMagic = 0x50494655u;  // "UFIP"
constexpr uint32_t kPartVersion = 1;

struct PartHeader {
	uint32_t magic, version, color, depth_levels, min_depth, pruned;
	uint64_t resolution_bits, n_bv, n_bricks, stream_bytes;
};
static_assert(sizeof(PartHeader) == 56, "the part header stays 56 bytes");

struct PartBrick {
	uint64_t code;
	BrickInfo info;
};
static_assert(sizeof(PartBrick) == 24, "a part's brick entry stays 24 bytes");

size_t part_bytes(const ImagePart& p)
{
	return sizeof(PartHeader) + sizeof(VolRec) * p.vol.size() + sizeof(PartBrick) * p.codes.size() + p.stream_bytes;
}

void put_part(const ImagePart& p, uint8_t* out)
{
	PartHeader h{kPartMagic, kPartVersion, p.color, p.depth_levels, p.min_depth, p.pruned, 0, p.vol.size(), p.codes.size(), p.stream_bytes};
	std::memcpy(&h.resolution_bits, &p.resolution, 8);
	std::memcpy(out, &h, sizeof h);
	out += sizeof h;
	if (!p.vol.empty()) std::memcpy(out, p.vol.data(), sizeof(VolRec) * p.vol.size());
	out += sizeof(VolRec) * p.vol.size();
	for (size_t i = 0; i < p.codes.size(); ++i) {
		const PartBrick b{p.codes[i], p.info[i]};
		std::memcpy(out, &b, sizeof b);
		out += sizeof b;
	}
	if (p.stream_bytes) std::memcpy(out, p.stream, p.stream_bytes);
}

// A part as put_part wrote it, or false: every field in range, sizes that add up, brick codes inside
// the tree and strictly ascending, BrickInfo of the shapes k_brick_stream produces.  The stream stays
// in the caller's blob.
bool parse_part(const void* blob, size_t size, ImagePart& p)
{
	if (!blob || size < sizeof(PartHeader)) return false;
	const uint8_t* b = static_cast<const uint8_t*>(blob);
	PartHeader h;
	std::memcpy(&h, b, sizeof h);
	if (h.magic != kPartMagic || h.version != kPartVersion) return false;
	if (h.color > 1 || h.pruned > 1 || h.min_depth > 4 || h.depth_levels < 5 || h.depth_levels > 21) return false;
	double res;
	std::memcpy(&res, &h.resolution_bits, 8);
	if (!(res > 0.0) || !std::isfinite(res)) return false;
	size_t rest = size - sizeof h;
	if (h.n_bv > 0xffffffffull || h.n_bv > rest / sizeof(VolRec)) return false;
	rest -= (size_t)h.n_bv * sizeof(VolRec);
	if (h.n_bricks > rest / sizeof(PartBrick)) return false;
	rest -= (size_t)h.n_bricks * sizeof(PartBrick);
	if (h.stream_bytes != rest) return false;
	p.color = h.color;
	p.depth_levels = h.depth_levels;
	p.min_depth = h.min_depth;
	p.pruned = h.pruned;
	p.resolution = res;
	b += sizeof h;
	p.vol.resize((size_t)h.n_bv);
	if (h.n_bv) std::memcpy(p.vol.data(), b, sizeof(VolRec) * (size_t)h.n_bv);
	for (const VolRec& r : p.vol)
		if (r.type >= kVolTypes) return false;
	b += sizeof(VolRec) * (size_t)h.n_bv;
	const unsigned long long code_end = 1ull << (3 * (h.depth_levels - 4));
	const uint32_t P = h.color ? 7u : 4u;
	unsigned long long record_bytes = 0;
	p.codes.resize((size_t)h.n_bricks);
	p.info.resize((size_t)h.n_bricks);
	for (size_t i = 0; i < p.codes.size(); ++i) {
		PartBrick e;
		std::memcpy(&e, b + i * sizeof e, sizeof e);
		if (e.code >= code_end || (i && e.code <= p.codes[i - 1])) return false;
		if (e.info.flags == 5u) {
			if (e.info.size == 0 || e.info.size > (uint32_t)kBrickStreamMax) return false;
			record_bytes += e.info.size;
		} else if (e.info.flags > 1u || (e.info.size != 0 && e.info.size != P)) {
			return false;
		}
		p.codes[i] = e.code;
		p.info[i] = e.info;
	}
	if (record_bytes != h.stream_bytes) return false;
	p.stream = b + sizeof(PartBrick) * p.codes.size();
	p.stream_bytes = (size_t)h.stream_bytes;
	return true;
}
}  // namespace

namespace
{
// the rejections shared by the two setValueVolume entry points
int set_value_volume_allowed(Map* m, uint32_t min_depth)
{
	if (min_depth > 4 || m->M.g.depth_levels < 5) {
		m->set_error("setValueVolume: min_depth %u > 4 (or depth_levels < 5) is not supported", min_depth);
		return UFO_B200_E_UNSUPPORTED;
	}
	if (m->M.color && min_depth > 0) {
		m->set_error("setValueVolume on a colour map is supported at min_depth 0 only");
		return UFO_B200_E_UNSUPPORTED;
	}
	if (m->M.shard_world > 1) {
		m->set_error("setValueVolume on a sharded map is not supported");
		return UFO_B200_E_UNSUPPORTED;
	}
	if (m->route_stage == 1) {
		m->set_error("setValueVolume between ufo_b200_route_mark and the last ufo_b200_route_apply of the pass");
		return UFO_B200_E_INVALID;
	}
	return UFO_B200_OK;
}

// marks the volume's voxels (k_volume_mark over the candidate bricks of v) and sets them to
// clamp(float(logit(occupancy))): setOccupancy(LogitType&, LogitType const&), OMB:1151-1157
int set_value_volume_run(Map* m, const VolumeArgs& v, double occupancy)
{
	const float lo = (float)m->cmin_log, hi = (float)m->cmax_log;
	float value = (float)to_logit(occupancy);
	value = value < lo ? lo : (hi < value ? hi : value);
	const double origin[3] = {0.0, 0.0, 0.0};
	return do_insert(m, origin, nullptr, false, 0, nullptr, UFO_B200_XYZ_F64, -1.0, 0, 0, 0, 0, 0, nullptr, &v, value);
}

constexpr uint32_t kVolumeBrickLimit = 1u << 22;
}  // namespace

extern "C" {

int ufo_b200_set_value_volume(ufo_b200_map* m, const double box6[6], double occupancy, uint32_t min_depth)
{
	if (!m || !box6) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		bump_revision(m);
		const int allowed = set_value_volume_allowed(m, min_depth);
		if (allowed != UFO_B200_OK) return allowed;
		const Geometry& g = m->M.g;
		const VolRec rec = aabb_record(box6);
		const Volume hv{&rec, 1, {}, {}};
		const double c0[3] = {0.0, 0.0, 0.0};
		if (!vol_hits(hv, c0, g.half_size[g.depth_levels])) return (int)UFO_B200_OK;  // no node intersects
		// candidate bricks: the key range of the box, one brick of slack on every side (the kernel
		// decides with the reference's own cube tests)
		const double ext = g.half_size[g.depth_levels];
		const long long top = (1ll << (g.depth_levels - 4)) - 1;
		uint32_t first[3], count[3];
		unsigned long long total = 1;
		for (int k = 0; k < 3; ++k) {
			const double blo = box6[k] - box6[3 + k], bhi = box6[k] + box6[3 + k];
			const double lo = std::max(blo, -ext), hi = std::min(bhi, ext);
			long long a = ((long long)std::floor(lo * g.resolution_factor) + (long long)g.max_value) >> 4;
			long long b = ((long long)std::floor(hi * g.resolution_factor) + (long long)g.max_value) >> 4;
			a = std::min(std::max(a - 1, 0ll), top);
			b = std::min(std::max(b + 1, 0ll), top);
			first[k] = (uint32_t)a;
			count[k] = (uint32_t)(b - a + 1);
			total *= count[k];
		}
		if (total > kVolumeBrickLimit) {
			m->set_error("setValueVolume: the box covers %llu bricks (limit 4194304)", total);
			return (int)UFO_B200_E_UNSUPPORTED;
		}
		CK(cudaSetDevice(m->device));
		DeviceVolume dvol;
		VolumeArgs v{};
		Volume box = hv;
		volume_is_general(box);  // one AABB: lo / hi for the inline test
		v.vol = dvol.upload(box, m->stream);
		v.min_depth = min_depth;
		v.bx0 = first[0];
		v.by0 = first[1];
		v.bz0 = first[2];
		v.nx = count[0];
		v.ny = count[1];
		v.nz = count[2];
		return set_value_volume_run(m, v, occupancy);
	});
}

int ufo_b200_set_value_volume_bv(ufo_b200_map* m, const ufo_b200_volume* bv, double occupancy, uint32_t min_depth)
{
	if (!m || !bv) return UFO_B200_E_INVALID;
	// argument checks that need no device
	if (!volume_ok(m, bv, 1)) return UFO_B200_E_INVALID;
	const int allowed = set_value_volume_allowed(m, min_depth);
	if (allowed != UFO_B200_OK) return allowed;
	return guarded(m, [&]() {
		bump_revision(m);
		const Geometry& g = m->M.g;
		const Volume hv{as_records(bv), 1, {}, {}};
		const double c0[3] = {0.0, 0.0, 0.0};
		if (!vol_hits(hv, c0, g.half_size[g.depth_levels])) return (int)UFO_B200_OK;  // no node intersects
		CK(cudaSetDevice(m->device));
		sync_map(m);
		cudaStream_t s = m->stream;
		DeviceVolume dvol;
		Volume hvk = hv;
		const int general = volume_is_general(hvk) ? 1 : 0;
		const Volume dv = dvol.upload(hvk, s);
		// descent from the root to the bricks, one level per launch; frontier = (key, centre)
		DevBuf b_key[2], b_c[2], b_n;
		unsigned long long* d_key[2] = {b_key[0].alloc<unsigned long long>(1), nullptr};
		double* d_c[2] = {b_c[0].alloc<double>(3), nullptr};
		unsigned int* d_n = b_n.alloc<unsigned int>(1);
		int rc = UFO_B200_OK;
		CK(cudaMemsetAsync(d_key[0], 0, 8, s));
		CK(cudaMemsetAsync(d_c[0], 0, 24, s));
		uint32_t n_in = 1, cur = 0;
		for (uint32_t d = g.depth_levels; d > 4 && n_in; --d) {
			// children of depth d - 1
			const uint32_t cap = (uint32_t)std::min<unsigned long long>(8ull * n_in, kVolumeBrickLimit);
			const uint32_t nxt = cur ^ 1u;
			d_key[nxt] = b_key[nxt].alloc<unsigned long long>(cap);
			d_c[nxt] = b_c[nxt].alloc<double>(3ull * cap);
			CK(cudaMemsetAsync(d_n, 0, sizeof(unsigned int), s));
			const unsigned long long threads = 8ull * n_in;
			k_volume_descend<<<(uint32_t)((threads + 255) / 256), 256, 0, s>>>(dv, d_key[cur], d_c[cur], n_in, g.half_size[d - 1],
			                                                                    d_key[nxt], d_c[nxt], cap, d_n);
			CK(cudaGetLastError());
			unsigned int got = 0;
			CK(cudaMemcpyAsync(&got, d_n, sizeof(unsigned int), cudaMemcpyDeviceToHost, s));
			CK(cudaStreamSynchronize(s));
			b_key[cur].release();
			b_c[cur].release();
			if (got > kVolumeBrickLimit) {
				m->set_error("setValueVolume: %u nodes of depth %u pass the volume (limit 4194304)", got, d - 1);
				return (int)UFO_B200_E_UNSUPPORTED;
			}
			n_in = got;
			cur = nxt;
		}
		if (n_in) {
			VolumeArgs v{};
			v.vol = dv;
			v.min_depth = min_depth;
			v.nx = n_in;
			v.ny = 1;
			v.nz = 1;
			v.cand = d_key[cur];
			v.general = general;
			rc = set_value_volume_run(m, v, occupancy);
			sync_map(m);
		}
		return rc;
	});
}

int ufo_b200_write_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, uint32_t min_depth, int expanded,
                      void* buf, size_t cap, size_t* size)
{
	if (!m || !size) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		uint8_t* out = static_cast<uint8_t*>(buf);
		size_t at = 0;
		unsigned long long total = 0;
		int rc = export_image(m, expanded ? 0 : 1, min_depth, Volume{as_records(bv), (uint32_t)n_bv, {}, {}}, true,
		                      [&](const void* p, size_t len) {
			                      if (out && at + len <= cap) std::memcpy(out + at, p, len);
			                      at += len;
		                      },
		                      &total);
		*size = (size_t)total;
		return rc;
	});
}

int ufo_b200_write(ufo_b200_map* m, const double* box6, uint32_t min_depth, int expanded, void* buf, size_t cap,
                   size_t* size)
{
	const VolRec r = box6 ? aabb_record(box6) : VolRec{};
	return ufo_b200_write_bv(m, reinterpret_cast<const ufo_b200_volume*>(&r), box6 ? 1 : 0, min_depth, expanded, buf, cap, size);
}

int ufo_b200_write_data_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, uint32_t min_depth, void* buf,
                           size_t cap, size_t* size)
{
	if (!m || !size) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		uint8_t* out = static_cast<uint8_t*>(buf);
		size_t at = 0;
		unsigned long long total = 0;
		int rc = export_image(m, 1, min_depth, Volume{as_records(bv), (uint32_t)n_bv, {}, {}}, false,
		                      [&](const void* p, size_t len) {
			                      if (out && at + len <= cap) std::memcpy(out + at, p, len);
			                      at += len;
		                      },
		                      &total);
		*size = (size_t)total;
		return rc;
	});
}

int ufo_b200_write_data(ufo_b200_map* m, const double* box6, uint32_t min_depth, void* buf, size_t cap,
                        size_t* size)
{
	const VolRec r = box6 ? aabb_record(box6) : VolRec{};
	return ufo_b200_write_data_bv(m, reinterpret_cast<const ufo_b200_volume*>(&r), box6 ? 1 : 0, min_depth, buf, cap, size);
}

int ufo_b200_write_file(ufo_b200_map* m, const char* filename, const double* box6, uint32_t min_depth,
                        int expanded)
{
	if (!m || !filename) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		FILE* f = fopen(filename, "wb");
		if (!f) {
			m->set_error("cannot open %s", filename);
			return (int)UFO_B200_E_INVALID;
		}
		const VolRec r = box6 ? aabb_record(box6) : VolRec{};
		unsigned long long total = 0;
		bool ok = true;
		int rc = export_image(m, expanded ? 0 : 1, min_depth, Volume{&r, box6 ? 1u : 0u, {}, {}}, true,
		                      [&](const void* p, size_t len) { ok = ok && fwrite(p, 1, len, f) == len; }, &total);
		ok = fclose(f) == 0 && ok;
		if (rc == UFO_B200_OK && !ok) {
			m->set_error("short write to %s", filename);
			return (int)UFO_B200_E_INVALID;
		}
		return rc;
	});
}

int ufo_b200_set_sensor_model(ufo_b200_map* m, const double p[6])
{
	if (!m || !p) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		bump_revision(m);
		sync_map(m);
		m->occ_thr_log = to_logit(p[0]);
		m->free_thr_log = to_logit(p[1]);
		m->hit_log = to_logit(p[2]);
		m->miss_log = to_logit(p[3]);
		m->cmin_log = to_logit(p[4]);
		m->cmax_log = to_logit(p[5]);
		refresh_model(m);
		rebuild_flags(m);
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_set_sensor_model_field(ufo_b200_map* m, int index, double probability)
{
	if (!m || index < 0 || index > 5) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		bump_revision(m);
		sync_map(m);
		double* field[6] = {&m->occ_thr_log, &m->free_thr_log, &m->hit_log, &m->miss_log, &m->cmin_log, &m->cmax_log};
		*field[index] = to_logit(probability);
		refresh_model(m);
		if (index <= 1) rebuild_flags(m);
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_sensor_model_logit(const ufo_b200_map* m, double o[6])
{
	if (!m || !o) return UFO_B200_E_INVALID;
	o[0] = m->occ_thr_log;
	o[1] = m->free_thr_log;
	o[2] = m->hit_log;
	o[3] = m->miss_log;
	o[4] = m->cmin_log;
	o[5] = m->cmax_log;
	return UFO_B200_OK;
}

int ufo_b200_change_bbox(ufo_b200_map* m, double mn[3], double mx[3])
{
	if (!m || !mn || !mx) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		sync_map(m);
		memcpy(mn, m->min_change, sizeof(m->min_change));
		memcpy(mx, m->max_change, sizeof(m->max_change));
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_reset_change_bbox(ufo_b200_map* m)
{
	if (!m) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		sync_map(m);
		reset_bbox(m);
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_last_scan_stats(ufo_b200_map* m, ufo_b200_scan_stats* out)
{
	if (!m || !out) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		sync_map(m);
		*out = m->stats;
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_last_walk_stats(ufo_b200_map* m, ufo_b200_walk_stats* out)
{
	if (!m || !out) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		sync_map(m);
		*out = m->walk_stats;
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_last_update_stats(ufo_b200_map* m, ufo_b200_update_stats* out)
{
	if (!m || !out) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		sync_map(m);
		*out = m->update_stats;
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_completed_scan_stats(ufo_b200_map* m, ufo_b200_scan_stats* out)
{
	if (!m || !out) return UFO_B200_E_INVALID;
	*out = m->done_stats;
	return UFO_B200_OK;
}

int ufo_b200_last_early_stats(ufo_b200_map* m, ufo_b200_early_stats* out)
{
	if (!m || !out) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		sync_map(m);
		*out = m->early_stats;
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_set_early_stopping(ufo_b200_map* m, int exact)
{
	if (!m) return UFO_B200_E_INVALID;
	if (exact != 0 && exact != 1) {
		m->set_error("ufo_b200_set_early_stopping: exact must be 0 or 1, got %d", exact);
		return UFO_B200_E_INVALID;
	}
	m->early_exact = exact;  // read when a scan is enqueued: the scan in flight keeps its own setting
	return UFO_B200_OK;
}

int ufo_b200_set_profiling(ufo_b200_map* m, int enable)
{
	if (!m) return UFO_B200_E_INVALID;
	m->profiling = enable < 0 ? 0 : enable;
	return UFO_B200_OK;
}

int ufo_b200_set_shard(ufo_b200_map* m, uint32_t rank, uint32_t world)
{
	if (!m || (world > 1 && rank >= world)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		bump_revision(m);
		sync_map(m);
		if (m->n_bricks != 0) {
			m->set_error("ufo_b200_set_shard must be called on an empty map");
			return (int)UFO_B200_E_INVALID;
		}
		m->M.shard_rank = world > 1 ? rank : 0;
		m->M.shard_world = world > 1 ? world : 1;
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_clear(ufo_b200_map* m)
{
	if (!m) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		bump_revision(m);
		CK(cudaSetDevice(m->device));
		try {
			sync_map(m);
		} catch (MapError&) {
			// a scan that failed half-way: its marks are wiped below
		}
		DeviceMap& M = m->M;
		cudaStream_t s = m->stream;
		CK(cudaMemsetAsync(M.bh_tab, 0xff, ((size_t)M.bh_mask + 1) * sizeof(ulonglong2), s));
		CK(cudaMemsetAsync(M.uh_keys, 0xff, ((size_t)M.uh_mask + 1) * 8, s));
		CK(cudaMemsetAsync(M.uh_vals, 0xff, ((size_t)M.uh_mask + 1) * 4, s));
		CK(cudaMemsetAsync(M.brick_stamp, 0, (size_t)m->n_bricks * 4, s));
		CK(cudaMemsetAsync(M.hit_stamp, 0, (size_t)m->n_bricks * 4, s));
		CK(cudaMemsetAsync(M.up_stamp, 0, (size_t)m->n_upper * 4, s));
		CK(cudaMemsetAsync(M.up_valid, 0, (size_t)m->n_upper * 4, s));
		CK(cudaMemsetAsync(M.up_parent, 0xff, (size_t)m->n_upper * 4, s));
		CK(cudaMemsetAsync(M.brick_parent, 0xff, (size_t)m->n_bricks * 4, s));
		const size_t nb = (size_t)m->n_bricks * 64;
		CK(cudaMemsetAsync(M.leaf, 0, nb * 64 * 4, s));
		CK(cudaMemsetAsync(M.miss_mask, 0, nb * 8, s));
		CK(cudaMemsetAsync(M.hit_mask, 0, nb * 8, s));
		CK(cudaMemsetAsync(M.line_max, 0, nb * sizeof(float2), s));
		CK(cudaMemsetAsync(M.meta, 0, nb * 4, s));
		if (M.color) CK(cudaMemsetAsync(M.leaf_rgb, 0, nb * 64 * 4, s));
		if (M.alias_miss) {
			CK(cudaMemsetAsync(M.alias_miss, 0, nb * 8, s));
			CK(cudaMemsetAsync(M.alias_hit, 0, nb * 8, s));
		}
		if (M.chg_mask) CK(cudaMemsetAsync(M.chg_mask, 0, nb * 8, s));
		wipe_volume(m);
		m->n_blocks = 0;
		m->n_bricks = 0;
		m->n_upper = 0;
		M.scan_id = 0;
		M.up_epoch = 0;
		m->poisoned = false;
		m->route_stage = 0;
		reset_bbox(m);
		set_value_floor(m, fminf(0.0f, M.clamp_min));  // no leaf left
		CK(cudaStreamSynchronize(s));
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_clear_resize(ufo_b200_map* m, double resolution, uint32_t depth_levels)
{
	if (!m) return UFO_B200_E_INVALID;
	if (depth_levels < 2 || depth_levels > 21 || !(resolution > 0)) return UFO_B200_E_INVALID;  // octree.h:931-935
	int rc = ufo_b200_clear(m);
	if (rc != UFO_B200_OK) return rc;
	return guarded(m, [&]() {
		bump_revision(m);
		m->params.resolution = resolution;
		m->params.depth_levels = depth_levels;
		m->M.g = make_geometry(resolution, depth_levels);
		refresh_model(m);
		reset_bbox(m);
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_route_inbox_bytes(uint32_t world, uint32_t cap_bricks, uint32_t cap_hits, size_t* bytes)
{
	if (!bytes || world < 2 || world > kMaxRanks || !cap_bricks || !cap_hits) return UFO_B200_E_INVALID;
	*bytes = route_layout(world, cap_bricks, cap_hits, 1, nullptr, nullptr, nullptr);
	return UFO_B200_OK;
}

int ufo_b200_route_inbox_bytes_color(uint32_t world, uint32_t cap_bricks, uint32_t cap_hits, size_t* bytes)
{
	if (!bytes || world < 2 || world > kMaxRanks || !cap_bricks || !cap_hits) return UFO_B200_E_INVALID;
	*bytes = route_layout(world, cap_bricks, cap_hits, 2, nullptr, nullptr, nullptr);
	return UFO_B200_OK;
}

int ufo_b200_route_setup(ufo_b200_map* m, uint32_t rank, uint32_t world, uint32_t cap_bricks, uint32_t cap_hits,
                         void** inbox)
{
	if (!m || !inbox || world < 2 || world > kMaxRanks || rank >= world || !cap_bricks || !cap_hits) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		CK(cudaSetDevice(m->device));
		sync_map(m);
		if (m->n_bricks != 0 || m->route_inbox.p || m->M.shard_world > 1) {
			m->set_error("ufo_b200_route_setup: needs an empty, unsharded map and may be called once");
			return (int)UFO_B200_E_INVALID;
		}
		const uint32_t hit_words = m->M.color ? 2u : 1u;
		const size_t total = route_layout(world, cap_bricks, cap_hits, hit_words, &m->route_region, &m->route_miss_off,
		                                  &m->route_hit_off);
		m->route_inbox.ensure(m, total, 0);
		m->route_table.ensure(m, sizeof(RouteTable), 0);
		m->M.route = m->route_table.p;
		CK(cudaHostAlloc(reinterpret_cast<void**>(&m->h_route), sizeof(RouteTable), cudaHostAllocDefault));
		CK(cudaHostAlloc(reinterpret_cast<void**>(&m->h_route_flag), 4 * sizeof(uint32_t), cudaHostAllocDefault));
		memset(m->h_route_flag, 0, 4 * sizeof(uint32_t));
		if (m->M.color) {
			// apply table: every hit record of every source of one apply call, at most half full
			m->route_tab_size = std::max(1u << 12, next_pow2(2ull * world * cap_hits));
			m->d_route_tab_keys.ensure(m, (size_t)m->route_tab_size * sizeof(unsigned long long), 0xff);
			m->d_route_tab_min.ensure(m, (size_t)m->route_tab_size * sizeof(uint32_t), 0xff);
		}
		CK(cudaStreamSynchronize(m->stream));  // peers write into the inbox as soon as they have its handle
		m->route_cap_m = cap_bricks;
		m->route_cap_h = cap_hits;
		m->M.route_rank = rank;
		m->M.route_world = world;
		*inbox = m->route_inbox.p;
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_route_connect(ufo_b200_map* m, void* const* peer_inboxes)
{
	if (!m || !peer_inboxes || m->M.route_world < 2) return UFO_B200_E_INVALID;
	for (uint32_t r = 0; r < m->M.route_world; ++r) {
		if (!peer_inboxes[r]) return UFO_B200_E_INVALID;
		m->route_peer[r] = peer_inboxes[r];
	}
	return UFO_B200_OK;
}

int ufo_b200_route_mark(ufo_b200_map* m, const double origin[3], const void* points, size_t n, int layout,
                        double max_range, int on_device, int self_too)
{
	return guarded(m, [&]() {
		bump_revision(m);
		return do_route_mark(m, origin, points, on_device != 0, n, layout, max_range, 0, 0, 0, 0, 0, 1, self_too, false);
	});
}

int ufo_b200_route_mark_ex(ufo_b200_map* m, const double origin[3], const void* points, size_t n, int layout,
                           double max_range, uint32_t depth, int simple_ray_casting, uint32_t early_stopping,
                           int discrete, uint64_t index_base, uint32_t index_stride, int on_device, int self_too)
{
	return guarded(m, [&]() {
		bump_revision(m);
		return do_route_mark(m, origin, points, on_device != 0, n, layout, max_range, depth, simple_ray_casting,
		                     early_stopping, discrete, index_base, index_stride, self_too, true);
	});
}

int ufo_b200_route_sent(ufo_b200_map* m, uint32_t counts[3])
{
	if (!m || !counts) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		if (!m->h_route_flag) {
			m->set_error("routed mode is not set up");
			return (int)UFO_B200_E_INVALID;
		}
		CK(cudaSetDevice(m->device));
		CK(cudaStreamSynchronize(m->stream));
		for (int i = 0; i < 3; ++i) counts[i] = m->h_route_flag[1 + i];
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_route_apply(ufo_b200_map* m, uint32_t first_source, uint32_t n_sources, int last)
{
	return guarded(m, [&]() { bump_revision(m); return do_route_apply(m, first_source, n_sources, last); });
}

int ufo_b200_ipc_export(void* dev_ptr, void* handle64)
{
	if (!dev_ptr || !handle64) return UFO_B200_E_INVALID;
	static_assert(sizeof(cudaIpcMemHandle_t) == 64, "handle size");
	cudaIpcMemHandle_t h;
	if (cudaIpcGetMemHandle(&h, dev_ptr) != cudaSuccess) return UFO_B200_E_CUDA;
	memcpy(handle64, &h, 64);
	return UFO_B200_OK;
}

int ufo_b200_ipc_open(const void* handle64, void** dev_ptr)
{
	if (!handle64 || !dev_ptr) return UFO_B200_E_INVALID;
	cudaIpcMemHandle_t h;
	memcpy(&h, handle64, 64);
	if (cudaIpcOpenMemHandle(dev_ptr, h, cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) return UFO_B200_E_CUDA;
	return UFO_B200_OK;
}

int ufo_b200_ipc_close(void* dev_ptr)
{
	if (!dev_ptr) return UFO_B200_E_INVALID;
	return cudaIpcCloseMemHandle(dev_ptr) == cudaSuccess ? UFO_B200_OK : UFO_B200_E_CUDA;
}

int ufo_b200_enable_change_detection(ufo_b200_map* m, int enable)
{
	if (!m) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		CK(cudaSetDevice(m->device));
		sync_map(m);
		// the reference keeps the recorded set when detection is switched off; so do we: the mask
		// array stays, recording stops
		m->chg_recording = enable != 0;
		if (enable) alloc_arrays(m, Pool::Brick, Have::Changes);
		m->M.chg_mask = m->chg_recording ? m->chg_mask : nullptr;
		CK(cudaStreamSynchronize(m->stream));
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_reset_change_detection(ufo_b200_map* m)
{
	if (!m) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		CK(cudaSetDevice(m->device));
		sync_map(m);
		if (m->chg_mask) CK(cudaMemsetAsync(m->chg_mask, 0, (size_t)m->M.brick_cap * 64 * 8, m->stream));
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_changed_codes(ufo_b200_map* m, uint32_t depth, uint64_t* codes, size_t cap, size_t* n)
{
	if (!m || !n) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		CK(cudaSetDevice(m->device));
		sync_map(m);
		*n = 0;
		DeviceMap M = m->M;
		M.chg_mask = m->chg_mask;  // recording or not
		if (!M.chg_mask || !m->n_bricks) return (int)UFO_B200_OK;
		if (depth > M.g.depth_levels) return (int)UFO_B200_E_INVALID;
		const uint32_t dd = std::min(depth, 4u);
		cudaStream_t s = m->stream;
		DevBuf b_count, b_codes;
		unsigned long long* d_count = b_count.alloc<unsigned long long>(1);
		const uint32_t grid = (uint32_t)(((size_t)m->n_bricks * 64 + 255) / 256);
		CK(cudaMemsetAsync(d_count, 0, 8, s));
		k_changed<<<grid, 256, 0, s>>>(M, m->n_bricks, dd, nullptr, 0, d_count);
		unsigned long long cnt = 0;
		CK(cudaMemcpyAsync(&cnt, d_count, 8, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		std::vector<unsigned long long> h(cnt);
		if (cnt) {
			unsigned long long* d_codes = b_codes.alloc<unsigned long long>(cnt);
			CK(cudaMemsetAsync(d_count, 0, 8, s));
			k_changed<<<grid, 256, 0, s>>>(M, m->n_bricks, dd, d_codes, cnt, d_count);
			CK(cudaMemcpyAsync(h.data(), d_codes, cnt * 8, cudaMemcpyDeviceToHost, s));
			CK(cudaStreamSynchronize(s));
		}
		if (depth >= 4) {
			// ancestors above the brick + duplicates: snap to `depth` (with the centre bits) and unique
			const unsigned long long lowmask = depth >= 21 ? ~0ull : ((1ull << (3 * depth)) - 1ull);
			const unsigned long long centre = key_to_code({1u << (depth - 1), 1u << (depth - 1), 1u << (depth - 1)});
			for (auto& c : h) c = (c & ~lowmask) | centre;
			std::sort(h.begin(), h.end());
			h.erase(std::unique(h.begin(), h.end()), h.end());
		}
		*n = h.size();
		if (codes) std::memcpy(codes, h.data(), std::min(cap, h.size()) * 8);
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_write_compressed_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, uint32_t min_depth,
                                 int data_only, int acceleration_level, int compression_level, void* buf, size_t cap,
                                 size_t* size, size_t* uncompressed_size)
{
	if (!m || !size) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		if (!lz4().ok) {
			m->set_error("liblz4.so.1 not found: compressed output is unavailable");
			return (int)UFO_B200_E_UNSUPPORTED;
		}
		ImagePart part;
		const int rc = make_part(m, 1, min_depth, Volume{as_records(bv), (uint32_t)n_bv, {}, {}}, part);
		if (rc != UFO_B200_OK) return rc;
		return image_to_buffer({&part}, !data_only, true, acceleration_level, compression_level, buf, cap, size,
		                       uncompressed_size, m);
	});
}

int ufo_b200_image_part_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, uint32_t min_depth, int expanded,
                           void* buf, size_t cap, size_t* size)
{
	if (!m || !size) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	if (m->route_stage == 1) {
		m->set_error("ufo_b200_image_part_bv between ufo_b200_route_mark and the last ufo_b200_route_apply of the pass");
		return UFO_B200_E_INVALID;
	}
	return guarded(m, [&]() {
		ImagePart part;
		const int rc = make_part(m, expanded ? 0 : 1, min_depth, Volume{as_records(bv), (uint32_t)n_bv, {}, {}}, part);
		if (rc != UFO_B200_OK) return rc;
		*size = part_bytes(part);
		if (buf && cap >= *size) put_part(part, static_cast<uint8_t*>(buf));
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_image_assemble(const void* const* parts, const size_t* sizes, size_t n_parts, int with_header, int compress,
                            int acceleration_level, int compression_level, void* buf, size_t cap, size_t* size,
                            size_t* uncompressed_size)
{
	if (!parts || !sizes || !n_parts || !size) return UFO_B200_E_INVALID;
	if (compress && !lz4().ok) return UFO_B200_E_UNSUPPORTED;
	try {
		std::vector<ImagePart> ps(n_parts);
		std::vector<const ImagePart*> ptrs(n_parts);
		for (size_t i = 0; i < n_parts; ++i) {
			if (!parse_part(parts[i], sizes[i], ps[i])) return (int)UFO_B200_E_INVALID;
			ptrs[i] = &ps[i];
		}
		return image_to_buffer(ptrs, with_header != 0, compress != 0, acceleration_level, compression_level, buf, cap, size,
		                       uncompressed_size, nullptr);
	} catch (std::bad_alloc&) {
		return (int)UFO_B200_E_NOMEM;
	}
}

int ufo_b200_write_compressed(ufo_b200_map* m, const double* box6, uint32_t min_depth, int data_only,
                              int acceleration_level, int compression_level, void* buf, size_t cap, size_t* size,
                              size_t* uncompressed_size)
{
	const VolRec r = box6 ? aabb_record(box6) : VolRec{};
	return ufo_b200_write_compressed_bv(m, reinterpret_cast<const ufo_b200_volume*>(&r), box6 ? 1 : 0, min_depth, data_only,
	                                    acceleration_level, compression_level, buf, cap, size, uncompressed_size);
}

int ufo_b200_cast_rays(ufo_b200_map* m, const double* origins, const double* directions, size_t n,
                       int ignore_unknown, double max_range, uint32_t depth, uint64_t* codes, uint8_t* hit)
{
	if (!m || (n && (!origins || !directions || !codes || !hit)) || n > 0x7fffffffull) return UFO_B200_E_INVALID;
	if (!n) return UFO_B200_OK;
	return guarded(m, [&]() {
		if (depth > m->M.g.depth_levels) return (int)UFO_B200_E_INVALID;
		CK(cudaSetDevice(m->device));
		sync_map(m);
		cudaStream_t s = m->stream;
		std::vector<double> rays(6 * n);
		for (size_t i = 0; i < n; ++i) {
			for (int k = 0; k < 3; ++k) {
				rays[6 * i + k] = origins[3 * i + k];
				rays[6 * i + 3 + k] = directions[3 * i + k];
			}
		}
		DevBuf b_rays, b_codes, b_hit;
		double* d_rays = b_rays.alloc<double>(rays.size());
		unsigned long long* d_codes = b_codes.alloc<unsigned long long>(n);
		uint8_t* d_hit = b_hit.alloc<uint8_t>(n);
		CK(cudaMemcpyAsync(d_rays, rays.data(), rays.size() * 8, cudaMemcpyHostToDevice, s));
		k_cast_rays<<<(uint32_t)((n + 127) / 128), 128, 0, s>>>(m->M, d_rays, (uint32_t)n, ignore_unknown, max_range, depth, d_codes, d_hit);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(codes, d_codes, n * 8, cudaMemcpyDeviceToHost, s));
		CK(cudaMemcpyAsync(hit, d_hit, n, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		return (int)UFO_B200_OK;
	});
}

}  // extern "C"

namespace
{
// Filtered leaf iteration (ufo_export.cuh, k_export_nodes / k_export_upper).  chain == false: the
// node's own cube is tested against the volume; chain == true: every cube on its path from the root.
int export_nodes(Map* m, uint32_t depth, int occupied, int free_space, int unknown, const Volume& vol, bool chain,
                 uint64_t* codes, float* logodds, uint8_t* rgb, size_t cap, size_t* n)
{
	CK(cudaSetDevice(m->device));
	sync_map(m);
	*n = 0;
	if (depth > m->M.g.depth_levels) return (int)UFO_B200_E_INVALID;
	NodeFilter f{};
	f.depth = depth;
	f.occupied = occupied;
	f.free_ = free_space;
	f.unknown = unknown;
	f.chain = chain && vol.n ? 1 : 0;
	if (f.chain) {
		const double c0[3] = {0.0, 0.0, 0.0};
		if (!vol_hits(vol, c0, m->M.g.half_size[m->M.g.depth_levels])) return (int)UFO_B200_OK;  // the root misses
	}
	{
		cudaStream_t s = m->stream;
		unsigned long long* d_codes = nullptr;
		float* d_occ = nullptr;
		uint32_t* d_rgb = nullptr;
		DevBuf b_count, b_codes, b_occ, b_rgb, b_ok, b_bc;
		DeviceVolume dvol;
		Volume hv = vol;
		volume_is_general(hv);  // lo / hi of a single box, tested inline without the chain
		f.vol = dvol.upload(hv, s);
		if (f.chain && depth <= 4 && m->n_bricks) {
			uint8_t* d_ok = b_ok.alloc<uint8_t>(m->n_bricks);
			double* d_bc = b_bc.alloc<double>(3ull * m->n_bricks);
			k_brick_chain<<<(m->n_bricks + 255) / 256, 256, 0, s>>>(m->M, m->n_bricks, f.vol, d_ok, d_bc);
			f.brick_ok = d_ok;
			f.brick_c = d_bc;
		}
		unsigned long long* d_count = b_count.alloc<unsigned long long>(1);
		const bool fill = codes != nullptr && cap > 0;
		if (fill) {
			d_codes = b_codes.alloc<unsigned long long>(cap);
			d_occ = b_occ.alloc<float>(cap);
			if (rgb) d_rgb = b_rgb.alloc<uint32_t>(cap);
		}
		CK(cudaMemsetAsync(d_count, 0, 8, s));
		if (depth <= 4) {
			const size_t threads = (size_t)m->n_bricks * 64;
			if (threads && f.chain)
				k_export_nodes<true><<<(uint32_t)((threads + 255) / 256), 256, 0, s>>>(m->M, m->n_bricks, f, d_codes, d_occ, d_rgb, fill ? cap : 0, d_count);
			else if (threads)
				k_export_nodes<false><<<(uint32_t)((threads + 255) / 256), 256, 0, s>>>(m->M, m->n_bricks, f, d_codes, d_occ, d_rgb, fill ? cap : 0, d_count);
		} else if (m->n_upper) {
			if (f.chain) k_export_upper<true><<<(m->n_upper + 255) / 256, 256, 0, s>>>(m->M, m->n_upper, f, d_codes, d_occ, d_rgb, fill ? cap : 0, d_count);
			else k_export_upper<false><<<(m->n_upper + 255) / 256, 256, 0, s>>>(m->M, m->n_upper, f, d_codes, d_occ, d_rgb, fill ? cap : 0, d_count);
		}
		CK(cudaGetLastError());
		unsigned long long cnt = 0;
		CK(cudaMemcpyAsync(&cnt, d_count, 8, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		*n = (size_t)cnt;
		if (fill) {
			const size_t k = std::min<size_t>(cnt, cap);
			CK(cudaMemcpy(codes, d_codes, k * 8, cudaMemcpyDeviceToHost));
			if (logodds) CK(cudaMemcpy(logodds, d_occ, k * 4, cudaMemcpyDeviceToHost));
			if (rgb) {
				std::vector<uint32_t> h(k);
				CK(cudaMemcpy(h.data(), d_rgb, k * 4, cudaMemcpyDeviceToHost));
				for (size_t i = 0; i < k; ++i) {
					rgb[3 * i] = h[i] & 0xff;
					rgb[3 * i + 1] = (h[i] >> 8) & 0xff;
					rgb[3 * i + 2] = (h[i] >> 16) & 0xff;
				}
			}
		}
	}
	return (int)UFO_B200_OK;
}
}  // namespace

extern "C" {

int ufo_b200_export_nodes(ufo_b200_map* m, uint32_t depth, int occupied, int free_space, int unknown, const double* box6,
                          uint64_t* codes, float* logodds, uint8_t* rgb, size_t cap, size_t* n)
{
	if (!m || !n) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		const VolRec r = box6 ? aabb_record(box6) : VolRec{};
		return export_nodes(m, depth, occupied, free_space, unknown, Volume{&r, box6 ? 1u : 0u, {}, {}}, false, codes, logodds, rgb, cap, n);
	});
}

int ufo_b200_export_nodes_bv(ufo_b200_map* m, uint32_t depth, int occupied, int free_space, int unknown,
                             const ufo_b200_volume* bv, size_t n_bv, uint64_t* codes, float* logodds, uint8_t* rgb,
                             size_t cap, size_t* n)
{
	if (!m || !n) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		return export_nodes(m, depth, occupied, free_space, unknown, Volume{as_records(bv), (uint32_t)n_bv, {}, {}}, true, codes, logodds,
		                    rgb, cap, n);
	});
}

}  // extern "C"

namespace
{
// ---- iteration (ufo_export.cuh, k_brick_iter): the levels above the bricks on the host ----
struct IterWalk {
	const ExportPlan* plan = nullptr;  // tree shape above the bricks (build_upper)
	IterArgs a{};                      // host volume records
	std::vector<float> occ;            // ufo_b200_query values of plan->nodes
	std::vector<uint8_t> flags;
	std::vector<uint32_t> rgb;
	uint32_t default_flags = 0;
	// the sequence: a record of a node above the bricks (brick == kNone), or the records of a brick
	std::vector<std::pair<IterRec, uint32_t>> pieces;
	std::vector<unsigned long long> offs;  // per brick slot: first record in the packed brick records, ~0 = not reached
	unsigned long long packed = 0, total = 0;
};

// code and depth of every node of the shape, for the value query
void upper_codes(const ExportPlan& plan, int32_t idx, uint32_t d, unsigned long long code, std::vector<unsigned long long>& codes,
                 std::vector<uint32_t>& depths)
{
	codes[idx] = code;
	depths[idx] = d;
	if (d == 5) return;
	for (uint32_t i = 0; i < 8; ++i)
		if (plan.nodes[idx].child[i] >= 0)
			upper_codes(plan, plan.nodes[idx].child[i], d - 1, code | ((unsigned long long)i << (3 * (d - 1))), codes, depths);
}

// node (idx into plan->nodes, -1: a default leaf) of depth d >= 4 whose parent is descended into
void iter_walk(IterWalk& w, int32_t idx, uint32_t d, unsigned long long code, const double c[3], float v, uint32_t fl, uint32_t rgb,
               bool leaf)
{
	const Geometry& g = *w.plan->g;
	if (!vol_hits(w.a.vol, c, g.half_size[d]) || !iter_valid(w.a, d, v, fl)) return;
	if (iter_returns(w.a, d, leaf, v, fl)) {
		w.pieces.emplace_back(iter_rec(code, v, rgb, d, fl, leaf), kNone);
		++w.total;
	}
	if (d <= w.a.min_depth || leaf) return;
	const UpNode& n = w.plan->nodes[idx];
	for (uint32_t i = 0; i < 8; ++i) {
		double cc[3];
		child_center(c, g.half_size[d - 1], i, cc);
		const unsigned long long ccode = code | ((unsigned long long)i << (3 * (d - 1)));
		const int32_t ch = n.child[i];
		if (ch < 0) {
			iter_walk(w, -1, d - 1, ccode, cc, 0.0f, w.default_flags, 0u, true);
		} else if (d == 5) {
			// the brick node and its subtree: validNode and the rest were evaluated by the size pass
			const uint32_t slot = w.plan->order[ch];
			const uint32_t k = w.plan->info[slot].size;
			if (!k) continue;
			w.offs[slot] = w.packed;
			w.packed += k;
			w.total += k;
			w.pieces.emplace_back(IterRec{}, slot);
		} else {
			const UpNode& cn = w.plan->nodes[ch];
			iter_walk(w, ch, d - 1, ccode, cc, cn.has ? w.occ[ch] : cn.occ, w.flags[ch], cn.has ? w.rgb[ch] : cn.rgb, !cn.has);
		}
	}
}

// What iterate, tree_info and the nearest search share: `pass(d_info)` enqueues the size pass over the
// live bricks; their info and keys come back, the bricks of the tree are sorted into Morton order, the
// shape above them is built (build_upper) and its nodes get their values (ufo_b200_query's) in occ /
// flags / rgb.  Returns false when no brick is part of the tree (plan.nodes stays empty).
template <class Pass>
bool build_shape(Map* m, ExportPlan& plan, std::vector<BrickInfo>& info, std::vector<unsigned long long>& keys,
                 std::vector<unsigned long long>& brick_codes, std::vector<float>& occ, std::vector<uint8_t>& flags,
                 std::vector<uint32_t>& rgb, Pass&& pass)
{
	cudaStream_t s = m->stream;
	const uint32_t nb = m->n_bricks;
	const uint32_t L = m->M.g.depth_levels;
	const bool color = m->M.color != 0;
	const double c0[3] = {0.0, 0.0, 0.0};
	plan.levels = L;
	plan.pruned = true;
	plan.g = &m->M.g;
	info.assign(nb, BrickInfo{});
	plan.info = info.data();
	DevBuf b_info, b_qcodes, b_qdepths, b_qocc, b_qflags, b_qrgb;
	keys.assign(nb, 0ull);
	if (nb) {
		BrickInfo* d_info = b_info.alloc<BrickInfo>(nb);
		pass(d_info);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(info.data(), d_info, sizeof(BrickInfo) * nb, cudaMemcpyDeviceToHost, s));
		CK(cudaMemcpyAsync(keys.data(), m->M.brick_key, 8ull * nb, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
	}
	// bricks in the tree, in Morton order (as make_part: a default leaf brick is untouched space)
	std::vector<std::pair<unsigned long long, uint32_t>> sorted;
	sorted.reserve(nb);
	for (uint32_t b = 0; b < nb; ++b) {
		const BrickInfo& bi = info[b];
		if (bi.flags & 2u) continue;
		if (!(bi.flags & 1u) && bi.occ == 0.0f && bi.rgb == 0u) continue;
		uint32_t x, y, z;
		unpack_key(keys[b], x, y, z);
		sorted.emplace_back(spread3_host(x) | (spread3_host(y) << 1) | (spread3_host(z) << 2), b);
	}
	std::sort(sorted.begin(), sorted.end());
	plan.order.resize(sorted.size());
	brick_codes.resize(sorted.size());
	for (size_t i = 0; i < sorted.size(); ++i) {
		brick_codes[i] = sorted[i].first;
		plan.order[i] = sorted[i].second;
	}
	plan.codes = brick_codes.data();
	if (sorted.empty()) return false;
	build_upper(plan, L, 0, sorted.size(), c0);
	// values of the nodes above the bricks: ufo_b200_query's, one batch
	const size_t nu = plan.nodes.size();
	std::vector<unsigned long long> qc(nu);
	std::vector<uint32_t> qd(nu), qrgb(nu, 0u);
	upper_codes(plan, 0, L, 0ull, qc, qd);
	occ.resize(nu);
	flags.resize(nu);
	unsigned long long* d_qcodes = b_qcodes.alloc<unsigned long long>(nu);
	uint32_t* d_qdepths = b_qdepths.alloc<uint32_t>(nu);
	float* d_qocc = b_qocc.alloc<float>(nu);
	uint8_t* d_qflags = b_qflags.alloc<uint8_t>(nu);
	uint32_t* d_qrgb = color ? b_qrgb.alloc<uint32_t>(nu) : nullptr;
	CK(cudaMemcpyAsync(d_qcodes, qc.data(), 8 * nu, cudaMemcpyHostToDevice, s));
	CK(cudaMemcpyAsync(d_qdepths, qd.data(), 4 * nu, cudaMemcpyHostToDevice, s));
	k_query<<<(uint32_t)((nu + 255) / 256), 256, 0, s>>>(m->M, d_qcodes, d_qdepths, (uint32_t)nu, d_qocc, d_qflags, d_qrgb);
	CK(cudaGetLastError());
	CK(cudaMemcpyAsync(occ.data(), d_qocc, 4 * nu, cudaMemcpyDeviceToHost, s));
	CK(cudaMemcpyAsync(flags.data(), d_qflags, nu, cudaMemcpyDeviceToHost, s));
	if (color) CK(cudaMemcpyAsync(qrgb.data(), d_qrgb, 4 * nu, cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	rgb = std::move(qrgb);
	return true;
}

// What iterate and tree_info share: build_shape, then iter_walk walks w.a over the shape.  w.plan must
// point at plan.
template <class Pass>
void walk_above_bricks(Map* m, IterWalk& w, ExportPlan& plan, std::vector<BrickInfo>& info, std::vector<unsigned long long>& keys,
                       std::vector<unsigned long long>& brick_codes, Pass&& pass)
{
	const uint32_t L = m->M.g.depth_levels;
	const double c0[3] = {0.0, 0.0, 0.0};
	w.a.occ_thr = m->M.occ_thr;
	w.a.free_thr = m->M.free_thr;
	w.default_flags = m->M.default_flags;
	w.offs.assign(m->n_bricks, ~0ull);
	if (!build_shape(m, plan, info, keys, brick_codes, w.occ, w.flags, w.rgb, pass)) {
		iter_walk(w, -1, L, 0ull, c0, 0.0f, w.default_flags, 0u, true);
		return;
	}
	const UpNode& r = plan.nodes[0];
	iter_walk(w, 0, L, 0ull, c0, r.has ? w.occ[0] : r.occ, w.flags[0], r.has ? w.rgb[0] : r.rgb, !r.has);
}

int iterate(Map* m, const IterArgs& args, uint64_t* codes, uint8_t* depths, float* logodds, uint8_t* flags, uint8_t* rgb, size_t cap,
            size_t* n)
{
	*n = 0;
	if (m->M.g.depth_levels < 5) {
		m->set_error("iteration needs depth_levels >= 5");
		return UFO_B200_E_UNSUPPORTED;
	}
	CK(cudaSetDevice(m->device));
	sync_map(m);
	const uint32_t L = m->M.g.depth_levels;
	const double c0[3] = {0.0, 0.0, 0.0};
	if (args.min_depth > L || !vol_hits(args.vol, c0, m->M.g.half_size[L])) return UFO_B200_OK;  // octree.h:200-208
	cudaStream_t s = m->stream;
	const uint32_t nb = m->n_bricks;
	const bool color = m->M.color != 0;
	ExportPlan plan;
	std::vector<BrickInfo> info;
	std::vector<unsigned long long> keys, brick_codes;
	IterWalk w;
	w.plan = &plan;
	w.a = args;
	DevBuf b_offs, b_out;
	DeviceVolume dvol;
	Volume hv = args.vol;
	const bool general = volume_is_general(hv);
	IterArgs da = args;
	da.occ_thr = m->M.occ_thr;
	da.free_thr = m->M.free_thr;
	da.vol = dvol.upload(hv, s);
	auto brick_iter = [&](BrickInfo* d_info, const unsigned long long* offs, IterRec* out) {
		if (color && general) k_brick_iter<true, true><<<nb, 64, 0, s>>>(m->M, nb, da, d_info, offs, out);
		else if (color) k_brick_iter<true, false><<<nb, 64, 0, s>>>(m->M, nb, da, d_info, offs, out);
		else if (general) k_brick_iter<false, true><<<nb, 64, 0, s>>>(m->M, nb, da, d_info, offs, out);
		else k_brick_iter<false, false><<<nb, 64, 0, s>>>(m->M, nb, da, d_info, offs, out);
	};
	walk_above_bricks(m, w, plan, info, keys, brick_codes, [&](BrickInfo* d_info) { brick_iter(d_info, nullptr, nullptr); });
	*n = (size_t)w.total;
	if (codes && w.total && w.total <= cap) {
		std::vector<IterRec> packed(w.packed);
		if (w.packed) {
			unsigned long long* d_offs = b_offs.alloc<unsigned long long>(nb);
			IterRec* d_out = b_out.alloc<IterRec>(w.packed);
			CK(cudaMemcpyAsync(d_offs, w.offs.data(), 8ull * nb, cudaMemcpyHostToDevice, s));
			brick_iter(nullptr, d_offs, d_out);
			CK(cudaGetLastError());
			CK(cudaMemcpyAsync(packed.data(), d_out, sizeof(IterRec) * w.packed, cudaMemcpyDeviceToHost, s));
			CK(cudaStreamSynchronize(s));
		}
		size_t at = 0;
		auto put = [&](const IterRec& r) {
			codes[at] = r.code;
			depths[at] = (uint8_t)((r.meta >> 24) & 31u);
			logodds[at] = r.occ;
			flags[at] = (uint8_t)(r.meta >> 29);
			if (rgb) {
				rgb[3 * at] = (uint8_t)r.meta;
				rgb[3 * at + 1] = (uint8_t)(r.meta >> 8);
				rgb[3 * at + 2] = (uint8_t)(r.meta >> 16);
			}
			++at;
		};
		for (const auto& p : w.pieces) {
			if (p.second == kNone) {
				put(p.first);
			} else {
				const IterRec* r = packed.data() + w.offs[p.second];
				for (uint32_t i = 0; i < info[p.second].size; ++i) put(r[i]);
			}
		}
	}
	return UFO_B200_OK;
}

// nodes with children at depth >= 5 of the shape above the bricks (a collapsed node has none below it)
void count_upper(const ExportPlan& plan, int32_t idx, uint32_t d, uint64_t* with_children)
{
	const UpNode& n = plan.nodes[idx];
	if (!n.has) return;
	++with_children[d];
	if (d == 5) return;
	for (uint32_t i = 0; i < 8; ++i)
		if (n.child[i] >= 0) count_upper(plan, n.child[i], d - 1, with_children);
}

// centre of the node `code` of depth d, accumulated from the root as the iterators accumulate it
void node_center(const Geometry& g, unsigned long long code, uint32_t d, double c[3])
{
	c[0] = c[1] = c[2] = 0.0;
	for (uint32_t l = g.depth_levels; l > d; --l) {
		double n[3];
		child_center(c, g.half_size[l - 1], (uint32_t)(code >> (3 * (l - 1))) & 7u, n);
		c[0] = n[0];
		c[1] = n[1];
		c[2] = n[2];
	}
}

// getNumLeafNodes / getNumInnerNodes / getKnownBBX of the pruned tree: k_brick_info over the live
// bricks, the levels above them as iterate walks them (beginLeaves(occupied, free, !unknown)).
int tree_info(Map* m, ufo_b200_tree_stats* out)
{
	*out = ufo_b200_tree_stats{};
	if (m->M.g.depth_levels < 5) {
		m->set_error("tree_info needs depth_levels >= 5");
		return UFO_B200_E_UNSUPPORTED;
	}
	CK(cudaSetDevice(m->device));
	sync_map(m);
	cudaStream_t s = m->stream;
	const uint32_t nb = m->n_bricks;
	const Geometry& g = m->M.g;
	ExportPlan plan;
	std::vector<BrickInfo> info;
	std::vector<unsigned long long> keys, brick_codes;
	IterWalk w;
	w.plan = &plan;
	w.a.leaves_only = 1;
	w.a.occupied = 1;
	w.a.free_ = 1;
	IterArgs da = w.a;
	da.occ_thr = m->M.occ_thr;
	da.free_thr = m->M.free_thr;
	TreeTotals tot{};
	for (int i = 0; i < 3; ++i) tot.box[i] = ~0ull;
	DevBuf b_tot;
	TreeTotals* d_tot = b_tot.alloc<TreeTotals>(1);
	Events ev;
	CK(cudaMemcpyAsync(d_tot, &tot, sizeof(tot), cudaMemcpyHostToDevice, s));
	walk_above_bricks(m, w, plan, info, keys, brick_codes, [&](BrickInfo* d_info) {
		CK(cudaEventRecord(ev.e[0], s));
		if (m->M.color) k_brick_info<true><<<nb, 64, 0, s>>>(m->M, nb, da, d_info, d_tot);
		else k_brick_info<false><<<nb, 64, 0, s>>>(m->M, nb, da, d_info, d_tot);
		CK(cudaEventRecord(ev.e[1], s));
		++m->launches;
	});
	CK(cudaMemcpyAsync(&tot, d_tot, sizeof(tot), cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	if (nb) CK(cudaEventElapsedTime(&out->ms_device, ev.e[0], ev.e[1]));

	const uint32_t L = g.depth_levels;
	for (uint32_t d = 1; d <= 4; ++d) out->with_children[d] = tot.with_children[d - 1];
	if (!plan.nodes.empty()) count_upper(plan, 0, L, out->with_children);
	uint64_t inner = 0;
	for (uint32_t d = 2; d <= L; ++d) inner += out->with_children[d];
	out->num_leaf_nodes = 8 * out->with_children[1];
	out->num_inner_nodes = 1 + 8 * inner;

	// occupancy_map_base.h:828-852: nothing but unknown space gives AABB((0,0,0), 0)
	const bool root_has = !plan.nodes.empty() && plan.nodes[0].has;
	const float root_v = plan.nodes.empty() ? 0.0f : (root_has ? w.occ[0] : plan.nodes[0].occ);
	const uint32_t root_fl = plan.nodes.empty() ? m->M.default_flags : w.flags[0];
	out->known = iter_contains(w.a, root_v, root_fl) ? 1 : 0;
	if (!out->known) return UFO_B200_OK;
	double lo[3], hi[3];
	for (int i = 0; i < 3; ++i) {
		lo[i] = tot.box[i] != ~0ull ? decode_ordered(tot.box[i]) : DBL_MAX;
		hi[i] = tot.box[3 + i] != 0ull ? decode_ordered(tot.box[3 + i]) : -DBL_MAX;
	}
	// the leaves above the brick level and the bricks that are leaves themselves
	for (const auto& p : w.pieces) {
		double c[3];
		uint32_t d = 4;
		if (p.second == kNone) {
			d = (p.first.meta >> 24) & 31u;
			node_center(g, p.first.code, d, c);
		} else {
			uint32_t x, y, z;
			unpack_key(keys[p.second], x, y, z);
			brick_center(g, x, y, z, c);
		}
		for (int i = 0; i < 3; ++i) {
			lo[i] = std::min(lo[i], dop::sub(c[i], g.half_size[d]));
			hi[i] = std::max(hi[i], dop::add(c[i], g.half_size[d]));
		}
	}
	for (int i = 0; i < 3; ++i) {
		out->known_min[i] = lo[i];
		out->known_max[i] = hi[i];
	}
	return UFO_B200_OK;
}
}  // namespace

// The pruned tree shape above the bricks with the values of its nodes (build_shape), kept on the map
// for the nearest search and valid while the map's revision stays `revision`.
struct TreeShape {
	uint64_t revision = 0;
	bool any = false;  // some brick is part of the tree (else the root is a default leaf)
	ExportPlan plan;
	std::vector<BrickInfo> info;
	std::vector<unsigned long long> keys, brick_codes;
	std::vector<float> occ;
	std::vector<uint8_t> flags;
	std::vector<uint32_t> rgb;
};

namespace
{
// the shape for the map's current revision: built by the first call after a change, kept after that
const TreeShape& current_shape(Map* m, bool* rebuilt)
{
	*rebuilt = false;
	if (m->shape && m->shape->revision == m->revision) return *m->shape;
	m->shape.reset();
	auto sh = std::make_shared<TreeShape>();
	const uint32_t nb = m->n_bricks;
	cudaStream_t s = m->stream;
	IterArgs da{};  // the size pass is run for the shape and the brick payloads only
	da.occ_thr = m->M.occ_thr;
	da.free_thr = m->M.free_thr;
	da.occupied = da.free_ = da.unknown = 1;
	sh->any = build_shape(m, sh->plan, sh->info, sh->keys, sh->brick_codes, sh->occ, sh->flags, sh->rgb, [&](BrickInfo* d_info) {
		if (m->M.color) k_brick_iter<true, false><<<nb, 64, 0, s>>>(m->M, nb, da, d_info, nullptr, nullptr);
		else k_brick_iter<false, false><<<nb, 64, 0, s>>>(m->M, nb, da, d_info, nullptr, nullptr);
		++m->launches;
	});
	sh->plan.info = sh->info.data();
	sh->plan.codes = sh->brick_codes.data();
	sh->revision = m->revision;
	m->shape = std::move(sh);
	*rebuilt = true;
	return *m->shape;
}

// One entry of the host search: a node above the bricks (idx into plan.nodes), a default leaf (idx < 0)
// or, at depth 4, a brick of the tree (idx = its slot).
struct NearItem {
	double d2;
	int32_t idx;
	uint32_t d;
	unsigned long long code;
	double c[3];
	bool operator>(const NearItem& o) const { return d2 > o.d2; }
};

struct NearOut {
	double d2;
	IterRec r;
};

bool near_less(const NearOut& x, const NearOut& y)
{
	if (x.d2 != y.d2) return x.d2 < y.d2;
	if (x.r.code != y.r.code) return x.r.code < y.r.code;
	return ((x.r.meta >> 24) & 31u) > ((y.r.meta >> 24) & 31u);
}

// One shell of the nearest-first iteration.  The host runs a best-first search over the cached shape
// above the bricks with iter_walk's rules: it keeps the returned nodes of depth >= 5 (and default leaves)
// and collects the bricks in order of their cube's distance.  It stops once the nodes and bricks it has
// taken reach a target count; hi is then the key of the nearest entry not taken.  A key is a lower bound
// of the distance of every node below the entry: the entry's own distance, lowered by a slack far above
// the rounding of the accumulated centres (a child's cube can stick out of its parent's by an ulp).  So
// every node nearer than hi lies in a taken brick or was taken itself, and the shell, cut at the nodes'
// own distances, never misses one.  k_brick_nearest takes the shell's records out of
// the taken bricks; when the shell holds fewer than `want` nodes the target doubles and the bricks are
// searched again with the larger hi.
int nearest(Map* m, const double p[3], const IterArgs& args, double lo, size_t want, std::vector<NearOut>& out, double* hi_out)
{
	out.clear();
	*hi_out = INFINITY;
	ufo_b200_nearest_stats& st = m->nearest_stats;
	st = ufo_b200_nearest_stats{};
	if (m->M.g.depth_levels < 5) {
		m->set_error("nearest iteration needs depth_levels >= 5");
		return UFO_B200_E_UNSUPPORTED;
	}
	CK(cudaSetDevice(m->device));
	sync_map(m);
	st.revision = m->revision;
	const uint32_t L = m->M.g.depth_levels;
	const Geometry& g = m->M.g;
	const double c0[3] = {0.0, 0.0, 0.0};
	if (args.min_depth > L || !vol_hits(args.vol, c0, g.half_size[L]) || !(lo < INFINITY)) return UFO_B200_OK;
	cudaStream_t s = m->stream;
	const auto t0 = std::chrono::steady_clock::now();
	bool rebuilt = false;
	const TreeShape& sh = current_shape(m, &rebuilt);
	st.rebuilt = rebuilt ? 1 : 0;
	if (rebuilt) st.ms_rebuild = std::chrono::duration<float, std::milli>(std::chrono::steady_clock::now() - t0).count();
	const ExportPlan& plan = sh.plan;
	IterArgs a = args;
	a.occ_thr = m->M.occ_thr;
	a.free_thr = m->M.free_thr;
	const uint32_t dfl = m->M.default_flags;

	const double slack = 1e-9 * (g.half_size[L] + std::max(std::fabs(p[0]), std::max(std::fabs(p[1]), std::fabs(p[2]))));
	auto key = [&](double d2) {
		const double r = std::sqrt(d2) - slack;
		return r > 0.0 ? r * r : 0.0;
	};
	std::priority_queue<NearItem, std::vector<NearItem>, std::greater<NearItem>> heap;
	heap.push(NearItem{key(node_d2(p, c0, g.half_size[L])), sh.any ? 0 : -1, L, 0ull, {0.0, 0.0, 0.0}});
	std::vector<uint32_t> bricks;  // taken, by slot
	size_t taken = 0, kept = 0;
	double last = -INFINITY;
	auto take = [&]() {
		const NearItem it = heap.top();
		heap.pop();
		last = it.d2;
		if (it.d == 4 && it.idx >= 0) {
			bricks.push_back((uint32_t)it.idx);
			if (it.d2 >= lo) ++taken;
			return;
		}
		++st.upper_visited;
		const UpNode* n = it.idx >= 0 ? &plan.nodes[it.idx] : nullptr;
		const bool leaf = !n || !n->has;
		const float v = !n ? 0.0f : (n->has ? sh.occ[it.idx] : n->occ);
		const uint32_t fl = n ? sh.flags[it.idx] : dfl;
		const uint32_t rgb = !n ? 0u : (n->has ? sh.rgb[it.idx] : n->rgb);
		if (!vol_hits(a.vol, it.c, g.half_size[it.d]) || !iter_valid(a, it.d, v, fl)) return;
		const double d2 = node_d2(p, it.c, g.half_size[it.d]);
		if (iter_returns(a, it.d, leaf, v, fl) && d2 >= lo) {
			out.push_back(NearOut{d2, iter_rec(it.code, v, rgb, it.d, fl, leaf)});
			++taken;
		}
		if (it.d <= a.min_depth || leaf) return;
		for (uint32_t i = 0; i < 8; ++i) {
			NearItem c{};
			c.d = it.d - 1;
			child_center(it.c, g.half_size[c.d], i, c.c);
			c.code = it.code | ((unsigned long long)i << (3 * c.d));
			c.d2 = key(node_d2(p, c.c, g.half_size[c.d]));
			const int32_t ch = n->child[i];
			c.idx = ch < 0 ? -1 : (it.d == 5 ? (int32_t)plan.order[ch] : ch);
			heap.push(c);
		}
	};

	const bool color = m->M.color != 0;
	Volume hv = args.vol;
	const bool general = volume_is_general(hv);
	DeviceVolume dvol;
	IterArgs da = a;
	da.vol = dvol.upload(hv, s);
	DevBuf b_bricks, b_count, b_keys[2], b_recs[2], b_tmp;
	unsigned long long* d_count = b_count.alloc<unsigned long long>(1);
	size_t rec_cap = 0;
	NearKey* d_keys[2] = {nullptr, nullptr};
	IterRec* d_recs[2] = {nullptr, nullptr};
	Events ev;
	bool timed = false;
	std::vector<IterRec> dev_recs;
	std::vector<NearKey> dev_keys;
	want = std::max<size_t>(want, 1);
	size_t target = want;
	double hi = INFINITY;
	for (;;) {
		while (!heap.empty() && taken < target) take();
		while (!heap.empty() && heap.top().d2 <= last) take();  // hi above every key taken
		hi = heap.empty() ? INFINITY : heap.top().d2;
		// the nodes taken above the bricks that lie beyond hi belong to a later shell
		kept = (size_t)std::count_if(out.begin(), out.end(), [&](const NearOut& r) { return r.d2 < hi; });
		unsigned long long cnt = 0;
		if (!bricks.empty()) {
			const uint32_t nbk = (uint32_t)bricks.size();
			uint32_t* d_bricks = b_bricks.alloc<uint32_t>(nbk);
			CK(cudaMemcpyAsync(d_bricks, bricks.data(), 4ull * nbk, cudaMemcpyHostToDevice, s));
			const NearShell q{{p[0], p[1], p[2]}, lo, hi};
			for (;;) {
				CK(cudaMemsetAsync(d_count, 0, 8, s));
				if (!timed) CK(cudaEventRecord(ev.e[0], s));
				timed = true;
				if (color && general)
					k_brick_nearest<true, true><<<nbk, 64, 0, s>>>(m->M, d_bricks, nbk, da, q, d_keys[0], d_recs[0], d_count, rec_cap);
				else if (color)
					k_brick_nearest<true, false><<<nbk, 64, 0, s>>>(m->M, d_bricks, nbk, da, q, d_keys[0], d_recs[0], d_count, rec_cap);
				else if (general)
					k_brick_nearest<false, true><<<nbk, 64, 0, s>>>(m->M, d_bricks, nbk, da, q, d_keys[0], d_recs[0], d_count, rec_cap);
				else
					k_brick_nearest<false, false><<<nbk, 64, 0, s>>>(m->M, d_bricks, nbk, da, q, d_keys[0], d_recs[0], d_count, rec_cap);
				CK(cudaGetLastError());
				++m->launches;
				st.bricks_visited += nbk;
				++st.shells;
				CK(cudaMemcpyAsync(&cnt, d_count, 8, cudaMemcpyDeviceToHost, s));
				CK(cudaStreamSynchronize(s));
				if (cnt <= rec_cap) break;
				rec_cap = std::max<size_t>(cnt, 2 * rec_cap);  // room for the whole shell, then again
				for (int i = 0; i < 2; ++i) {
					d_keys[i] = b_keys[i].alloc<NearKey>(rec_cap);
					d_recs[i] = b_recs[i].alloc<IterRec>(rec_cap);
				}
			}
		}
		if (kept + cnt >= want || heap.empty()) {
			*hi_out = hi;
			if (cnt) {
				// (d2, code, ~depth), then one copy back
				size_t tmp_bytes = 0;
				CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_keys[0], d_keys[1], d_recs[0], d_recs[1], (int)cnt,
				                                   NearKeyParts{}, s));
				void* d_tmp = b_tmp.alloc<unsigned char>(tmp_bytes);
				CK(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_keys[0], d_keys[1], d_recs[0], d_recs[1], (int)cnt,
				                                   NearKeyParts{}, s));
				++m->launches;
				dev_keys.resize(cnt);
				dev_recs.resize(cnt);
				CK(cudaMemcpyAsync(dev_keys.data(), d_keys[1], sizeof(NearKey) * cnt, cudaMemcpyDeviceToHost, s));
				CK(cudaMemcpyAsync(dev_recs.data(), d_recs[1], sizeof(IterRec) * cnt, cudaMemcpyDeviceToHost, s));
			}
			if (timed) CK(cudaEventRecord(ev.e[1], s));
			CK(cudaStreamSynchronize(s));
			if (timed) CK(cudaEventElapsedTime(&st.ms_device, ev.e[0], ev.e[1]));
			break;
		}
		target = 2 * std::max(target, taken);
	}
	// merge the records of the levels above the bricks (few) into the sorted brick records
	out.erase(std::remove_if(out.begin(), out.end(), [&](const NearOut& r) { return !(r.d2 < hi); }), out.end());
	std::sort(out.begin(), out.end(), near_less);
	std::vector<NearOut> dev(dev_recs.size());
	for (size_t i = 0; i < dev.size(); ++i) {
		double d2;
		std::memcpy(&d2, &dev_keys[i].d2, 8);
		dev[i] = NearOut{d2, dev_recs[i]};
	}
	std::vector<NearOut> merged(out.size() + dev.size());
	std::merge(out.begin(), out.end(), dev.begin(), dev.end(), merged.begin(), near_less);
	out.swap(merged);
	return UFO_B200_OK;
}
}  // namespace

extern "C" {

int ufo_b200_iterate(ufo_b200_map* m, int leaves_only, int occupied, int free_space, int unknown, int contains, uint32_t min_depth,
                     const ufo_b200_volume* bv, size_t n_bv, uint64_t* codes, uint8_t* depths, float* logodds, uint8_t* flags,
                     uint8_t* rgb, size_t cap, size_t* n)
{
	if (!m || !n) return UFO_B200_E_INVALID;
	*n = 0;
	if (cap && (!codes || !depths || !logodds || !flags)) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		IterArgs a{};
		a.vol = Volume{as_records(bv), (uint32_t)n_bv, {}, {}};
		a.min_depth = min_depth;
		a.leaves_only = leaves_only != 0;
		a.occupied = occupied != 0;
		a.free_ = free_space != 0;
		a.unknown = unknown != 0;
		a.contains = contains != 0;
		return iterate(m, a, codes, depths, logodds, flags, rgb, cap, n);
	});
}

int ufo_b200_tree_info(ufo_b200_map* m, ufo_b200_tree_stats* out)
{
	if (!m || !out) return UFO_B200_E_INVALID;
	return guarded(m, [&]() { return tree_info(m, out); });
}

int ufo_b200_nearest(ufo_b200_map* m, const double point[3], const ufo_b200_volume* bv, size_t n_bv, int leaves_only,
                     int occupied, int free_space, int unknown, int contains, uint32_t min_depth, double d2_from,
                     size_t want, uint64_t* codes, uint8_t* depths, float* logodds, uint8_t* flags, uint8_t* rgb,
                     double* d2, size_t cap, size_t* n, double* d2_next)
{
	if (!m || !n || !d2_next || !point) return UFO_B200_E_INVALID;
	*n = 0;
	*d2_next = INFINITY;
	if (cap && (!codes || !depths || !logodds || !flags || !d2)) return UFO_B200_E_INVALID;
	if (!std::isfinite(point[0]) || !std::isfinite(point[1]) || !std::isfinite(point[2]) || std::isnan(d2_from)) {
		m->set_error("nearest: the point must be finite and d2_from a number");
		return UFO_B200_E_INVALID;
	}
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		IterArgs a{};
		a.vol = Volume{as_records(bv), (uint32_t)n_bv, {}, {}};
		a.min_depth = min_depth;
		a.leaves_only = leaves_only != 0;
		a.occupied = occupied != 0;
		a.free_ = free_space != 0;
		a.unknown = unknown != 0;
		a.contains = contains != 0;
		std::vector<NearOut> recs;
		double hi = INFINITY;
		const int rc = nearest(m, point, a, d2_from, want, recs, &hi);
		if (rc != UFO_B200_OK) return rc;
		*n = recs.size();
		*d2_next = hi;
		if (codes && !recs.empty() && recs.size() <= cap) {
			for (size_t i = 0; i < recs.size(); ++i) {
				const IterRec& r = recs[i].r;
				codes[i] = r.code;
				depths[i] = (uint8_t)((r.meta >> 24) & 31u);
				logodds[i] = r.occ;
				flags[i] = (uint8_t)(r.meta >> 29);
				d2[i] = recs[i].d2;
				if (rgb) {
					rgb[3 * i] = (uint8_t)r.meta;
					rgb[3 * i + 1] = (uint8_t)(r.meta >> 8);
					rgb[3 * i + 2] = (uint8_t)(r.meta >> 16);
				}
			}
		}
		return (int)UFO_B200_OK;
	});
}

int ufo_b200_last_nearest_stats(ufo_b200_map* m, ufo_b200_nearest_stats* out)
{
	if (!m || !out) return UFO_B200_E_INVALID;
	*out = m->nearest_stats;
	return UFO_B200_OK;
}

}  // extern "C"

namespace
{
Vec3 vec_of(const double* p) { return Vec3{p[0], p[1], p[2]}; }
Vec3 vcross(Vec3 a, Vec3 b)
{
	return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x};
}
double vdot(Vec3 a, Vec3 b) { return (a.x * b.x + a.y * b.y) + a.z * b.z; }
Vec3 vnormalized(Vec3 a) { return vdiv(a, vnorm(a)); }

// Plane(v1, v2, v3): normal = normalised (v3 - v2) x (v1 - v2), distance = -normal . v2
void plane_of(Vec3 v1, Vec3 v2, Vec3 v3, double* out)
{
	const Vec3 n = vnormalized(vcross(vsub(v3, v2), vsub(v1, v2)));
	out[0] = n.x;
	out[1] = n.y;
	out[2] = n.z;
	out[3] = -vdot(n, v2);
}
}  // namespace

extern "C" {

int ufo_b200_geometry_frustum(const double pos_in[3], const double target[3], const double up[3], double vertical_angle,
                              double horizontal_angle, double near_distance, double far_distance, double planes[24])
{
	if (!pos_in || !target || !up || !planes) return UFO_B200_E_INVALID;
	const double ratio = horizontal_angle / vertical_angle;
	const double tang = std::tan(vertical_angle * 0.5);
	const double near_h = near_distance * tang, near_w = near_h * ratio;
	const double far_h = far_distance * tang, far_w = far_h * ratio;
	const Vec3 pos = vec_of(pos_in);
	const Vec3 Z = vnormalized(vsub(pos, vec_of(target)));
	const Vec3 X = vnormalized(vcross(vec_of(up), Z));
	const Vec3 Y = vcross(Z, X);
	const Vec3 nc = vsub(pos, vscale(Z, near_distance)), fc = vsub(pos, vscale(Z, far_distance));
	// corner = centre (+/-) Y * height (+/-) X * width, summed left to right
	auto corner = [&](Vec3 c, double ys, double h, double xs, double w) {
		const Vec3 a = ys > 0 ? vadd(c, vscale(Y, h)) : vsub(c, vscale(Y, h));
		return xs > 0 ? vadd(a, vscale(X, w)) : vsub(a, vscale(X, w));
	};
	const Vec3 ntl = corner(nc, 1, near_h, -1, near_w), ntr = corner(nc, 1, near_h, 1, near_w);
	const Vec3 nbl = corner(nc, -1, near_h, -1, near_w), nbr = corner(nc, -1, near_h, 1, near_w);
	const Vec3 ftl = corner(fc, 1, far_h, -1, far_w), ftr = corner(fc, 1, far_h, 1, far_w);
	const Vec3 fbl = corner(fc, -1, far_h, -1, far_w), fbr = corner(fc, -1, far_h, 1, far_w);
	plane_of(ntr, ntl, ftl, planes);       // top
	plane_of(nbl, nbr, fbr, planes + 4);   // bottom
	plane_of(ntl, nbl, fbl, planes + 8);   // left
	plane_of(nbr, ntr, fbr, planes + 12);  // right
	plane_of(ntl, ntr, nbr, planes + 16);  // near
	plane_of(ftr, ftl, fbl, planes + 20);  // far
	return UFO_B200_OK;
}

int ufo_b200_geometry_plane(const double v1[3], const double v2[3], const double v3[3], double plane[4])
{
	if (!v1 || !v2 || !v3 || !plane) return UFO_B200_E_INVALID;
	plane_of(vec_of(v1), vec_of(v2), vec_of(v3), plane);
	return UFO_B200_OK;
}

int ufo_b200_geometry_ray(const double origin[3], const double direction[3], double ray[6])
{
	if (!origin || !direction || !ray) return UFO_B200_E_INVALID;
	const Vec3 d = vnormalized(vec_of(direction));
	ray[0] = origin[0];
	ray[1] = origin[1];
	ray[2] = origin[2];
	ray[3] = d.x;
	ray[4] = d.y;
	ray[5] = d.z;
	return UFO_B200_OK;
}

int ufo_b200_volume_intersects(const ufo_b200_volume* bv, size_t n_bv, const double* centres, const double* half_sizes,
                               size_t n, uint8_t* out)
{
	if ((n && (!centres || !half_sizes || !out)) || !volume_ok(nullptr, bv, n_bv)) return UFO_B200_E_INVALID;
	const VolRec* r = as_records(bv);
	for (size_t i = 0; i < n; ++i)
		out[i] = (n_bv == 0 || volume_hits_any(r, (uint32_t)n_bv, centres + 3 * i, half_sizes + 3 * i)) ? 1 : 0;
	return UFO_B200_OK;
}

}  // extern "C"

namespace
{
// Pinned staging for the sections of a page: two chunks of a bounded size on each side, so that the
// host's copy of one chunk overlaps the device's work on the next and a page of any size needs
// 2 x kPageChunk of pinned memory.
constexpr size_t kPageChunk = 16u << 20;
struct PageStage {
	uint8_t* pin[2] = {};
	DevBuf dev_buf[2];
	uint8_t* dev[2] = {};
	cudaEvent_t ev[2] = {};
	PageStage()
	{
		for (int b = 0; b < 2; ++b) {
			CK(cudaHostAlloc(reinterpret_cast<void**>(&pin[b]), kPageChunk, cudaHostAllocDefault));
			dev[b] = dev_buf[b].alloc<uint8_t>(kPageChunk);
			CK(cudaEventCreateWithFlags(&ev[b], cudaEventDisableTiming));
		}
	}
	PageStage(const PageStage&) = delete;
	PageStage& operator=(const PageStage&) = delete;
	~PageStage()
	{
		for (int b = 0; b < 2; ++b) {
			if (pin[b]) cudaFreeHost(pin[b]);
			if (ev[b]) cudaEventDestroy(ev[b]);
		}
	}
};

struct StreamReader {
	const uint8_t* p;
	size_t n, at = 0;
	bool ok = true;
	bool skip(size_t len)
	{
		if (at + len > n) {
			ok = false;
			at = n + 1;
			return false;
		}
		at += len;
		return true;
	}
	bool get(void* out, size_t len)
	{
		const size_t from = at;
		if (!skip(len)) {
			std::memset(out, 0, len);
			return false;
		}
		std::memcpy(out, p + from, len);
		return true;
	}
};

// a depth-4 node with children: its bytes in the stream
struct SubStream {
	unsigned long long code;
	size_t at;
	uint32_t len;
};

struct ImportPlan {
	std::vector<ImportRec> bricks, wipe;  // depth 4, depth >= 5
	std::vector<SubStream> subs;          // of the bricks this map owns, in stream order
	std::vector<size_t> cuts;             // upload chunk k holds subs[cuts[k], cuts[k + 1])
	Geometry g{};
	Volume vol{nullptr, 0, {}, {}};  // host records
	uint32_t P = 4;
	uint64_t budget = 1ull << 20;  // bricks a stream may create through collapsed nodes above the brick level
	bool too_big = false;
	bool none = false;  // the volume misses the root: nothing to read
	uint32_t route_world = 1, route_rank = 0;  // a routed rank expands only the bricks it owns
	bool owns(uint64_t brick_key) const { return route_world <= 1 || brick_owner(brick_key, route_world) == route_rank; }
};

// a leaf at depth >= 4 (the walk hands the levels below to k_import_parse)
void import_leaf(ImportPlan& plan, uint64_t code, uint32_t depth, float occ, uint32_t rgb)
{
	const ImportRec r{code, depth, occ, rgb, 0u};
	if (depth == 4) {
		plan.bricks.push_back(r);
		return;
	}
	// existing bricks below the node take the payload; if it is not the default, the bricks that
	// do not exist yet have to be created as well (the value field has no collapsed nodes).  The
	// budget counts every brick of the node on every rank, so that all ranks of a routed map
	// reach the same decision.
	plan.wipe.push_back(r);
	if (occ != 0.0f || rgb != 0u) {
		const uint64_t nb = depth >= 11 ? ~0ull : 1ull << (3 * (depth - 4));
		if (nb > plan.budget) {
			plan.too_big = true;
			return;
		}
		plan.budget -= nb;
		for (uint64_t i = 0; i < nb; ++i) {
			const uint64_t c = code + (i << 12);
			if (plan.owns(record_brick(c))) plan.bricks.push_back(ImportRec{c, 4u, occ, rgb, 0u});
		}
	}
}

void read_payload(StreamReader& in, uint32_t P, float& occ, uint32_t& rgb)
{
	uint8_t b[7] = {0, 0, 0, 0, 0, 0, 0};
	in.get(b, P);
	std::memcpy(&occ, b, 4);
	rgb = P == 7 ? ((uint32_t)b[4] | ((uint32_t)b[5] << 8) | ((uint32_t)b[6] << 16)) : 0u;
}

// The bytes of the depth-4 node with children at in.at (first voxel `code`, centre c): reads its
// children bytes only and steps over the payloads, whose number the children bytes and the volume
// decide (readNodesRecurs reads no bytes for a child whose cube misses the volume).  Without a
// volume no cube is tested and a depth-2 node costs one step.
void walk_brick(ImportPlan& plan, StreamReader& in, uint64_t code, const double c[3])
{
	const size_t at0 = in.at;
	const uint32_t P = plan.P;
	const bool filtered = plan.vol.n != 0;
	const double* hs = plan.g.half_size;
	auto hits = [&](const double* pc, uint32_t d, uint32_t i, double out[3]) {
		if (!filtered) return true;
		child_center(pc, hs[d], i, out);
		return vol_hits(plan.vol, out, hs[d]);
	};
	uint8_t c4 = 0;
	if (!in.get(&c4, 1)) return;
	for (uint32_t j = 0; j < 8; ++j) {
		double c3c[3];
		if (!hits(c, 3, j, c3c)) continue;
		if (!((c4 >> j) & 1u)) {
			in.skip(P);
			continue;
		}
		uint8_t c3 = 0;
		if (!in.get(&c3, 1)) return;
		for (uint32_t k = 0; k < 8; ++k) {
			double c2c[3];
			if (!hits(c3c, 2, k, c2c)) continue;
			if (!((c3 >> k) & 1u)) {
				in.skip(P);
				continue;
			}
			uint8_t c2 = 0;
			if (!in.get(&c2, 1)) return;
			if (!filtered) {
				in.skip((size_t)P * (8 + 7 * __builtin_popcount(c2)));
				continue;
			}
			for (uint32_t o = 0; o < 8; ++o) {
				double c1c[3];
				if (!hits(c2c, 1, o, c1c)) continue;
				if (!((c2 >> o) & 1u)) {
					in.skip(P);
					continue;
				}
				uint32_t nv = 0;
				for (uint32_t v = 0; v < 8; ++v) {
					double c0c[3];
					nv += hits(c1c, 0, v, c0c) ? 1u : 0u;
				}
				in.skip((size_t)P * nv);
			}
		}
	}
	if (in.ok && plan.owns(record_brick(code))) plan.subs.push_back(SubStream{code, at0, (uint32_t)(in.at - at0)});
}

// readNodesRecurs (occupancy_map_base.h:1403-1456) above the brick level: `code` = first voxel of
// the node of depth `depth` (> 4)
void import_rec(ImportPlan& plan, StreamReader& in, uint64_t code, uint32_t depth, const double c[3])
{
	const uint32_t cd = depth - 1;
	const double chs = plan.g.half_size[cd];
	uint8_t children = 0;
	if (!in.get(&children, 1)) return;
	for (uint32_t i = 0; i < 8 && in.ok; ++i) {
		double cc[3];
		child_center(c, chs, i, cc);
		if (!vol_hits(plan.vol, cc, chs)) continue;
		const uint64_t ccode = code + ((uint64_t)i << (3 * cd));
		if ((children >> i) & 1u) {
			if (cd == 4) walk_brick(plan, in, ccode, cc);
			else import_rec(plan, in, ccode, cd, cc);
		} else {
			float occ;
			uint32_t rgb;
			read_payload(in, plan.P, occ, rgb);
			import_leaf(plan, ccode, cd, occ, rgb);
		}
	}
}

// Upload chunks: records, then the sub-streams, and the 16 bytes k_import_parse may read past the
// last one (it copies whole 16-byte words), within one staging chunk.
void cut_chunks(ImportPlan& plan)
{
	plan.cuts.assign(1, 0);
	size_t bytes = 16;
	for (size_t i = 0; i < plan.subs.size(); ++i) {
		const size_t add = sizeof(ImportSub) + plan.subs[i].len;
		if (bytes + add > kPageChunk) {
			plan.cuts.push_back(i);
			bytes = 16;
		}
		bytes += add;
	}
	if (!plan.subs.empty()) plan.cuts.push_back(plan.subs.size());
}

// The host part of readData: walks the stream with plan.g, plan.vol, plan.P and the routing set,
// deciding every rejection before any device work.
int plan_import(Map* m, ImportPlan& plan, const uint8_t* data, size_t size)
{
	const double c0[3] = {0.0, 0.0, 0.0};
	if (!vol_hits(plan.vol, c0, plan.g.half_size[plan.g.depth_levels])) {  // no node intersects
		plan.none = true;
		return UFO_B200_OK;
	}
	StreamReader in{data, size};
	uint8_t children = 0;
	in.get(&children, 1);
	if (0 == children) {
		float occ;
		uint32_t rgb;
		read_payload(in, plan.P, occ, rgb);
		import_leaf(plan, 0, plan.g.depth_levels, occ, rgb);
	} else {
		import_rec(plan, in, 0, plan.g.depth_levels, c0);
	}
	if (!in.ok) {
		m->set_error("readData: the node stream is truncated");
		return UFO_B200_E_INVALID;
	}
	if (plan.too_big) {
		m->set_error("readData: a collapsed node above the brick level would expand into more than 2^20 bricks");
		return UFO_B200_E_UNSUPPORTED;
	}
	cut_chunks(plan);
	return UFO_B200_OK;
}

// the checks of readData that need no stream; plan set up for this map
int import_allowed(Map* m, uint32_t depth_levels, ImportPlan& plan, const Volume& vol)
{
	if (depth_levels < 5) {
		m->set_error("readData needs depth_levels >= 5");
		return UFO_B200_E_UNSUPPORTED;
	}
	if (m->M.shard_world > 1) {
		m->set_error("readData on a sharded map is not supported");
		return UFO_B200_E_UNSUPPORTED;
	}
	plan.P = m->M.color ? 7 : 4;
	plan.vol = vol;
	plan.route_world = m->M.route_world;
	plan.route_rank = m->M.route_rank;
	return UFO_B200_OK;
}

// The device part of readData.  The sub-streams travel in pinned chunks on the copy stream while
// the map's stream parses the chunk before; writing leaves is idempotent, so a grown pool runs the
// whole import again.
int apply_import(Map* m, const ImportPlan& plan, const uint8_t* data)
{
	if (plan.none) return UFO_B200_OK;
	DeviceMap& M = m->M;
	CK(cudaSetDevice(m->device));
	finalize_scan(m);
	cudaStream_t s = m->stream;
	const size_t n_bricks = plan.bricks.size(), n_wipe = plan.wipe.size();
	DevBuf b_bricks, b_wipe;
	ImportRec *d_bricks = nullptr, *d_wipe = nullptr;
	if (n_bricks) {
		d_bricks = b_bricks.alloc<ImportRec>(n_bricks);
		CK(cudaMemcpyAsync(d_bricks, plan.bricks.data(), n_bricks * sizeof(ImportRec), cudaMemcpyHostToDevice, s));
	}
	if (n_wipe) {
		d_wipe = b_wipe.alloc<ImportRec>(n_wipe);
		CK(cudaMemcpyAsync(d_wipe, plan.wipe.data(), n_wipe * sizeof(ImportRec), cudaMemcpyHostToDevice, s));
	}
	Volume hv = plan.vol;
	const bool general = volume_is_general(hv);
	DeviceVolume dvol;
	const Volume dv = dvol.upload(hv, s);
	std::unique_ptr<PageStage> st;
	Events ev;  // e[0..1]: chunk copied to the device, e[2..3]: chunk parsed
	if (!plan.subs.empty()) st.reset(new PageStage());
	auto parse = [&](uint32_t grid, const ImportSub* subs, uint32_t n, const uint8_t* bytes) {
		if (M.color && general) k_import_parse<true, true><<<grid, 64, 0, s>>>(M, dv, subs, n, bytes);
		else if (M.color) k_import_parse<true, false><<<grid, 64, 0, s>>>(M, dv, subs, n, bytes);
		else if (general) k_import_parse<false, true><<<grid, 64, 0, s>>>(M, dv, subs, n, bytes);
		else k_import_parse<false, false><<<grid, 64, 0, s>>>(M, dv, subs, n, bytes);
	};
	set_value_floor(m, -INFINITY);  // the stream's values are not clamped to this map's sensor model
	return run_growing(m, "readData", [&]() {
		new_scan_id(m);
		new_up_epoch(m);
		M.dense = 0;
		M.mask_base = M.miss_mask;
		if (n_wipe && m->n_bricks)
			k_import_wipe<<<(uint32_t)(((size_t)m->n_bricks * 64 + 255) / 256), 256, 0, s>>>(M, m->n_bricks, d_wipe, (uint32_t)n_wipe);
		if (n_bricks) k_import_bricks<<<(uint32_t)std::min<size_t>(n_bricks, (size_t)m->sm_count * 16), 64, 0, s>>>(M, d_bricks, (uint32_t)n_bricks);
		for (size_t k = 0; k + 1 < plan.cuts.size(); ++k) {
			const int b = (int)(k & 1);
			const size_t first = plan.cuts[k], n = plan.cuts[k + 1] - first;
			if (k >= 2) CK(cudaEventSynchronize(ev.e[b]));  // the pinned chunk has gone to the device
			ImportSub* recs = reinterpret_cast<ImportSub*>(st->pin[b]);
			uint8_t* bytes = st->pin[b] + n * sizeof(ImportSub);
			uint32_t off = 0;
			for (size_t i = 0; i < n; ++i) {
				const SubStream& sub = plan.subs[first + i];
				recs[i] = ImportSub{sub.code, off, sub.len};
				memcpy(bytes + off, data + sub.at, sub.len);
				off += sub.len;
			}
			if (k >= 2) CK(cudaStreamWaitEvent(m->copy_stream, ev.e[2 + b], 0));  // the device chunk is parsed
			CK(cudaMemcpyAsync(st->dev[b], st->pin[b], n * sizeof(ImportSub) + off, cudaMemcpyHostToDevice, m->copy_stream));
			CK(cudaEventRecord(ev.e[b], m->copy_stream));
			CK(cudaStreamWaitEvent(s, ev.e[b], 0));
			parse((uint32_t)std::min<size_t>(n, (size_t)m->sm_count * 7), reinterpret_cast<const ImportSub*>(st->dev[b]),
			      (uint32_t)n, st->dev[b] + n * sizeof(ImportSub));
			CK(cudaEventRecord(ev.e[2 + b], s));
		}
		launch_leaf_refresh(m);
		launch_upper(m);
	});
}

int import_stream(Map* m, const uint8_t* data, size_t size, const Volume& vol)
{
	// the stream is parsed and every rejection decided before any device work, so that the ranks
	// of a routed map, which take the same call, reach the same status and a rejected call changes
	// nothing
	ImportPlan plan;
	plan.g = m->M.g;
	int rc = import_allowed(m, m->M.g.depth_levels, plan, vol);
	if (rc == UFO_B200_OK) rc = plan_import(m, plan, data, size);
	return rc == UFO_B200_OK ? apply_import(m, plan, data) : rc;
}

// the node stream of a compressed input: one LZ4 block of uncompressed_size bytes
int decompress_stream(Map* m, const void* data, size_t size, size_t uncompressed_size, std::vector<uint8_t>& raw)
{
	if (!lz4().ok) {
		m->set_error("liblz4.so.1 not found: compressed input is unavailable");
		return UFO_B200_E_UNSUPPORTED;
	}
	if (size > (size_t)INT_MAX || uncompressed_size > (size_t)INT_MAX) {
		m->set_error("readData: an LZ4 block is at most 2^31 - 1 bytes");
		return UFO_B200_E_INVALID;
	}
	raw.resize(std::max<size_t>(uncompressed_size, 1));
	const int n = lz4().decompress(static_cast<const char*>(data), reinterpret_cast<char*>(raw.data()), (int)size, (int)uncompressed_size);
	if (n < 0) {
		m->set_error("readData: LZ4 decompression failed");
		return UFO_B200_E_INVALID;
	}
	raw.resize((size_t)n);
	return UFO_B200_OK;
}

// ---- file images: readHeader (octree.h:1338-1417) ----
const char kFileHeader[] = "# UFOMap file";

// The token loop of an istream over the image: operator>> skips whitespace and reads up to the next
// one; numbers are the longest prefix of the token num_get would take.
struct HeaderReader {
	const char* p;
	size_t n, at = 0;
	bool good = true;
	static bool space(char c) { return c == ' ' || c == '\t' || c == '\n' || c == '\v' || c == '\f' || c == '\r'; }
	bool skip_space()
	{
		while (at < n && space(p[at])) ++at;
		if (at == n) good = false;
		return good;
	}
	std::string token()
	{
		if (!skip_space()) return std::string();
		const size_t from = at;
		while (at < n && !space(p[at])) ++at;
		if (at == n) good = false;  // eof while reading: the token stands, the stream is no longer good
		return std::string(p + from, at - from);
	}
	void skip_line()
	{
		while (at < n && p[at++] != '\n') {}
		if (at == n && (n == 0 || p[n - 1] != '\n')) good = false;
	}
	// [+-]digits[.digits][e[+-]digits] with at least one digit; false (and not good) otherwise
	bool number(std::string& out, bool fraction)
	{
		if (!skip_space()) return false;
		const size_t from = at;
		auto digits = [&]() {
			size_t k = 0;
			while (at < n && p[at] >= '0' && p[at] <= '9') ++at, ++k;
			return k;
		};
		if (at < n && (p[at] == '+' || p[at] == '-')) ++at;
		size_t nd = digits();
		if (fraction && at < n && p[at] == '.') {
			++at;
			nd += digits();
		}
		if (fraction && nd && at < n && (p[at] == 'e' || p[at] == 'E')) {
			const size_t e = at++;
			if (at < n && (p[at] == '+' || p[at] == '-')) ++at;
			if (!digits()) at = e;
		}
		if (!nd) {
			good = false;
			return false;
		}
		out.assign(p + from, at - from);
		if (at == n) good = false;
		return true;
	}
};

// readHeader without the tree-type test; `id` in full.  Returns OK or E_INVALID, and fills `out`
// with what it read either way.
int parse_header(const void* image, size_t size, ufo_b200_file_header* out, std::string& id)
{
	memset(out, 0, sizeof(*out));
	out->uncompressed_data_size = -1;
	id.clear();
	const char* p = static_cast<const char*>(image);
	size_t eol = 0;
	while (eol < size && p[eol] != '\n') ++eol;
	if (eol < sizeof kFileHeader - 1 || memcmp(p, kFileHeader, sizeof kFileHeader - 1) != 0) return UFO_B200_E_INVALID;
	HeaderReader s{p, size, eol < size ? eol + 1 : size};
	if (s.at == size) s.good = false;
	std::string version;
	bool header_read = false;
	while (s.good && !header_read) {
		const std::string token = s.token();
		std::string num;
		if (token.empty()) break;
		if (token == "data") {
			header_read = true;
			s.skip_line();
			out->data_offset = s.at;
		} else if (token[0] == '#') {
			s.skip_line();
		} else if (token == "version") {
			version = s.token();
		} else if (token == "id") {
			id = s.token();
		} else if (token == "resolution") {
			if (s.number(num, true)) out->resolution = strtod(num.c_str(), nullptr);
		} else if (token == "depth_levels") {
			if (s.number(num, false)) {
				const long long v = strtoll(num.c_str(), nullptr, 10);
				if (v > (long long)UINT32_MAX || v < -(long long)UINT32_MAX) s.good = false;
				else out->depth_levels = (uint32_t)v;
			}
		} else if (token == "compressed") {
			if (s.number(num, false)) {
				const long long v = strtoll(num.c_str(), nullptr, 10);
				if (v != 0 && v != 1) s.good = false;
				else out->compressed = (int32_t)v;
			}
		} else if (token == "uncompressed_data_size") {
			if (s.number(num, false)) {
				const long long v = strtoll(num.c_str(), nullptr, 10);
				if (v > INT_MAX || v < INT_MIN) s.good = false;
				else out->uncompressed_data_size = v;
			}
		} else {
			s.skip_line();
		}
	}
	snprintf(out->version, sizeof out->version, "%s", version.c_str());
	snprintf(out->id, sizeof out->id, "%s", id.c_str());
	if (!header_read || version.empty() || id.empty() || !(out->resolution > 0.0) || out->depth_levels == 0 ||
	    out->uncompressed_data_size < 0)
		return UFO_B200_E_INVALID;
	return UFO_B200_OK;
}

// Octree::read (octree.h:700-729) of a file image
int read_image(Map* m, const uint8_t* image, size_t size)
{
	ufo_b200_file_header h;
	std::string id;
	if (parse_header(image, size, &h, id) != UFO_B200_OK) {
		m->set_error("read: not a valid UFOMap file header");
		return UFO_B200_E_INVALID;
	}
	const char* type = m->M.color ? "occupancy_map_color" : "occupancy_map";
	if (id != type) {
		m->set_error("read: a file of type '%s' does not go into an %s", h.id, type);
		return UFO_B200_E_INVALID;
	}
	if (h.depth_levels > 21) {
		m->set_error("read: depth_levels %u (at most 21)", h.depth_levels);
		return UFO_B200_E_INVALID;
	}
	ImportPlan plan;
	plan.g = make_geometry(h.resolution, h.depth_levels);
	int rc = import_allowed(m, h.depth_levels, plan, Volume{nullptr, 0, {}, {}});
	if (rc != UFO_B200_OK) return rc;
	const bool resize = h.resolution != m->M.g.resolution || h.depth_levels != m->M.g.depth_levels;
	if (resize && m->M.route_world > 1) {
		m->set_error("read: a routed map cannot be re-created with the file's resolution / depth_levels");
		return UFO_B200_E_UNSUPPORTED;
	}
	const uint8_t* body = image + h.data_offset;
	size_t body_size = size - h.data_offset;
	std::vector<uint8_t> raw;
	if (h.compressed) {
		// decompressed once: the reference decompresses a second time in readData (DESIGN.md section 7)
		rc = decompress_stream(m, body, body_size, (size_t)h.uncompressed_data_size, raw);
		if (rc != UFO_B200_OK) return rc;
		body = raw.data();
		body_size = raw.size();
	}
	rc = plan_import(m, plan, body, body_size);
	if (rc != UFO_B200_OK) return rc;
	if (resize) {
		rc = ufo_b200_clear_resize(m, h.resolution, h.depth_levels);
		if (rc != UFO_B200_OK) return rc;
	}
	return apply_import(m, plan, body);
}
}  // namespace

extern "C" {

int ufo_b200_read_data_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, const void* data, size_t size,
                          int compressed, size_t uncompressed_size)
{
	if (!m || (!data && size)) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	if (m->route_stage == 1) {
		m->set_error("readData between ufo_b200_route_mark and the last ufo_b200_route_apply of the pass");
		return UFO_B200_E_INVALID;
	}
	return guarded(m, [&]() {
		bump_revision(m);
		const Volume vol{as_records(bv), (uint32_t)n_bv};
		if (!compressed) return import_stream(m, static_cast<const uint8_t*>(data), size, vol);
		std::vector<uint8_t> raw;
		const int rc = decompress_stream(m, data, size, uncompressed_size, raw);
		return rc != UFO_B200_OK ? rc : import_stream(m, raw.data(), raw.size(), vol);
	});
}

int ufo_b200_read_data(ufo_b200_map* m, const double* box6, const void* data, size_t size, int compressed,
                       size_t uncompressed_size)
{
	const VolRec r = box6 ? aabb_record(box6) : VolRec{};
	return ufo_b200_read_data_bv(m, reinterpret_cast<const ufo_b200_volume*>(&r), box6 ? 1 : 0, data, size, compressed,
	                             uncompressed_size);
}

int ufo_b200_read_header(const void* image, size_t size, ufo_b200_file_header* out)
{
	if (!out || (!image && size)) return UFO_B200_E_INVALID;
	std::string id;
	return parse_header(image, size, out, id);
}

int ufo_b200_read(ufo_b200_map* m, const void* image, size_t size)
{
	if (!m || (!image && size)) return UFO_B200_E_INVALID;
	if (m->route_stage == 1) {
		m->set_error("read between ufo_b200_route_mark and the last ufo_b200_route_apply of the pass");
		return UFO_B200_E_INVALID;
	}
	return guarded(m, [&]() { bump_revision(m); return read_image(m, static_cast<const uint8_t*>(image), size); });
}

int ufo_b200_read_file(ufo_b200_map* m, const char* filename)
{
	if (!m || !filename) return UFO_B200_E_INVALID;
	if (m->route_stage == 1) {
		m->set_error("read between ufo_b200_route_mark and the last ufo_b200_route_apply of the pass");
		return UFO_B200_E_INVALID;
	}
	return guarded(m, [&]() {
		bump_revision(m);
		FILE* f = fopen(filename, "rb");
		if (!f) {
			m->set_error("cannot open %s", filename);
			return (int)UFO_B200_E_INVALID;
		}
		std::vector<uint8_t> image;
		bool ok = fseeko(f, 0, SEEK_END) == 0;
		const off_t n = ok ? ftello(f) : -1;
		ok = ok && n >= 0 && fseeko(f, 0, SEEK_SET) == 0;
		if (ok) {
			image.resize((size_t)n);
			ok = fread(image.data(), 1, image.size(), f) == image.size();
		}
		fclose(f);
		if (!ok) {
			m->set_error("cannot read %s", filename);
			return (int)UFO_B200_E_INVALID;
		}
		return read_image(m, image.data(), image.size());
	});
}

}  // extern "C"

namespace
{
// checks shared by the two write entry points (they need no device); returns OK or the status to
// reject the batch with
int write_allowed(Map* m, uint32_t depth)
{
	if (depth > 6) {
		m->set_error("write depth %u > 6 is not supported (a node of depth 7 covers 512 bricks of the dense value field)", depth);
		return UFO_B200_E_UNSUPPORTED;
	}
	if (depth > m->M.g.depth_levels) {
		m->set_error("write depth %u exceeds the tree's depth_levels %u", depth, m->M.g.depth_levels);
		return UFO_B200_E_INVALID;
	}
	if (m->M.shard_world > 1) {
		m->set_error("per-node writes on a sharded map are not supported");
		return UFO_B200_E_UNSUPPORTED;
	}
	if (m->route_stage == 1) {
		m->set_error("a write between ufo_b200_route_mark and the last ufo_b200_route_apply of the pass");
		return UFO_B200_E_INVALID;
	}
	if (m->poisoned) {
		m->set_error("an earlier scan failed half-way; ufo_b200_clear() the map before writing again");
		return UFO_B200_E_INVALID;
	}
	return UFO_B200_OK;
}

bool depth0_key_ok(const Geometry& g, const double p[3])
{
	for (int k = 0; k < 3; ++k) {
		const double kv = std::floor(p[k] * g.resolution_factor) + (double)g.max_value;  // toKey at depth 0
		if (!(kv >= 0.0 && kv < (double)(1ull << g.depth_levels))) return false;
	}
	return true;
}

// Copies a batch's inputs and record offsets to the device and enqueues it (ufo_write.cuh).
// `blobs`: host arrays copied back to back into the map's input buffer, each 8-byte aligned;
// `bind` receives the device address of each blob and stores it into the batch's arguments.
template <class Bind>
int do_write(Map* m, WriteArgs w, const std::vector<std::pair<const void*, size_t>>& blobs,
             const std::vector<unsigned long long>& offs, int async, Bind&& bind)
{
	finalize_scan(m);
	const unsigned long long n_rec = offs.back();
	if (n_rec > 0x7fffffffull) {
		m->set_error("write batch needs %llu records (limit 2^31 - 1)", n_rec);
		return UFO_B200_E_UNSUPPORTED;
	}
	cudaStream_t s = m->stream;
	size_t total = offs.size() * 8;
	for (const auto& b : blobs) total += (b.second + 7) & ~size_t(7);
	ensure_spare(m, m->d_w_in, total, 1 << 12);
	unsigned char* in = m->d_w_in.p;
	size_t at = 0;
	std::vector<const void*> ptrs;
	for (const auto& b : blobs) {
		if (b.second) CK(cudaMemcpyAsync(in + at, b.first, b.second, cudaMemcpyHostToDevice, s));
		ptrs.push_back(in + at);
		at += (b.second + 7) & ~size_t(7);
	}
	CK(cudaMemcpyAsync(in + at, offs.data(), offs.size() * 8, cudaMemcpyHostToDevice, s));
	bind(w, ptrs);
	w.offs = reinterpret_cast<const unsigned long long*>(in + at);
	w.n_rec = n_rec;
	if (n_rec > m->w_rec_cap) {
		m->w_rec_cap = 0;
		const size_t cap = std::max<size_t>(n_rec + n_rec / 8, 1 << 12);
		for (int i = 0; i < 2; ++i) {
			m->d_w_keys[i].ensure(m, cap * sizeof(unsigned long long), 0);
			m->d_w_idx[i].ensure(m, cap * sizeof(uint32_t), 0);
		}
		m->d_w_recs.ensure(m, cap * sizeof(WriteRec), 0);
		m->w_rec_cap = cap;
	}
	PendingScan& p = m->pending;
	p = PendingScan{};
	p.write = true;
	p.w = w;
	m->stats = ufo_b200_scan_stats{};
	m->stats.points = w.n;
	m->launches = 0;
	m->h2d_valid = false;
	CK(cudaEventRecord(m->ev[0], s));
	// the inputs above were staged from pageable memory: the caller's arrays are free again here
	enqueue_scan(m, p);
	if (!async) return sync_map(m);
	return UFO_B200_OK;
}

bool code_in_map(const Geometry& g, uint64_t code, uint32_t d)
{
	const Key3 k = code_to_key(code);
	return !((((k.x >> d) << d) | ((k.y >> d) << d) | ((k.z >> d) << d)) & ~g.key_mask);
}

// The body of ufo_b200_update_nodes (rgb == NULL) and of ufo_b200_update_nodes_color for a batch
// that holds a colour op (rgb != NULL, every entry already checked).
int write_nodes(Map* m, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops, const float* values,
                const uint8_t* rgb, size_t n, int async)
{
	return guarded(m, [&]() {
		bump_revision(m);
		CK(cudaSetDevice(m->device));
		const Geometry& g = m->M.g;
		std::vector<unsigned long long> offs(n + 1);
		unsigned long long tot = 0;
		for (size_t i = 0; i < n; ++i) {
			const uint32_t d = depths[i];
			if (ops[i] > (rgb ? 3 : 1)) {
				m->set_error("entry %zu: op %u is neither ADD (0) nor SET (1)", i, (unsigned)ops[i]);
				return (int)UFO_B200_E_INVALID;
			}
			if (ops[i] == 1 && d > 0 && m->M.color) {
				m->set_error("SET on a colour map is supported at depth 0 only");
				return (int)UFO_B200_E_UNSUPPORTED;
			}
			if (!code_in_map(g, codes[i], d)) {
				m->set_error("entry %zu: code %llu lies outside the map", i, (unsigned long long)codes[i]);
				return (int)UFO_B200_E_INVALID;
			}
			offs[i] = tot;
			tot += d <= 4 ? 1ull : 1ull << (3 * (d - 4));
		}
		offs[n] = tot;
		if (!n) {
			finalize_scan(m);
			return (int)UFO_B200_OK;
		}
		WriteArgs w{};
		w.n = (uint32_t)n;
		std::vector<std::pair<const void*, size_t>> blobs = {{codes, n * 8}, {values, n * 4}, {depths, n * 4}, {ops, n}};
		if (rgb) blobs.push_back({rgb, n * 3});
		return do_write(m, w, blobs, offs, async, [](WriteArgs& a, const std::vector<const void*>& p) {
			a.codes = static_cast<const unsigned long long*>(p[0]);
			a.values = static_cast<const float*>(p[1]);
			a.depths = static_cast<const uint32_t*>(p[2]);
			a.ops = static_cast<const uint8_t*>(p[3]);
			a.rgb = p.size() > 4 ? static_cast<const uint8_t*>(p[4]) : nullptr;
		});
	});
}
}  // namespace

extern "C" {

int ufo_b200_update_nodes(ufo_b200_map* m, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                          const float* values, size_t n, int async)
{
	if (!m || (n && (!codes || !depths || !ops || !values)) || n > 0x7fffffffull) return UFO_B200_E_INVALID;
	for (size_t i = 0; i < n; ++i) {
		const int rc = write_allowed(m, depths[i]);
		if (rc != UFO_B200_OK) return rc;
	}
	return write_nodes(m, codes, depths, ops, values, nullptr, n, async);
}

int ufo_b200_update_nodes_color(ufo_b200_map* m, const uint64_t* codes, const uint32_t* depths, const uint8_t* ops,
                                const float* values, const uint8_t* rgb, size_t n, int async)
{
	if (!m || (n && (!codes || !depths || !ops || !values)) || n > 0x7fffffffull) return UFO_B200_E_INVALID;
	// every check runs on the host before any device work, so a rejected batch applies nothing
	bool has_color = false;
	for (size_t i = 0; i < n; ++i) {
		const uint32_t d = depths[i];
		if (ops[i] > 3) {
			m->set_error("entry %zu: op %u is not ADD (0), SET (1), ADD_COLOR (2) or SET_COLOR (3)", i, (unsigned)ops[i]);
			return UFO_B200_E_INVALID;
		}
		if (ops[i] >= 2 && !m->params.color) {
			m->set_error("entry %zu: colour op %u on a map without colour", i, (unsigned)ops[i]);
			return UFO_B200_E_INVALID;
		}
		const int rc = write_allowed(m, d);
		if (rc != UFO_B200_OK) return rc;
		if (!code_in_map(m->M.g, codes[i], d)) {
			m->set_error("entry %zu: code %llu lies outside the map", i, (unsigned long long)codes[i]);
			return UFO_B200_E_INVALID;
		}
		if (ops[i] >= 2 && d > 0) {
			// the reference's result depends on whether the node has children, which the value
			// field does not record (DESIGN.md section 8)
			m->set_error("entry %zu: colour ops are supported at depth 0 only", i);
			return UFO_B200_E_UNSUPPORTED;
		}
		if (ops[i] == 1 && d > 0 && m->params.color) {
			m->set_error("SET on a colour map is supported at depth 0 only");
			return UFO_B200_E_UNSUPPORTED;
		}
		has_color |= ops[i] >= 2;
	}
	if (has_color && !rgb) {
		m->set_error("the batch holds a colour op but rgb is NULL");
		return UFO_B200_E_INVALID;
	}
	return write_nodes(m, codes, depths, ops, values, has_color ? rgb : nullptr, n, async);
}

int ufo_b200_insert_rays(ufo_b200_map* m, const double* origins, const double* ends, size_t n, double max_range,
                         uint32_t depth, int hit_end, int async)
{
	if (!m || (n && (!origins || !ends)) || n > 0x7fffffffull) return UFO_B200_E_INVALID;
	const int rc = write_allowed(m, depth);
	if (rc != UFO_B200_OK) return rc;
	return guarded(m, [&]() {
		bump_revision(m);
		CK(cudaSetDevice(m->device));
		const Geometry& g = m->M.g;
		// record region of every ray: an upper bound of the walk's records.  Every step of the walk
		// moves one axis by one node, so a walk from key a to key b visits |a - b|_1 + 1 nodes and
		// enters |a/4 - b/4|_1 + 1 blocks (depth <= 2, one record per block); 2 spare records cover a
		// walk that stops on the range test instead of on the end node.
		const uint32_t shift = depth <= 2 ? 2u : depth;
		const unsigned long long per = depth <= 4 ? 1ull : 1ull << (3 * (depth - 4));
		std::vector<unsigned long long> offs(n + 1);
		unsigned long long tot = 0;
		for (size_t i = 0; i < n; ++i) {
			const double* po = origins + 3 * i;
			const double* pe = ends + 3 * i;
			if (!depth0_key_ok(g, po) || !depth0_key_ok(g, pe)) {
				m->set_error("ray %zu: origin or end lies outside the map", i);
				return (int)UFO_B200_E_INVALID;
			}
			const Vec3 o = {po[0], po[1], po[2]};
			Vec3 e = {pe[0], pe[1], pe[2]};
			Vec3 dir = vsub(e, o);
			const double dist = vnorm(dir);
			dir = vdiv(dir, dist);
			if (0 <= max_range && dist > max_range) e = vadd(o, vscale(dir, max_range));
			const Key3 a = point_to_key(g, o, depth), b = point_to_key(g, e, depth);
			const unsigned long long steps = (unsigned long long)std::llabs((long long)(a.x >> shift) - (long long)(b.x >> shift)) +
			                                 (unsigned long long)std::llabs((long long)(a.y >> shift) - (long long)(b.y >> shift)) +
			                                 (unsigned long long)std::llabs((long long)(a.z >> shift) - (long long)(b.z >> shift));
			offs[i] = tot;
			tot += (steps + 3) * per + (hit_end ? 1 : 0);
		}
		offs[n] = tot;
		if (!n) {
			finalize_scan(m);
			return (int)UFO_B200_OK;
		}
		WriteArgs w{};
		w.n = (uint32_t)n;
		w.rays = 1;
		w.max_range = max_range;
		w.depth = depth;
		w.hit_end = hit_end ? 1u : 0u;
		// integrateMiss / integrateHit: updateValue(code, float(prob_miss_log_ / prob_hit_log_))
		w.miss = (float)m->miss_log;
		w.hit = (float)m->hit_log;
		return do_write(m, w, {{origins, n * 24}, {ends, n * 24}}, offs, async,
		                [](WriteArgs& a, const std::vector<const void*>& p) {
			                a.origins = static_cast<const double*>(p[0]);
			                a.ends = static_cast<const double*>(p[1]);
		                });
	});
}

}  // extern "C"

// ---------------------------------------------------------------------------
// retain / page out / page in (ufo_page.cuh)
// ---------------------------------------------------------------------------
namespace
{
// One section of a page-out: gather(device chunk, first brick, bricks) fills a device chunk, which
// goes to pinned memory and from there into the caller's buffer.
template <class Gather>
void page_section_out(cudaStream_t s, PageStage& st, size_t n, size_t brick_bytes, uint8_t* dst, Gather&& gather)
{
	const size_t chunk = kPageChunk / brick_bytes;
	int wait_b = -1;
	size_t wait_first = 0, wait_n = 0;
	auto drain = [&]() {
		if (wait_b < 0) return;
		CK(cudaEventSynchronize(st.ev[wait_b]));
		memcpy(dst + wait_first * brick_bytes, st.pin[wait_b], wait_n * brick_bytes);
	};
	for (size_t first = 0, i = 0; first < n; first += chunk, ++i) {
		const int b = (int)(i & 1);
		const size_t cnt = std::min(chunk, n - first);
		gather(st.dev[b], first, cnt);
		CK(cudaGetLastError());
		CK(cudaMemcpyAsync(st.pin[b], st.dev[b], cnt * brick_bytes, cudaMemcpyDeviceToHost, s));
		CK(cudaEventRecord(st.ev[b], s));
		drain();
		wait_b = b;
		wait_first = first;
		wait_n = cnt;
	}
	drain();
}

// One section of a page-in: the caller's bytes go through pinned memory into a device chunk, which
// scatter(device chunk, first brick, bricks) applies.
template <class Scatter>
void page_section_in(cudaStream_t s, PageStage& st, size_t n, size_t brick_bytes, const uint8_t* src, Scatter&& scatter)
{
	const size_t chunk = kPageChunk / brick_bytes;
	bool used[2] = {false, false};
	for (size_t first = 0, i = 0; first < n; first += chunk, ++i) {
		const int b = (int)(i & 1);
		const size_t cnt = std::min(chunk, n - first);
		if (used[b]) CK(cudaEventSynchronize(st.ev[b]));  // the copy out of this pinned chunk has finished
		memcpy(st.pin[b], src + first * brick_bytes, cnt * brick_bytes);
		CK(cudaMemcpyAsync(st.dev[b], st.pin[b], cnt * brick_bytes, cudaMemcpyHostToDevice, s));
		CK(cudaEventRecord(st.ev[b], s));
		used[b] = true;
		scatter(st.dev[b], first, cnt);
		CK(cudaGetLastError());
	}
	CK(cudaStreamSynchronize(s));
}

// checks shared by retain, page-out and page-in; they need no device
int page_allowed(Map* m, const char* what)
{
	if (m->M.g.depth_levels < 5) {
		m->set_error("%s needs depth_levels >= 5", what);
		return UFO_B200_E_UNSUPPORTED;
	}
	if (m->M.route_world > 1 || m->route_stage != 0) {
		m->set_error("%s on a routed map is not supported", what);
		return UFO_B200_E_UNSUPPORTED;
	}
	if (m->poisoned) {
		m->set_error("an earlier scan failed half-way; ufo_b200_clear() the map first");
		return UFO_B200_E_INVALID;
	}
	return UFO_B200_OK;
}

// keep flags of the live bricks and, for a page-out, the sort keys / slots / count of the bricks to write
void launch_page_classify(Map* m, const Volume& vol, DeviceVolume& dvol, uint32_t* d_keep, unsigned long long* d_skey,
                          uint32_t* d_slot, uint32_t* d_count)
{
	const double c0[3] = {0.0, 0.0, 0.0};
	const int none = vol_hits(vol, c0, m->M.g.half_size[m->M.g.depth_levels]) ? 0 : 1;  // the root misses
	Volume hv = vol;
	volume_is_general(hv);
	const Volume dv = dvol.upload(hv, m->stream);
	k_page_classify<<<(m->n_bricks + 255) / 256, 256, 0, m->stream>>>(m->M, m->n_bricks, dv, none, d_keep, d_skey, d_slot, d_count);
	CK(cudaGetLastError());
	++m->launches;
}

void fill_pool_state(Map* m, uint64_t& bricks, uint64_t& cap, uint64_t& bytes)
{
	bricks = m->n_bricks;
	cap = m->M.brick_cap;
	bytes = m->device_bytes;
}

// The levels above the bricks from the depth-4 aggregates of bricks slot[0..n) (nullptr: 0..n): the
// scan's push-up pass with these bricks as its touched list.  `derived`: first recompute the bricks'
// own depth 1-4 values from their leaves, as an import does.
void page_propagate(Map* m, const uint32_t* d_slot, uint32_t n, bool derived)
{
	const int rc = run_growing(m, "upper-node propagation", [&]() {
		new_up_epoch(m);
		k_page_touch<<<std::max(1u, std::min((n + 255) / 256, (uint32_t)m->sm_count * 4)), 256, 0, m->stream>>>(m->M, d_slot, n);
		if (derived) launch_leaf_refresh(m);
		launch_upper(m);
	});
	if (rc != UFO_B200_OK) {
		m->poisoned = true;
		throw MapError{rc};
	}
}

int retain(Map* m, const Volume& vol, ufo_b200_retain_stats* out)
{
	const int allowed = page_allowed(m, "retain");
	if (allowed != UFO_B200_OK) return allowed;
	CK(cudaSetDevice(m->device));
	sync_map(m);
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	ufo_b200_retain_stats st{};
	fill_pool_state(m, st.bricks_before, st.brick_cap_before, st.device_bytes_before);
	st.bricks_kept = st.bricks_before;
	fill_pool_state(m, st.bricks_kept, st.brick_cap_after, st.device_bytes_after);
	const uint32_t n = m->n_bricks;
	uint32_t kept = n;
	DevBuf b_keep, b_new, b_src, b_tmp;
	uint32_t* d_src = nullptr;
	Events ev;
	if (vol.n && n) {
		uint32_t* d_keep = b_keep.alloc<uint32_t>(n);
		uint32_t* d_new = b_new.alloc<uint32_t>(n);
		d_src = b_src.alloc<uint32_t>(n);
		size_t tmp_bytes = 0;
		CK(cub::DeviceScan::ExclusiveSum(nullptr, tmp_bytes, d_keep, d_new, (int)n, s));
		void* d_tmp = b_tmp.alloc<uint8_t>(tmp_bytes);
		DeviceVolume dvol;
		CK(cudaEventRecord(ev.e[0], s));
		launch_page_classify(m, vol, dvol, d_keep, nullptr, nullptr, nullptr);
		CK(cub::DeviceScan::ExclusiveSum(d_tmp, tmp_bytes, d_keep, d_new, (int)n, s));
		k_page_sources<<<(n + 255) / 256, 256, 0, s>>>(n, d_keep, d_new, d_src);
		CK(cudaGetLastError());
		m->launches += 2;
		CK(cudaEventRecord(ev.e[1], s));
		uint32_t last[2] = {0, 0};
		CK(cudaMemcpyAsync(&last[0], d_new + (n - 1), 4, cudaMemcpyDeviceToHost, s));
		CK(cudaMemcpyAsync(&last[1], d_keep + (n - 1), 4, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		kept = last[0] + last[1];
		CK(cudaEventElapsedTime(&st.ms_classify, ev.e[0], ev.e[1]));
	}
	if (kept == n) {  // nothing to remove: the map stays as it is, bit for bit
		if (out) *out = st;
		return UFO_B200_OK;
	}

	uint32_t cap0, up0;
	initial_caps(m->params, cap0, up0);
	const uint32_t oc = M.brick_cap;
	const uint32_t nc = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(cap0, 2ull * kept), 0x3ffffffull);
	// One array at a time (each_array's order): allocate the new one, gather the survivors, free the
	// old one.  A failure before the first array is replaced leaves the map as it was.
	bool changed = false;
	auto each = [&](Pool pool, Retain retain, uint32_t old_cap, uint32_t new_cap, uint32_t keep) {
		each_array(m, pool, [&](const PoolArray& a) {
			if (a.retain != retain) return;
			reshape(m, a, old_cap, new_cap, keep, d_src);
			changed = true;
		});
	};
	CK(cudaEventRecord(ev.e[1], s));
	try {
		each(Pool::Brick, Retain::Compact, oc, nc, kept);
		CK(cudaEventRecord(ev.e[2], s));
		// per-scan lists and everything above the bricks start from their initial state
		each(Pool::Brick, Retain::Renew, oc, nc, 0);
		M.brick_cap = nc;
		brick_hash(m, kept);
		// the upper-node pool, in proportion, rebuilt from the survivors' depth-4 aggregates: a child
		// that never reports counts as never-touched space, which is what a removed brick now is
		const uint32_t ou = M.up_cap, nu = std::max(up0, nc / 2);
		each(Pool::Upper, Retain::Renew, ou, nu, 0);
		M.up_cap = nu;
		upper_hash(m, 0);
		m->n_bricks = kept;
		m->n_upper = 0;
		page_propagate(m, nullptr, kept, false);
		CK(cudaEventRecord(ev.e[3], s));
		// blocks that hold a written octet, for the statistics of later scans
		DevBuf b_cnt;
		unsigned long long* d_cnt = b_cnt.alloc<unsigned long long>(1);
		unsigned long long blocks = 0;
		CK(cudaMemsetAsync(d_cnt, 0, 8, s));
		if (kept) k_page_count_blocks<<<m->sm_count * 4, 256, 0, s>>>(M.meta, (size_t)kept * 64, d_cnt);
		CK(cudaMemcpyAsync(&blocks, d_cnt, 8, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
		m->n_blocks = (uint32_t)blocks;
	} catch (...) {
		if (!changed) throw;
		// the arrays no longer agree on their slots
		m->poisoned = true;
		m->set_error("retain failed after the leaves were compacted; the map is unusable");
		throw;
	}
	CK(cudaEventElapsedTime(&st.ms_compact, ev.e[1], ev.e[2]));
	CK(cudaEventElapsedTime(&st.ms_upper, ev.e[2], ev.e[3]));
	st.bricks_kept = kept;
	st.bricks_removed = n - kept;
	fill_pool_state(m, st.bricks_kept, st.brick_cap_after, st.device_bytes_after);
	if (out) *out = st;
	return UFO_B200_OK;
}

int page_out(Map* m, const Volume& vol, void* buf, size_t cap, size_t* size)
{
	const int allowed = page_allowed(m, "page_out");
	if (allowed != UFO_B200_OK) return allowed;
	CK(cudaSetDevice(m->device));
	sync_map(m);
	DeviceMap& M = m->M;
	cudaStream_t s = m->stream;
	const uint32_t n = m->n_bricks;
	const bool color = M.color != 0;
	uint32_t cnt = 0;
	DevBuf b_key[2], b_slot[2], b_cnt, b_tmp;
	unsigned long long* d_key[2] = {nullptr, nullptr};
	uint32_t* d_slot[2] = {nullptr, nullptr};
	if (vol.n && n) {
		for (int k = 0; k < 2; ++k) {
			d_key[k] = b_key[k].alloc<unsigned long long>(n);
			d_slot[k] = b_slot[k].alloc<uint32_t>(n);
		}
		uint32_t* d_cnt = b_cnt.alloc<uint32_t>(1);
		CK(cudaMemsetAsync(d_cnt, 0, 4, s));
		DeviceVolume dvol;
		launch_page_classify(m, vol, dvol, nullptr, d_key[0], d_slot[0], d_cnt);
		CK(cudaMemcpyAsync(&cnt, d_cnt, 4, cudaMemcpyDeviceToHost, s));
		CK(cudaStreamSynchronize(s));
	}
	*size = page_bytes(cnt, color);
	if (!buf || cap < *size) return UFO_B200_OK;

	uint8_t* o = static_cast<uint8_t*>(buf);
	PageHeader h{};
	h.magic = kPageMagic;
	h.version = kPageVersion;
	h.color = color ? 1u : 0u;
	memcpy(&h.resolution_bits, &m->params.resolution, 8);
	h.depth_levels = M.g.depth_levels;
	h.n_bricks = cnt;
	memcpy(o, &h, sizeof(h));
	if (!cnt) return UFO_B200_OK;
	// ascending packed key: equal maps give equal blobs whatever their slot order
	size_t tmp_bytes = 0;
	CK(cub::DeviceRadixSort::SortPairs(nullptr, tmp_bytes, d_key[0], d_key[1], d_slot[0], d_slot[1], (int)n, 0, 64, s));
	void* d_tmp = b_tmp.alloc<uint8_t>(tmp_bytes);
	CK(cub::DeviceRadixSort::SortPairs(d_tmp, tmp_bytes, d_key[0], d_key[1], d_slot[0], d_slot[1], (int)n, 0, 64, s));
	++m->launches;
	const uint32_t* slots = d_slot[1];
	o += sizeof(h);
	CK(cudaMemcpyAsync(o, d_key[1], (size_t)cnt * 8, cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	o += (size_t)cnt * 8;
	PageStage stage;
	page_section_out(s, stage, cnt, kPageLeafBytes, o, [&](uint8_t* d, size_t first, size_t k) {
		launch_page_move<false>(m, d, M.leaf, slots + first, k, kPageLeafBytes);
	});
	o += (size_t)cnt * kPageLeafBytes;
	page_section_out(s, stage, cnt, kPageBitsBytes, o, [&](uint8_t* d, size_t first, size_t k) {
		k_page_bits_out<<<(uint32_t)std::min<size_t>((k * 64 + 255) / 256, (size_t)m->sm_count * 8), 256, 0, s>>>(M.meta, slots + first, k * 64, d);
		++m->launches;
	});
	o += (size_t)cnt * kPageBitsBytes;
	if (color)
		page_section_out(s, stage, cnt, kPageLeafBytes, o, [&](uint8_t* d, size_t first, size_t k) {
			launch_page_move<false>(m, d, M.leaf_rgb, slots + first, k, kPageLeafBytes);
		});
	return UFO_B200_OK;
}

int page_header_ok(const void* blob, size_t size, PageHeader& h)
{
	if (!blob || size < sizeof(PageHeader)) return 1;
	memcpy(&h, blob, sizeof(h));
	if (h.magic != kPageMagic) return 2;
	if (h.version != kPageVersion) return 3;
	return 0;
}

int page_in(Map* m, const void* blob, size_t size, ufo_b200_retain_stats* out)
{
	const int allowed = page_allowed(m, "page_in");
	if (allowed != UFO_B200_OK) return allowed;
	DeviceMap& M = m->M;
	PageHeader h{};
	switch (page_header_ok(blob, size, h)) {
		case 0: break;
		case 1: m->set_error("page_in: %zu bytes are less than a page header", size); return UFO_B200_E_INVALID;
		case 2: m->set_error("page_in: not a page blob (bad magic)"); return UFO_B200_E_INVALID;
		default: m->set_error("page_in: page format version %u, this library reads version %u", h.version, kPageVersion); return UFO_B200_E_INVALID;
	}
	const bool color = M.color != 0;
	unsigned long long res_bits;
	memcpy(&res_bits, &m->params.resolution, 8);
	if ((h.color != 0) != color || h.color > 1) {
		m->set_error("page_in: the blob is from a %s map, this is a %s map", h.color ? "colour" : "mono", color ? "colour" : "mono");
		return UFO_B200_E_INVALID;
	}
	if (h.resolution_bits != res_bits || h.depth_levels != M.g.depth_levels) {
		double r;
		memcpy(&r, &h.resolution_bits, 8);
		m->set_error("page_in: the blob is from a map of resolution %.17g and %u depth levels, this map has %.17g and %u", r,
		             h.depth_levels, m->params.resolution, M.g.depth_levels);
		return UFO_B200_E_INVALID;
	}
	if (h.n_bricks > 0x3ffffffull || size != page_bytes(h.n_bricks, color)) {
		m->set_error("page_in: the header says %llu bricks, which does not match the blob's %zu bytes", h.n_bricks, size);
		return UFO_B200_E_INVALID;
	}
	CK(cudaSetDevice(m->device));
	sync_map(m);
	cudaStream_t s = m->stream;
	ufo_b200_retain_stats st{};
	fill_pool_state(m, st.bricks_before, st.brick_cap_before, st.device_bytes_before);
	fill_pool_state(m, st.bricks_kept, st.brick_cap_after, st.device_bytes_after);
	const uint32_t n = (uint32_t)h.n_bricks;
	if (!n) {
		if (out) *out = st;
		return UFO_B200_OK;
	}
	set_value_floor(m, -INFINITY);  // the blob may come from a map with another sensor model
	const uint8_t* p_keys = static_cast<const uint8_t*>(blob) + sizeof(PageHeader);
	const uint8_t* p_leaf = p_keys + (size_t)n * 8;
	const uint8_t* p_bits = p_leaf + (size_t)n * kPageLeafBytes;
	const uint8_t* p_rgb = p_bits + (size_t)n * kPageBitsBytes;

	DevBuf b_keys, b_slot, b_cnt, b_bits;
	unsigned long long* d_keys = b_keys.alloc<unsigned long long>(n);
	uint32_t* d_slot = b_slot.alloc<uint32_t>(n);
	uint32_t* d_cnt = b_cnt.alloc<uint32_t>(2);
	Events ev;
	CK(cudaEventRecord(ev.e[0], s));
	CK(cudaMemcpyAsync(d_keys, p_keys, (size_t)n * 8, cudaMemcpyHostToDevice, s));
	CK(cudaMemsetAsync(d_cnt, 0, 8, s));
	// its own pass, before anything is created: a refusal leaves no brick behind
	k_page_lookup<<<(n + 255) / 256, 256, 0, s>>>(M, d_keys, n, d_cnt);
	CK(cudaGetLastError());
	++m->launches;
	uint32_t counts[2] = {0, 0};
	CK(cudaMemcpyAsync(counts, d_cnt, 8, cudaMemcpyDeviceToHost, s));
	CK(cudaStreamSynchronize(s));
	if (counts[1]) {
		m->set_error("page_in: %u of the blob's %u brick keys lie outside the map or are out of order", counts[1], n);
		return UFO_B200_E_INVALID;
	}
	if (counts[0]) {
		m->set_error("page_in: %u of the blob's %u bricks exist in the map; a page cannot be merged into existing bricks", counts[0], n);
		return UFO_B200_E_INVALID;
	}
	// Every brick first, nothing written until all exist: creation is idempotent, so a pass that
	// ran into a full pool is repeated as a whole after the pool has grown.
	const int rc = run_growing(m, "page_in", [&]() {
		k_page_create<<<(n + 255) / 256, 256, 0, s>>>(M, d_keys, n, d_slot);
		++m->launches;
	});
	if (rc != UFO_B200_OK) return rc;
	CK(cudaEventRecord(ev.e[1], s));
	{
		PageStage stage;
		page_section_in(s, stage, n, kPageLeafBytes, p_leaf, [&](uint8_t* d, size_t first, size_t k) {
			launch_page_move<true>(m, M.leaf, d, d_slot + first, k, kPageLeafBytes);
		});
		if (color)
			page_section_in(s, stage, n, kPageLeafBytes, p_rgb, [&](uint8_t* d, size_t first, size_t k) {
				launch_page_move<true>(m, M.leaf_rgb, d, d_slot + first, k, kPageLeafBytes);
			});
		page_section_in(s, stage, n, kPageBitsBytes, p_bits, [&](uint8_t* d, size_t first, size_t k) {
			k_page_bits_in<<<(uint32_t)std::min<size_t>((k * 64 + 255) / 256, (size_t)m->sm_count * 8), 256, 0, s>>>(M.meta, d_slot + first, k * 64, d);
			++m->launches;
		});
	}
	CK(cudaEventRecord(ev.e[2], s));
	// line maxima, flags, inner colours, depth 3 / 4 and the levels above, under the current sensor model
	page_propagate(m, d_slot, n, true);
	CK(cudaEventRecord(ev.e[3], s));
	CK(cudaStreamSynchronize(s));
	size_t blocks = 0;
	for (size_t i = 0; i < (size_t)n * 64; ++i) blocks += p_bits[i] ? 1 : 0;
	m->n_blocks += (uint32_t)blocks;
	CK(cudaEventElapsedTime(&st.ms_classify, ev.e[0], ev.e[1]));
	CK(cudaEventElapsedTime(&st.ms_compact, ev.e[1], ev.e[2]));
	CK(cudaEventElapsedTime(&st.ms_upper, ev.e[2], ev.e[3]));
	fill_pool_state(m, st.bricks_kept, st.brick_cap_after, st.device_bytes_after);
	if (out) *out = st;
	return UFO_B200_OK;
}

// A device copy of src, built the way retain rebuilds a map after its compaction: the first n_bricks
// entries of every Compact brick array copied (every slot below n_bricks is live), the Renew arrays at
// their fill, the change masks left out, the brick hash and the levels above the bricks rebuilt.
void clone_into(Map* m, Map* src)
{
	ufo_b200_params p = src->params;
	p.device = src->device;
	init_map(m, &p);
	m->params = src->params;
	m->occ_thr_log = src->occ_thr_log;
	m->free_thr_log = src->free_thr_log;
	m->hit_log = src->hit_log;
	m->miss_log = src->miss_log;
	m->cmin_log = src->cmin_log;
	m->cmax_log = src->cmax_log;
	m->value_floor = src->value_floor;
	refresh_model(m);
	m->no_dense = src->no_dense;
	m->M.scan_id = src->M.scan_id;  // the copied brick stamps hold scan ids of the source
	reset_bbox(m);
	DeviceMap& M = m->M;
	const uint32_t n = src->n_bricks;
	uint32_t cap0, up0;
	initial_caps(m->params, cap0, up0);
	M.brick_cap = (uint32_t)std::min<uint64_t>(std::max<uint64_t>(cap0, 2ull * n), 0x3ffffffull);
	M.up_cap = std::max(up0, M.brick_cap / 2);
	for (const Pool pool : {Pool::Brick, Pool::Upper})
		each_array(src, pool, [&](const PoolArray& a) {
			if (a.have == Have::Changes) return;
			const uint32_t keep = (pool == Pool::Brick && a.retain == Retain::Compact) ? n : 0u;
			reshape(m, a, 0, pool_cap(m, pool), keep, nullptr, src);
		});
	m->ctr.ensure(m, sizeof(Counters), 0);
	M.ctr = m->ctr.p;
	brick_hash(m, n);
	upper_hash(m, 0);
	m->n_blocks = src->n_blocks;
	m->n_bricks = n;
	m->n_upper = 0;
	page_propagate(m, nullptr, n, false);
	CK(cudaStreamSynchronize(m->stream));
}

int clone(Map* src, Map** out)
{
	if (src->M.route_world > 1 || src->route_inbox.p || src->M.shard_world > 1) {
		src->set_error("ufo_b200_clone: a routed or sharded map holds one rank's part and cannot be copied");
		return UFO_B200_E_UNSUPPORTED;
	}
	CK(cudaSetDevice(src->device));
	sync_map(src);
	if (src->poisoned) {
		src->set_error("an earlier scan failed half-way; ufo_b200_clear() the map first");
		return UFO_B200_E_INVALID;
	}
	Map* m = new Map;
	try {
		clone_into(m, src);
	} catch (...) {
		// a failed cudaMalloc is the runtime's last error: read and clear it, so that later calls on the
		// source do not report it
		const bool oom = cudaGetLastError() == cudaErrorMemoryAllocation;
		const std::string why = m->err;
		ufo_b200_destroy(m);
		if (oom) {
			src->set_error("ufo_b200_clone: the device cannot hold the copy");
			return UFO_B200_E_NOMEM;
		}
		if (!why.empty()) src->err = why;
		throw;
	}
	*out = m;
	return UFO_B200_OK;
}
}  // namespace

extern "C" {

int ufo_b200_clone(ufo_b200_map* src, ufo_b200_map** out)
{
	if (out) *out = nullptr;
	if (!src || !out) return UFO_B200_E_INVALID;
	return guarded(src, [&]() { return clone(src, out); });
}

int ufo_b200_retain_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, ufo_b200_retain_stats* out)
{
	if (!m) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() { bump_revision(m); return retain(m, Volume{as_records(bv), (uint32_t)n_bv, {}, {}}, out); });
}

int ufo_b200_retain(ufo_b200_map* m, const double box6[6], ufo_b200_retain_stats* out)
{
	if (!m || !box6) return UFO_B200_E_INVALID;
	const VolRec r = aabb_record(box6);
	return ufo_b200_retain_bv(m, reinterpret_cast<const ufo_b200_volume*>(&r), 1, out);
}

int ufo_b200_page_out_bv(ufo_b200_map* m, const ufo_b200_volume* bv, size_t n_bv, void* buf, size_t cap, size_t* size)
{
	if (!m || !size) return UFO_B200_E_INVALID;
	if (!volume_ok(m, bv, n_bv)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() { return page_out(m, Volume{as_records(bv), (uint32_t)n_bv, {}, {}}, buf, cap, size); });
}

int ufo_b200_page_in(ufo_b200_map* m, const void* blob, size_t size, ufo_b200_retain_stats* out)
{
	if (!m || (!blob && size)) return UFO_B200_E_INVALID;
	return guarded(m, [&]() { bump_revision(m); return page_in(m, blob, size, out); });
}

int ufo_b200_page_info(const void* blob, size_t size, ufo_b200_page_header* out)
{
	if (!out) return UFO_B200_E_INVALID;
	PageHeader h{};
	if (page_header_ok(blob, size, h) || h.color > 1 || h.n_bricks > 0x3ffffffull) return UFO_B200_E_INVALID;
	*out = ufo_b200_page_header{};
	out->version = h.version;
	out->color = h.color;
	out->depth_levels = h.depth_levels;
	memcpy(&out->resolution, &h.resolution_bits, 8);
	out->n_bricks = h.n_bricks;
	out->bytes = page_bytes(h.n_bricks, h.color != 0);
	return UFO_B200_OK;
}

int ufo_b200_pool_stats(ufo_b200_map* m, ufo_b200_pool_counts* out)
{
	if (!m || !out) return UFO_B200_E_INVALID;
	return guarded(m, [&]() {
		CK(cudaSetDevice(m->device));
		sync_map(m);
		*out = ufo_b200_pool_counts{m->n_bricks, m->M.brick_cap, m->n_upper, m->M.up_cap, m->device_bytes};
		return (int)UFO_B200_OK;
	});
}

}  // extern "C"
