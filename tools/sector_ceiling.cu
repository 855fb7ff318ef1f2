// sector_ceiling.cu -- what HBM delivers for K3's access pattern: read-modify-write of a
// SPARSE set of 32 B sectors (the touched octets of a scan: ~24 % of the 512 leaf sectors of
// each touched 16 KB brick), with nothing else to do per sector.  K3's leaf traffic is compared
// against this number instead of the streaming-copy peak.
//
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o tools/sector_ceiling tools/sector_ceiling.cu
//   tools/sector_ceiling            (prints one JSON line per pattern)
//
// Patterns over B bricks of 16 KB in a pool of P bricks, each touched brick with a random set of
// sectors of density d:
//   rmw      every listed sector: 2 x LDG.128, add, 2 x STG.128  (thread per sector, 4 in flight)
//   read     loads only (sum kept alive)
// and the sector set of K3 itself ("k3_leaf", "k3_all"), shaped by the counters of the bench
// workload: in every touched brick 53 % of the 64 blocks are marked (D_2 / 64 D_4); a marked block
// has touched octets in ONE of its two 128 B lines with probability 0.86, in both otherwise
// (touched_lines / D_2 = 1.14), and 81 % of the 4 octets of a touched line are touched
// (D_1 / touched_lines = 3.2); k3_all adds, per brick, the depth-1 sector of every marked block
// (own region), the mask / meta slab (1280 B) and the depth-2 aggregates (512 B) -- the metadata of
// the layout with per-octet maxima; k3_pairs the layout with pair maxima: the leaf sectors, the untouched
// partner (2k, 2k+1) of every touched octet (read-modify-written here, only read by K3: an upper
// bound), the mask / meta slab and the brick's pair maxima (1 KB); k3_lines is the layout with one
// maximum per 128 B line: the leaf sectors, every other octet of each touched line (again
// read-modify-written), the mask / meta slab and the brick's line maxima (512 B).  The "_ro"
// variants of the last two only read the untouched partners / line-mates, as K3 does.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#define CK(x)                                                                      \
	do {                                                                             \
		cudaError_t e = (x);                                                           \
		if (e != cudaSuccess) {                                                        \
			fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e));    \
			exit(1);                                                                     \
		}                                                                              \
	} while (0)

constexpr uint32_t kReadOnly = 0x80000000u;  // list flag (mode 0): load the sector, do not write it back

template <int MODE>  // 0 rmw, 1 read
__global__ void __launch_bounds__(256) k_sectors(float4* __restrict__ pool, const uint32_t* __restrict__ list, uint32_t n, float* sink)
{
	constexpr int U = 4;
	float acc = 0.f;
	const uint32_t stride = gridDim.x * blockDim.x;
	for (uint32_t i0 = blockIdx.x * blockDim.x + threadIdx.x; i0 < n; i0 += U * stride) {
		float4 a[U], b[U];
		uint32_t s[U];
#pragma unroll
		for (int u = 0; u < U; ++u) {
			const uint32_t i = i0 + u * stride;
			s[u] = i < n ? list[i] : 0xffffffffu;
		}
#pragma unroll
		for (int u = 0; u < U; ++u) {
			if (s[u] != 0xffffffffu) {
				const size_t q = s[u] & ~kReadOnly;
				a[u] = pool[q * 2];
				b[u] = pool[q * 2 + 1];
			}
		}
#pragma unroll
		for (int u = 0; u < U; ++u) {
			if (s[u] == 0xffffffffu) continue;
			if (MODE == 0 && (s[u] & kReadOnly)) {
				acc += a[u].y + b[u].z;
			} else if (MODE == 0) {
				a[u].x += 1.f; a[u].y += 1.f; a[u].z += 1.f; a[u].w += 1.f;
				b[u].x += 1.f; b[u].y += 1.f; b[u].z += 1.f; b[u].w += 1.f;
				pool[(size_t)s[u] * 2] = a[u];
				pool[(size_t)s[u] * 2 + 1] = b[u];
			} else {
				acc += a[u].x + b[u].w;
			}
		}
	}
	if (acc == 123.456f) *sink = acc;
}

int main(int argc, char** argv)
{
	const uint32_t pool_bricks = argc > 1 ? (uint32_t)atoi(argv[1]) : 330000u;
	const uint32_t touched = argc > 2 ? (uint32_t)atoi(argv[2]) : 244000u;
	cudaDeviceProp prop;
	CK(cudaGetDeviceProperties(&prop, 0));
	float4* pool;
	CK(cudaMalloc(&pool, (size_t)pool_bricks * 16384));
	CK(cudaMemset(pool, 0, (size_t)pool_bricks * 16384));
	float* sink;
	CK(cudaMalloc(&sink, 4));
	std::mt19937_64 rng(12345);
	std::vector<uint32_t> perm(pool_bricks);
	for (uint32_t i = 0; i < pool_bricks; ++i) perm[i] = i;
	std::shuffle(perm.begin(), perm.end(), rng);
	cudaEvent_t e0, e1;
	CK(cudaEventCreate(&e0));
	CK(cudaEventCreate(&e1));
	const double dens[] = {0.06, 0.12, 0.24, 0.5, 1.0};
	for (int order = 0; order < 2; ++order) {
		for (double d : dens) {
			std::vector<uint32_t> list;
			list.reserve((size_t)(touched * 512 * d * 1.05) + 1024);
			std::uniform_real_distribution<double> uni(0.0, 1.0);
			for (uint32_t t = 0; t < touched; ++t) {
				const uint32_t brick = order == 0 ? perm[t] : t;  // scattered bricks / a contiguous run of bricks
				for (uint32_t s = 0; s < 512; ++s)
					if (uni(rng) < d) list.push_back(brick * 512u + s);
			}
			const uint32_t n = (uint32_t)list.size();
			uint32_t* dl;
			CK(cudaMalloc(&dl, (size_t)n * 4));
			CK(cudaMemcpy(dl, list.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
			for (int mode = 0; mode < 2; ++mode) {
				const int grid = prop.multiProcessorCount * 8;
				float best = 1e30f;
				for (int rep = 0; rep < 5; ++rep) {
					CK(cudaEventRecord(e0));
					if (mode == 0) k_sectors<0><<<grid, 256>>>(pool, dl, n, sink);
					else k_sectors<1><<<grid, 256>>>(pool, dl, n, sink);
					CK(cudaEventRecord(e1));
					CK(cudaEventSynchronize(e1));
					float ms;
					CK(cudaEventElapsedTime(&ms, e0, e1));
					if (rep >= 1) best = std::min(best, ms);
				}
				const double bytes = (double)n * (mode == 0 ? 64.0 : 32.0);
				printf("{\"pattern\": \"%s\", \"bricks\": \"%s\", \"density\": %.2f, \"sectors\": %u, \"ms\": %.4f, \"sectors_per_s\": %.4g, \"GBps\": %.1f}\n",
				       mode == 0 ? "rmw" : "read", order == 0 ? "scattered" : "contiguous", d, n, best, n / (best * 1e-3), bytes / (best * 1e-3) / 1e9);
			}
			CK(cudaFree(dl));
		}
	}
	// K3's own sector set
	{
		const double pb = argc > 3 ? atof(argv[3]) : 0.53, p_both = argc > 4 ? atof(argv[4]) : 0.14, po = argc > 5 ? atof(argv[5]) : 0.81;
		std::uniform_real_distribution<double> uni(0.0, 1.0);
		// regions inside the pool, in 32 B sectors: leaves [0, T*512), depth-1 [T*512, T*576), slab + depth-2
		// [T*576, T*632); k3_pairs: slab + pair maxima [T*576, T*648); k3_lines: slab + line maxima [T*576, T*632)
		const uint32_t T = std::min(touched, (uint32_t)((size_t)pool_bricks * 512 / 648));
		const char* names[] = {"k3_leaf", "k3_all", "k3_pairs", "k3_lines", "k3_pairs_ro", "k3_lines_ro"};
		std::vector<uint32_t> pt(T);
		for (uint32_t i = 0; i < T; ++i) pt[i] = i;
		std::shuffle(pt.begin(), pt.end(), rng);
		for (int all = 0; all < 6; ++all) {
			const bool pairs = all == 2 || all == 4, lines_ = all == 3 || all == 5, ro = all >= 4;
			std::vector<uint32_t> list;
			size_t leaf_sectors = 0, lines = 0;
			for (uint32_t t = 0; t < T; ++t) {
				const uint32_t brick = pt[t];
				for (uint32_t blk = 0; blk < 64; ++blk) {
					if (uni(rng) >= pb) continue;
					uint32_t t8 = 0;
					const bool both = uni(rng) < p_both;
					const uint32_t first = uni(rng) < 0.5 ? 0u : 1u;
					for (uint32_t h = 0; h < 2; ++h) {
						if (!both && h != first) continue;
						uint32_t l4 = 0;
						for (uint32_t o = 0; o < 4; ++o)
							if (uni(rng) < po) l4 |= 1u << o;
						if (!l4) l4 = 1u << (blk & 3);
						t8 |= l4 << (4 * h);
					}
					const uint32_t ld = pairs    ? t8 | ((t8 & 0x55u) << 1) | ((t8 & 0xaau) >> 1)
					                    : lines_ ? ((t8 & 0x0fu) ? 0x0fu : 0u) | ((t8 & 0xf0u) ? 0xf0u : 0u)
					                             : t8;
					for (uint32_t o = 0; o < 8; ++o)
						if ((ld >> o) & 1u) list.push_back((brick * 512u + blk * 8u + o) | (ro && !((t8 >> o) & 1u) ? kReadOnly : 0u));
					leaf_sectors += __builtin_popcount(t8);
					lines += ((t8 & 0x0f) ? 1 : 0) + ((t8 & 0xf0) ? 1 : 0);
					if (all == 1) list.push_back(T * 512u + brick * 64u + blk);
				}
				if (all == 1)
					for (uint32_t q = 0; q < 56; ++q) list.push_back(T * 576u + brick * 56u + q);
				if (pairs)
					for (uint32_t q = 0; q < 72; ++q) list.push_back(T * 576u + brick * 72u + q);
				if (lines_)
					for (uint32_t q = 0; q < 56; ++q) list.push_back(T * 576u + brick * 56u + q);
			}
			const uint32_t n = (uint32_t)list.size();
			for (uint32_t e : list)
				if ((e & ~kReadOnly) >= pool_bricks * 512u) {
					fprintf(stderr, "%s: sector %u outside the pool\n", names[all], e & ~kReadOnly);
					return 1;
				}
			uint32_t* dl;
			CK(cudaMalloc(&dl, (size_t)n * 4));
			CK(cudaMemcpy(dl, list.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
			float best = 1e30f;
			for (int rep = 0; rep < 5; ++rep) {
				CK(cudaEventRecord(e0));
				k_sectors<0><<<prop.multiProcessorCount * 8, 256>>>(pool, dl, n, sink);
				CK(cudaEventRecord(e1));
				CK(cudaEventSynchronize(e1));
				float ms;
				CK(cudaEventElapsedTime(&ms, e0, e1));
				if (rep >= 1) best = std::min(best, ms);
			}
			printf("{\"pattern\": \"%s\", \"bricks\": %u, \"p_block\": %.2f, \"p_both_lines\": %.2f, \"p_octet_in_line\": %.2f, \"sectors\": %u, \"leaf_sectors\": %zu, \"leaf_lines_128B\": %zu, \"ms\": %.4f, \"GBps\": %.1f}\n",
			       names[all], T, pb, p_both, po, n, leaf_sectors, lines, best, (double)n * 64.0 / (best * 1e-3) / 1e9);
			CK(cudaFree(dl));
		}
	}
	return 0;
}
