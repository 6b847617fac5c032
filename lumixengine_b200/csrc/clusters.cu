// PipelineImpl::fillClusters (src/renderer/pipeline.cpp:3327-3684) on the device, for the LOCAL_LIGHT segment a view's cull left in HBM.
//
//   clusters_items_kernel  one cooperative launch.  Items are the lights of the segment, then the env probes, then the refl probes; block b
//             owns one contiguous run of them.  Pass 1: a light's ClusterLight (:3388-3396), its entity, its shadow priority (:3322-3325)
//             and flags; every item's range() per axis (:3540-3561) and its cluster count.  Block totals -> grid barrier -> every block
//             sums the totals before it.  Pass 2: per tile of CL_THREADS items a block scan of the counts, then the tile's (cluster, item)
//             pairs are written by all threads at their scanned positions, so pairs lie in item order.
//   clusters_atlas_kernel  one block: the list AtlasSorter::push (:2375-2401) leaves over the lights in order, by a radix select of the
//             64 best casters, or by replaying the pushes when a priority is NaN.  Also the lights without CAST_SHADOWS that have an
//             atlas entry (:3405-3407), in light order.
//   radix_sort_kernel (radix_sort.cu)  the stable sort of the pairs by cluster: within a cluster the pairs keep item order, which is the
//             order of the reference's three scatter passes (lights, env probes, refl probes, each in increasing index).
//   clusters_tables_kernel  map[] = the sorted items; clusters[c] from binary searches of the sorted keys (start of the run = offset, the
//             kind boundaries inside it = the three counts).
// The planes (:3468-3495) are built on the host with the reference's fp32 arithmetic and powf and go to the items kernel as a parameter.
#include "grid_barrier.cuh"
#include "lb200_internal.h"

#include <algorithm>
#include <math.h>
#include <memory>
#include <new>
#include <unordered_map>
#include <vector>

static_assert(sizeof(lb200_point_light) == 32, "PointLight fields, render_module.h:156-171");
static_assert(sizeof(lb200_cluster_light) == 64, "ClusterLight, pipeline.cpp:3331-3341");
static_assert(sizeof(lb200_cluster) == 16, "Cluster, pipeline.cpp:3343-3348");
static_assert(sizeof(lb200_cluster_env_probe) == 208, "ClusterEnvProbe, pipeline.cpp:3350-3359");
static_assert(sizeof(lb200_cluster_refl_probe) == 48, "ClusterReflProbe, pipeline.cpp:3361-3367");
static_assert(sizeof(lb200_shadow_candidate) == 12, "AtlasSorter::Light, pipeline.cpp:2394-2398");

namespace {

using namespace lb;

constexpr int CL_THREADS = 256;
constexpr int CL_ATLAS_THREADS = 1024;
constexpr uint32_t CL_MAX_DIM = 4096;                      // w, h: (4096 + 63) / 64 + 1 = 65 planes, the reference's xplanes[65]
constexpr int CL_ZS = 16;                                  // size.z
constexpr int CL_PLANES = 65 + 65 + 17;                    // xplanes, yplanes, zplanes
constexpr uint32_t RT_LOCAL_LIGHT = 2;                     // render_module.h:293-301
constexpr uint8_t LF_CASTER = 1, LF_UNCAST_IN_ATLAS = 2;   // per-light flags of pass 1
constexpr uint32_t CL_NONE = 0xffffffffu;

struct Planes { float4 p[CL_PLANES]; }; // x at [0, sx], y at [65, 65 + sy], z at [130, 146]

// What the device leaves for the one read-back of a fill
struct DevResult {
	uint32_t n_lights, n_sort;        // lights of the segment; pairs the sort takes (min(pairs, capacity))
	unsigned long long n_pairs;
	uint32_t n_shadow, n_uncast;
	lb200_shadow_candidate shadow[LB200_CLUSTERS_MAX_ATLAS];
	int32_t uncast[LB200_CLUSTERS_MAX_ATLAS];
};

struct ItemsParams {
	Planes planes;
	double cam[3];
	int sx, sy;                                 // size.x, size.y
	const uint32_t* ids;                        // the segment
	const uint32_t* n_lights_dev;               // its count, the cull's counter
	uint32_t light_cap;                         // the segment's size: no cull writes more
	uint32_t n_env, n_refl;
	const float4* probes;                       // n_env then n_refl: pos, radius
	const SkEntity* ent;
	const lb200_point_light* pl;
	const int32_t* atlas;
	lb200_cluster_light* lights;
	int32_t* light_entities;
	float* prio;
	uint8_t* lflags;
	unsigned long long* item_range;             // per item: x0, x1, y0, y1, z0, z1 as bytes (+1, so -1 is 0)
	unsigned long long* block_total;            // [gridDim]
	uint64_t* keys;                             // cluster
	uint64_t* values;                           // kind << 32 | index of the item within its kind
	uint32_t pair_cap;
	DevResult* res;
	GridBar* bar;
};

// planeDist (geometry.cpp:826-828), in the reference's order
__device__ __forceinline__ float plane_dist(const float4& pl, const float3& p) { return pl.x * p.x + pl.y * p.y + pl.z * p.z + pl.w; }

// range() of fillClusters (:3540-3561), statement for statement: {-1, -1} or [x, y) of clusters the sphere may touch
__device__ __forceinline__ int2 cluster_range(const float3& p, float r, int size, const float4* planes) {
	int2 range = make_int2(-1, -1);
	if (plane_dist(planes[0], p) < -r) return range;
	for (int i = 0; i < size; ++i) {
		const float dist = plane_dist(planes[i + 1], p);
		if (dist > r) continue;
		range.x = i;
		for (int i2 = i + 1; i2 < size + 1; ++i2) {
			const float d = plane_dist(planes[i2], p);
			if (d < -r) {
				range.y = i2;
				return range;
			}
		}
		range.y = size;
		return range;
	}
	return range;
}

__device__ __forceinline__ unsigned long long pack_ranges(int2 x, int2 y, int2 z) {
	return (unsigned long long)(uint8_t)(x.x + 1) | (unsigned long long)(uint8_t)(x.y + 1) << 8 | (unsigned long long)(uint8_t)(y.x + 1) << 16 |
	       (unsigned long long)(uint8_t)(y.y + 1) << 24 | (unsigned long long)(uint8_t)(z.x + 1) << 32 | (unsigned long long)(uint8_t)(z.y + 1) << 40;
}
__device__ __forceinline__ int range_at(unsigned long long r, int k) { return (int)((r >> (8 * k)) & 0xffu) - 1; }
// the pairs of :3566-3576 for one item: (x1 - x0) (y1 - y0) (z1 - z0), 0 when any axis is {-1, -1}
__device__ __forceinline__ uint32_t range_count(unsigned long long r) {
	return (uint32_t)((range_at(r, 1) - range_at(r, 0)) * (range_at(r, 3) - range_at(r, 2)) * (range_at(r, 5) - range_at(r, 4)));
}

// exclusive scan of one value per thread over the block; *total = the sum (all threads)
template <int THREADS> __device__ __forceinline__ uint32_t block_scan(uint32_t v, uint32_t* s_warp, uint32_t* total) {
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	uint32_t x = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (uint32_t)o) x += y; }
	if (lane == 31) s_warp[warp] = x;
	__syncthreads();
	uint32_t before = 0, sum = 0;
	for (int w = 0; w < THREADS / 32; ++w) { const uint32_t t = s_warp[w]; if (w < (int)warp) before += t; sum += t; }
	__syncthreads();
	*total = sum;
	return before + x - v;
}

__global__ void __launch_bounds__(CL_THREADS) clusters_items_kernel(const __grid_constant__ ItemsParams P) {
	__shared__ float4 s_planes[CL_PLANES];
	__shared__ uint32_t s_warp[CL_THREADS / 32];
	__shared__ uint32_t s_off[CL_THREADS + 1];
	__shared__ unsigned long long s_rng[CL_THREADS];
	__shared__ unsigned long long s_red[CL_THREADS / 32];
	const uint32_t tid = threadIdx.x;
	for (uint32_t i = tid; i < CL_PLANES; i += CL_THREADS) s_planes[i] = P.planes.p[i];
	__syncthreads();
	const float4* xpl = s_planes;
	const float4* ypl = s_planes + 65;
	const float4* zpl = s_planes + 130;
	const uint32_t n_lights = min(__ldg(P.n_lights_dev), P.light_cap);
	const uint32_t n_items = n_lights + P.n_env + P.n_refl;
	const uint32_t chunk = (n_items + gridDim.x - 1) / gridDim.x;
	const uint32_t begin = min(blockIdx.x * chunk, n_items), end = min(begin + chunk, n_items);

	// pass 1
	unsigned long long mine = 0;
	for (uint32_t g = begin + tid; g < end; g += CL_THREADS) {
		float3 p;
		float r;
		if (g < n_lights) {
			const uint32_t e = __ldg(P.ids + g);
			const SkEntity& rec = P.ent[e];
			const lb200_point_light pl = P.pl[e];
			const int32_t atlas = __ldg(P.atlas + e);
			const double lx = rec.pos[0], ly = rec.pos[1], lz = rec.pos[2];
			const float4 rot = *reinterpret_cast<const float4*>(rec.rot);
			p = make_float3((float)(lx - P.cam[0]), (float)(ly - P.cam[1]), (float)(lz - P.cam[2]));
			r = pl.range;
			const bool cast = (pl.flags & LB200_LIGHT_CAST_SHADOWS) != 0;
			float4* out = reinterpret_cast<float4*>(P.lights + g);
			out[0] = make_float4(p.x, p.y, p.z, r);
			out[1] = rot;
			out[2] = make_float4(pl.color[0] * pl.intensity, pl.color[1] * pl.intensity, pl.color[2] * pl.intensity, pl.attenuation_param);
			out[3] = make_float4(__uint_as_float(cast && atlas >= 0 ? (uint32_t)atlas : CL_NONE), pl.fov, 0.0f, 0.0f);
			P.light_entities[g] = (int32_t)e;
			float prio = 0.0f;
			if (cast) { // computeShadowPriority(fov, radius, light_pos, cam_pos)
				const float lr3 = r * r * r;
				const double dx = P.cam[0] - lx, dy = P.cam[1] - ly, dz = P.cam[2] - lz;
				prio = (float)((double)(pl.fov * lr3) / sqrt(dx * dx + dy * dy + dz * dz));
			}
			P.prio[g] = prio;
			P.lflags[g] = cast ? LF_CASTER : atlas >= 0 ? LF_UNCAST_IN_ATLAS : 0;
		} else {
			const float4 q = __ldg(P.probes + (g - n_lights));
			p = make_float3(q.x, q.y, q.z);
			r = q.w;
		}
		const int2 xr = cluster_range(p, r, P.sx, xpl);
		const int2 yr = cluster_range(p, r, P.sy, ypl);
		const int2 zr = cluster_range(p, r, CL_ZS, zpl);
		const unsigned long long packed = pack_ranges(xr, yr, zr);
		P.item_range[g] = packed;
		mine += range_count(packed);
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
	if ((tid & 31u) == 0) s_red[tid >> 5] = mine;
	__syncthreads();
	if (tid == 0) {
		unsigned long long t = 0;
		for (int w = 0; w < CL_THREADS / 32; ++w) t += s_red[w];
		P.block_total[blockIdx.x] = t;
	}
	uint32_t passed = 0;
	grid_barrier(P.bar, passed);

	// where this block's pairs start; block 0 also publishes the total
	unsigned long long before = 0, all = 0;
	for (uint32_t b = tid; b < gridDim.x; b += CL_THREADS) {
		const unsigned long long t = __ldcg(P.block_total + b);
		if (b < blockIdx.x) before += t;
		all += t;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) { before += __shfl_xor_sync(0xffffffffu, before, o); all += __shfl_xor_sync(0xffffffffu, all, o); }
	__syncthreads();
	if ((tid & 31u) == 0) s_red[tid >> 5] = before;
	__syncthreads();
	unsigned long long base = 0;
	for (int w = 0; w < CL_THREADS / 32; ++w) base += s_red[w];
	__syncthreads();
	if ((tid & 31u) == 0) s_red[tid >> 5] = all;
	__syncthreads();
	if (blockIdx.x == 0 && tid == 0) {
		unsigned long long total = 0;
		for (int w = 0; w < CL_THREADS / 32; ++w) total += s_red[w];
		P.res->n_lights = n_lights;
		P.res->n_pairs = total;
		P.res->n_sort = (uint32_t)min(total, (unsigned long long)P.pair_cap);
	}

	// pass 2: tiles of CL_THREADS items, their pairs at base + the scanned counts
	const uint32_t stride = (uint32_t)P.sx * (uint32_t)P.sy;
	for (uint32_t t0 = begin; t0 < end; t0 += CL_THREADS) {
		const uint32_t g = t0 + tid;
		const unsigned long long rng = g < end ? __ldcg(P.item_range + g) : 0ull;
		const uint32_t cnt = g < end ? range_count(rng) : 0u;
		uint32_t tile_total;
		const uint32_t off = block_scan<CL_THREADS>(cnt, s_warp, &tile_total);
		s_off[tid] = off;
		s_rng[tid] = rng;
		if (tid == 0) s_off[CL_THREADS] = tile_total;
		__syncthreads();
		for (uint32_t k = tid; k < tile_total; k += CL_THREADS) {
			int lo = 0, hi = CL_THREADS; // the last item whose first pair is at or before k (items without pairs share their offset)
			while (hi - lo > 1) { const int mid = (lo + hi) >> 1; if (s_off[mid] <= k) lo = mid; else hi = mid; }
			const unsigned long long rr = s_rng[lo];
			const uint32_t local = k - s_off[lo];
			const int x0 = range_at(rr, 0), y0 = range_at(rr, 2), z0 = range_at(rr, 4);
			const uint32_t nx = (uint32_t)(range_at(rr, 1) - x0), ny = (uint32_t)(range_at(rr, 3) - y0);
			const uint32_t x = (uint32_t)x0 + local % nx, y = (uint32_t)y0 + (local / nx) % ny, z = (uint32_t)z0 + local / (nx * ny);
			const unsigned long long at = base + k;
			if (at < P.pair_cap) {
				const uint32_t item = t0 + (uint32_t)lo;
				const uint32_t kind = item < n_lights ? 0u : item < n_lights + P.n_env ? 1u : 2u;
				const uint32_t index = kind == 0 ? item : kind == 1 ? item - n_lights : item - n_lights - P.n_env;
				P.keys[at] = x + y * (uint32_t)P.sx + z * stride;
				P.values[at] = (uint64_t)kind << 32 | index;
			}
		}
		base += tile_total;
		__syncthreads();
	}
}

// AtlasSorter::push (:2375-2401) for every CAST_SHADOWS light in light order, one block.
//
// Without NaN priorities the list AtlasSorter leaves is the first 64 casters ordered by (priority descending, light index ascending):
// a push lands after every entry that is not below it, and a full list drops its last entry.  The key (~orderable(priority) << 32 |
// index) orders casters that way, with -0 and +0 equal as the reference's `<` has them, and the 64 smallest keys are found by a radix
// select over the keys (8-bit digits from the top, stopping once the digits so far single out exactly the keys wanted), then ranked.
//
// A NaN priority never compares below anything, so with one among the casters the list depends on the push order itself.  Then warp 0
// replays the pushes, in order: it holds entry s at lane s % 32, slot s / 32.  Once the list is full a push changes it only if some entry
// is below its priority (:2378-2381), and the smallest non-NaN entry never decreases from then on, so a light whose priority is not above
// that minimum is skipped without being pushed: the result is the same.  Priorities that rise along the light order leave little to skip.
__device__ __forceinline__ unsigned long long caster_key(float p, uint32_t i) {
	uint32_t b = __float_as_uint(p);
	if ((b & 0x7fffffffu) == 0) b = 0;                      // -0 == +0
	const uint32_t asc = b ^ ((b >> 31) ? 0xffffffffu : 0x80000000u); // increasing with p
	return (unsigned long long)~asc << 32 | i;
}

__global__ void __launch_bounds__(CL_ATLAS_THREADS) clusters_atlas_kernel(const float* __restrict__ prio, const uint8_t* __restrict__ lflags,
	const int32_t* __restrict__ light_entities, DevResult* res)
{
	__shared__ uint32_t s_cand[CL_ATLAS_THREADS / 32], s_unc[CL_ATLAS_THREADS / 32];
	__shared__ int s_full, s_has_min;
	__shared__ float s_min;
	__shared__ uint32_t s_n_uncast, s_hist[256], s_k, s_n_sel;
	__shared__ unsigned long long s_prefix, s_mask, s_sel[LB200_CLUSTERS_MAX_ATLAS];
	const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
	const uint32_t n_lights = res->n_lights;
	if (tid == 0) { s_full = 0; s_has_min = 0; s_min = 0.0f; s_n_uncast = 0; }
	__syncthreads();

	// the uncast lights with an atlas entry, in order; whether a caster has a NaN priority; how many casters there are
	bool any_nan = false;
	uint32_t n_casters = 0;
	for (uint32_t b = 0; b < n_lights; b += CL_ATLAS_THREADS) {
		const uint32_t i = b + tid;
		const uint8_t f = i < n_lights ? lflags[i] : 0;
		const bool caster = (f & LF_CASTER) != 0;
		any_nan |= __syncthreads_or(caster && isnan(prio[i])) != 0;
		n_casters += (uint32_t)__syncthreads_count(caster);
		const uint32_t um = __ballot_sync(0xffffffffu, (f & LF_UNCAST_IN_ATLAS) != 0);
		if (lane == 0) s_unc[warp] = um;
		__syncthreads();
		if (warp == 0) {
			const uint32_t um_l = s_unc[lane];
			uint32_t x = __popc(um_l);
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (uint32_t)o) x += y; }
			uint32_t at = s_n_uncast + x - __popc(um_l);
			for (uint32_t m = um_l; m; m &= m - 1) {
				const uint32_t j = b + lane * 32 + (uint32_t)(__ffs((int)m) - 1);
				if (at < LB200_CLUSTERS_MAX_ATLAS) res->uncast[at] = light_entities[j];
				++at;
			}
			const uint32_t chunk_uncast = __shfl_sync(0xffffffffu, x, 31);
			if (lane == 0) s_n_uncast += chunk_uncast;
		}
		__syncthreads();
	}
	if (tid == 0) res->n_uncast = s_n_uncast;

	if (!any_nan) {
		const uint32_t want = min(n_casters, (uint32_t)LB200_CLUSTERS_MAX_ATLAS);
		if (tid == 0) { s_prefix = 0; s_mask = 0; s_k = want; s_n_sel = 0; }
		__syncthreads();
		unsigned long long limit = ~0ull; // the selection: casters whose key is <= limit
		for (int shift = 56; want && want < n_casters && shift >= 0; shift -= 8) {
			for (uint32_t d = tid; d < 256; d += CL_ATLAS_THREADS) s_hist[d] = 0;
			__syncthreads();
			const unsigned long long prefix = s_prefix, mask = s_mask;
			for (uint32_t b = 0; b < n_lights; b += CL_ATLAS_THREADS) { // whole warps: lanes without a key match only themselves
				const uint32_t i = b + tid;
				bool in = i < n_lights && (lflags[i] & LF_CASTER);
				const unsigned long long key = in ? caster_key(prio[i], i) : 0ull;
				in = in && (key & mask) == prefix;
				const uint32_t d = in ? (uint32_t)(key >> shift) & 255u : 256u + lane;
				const uint32_t peers = __match_any_sync(0xffffffffu, d);
				if (in && (int)lane == __ffs((int)peers) - 1) atomicAdd(&s_hist[d], (uint32_t)__popc(peers));
			}
			__syncthreads();
			if (tid == 0) {
				uint32_t below = 0, d = 0;
				while (below + s_hist[d] < s_k) below += s_hist[d++];
				s_k -= below;
				s_prefix = prefix | (unsigned long long)d << shift;
				s_mask = mask | 255ull << shift;
				s_hist[0] = s_hist[d]; // the keys that share the new prefix
			}
			__syncthreads();
			limit = s_prefix | ~s_mask;
			if (s_hist[0] == s_k) break; // every key with this prefix is wanted: the keys up to its last are the selection
			__syncthreads();
		}
		for (uint32_t i = tid; i < n_lights && want; i += CL_ATLAS_THREADS) {
			if (!(lflags[i] & LF_CASTER)) continue;
			const unsigned long long key = caster_key(prio[i], i);
			if (key <= limit) s_sel[atomicAdd(&s_n_sel, 1u)] = key;
		}
		__syncthreads();
		if (tid < want) {
			const unsigned long long key = s_sel[tid];
			uint32_t rank = 0;
			for (uint32_t t = 0; t < want; ++t) rank += s_sel[t] < key;
			const uint32_t j = (uint32_t)key;
			res->shadow[rank] = {j, prio[j], light_entities[j]};
		}
		if (tid == 0) res->n_shadow = want;
		return;
	}

	float p0 = 0.0f, p1 = 0.0f;      // warp 0: entries lane and lane + 32
	uint32_t i0 = 0, i1 = 0;
	int32_t e0 = 0, e1 = 0;
	uint32_t count = 0;
	for (uint32_t b = 0; b < n_lights; b += CL_ATLAS_THREADS) {
		const uint32_t i = b + tid;
		const uint8_t f = i < n_lights ? lflags[i] : 0;
		const float p = i < n_lights ? prio[i] : 0.0f;
		const bool cand = (f & LF_CASTER) && (!s_full || (s_has_min && s_min < p));
		const uint32_t cm = __ballot_sync(0xffffffffu, cand);
		if (lane == 0) s_cand[warp] = cm;
		__syncthreads();
		if (warp == 0) {
			for (uint32_t w = 0; w < CL_ATLAS_THREADS / 32; ++w) {
				for (uint32_t m = s_cand[w]; m; m &= m - 1) {
					const uint32_t j = b + w * 32 + (uint32_t)(__ffs((int)m) - 1);
					const float pj = prio[j];
					const uint32_t lt0 = __ballot_sync(0xffffffffu, lane < count && p0 < pj);
					const uint32_t lt1 = __ballot_sync(0xffffffffu, lane + 32 < count && p1 < pj);
					const uint32_t idx = lt0 ? (uint32_t)(__ffs((int)lt0) - 1) : lt1 ? 32u + (uint32_t)(__ffs((int)lt1) - 1) : count;
					if (idx == LB200_CLUSTERS_MAX_ATLAS) continue;
					if (count == LB200_CLUSTERS_MAX_ATLAS) --count;
					const int32_t ej = light_entities[j];
					// memmove(&lights[idx + 1], &lights[idx], count - idx) and the new entry at idx
					const float up_p0 = __shfl_up_sync(0xffffffffu, p0, 1), up_p1 = __shfl_up_sync(0xffffffffu, p1, 1);
					const uint32_t up_i0 = __shfl_up_sync(0xffffffffu, i0, 1), up_i1 = __shfl_up_sync(0xffffffffu, i1, 1);
					const int32_t up_e0 = __shfl_up_sync(0xffffffffu, e0, 1), up_e1 = __shfl_up_sync(0xffffffffu, e1, 1);
					const float c_p = __shfl_sync(0xffffffffu, p0, 31);
					const uint32_t c_i = __shfl_sync(0xffffffffu, i0, 31);
					const int32_t c_e = __shfl_sync(0xffffffffu, e0, 31);
					const uint32_t s0 = lane, s1 = lane + 32;
					if (s0 == idx) { p0 = pj; i0 = j; e0 = ej; }
					else if (s0 > idx && s0 <= count) { p0 = up_p0; i0 = up_i0; e0 = up_e0; }
					if (s1 == idx) { p1 = pj; i1 = j; e1 = ej; }
					else if (s1 > idx && s1 <= count) { p1 = lane ? up_p1 : c_p; i1 = lane ? up_i1 : c_i; e1 = lane ? up_e1 : c_e; }
					++count;
				}
			}
			// the screen of the next chunk: full, and the smallest non-NaN entry
			float mn = INFINITY;
			bool any = false;
			if (lane < count && p0 == p0) { mn = fminf(mn, p0); any = true; }
			if (lane + 32 < count && p1 == p1) { mn = fminf(mn, p1); any = true; }
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
			const bool has = __any_sync(0xffffffffu, any);
			if (lane == 0) { s_full = count == LB200_CLUSTERS_MAX_ATLAS; s_has_min = has; s_min = mn; }
		}
		__syncthreads();
	}
	if (warp == 0) {
		if (lane < count) res->shadow[lane] = {i0, p0, e0};
		if (lane + 32 < count) res->shadow[lane + 32] = {i1, p1, e1};
		if (lane == 0) res->n_shadow = count;
	}
}

// first position in [lo, hi) whose key is >= c
__device__ __forceinline__ uint32_t lower_key(const uint64_t* keys, uint32_t lo, uint32_t hi, uint64_t c) {
	while (lo < hi) { const uint32_t mid = lo + ((hi - lo) >> 1); if (__ldg(keys + mid) < c) lo = mid + 1; else hi = mid; }
	return lo;
}
// first position in [lo, hi) whose item is of kind >= k (kinds do not decrease inside a cluster's run)
__device__ __forceinline__ uint32_t lower_kind(const uint64_t* values, uint32_t lo, uint32_t hi, uint32_t k) {
	while (lo < hi) { const uint32_t mid = lo + ((hi - lo) >> 1); if ((uint32_t)(__ldg(values + mid) >> 32) < k) lo = mid + 1; else hi = mid; }
	return lo;
}

__global__ void __launch_bounds__(CL_THREADS) clusters_tables_kernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ values, const DevResult* __restrict__ res,
	uint32_t n_clusters, lb200_cluster* __restrict__ clusters, int32_t* __restrict__ map)
{
	const uint32_t n = res->n_sort;
	const uint32_t total = max(n, n_clusters);
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < total; i += gridDim.x * blockDim.x) {
		if (i < n) map[i] = (int32_t)(uint32_t)__ldg(values + i);
		if (i < n_clusters) {
			const uint32_t lo = lower_key(keys, 0, n, i), hi = lower_key(keys, lo, n, (uint64_t)i + 1);
			const uint32_t m1 = lower_kind(values, lo, hi, 1), m2 = lower_kind(values, m1, hi, 2);
			lb200_cluster c;
			c.offset = lo; c.lights_count = m1 - lo; c.env_probes_count = m2 - m1; c.refl_probes_count = hi - m2;
			clusters[i] = c;
		}
	}
}

__global__ void __launch_bounds__(256) clusters_set_lights_kernel(lb200_point_light* pl, const int32_t* __restrict__ entities, const lb200_point_light* __restrict__ rec, uint32_t n) {
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) pl[entities[i]] = rec[i];
}
__global__ void __launch_bounds__(256) clusters_set_atlas_kernel(int32_t* atlas, const int32_t* __restrict__ entities, const int32_t* __restrict__ idx, uint32_t n) {
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) atlas[entities[i]] = idx[i];
}
constexpr uint32_t CL_PATCH = 64;
struct PatchParams { uint32_t light[CL_PATCH]; int32_t atlas[CL_PATCH]; uint32_t n; };
__global__ void clusters_patch_kernel(lb200_cluster_light* lights, const __grid_constant__ PatchParams P) {
	if (threadIdx.x == 0) for (uint32_t i = 0; i < P.n; ++i) lights[P.light[i]].atlas_idx = (uint32_t)P.atlas[i];
}
__global__ void __launch_bounds__(256) clusters_init_kernel(lb200_point_light* pl, int32_t* atlas, uint32_t n) {
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) { pl[i] = lb200_point_light{}; atlas[i] = -1; }
}

// ---- host: the planes of :3468-3495 in fp32, the operations in the reference's order (math.cpp lerp / cross / normalize / dot,
// geometry.cpp makePlane); compiled without FMA contraction (Makefile) like the reference ----
struct V3 { float x, y, z; };
V3 sub(V3 a, V3 b) { return {a.x - b.x, a.y - b.y, a.z - b.z}; }
V3 mul(V3 a, float s) { return {a.x * s, a.y * s, a.z * s}; }
V3 cross(V3 a, V3 b) { return {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; }
float dot(V3 a, V3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
V3 normalize(V3 v) {
	const float inv_len = 1 / sqrtf(v.x * v.x + v.y * v.y + v.z * v.z);
	return {v.x * inv_len, v.y * inv_len, v.z * inv_len};
}
V3 lerp(V3 a, V3 b, float t) {
	const float invt = 1.0f - t;
	return {a.x * invt + b.x * t, a.y * invt + b.y * t, a.z * invt + b.z * t};
}
float4 make_plane(V3 n, V3 p) { return make_float4(n.x, n.y, n.z, -dot(n, p)); }

void build_planes(const lb200_shifted_frustum& f, int sx, int sy, Planes& out) {
	V3 pt[8];
	for (int i = 0; i < 8; ++i) pt[i] = {f.points[i][0], f.points[i][1], f.points[i][2]};
	memset(&out, 0, sizeof(out));
	const V3 cam_dir = normalize(cross(sub(pt[2], pt[0]), sub(pt[1], pt[0])));
	for (int i = 0; i < CL_ZS + 1; ++i) {
		const float znear = 0.1f, zfar = 10000.0f;
		const float z = znear * powf(zfar / znear, i / (float)CL_ZS);
		out.p[130 + i] = make_plane(cam_dir, mul(cam_dir, z));
	}
	for (int i = 0; i < sy + 1; ++i) {
		const float t = i / (float)sy;
		const V3 a = lerp(pt[0], pt[3], t), b = lerp(pt[1], pt[2], t), c = lerp(pt[4], pt[7], t);
		out.p[65 + i] = make_plane(normalize(cross(sub(b, a), sub(c, a))), a);
	}
	for (int i = 0; i < sx + 1; ++i) {
		const float t = i / (float)sx;
		const V3 a = lerp(pt[1], pt[0], t), b = lerp(pt[2], pt[3], t), c = lerp(pt[5], pt[4], t);
		out.p[i] = make_plane(normalize(cross(sub(b, a), sub(c, a))), a);
	}
}

} // namespace

struct lb200_clusters {
	lb200_ctx* ctx = nullptr;
	uint32_t max_entities = 0;
	DeviceArray<lb200_point_light> d_pl;   // per entity
	DeviceArray<int32_t> d_atlas;          // per entity, -1 = no entry
	std::unordered_map<int32_t, int32_t> atlas; // the same entries on the host (the limit of LB200_CLUSTERS_MAX_ATLAS)
	// outputs, per light / cluster / pair
	DeviceArray<lb200_cluster_light> d_lights; DeviceArray<int32_t> d_light_entities;
	DeviceArray<lb200_cluster> d_clusters; DeviceArray<int32_t> d_map;
	// scratch: per light, per item, per block, per pair
	DeviceArray<float> d_prio; DeviceArray<uint8_t> d_lflags;
	DeviceArray<unsigned long long> d_item_range, d_block_total;
	DeviceArray<uint64_t> d_keys, d_values, d_keys_alt, d_values_alt;
	DeviceArray<float4> d_probes;
	DeviceArray<DevResult> d_res; PinnedArray<DevResult> h_res;
	DeviceArray<GridBar> d_bar;
	RadixSortScratch sort;
	uint32_t items_limit = 0; // co-resident blocks of clusters_items_kernel
	// lb200_clusters_set_launch (0 = the default rule, -1 = every co-resident block, n > 0 = min(n, co-resident)) and what the last fill
	// launched (lb200_clusters_get_launch)
	int launch_blocks = 0;
	uint32_t last_grid = 0, last_tiles = 0;
	bool filled = false;
	uint32_t n_lights = 0;    // of the last fill
};

namespace {

// the per-light and per-item scratch for `lights` lights and `items` items, grown (by doubling) when short; contents are not kept
int ensure_items(lb200_clusters* cl, size_t lights, size_t items) {
	lb200_ctx* ctx = cl->ctx;
	if (lights > cl->d_lights.size() || !cl->d_lights) {
		const size_t cap = grownCapacity(cl->d_lights.size(), 1024, lights);
		LB200_CUDA(ctx, cl->d_lights.alloc(cap)); LB200_CUDA(ctx, cl->d_light_entities.alloc(cap));
		LB200_CUDA(ctx, cl->d_prio.alloc(cap)); LB200_CUDA(ctx, cl->d_lflags.alloc(cap));
	}
	if (items > cl->d_item_range.size() || !cl->d_item_range) LB200_CUDA(ctx, cl->d_item_range.alloc(grownCapacity(cl->d_item_range.size(), 1024, items)));
	return LB200_OK;
}
int ensure_pairs(lb200_clusters* cl, size_t pairs) {
	lb200_ctx* ctx = cl->ctx;
	if (pairs <= cl->d_keys.size() && cl->d_keys) return LB200_OK;
	const size_t cap = grownCapacity(cl->d_keys.size(), 1 << 16, pairs);
	if (cap > 0x7fffffffu) { lb200_set_error(ctx, "clusters_fill: a map of %zu entries does not fit", pairs); return LB200_ERR_CUDA; }
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // the earlier map may still be read
	cl->d_keys.reset(); cl->d_values.reset(); cl->d_keys_alt.reset(); cl->d_values_alt.reset(); cl->d_map.reset();
	LB200_CUDA(ctx, cl->d_keys.alloc(cap)); LB200_CUDA(ctx, cl->d_values.alloc(cap));
	LB200_CUDA(ctx, cl->d_keys_alt.alloc(cap)); LB200_CUDA(ctx, cl->d_values_alt.alloc(cap));
	LB200_CUDA(ctx, cl->d_map.alloc(cap));
	return LB200_OK;
}

// the four launches of one fill, on the context stream; *items_grid = the items kernel's grid
int launch_fill(lb200_clusters* cl, ItemsParams& P, uint32_t n_items_bound, uint32_t n_clusters, uint32_t* items_grid) {
	lb200_ctx* ctx = cl->ctx;
	cudaStream_t s = ctx->stream;
	P.keys = cl->d_keys; P.values = cl->d_values; P.pair_cap = (uint32_t)cl->d_keys.size();
	P.item_range = cl->d_item_range; P.block_total = cl->d_block_total;
	P.lights = cl->d_lights; P.light_entities = cl->d_light_entities; P.prio = cl->d_prio; P.lflags = cl->d_lflags;
	P.res = cl->d_res; P.bar = cl->d_bar;
	LB200_CUDA(ctx, cudaMemsetAsync(cl->d_res, 0, sizeof(DevResult), s));
	LB200_CUDA(ctx, cudaMemsetAsync(cl->d_bar, 0, sizeof(GridBar), s));
	uint32_t grid = std::max(1u, std::min(cl->items_limit, (n_items_bound + CL_THREADS - 1) / CL_THREADS));
	if (cl->launch_blocks < 0) grid = cl->items_limit; // not capped by the work: blocks without items still take part
	else if (cl->launch_blocks > 0) grid = std::min((uint32_t)cl->launch_blocks, cl->items_limit);
	*items_grid = grid;
	void* args[] = {&P};
	LB200_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)clusters_items_kernel, dim3(grid), dim3(CL_THREADS), args, 0, s));
	LB200_CHECK_LAUNCH(ctx);
	clusters_atlas_kernel<<<1, CL_ATLAS_THREADS, 0, s>>>(cl->d_prio, cl->d_lflags, cl->d_light_entities, cl->d_res);
	LB200_CHECK_LAUNCH(ctx);
	{
		lb200_range r("fill clusters: sort");
		const int rc = lb200_radix_sort_pairs(ctx, s, cl->d_keys, cl->d_keys_alt, cl->d_values, cl->d_values_alt, &cl->d_res.get()->n_sort,
			(uint32_t)cl->d_keys.size(), cl->sort, 0, false, nullptr);
		if (rc) return rc;
	}
	const uint32_t tgrid = std::max(1u, std::min((uint32_t)ctx->sm_count * 8, (uint32_t)((std::max<size_t>(cl->d_keys.size(), n_clusters) + CL_THREADS - 1) / CL_THREADS)));
	clusters_tables_kernel<<<tgrid, CL_THREADS, 0, s>>>(cl->d_keys, cl->d_values, cl->d_res, n_clusters, cl->d_clusters, cl->d_map);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaMemcpyAsync(cl->h_res, cl->d_res, sizeof(DevResult), cudaMemcpyDeviceToHost, s));
	LB200_CUDA(ctx, cudaStreamSynchronize(s));
	return LB200_OK;
}

// host array -> temporary device buffer on the context stream (setters are not on the per-frame path)
template <typename T> int upload_temp(lb200_ctx* ctx, const T* host, size_t n, DeviceArray<T>& dev) {
	LB200_CUDA(ctx, dev.alloc(n));
	LB200_CUDA(ctx, cudaMemcpyAsync(dev, host, sizeof(T) * n, cudaMemcpyHostToDevice, ctx->stream));
	return LB200_OK;
}

} // namespace

extern "C" {

int lb200_clusters_create(lb200_ctx* ctx, uint32_t max_entities, lb200_clusters** out) {
	if (!ctx || !out || !max_entities) return LB200_ERR_INVALID;
	*out = nullptr;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	std::unique_ptr<lb200_clusters, decltype(&lb200_clusters_destroy)> cl(new (std::nothrow) lb200_clusters, lb200_clusters_destroy);
	if (!cl) return LB200_ERR_CUDA;
	cl->ctx = ctx;
	cl->max_entities = max_entities;
	LB200_CUDA(ctx, cl->d_pl.alloc(max_entities));
	LB200_CUDA(ctx, cl->d_atlas.alloc(max_entities));
	clusters_init_kernel<<<std::min((max_entities + 255) / 256, 4096u), 256, 0, ctx->stream>>>(cl->d_pl, cl->d_atlas, max_entities);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cl->d_clusters.alloc(64 * 64 * CL_ZS));
	LB200_CUDA(ctx, cl->d_res.alloc(1));
	LB200_CUDA(ctx, cl->h_res.alloc(1));
	LB200_CUDA(ctx, cl->d_bar.alloc(1));
	LB200_CUDA(ctx, cl->d_probes.alloc(0, sizeof(float4)));
	int rc = lb200_coop_grid_limit(ctx, (const void*)clusters_items_kernel, CL_THREADS, 0, &cl->items_limit);
	if (rc) return rc;
	LB200_CUDA(ctx, cl->d_block_total.alloc(cl->items_limit));
	rc = lb200_radix_sort_alloc_scratch(ctx, (uint32_t)ctx->sm_count * 2, cl->sort);
	if (rc) return rc;
	rc = ensure_items(cl.get(), 1024, 1024);
	if (rc) return rc;
	rc = ensure_pairs(cl.get(), 1 << 16);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	*out = cl.release();
	return LB200_OK;
}

void lb200_clusters_destroy(lb200_clusters* cl) {
	if (!cl) return;
	if (cl->ctx) {
		cudaSetDevice(cl->ctx->device);
		cudaStreamSynchronize(cl->ctx->stream);
	}
	delete cl;
}

int lb200_clusters_set_point_lights(lb200_clusters* cl, const int32_t* entities, const lb200_point_light* records, uint32_t n) {
	if (!cl) return LB200_ERR_INVALID;
	lb200_ctx* ctx = cl->ctx;
	if (!n) return LB200_OK;
	if (!entities || !records) { lb200_set_error(ctx, "clusters_set_point_lights: NULL arrays for %u lights", n); return LB200_ERR_INVALID; }
	std::vector<uint8_t> seen(cl->max_entities, 0);
	for (uint32_t i = 0; i < n; ++i) {
		const int32_t e = entities[i];
		if (e < 0 || (uint32_t)e >= cl->max_entities) { lb200_set_error(ctx, "clusters_set_point_lights: entity %d is outside [0, %u)", e, cl->max_entities); return LB200_ERR_INVALID; }
		if (seen[e]++) { lb200_set_error(ctx, "clusters_set_point_lights: entity %d is listed twice", e); return LB200_ERR_INVALID; }
	}
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	DeviceArray<int32_t> e; DeviceArray<lb200_point_light> r;
	int rc = upload_temp(ctx, entities, n, e);
	if (!rc) rc = upload_temp(ctx, records, n, r);
	if (rc) return rc;
	clusters_set_lights_kernel<<<std::min((n + 255) / 256, 4096u), 256, 0, ctx->stream>>>(cl->d_pl, e, r, n);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // before the temporaries are freed
	return LB200_OK;
}

int lb200_clusters_set_atlas(lb200_clusters* cl, const int32_t* entities, const int32_t* atlas_idx, uint32_t n) {
	if (!cl) return LB200_ERR_INVALID;
	lb200_ctx* ctx = cl->ctx;
	if (!n) return LB200_OK;
	if (!entities || !atlas_idx) { lb200_set_error(ctx, "clusters_set_atlas: NULL arrays for %u entries", n); return LB200_ERR_INVALID; }
	std::unordered_map<int32_t, int32_t> next = cl->atlas;
	std::unordered_map<int32_t, int32_t> last; // per entity its final value: one device write each, so that list order holds
	for (uint32_t i = 0; i < n; ++i) {
		const int32_t e = entities[i], a = atlas_idx[i];
		if (e < 0 || (uint32_t)e >= cl->max_entities) { lb200_set_error(ctx, "clusters_set_atlas: entity %d is outside [0, %u)", e, cl->max_entities); return LB200_ERR_INVALID; }
		if (a < -1 || a >= LB200_CLUSTERS_MAX_ATLAS) { lb200_set_error(ctx, "clusters_set_atlas: atlas index %d is outside -1 .. %d", a, LB200_CLUSTERS_MAX_ATLAS - 1); return LB200_ERR_INVALID; }
		if (a < 0) next.erase(e); else next[e] = a;
		last[e] = a;
	}
	if (next.size() > LB200_CLUSTERS_MAX_ATLAS) { lb200_set_error(ctx, "clusters_set_atlas: %zu entities would have an atlas entry, the atlas holds %d", next.size(), LB200_CLUSTERS_MAX_ATLAS); return LB200_ERR_INVALID; }
	std::vector<int32_t> ue, ua;
	for (const auto& kv : last) { ue.push_back(kv.first); ua.push_back(kv.second); }
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	DeviceArray<int32_t> de, da;
	int rc = upload_temp(ctx, ue.data(), ue.size(), de);
	if (!rc) rc = upload_temp(ctx, ua.data(), ua.size(), da);
	if (rc) return rc;
	const uint32_t m = (uint32_t)ue.size();
	clusters_set_atlas_kernel<<<(m + 255) / 256, 256, 0, ctx->stream>>>(cl->d_atlas, de, da, m);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	cl->atlas = std::move(next);
	return LB200_OK;
}

int lb200_clusters_fill(lb200_clusters* cl, lb200_sortkeys* sk, lb200_culling* cs, const lb200_cluster_view* view,
                        const lb200_cluster_env_probe* env_probes, uint32_t n_env, const lb200_cluster_refl_probe* refl_probes,
                        uint32_t n_refl, lb200_cluster_result* result)
{
	if (!cl || !sk || !cs || !view || !result) return LB200_ERR_INVALID;
	lb200_ctx* ctx = cl->ctx;
	lb200_range range("fill clusters"); // pipeline.cpp:3328 PROFILE_FUNCTION
	if ((n_env && !env_probes) || (n_refl && !refl_probes)) { lb200_set_error(ctx, "clusters_fill: NULL probes with a count"); return LB200_ERR_INVALID; }
	if (view->w == 0 || view->h == 0 || view->w > CL_MAX_DIM || view->h > CL_MAX_DIM) {
		lb200_set_error(ctx, "clusters_fill: viewport %u x %u is not 1 .. %u each", view->w, view->h, CL_MAX_DIM);
		return LB200_ERR_INVALID;
	}
	SortKeysRecords recs;
	lb200_sortkeys_internal_records(sk, &recs);
	if (recs.ctx != ctx) { lb200_set_error(ctx, "clusters_fill: sort keys of another context"); return LB200_ERR_INVALID; }
	if (lb200_culling_internal_ctx(cs) != ctx) { lb200_set_error(ctx, "clusters_fill: a culling system of another context"); return LB200_ERR_INVALID; }
	if (!recs.have_transforms) { lb200_set_error(ctx, "clusters_fill: the sort keys hold no transforms yet"); return LB200_ERR_INVALID; }
	const uint32_t entity_range = lb200_culling_internal_entity_range(cs);
	if (entity_range > recs.max_entities || entity_range > cl->max_entities) {
		lb200_set_error(ctx, "clusters_fill: the culling system holds entity ids up to %u, the sort keys %u and the clusters %u", entity_range - 1, recs.max_entities, cl->max_entities);
		return LB200_ERR_INVALID;
	}
	const uint32_t* ids = nullptr;
	const uint32_t* counters = nullptr;
	const uint32_t* type_base = nullptr;
	int rc;
	if (view->view == LB200_CLUSTERS_LAST_CULL) {
		const uint32_t* type_counts = nullptr;
		rc = lb200_culling_internal_last(cs, &ids, &counters, &type_base, &type_counts);
		if (rc) return rc;
	} else {
		CullViewsResult cv;
		rc = lb200_culling_internal_views(cs, &cv);
		if (rc) return rc;
		if (view->view >= cv.n_views) { lb200_set_error(ctx, "clusters_fill: view %u of a cull_views call of %u views", view->view, cv.n_views); return LB200_ERR_INVALID; }
		ids = cv.ids + (size_t)view->view * cv.id_stride;
		counters = cv.counters + (size_t)view->view * cv.counter_stride;
		type_base = cv.type_base;
	}
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const uint32_t light_cap = type_base[RT_LOCAL_LIGHT + 1] - type_base[RT_LOCAL_LIGHT];
	const int sx = (int)((view->w + 63) / 64), sy = (int)((view->h + 63) / 64);
	const uint32_t n_clusters = (uint32_t)(sx * sy * CL_ZS);
	const size_t n_items = (size_t)light_cap + n_env + n_refl;
	rc = ensure_items(cl, light_cap, n_items);
	if (rc) return rc;
	// the probes' positions and radii (length(outer_range), length(half_extents)), in fp32 as :3583, :3606
	std::vector<float4> probes((size_t)n_env + n_refl);
	for (uint32_t i = 0; i < n_env; ++i) {
		const float* r = env_probes[i].outer_range;
		probes[i] = make_float4(env_probes[i].pos[0], env_probes[i].pos[1], env_probes[i].pos[2], sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]));
	}
	for (uint32_t i = 0; i < n_refl; ++i) {
		const float* r = refl_probes[i].half_extents;
		probes[n_env + i] = make_float4(refl_probes[i].pos[0], refl_probes[i].pos[1], refl_probes[i].pos[2], sqrtf(r[0] * r[0] + r[1] * r[1] + r[2] * r[2]));
	}
	if (probes.size() > cl->d_probes.size()) LB200_CUDA(ctx, cl->d_probes.alloc(grownCapacity(cl->d_probes.size(), 64, probes.size())));
	if (!probes.empty()) LB200_CUDA(ctx, cudaMemcpyAsync(cl->d_probes, probes.data(), sizeof(float4) * probes.size(), cudaMemcpyHostToDevice, ctx->stream));

	ItemsParams P;
	memset(&P, 0, sizeof(P));
	build_planes(view->frustum, sx, sy, P.planes);
	for (int c = 0; c < 3; ++c) P.cam[c] = view->cam_pos[c];
	P.sx = sx; P.sy = sy;
	P.ids = ids + type_base[RT_LOCAL_LIGHT];
	P.n_lights_dev = counters + RT_LOCAL_LIGHT;
	P.light_cap = light_cap;
	P.n_env = n_env; P.n_refl = n_refl;
	P.probes = cl->d_probes;
	P.ent = recs.records; P.pl = cl->d_pl; P.atlas = cl->d_atlas;
	uint32_t grid = 0;
	rc = launch_fill(cl, P, (uint32_t)n_items, n_clusters, &grid);
	if (rc) return rc;
	if (cl->h_res.get()->n_pairs > cl->d_keys.size()) { // the map grows: the same work again into room for all of it
		rc = ensure_pairs(cl, (size_t)cl->h_res.get()->n_pairs);
		if (!rc) rc = launch_fill(cl, P, (uint32_t)n_items, n_clusters, &grid);
		if (rc) { cl->filled = false; return rc; }
	}
	const DevResult& d = *cl->h_res.get();
	const uint32_t items = d.n_lights + n_env + n_refl, chunk = (items + grid - 1) / grid; // as the items kernel splits them
	cl->last_grid = grid;
	cl->last_tiles = (chunk + CL_THREADS - 1) / CL_THREADS;
	memset(result, 0, sizeof(*result));
	result->n_lights = d.n_lights;
	result->n_clusters = n_clusters;
	result->n_map = (uint32_t)d.n_pairs;
	result->size[0] = (uint32_t)sx; result->size[1] = (uint32_t)sy; result->size[2] = CL_ZS;
	result->n_shadow = d.n_shadow;
	memcpy(result->shadow, d.shadow, sizeof(d.shadow[0]) * std::min<uint32_t>(d.n_shadow, LB200_CLUSTERS_MAX_ATLAS));
	result->n_uncast = std::min<uint32_t>(d.n_uncast, LB200_CLUSTERS_MAX_ATLAS);
	memcpy(result->uncast, d.uncast, sizeof(d.uncast[0]) * result->n_uncast);
	cl->filled = true;
	cl->n_lights = d.n_lights;
	return LB200_OK;
}

int lb200_clusters_patch_atlas(lb200_clusters* cl, const uint32_t* light_idx, const int32_t* atlas_idx, uint32_t n) {
	if (!cl) return LB200_ERR_INVALID;
	lb200_ctx* ctx = cl->ctx;
	if (!cl->filled) { lb200_set_error(ctx, "clusters_patch_atlas: no fill yet"); return LB200_ERR_STATE; }
	if (!n) return LB200_OK;
	if (!light_idx || !atlas_idx) { lb200_set_error(ctx, "clusters_patch_atlas: NULL arrays for %u entries", n); return LB200_ERR_INVALID; }
	for (uint32_t i = 0; i < n; ++i) {
		if (light_idx[i] >= cl->n_lights) { lb200_set_error(ctx, "clusters_patch_atlas: light %u of %u", light_idx[i], cl->n_lights); return LB200_ERR_INVALID; }
		if (atlas_idx[i] < -1 || atlas_idx[i] >= LB200_CLUSTERS_MAX_ATLAS) {
			lb200_set_error(ctx, "clusters_patch_atlas: atlas index %d is outside -1 .. %d", atlas_idx[i], LB200_CLUSTERS_MAX_ATLAS - 1);
			return LB200_ERR_INVALID;
		}
	}
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	for (uint32_t b = 0; b < n; b += CL_PATCH) {
		PatchParams P;
		P.n = std::min(CL_PATCH, n - b);
		for (uint32_t i = 0; i < P.n; ++i) { P.light[i] = light_idx[b + i]; P.atlas[i] = atlas_idx[b + i]; }
		clusters_patch_kernel<<<1, 32, 0, ctx->stream>>>(cl->d_lights, P);
		LB200_CHECK_LAUNCH(ctx);
	}
	return LB200_OK;
}

int lb200_clusters_set_launch(lb200_clusters* cl, int blocks) {
	if (!cl) return LB200_ERR_INVALID;
	if (blocks < -1) { lb200_set_error(cl->ctx, "clusters_set_launch: blocks %d is not -1, 0 or a block count", blocks); return LB200_ERR_INVALID; }
	cl->launch_blocks = blocks;
	return LB200_OK;
}

int lb200_clusters_get_launch(lb200_clusters* cl, uint32_t* grid, uint32_t* tiles_per_block) {
	if (!cl) return LB200_ERR_INVALID;
	if (grid) *grid = cl->last_grid;
	if (tiles_per_block) *tiles_per_block = cl->last_tiles;
	return LB200_OK;
}

int lb200_clusters_outputs(lb200_clusters* cl, lb200_cluster_outputs* out) {
	if (!cl || !out) return LB200_ERR_INVALID;
	if (!cl->filled) { lb200_set_error(cl->ctx, "clusters_outputs: no fill yet"); return LB200_ERR_STATE; }
	out->lights = cl->d_lights; out->clusters = cl->d_clusters; out->map = cl->d_map; out->light_entities = cl->d_light_entities;
	return LB200_OK;
}

} // extern "C"
