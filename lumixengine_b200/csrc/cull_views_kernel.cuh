// cull_views_kernel — several views of one scene (a frame's main camera and shadow cascades) culled in ONE pass over the pages.
//
// The phases are cull_pages_kernel's (cull_kernel.cuh), with each page's work split into (page, view) items:
//   A1  one THREAD per page: the 32-byte descriptor is read once; the type filter and the "definitely outside" test run per view with
//       the single cull's margin expression.  A page is a candidate if any view keeps it; per-view pages_filtered / pages_outside count
//       as a lone cull of that view counts them.
//   A2  one THREAD per candidate page: the exact classification (contains, intersects, is_big, getRelative offsets, plane mask) per view
//       that kept the page, with the single cull's expressions.  Every view that works the page gets an item; the TEST items of one page
//       take consecutive slots, so that phase B finds them together.
//   B   one WARP per page that some view must TEST: the <= 200 spheres are loaded once, as the single cull's 7 x 128-bit streaming loads,
//       then each TEST view's needed planes are walked over the rows held in registers; ballots go to shared memory per item.
//   C   claim: one global atomic per (warp, view, renderable type) reserves the output range in that view's id buffer.
//   D   write: per item, the visible ids gathered into that view's buffer and the page's 32-byte row written into that view's mask.  Pages
//       that end without work for a view get a zero row in that view's mask.
// Shared memory per (page, view) item bounds a round: chunk <= MAX_ITEMS / n_views pages (viewsChunkBound).  B deals pages to the warps
// and C / D deal items, so a block barrier separates B from C (the single cull's warps run B, C and D without one).
// Like the single cull, everything before cudaGridDependencySynchronize() only READS scene data, so the kernel may be launched with
// programmatic stream serialization behind another cull.
// Bytes: 32 B descriptor per page + 16 B per sphere of a page some view tests (each page's rows once) + per view 4 B read + 4 B write per
// visible id and a 32 B mask row per page.
#pragma once

#include "culling_internal.h" // counter layout, statistics
#include "lb200_internal.h"
#include "lb200_math.cuh"

namespace lbviews {

using namespace lb;
using lbcull::COUNTER_WORDS;
using lbcull::N_STATS;

constexpr int ROWS = 7;            // ceil(200 / 32)
constexpr int VIEW_THREADS = 256;  // 4 blocks/SM at 64 registers
constexpr int VIEW_WARPS = VIEW_THREADS / 32;
constexpr int MAX_VIEWS = LB200_CULL_MAX_VIEWS;
constexpr int MAX_CHUNK = VIEW_THREADS; // one A1 thread per page
constexpr int MAX_ITEMS = 512;          // (page, view) items of one block and round
static_assert(MAX_VIEWS <= 8, "a view index takes 3 bits of an item, a view set 8 bits");
// Counters of one call: [view][COUNTER_WORDS] (cull_kernel.cuh's layout per view), then CALL_WORDS words for the call itself
constexpr int CALL_WORDS = 8;
enum { CALL_STREAMED = 0 }; // spheres read: each page that some view tests counted once (the union over the views)
constexpr int CALL_COUNTER_WORDS = MAX_VIEWS * COUNTER_WORDS + CALL_WORDS;

inline uint32_t viewsChunkBound(uint32_t n_views) { return (uint32_t)(MAX_ITEMS / n_views < MAX_CHUNK ? MAX_ITEMS / n_views : MAX_CHUNK); }

struct ViewsParams {
	// per view: planes NEAR, FAR, LEFT, RIGHT, TOP, BOTTOM relative to its origin, and the points getRelative re-anchors them on
	float nx[MAX_VIEWS][6], ny[MAX_VIEWS][6], nz[MAX_VIEWS][6], d[MAX_VIEWS][6];
	float px[MAX_VIEWS][6], py[MAX_VIEWS][6], pz[MAX_VIEWS][6];
	double ox[MAX_VIEWS], oy[MAX_VIEWS], oz[MAX_VIEWS];
	uint32_t type_filter[MAX_VIEWS]; // 0xff = all
	uint32_t n_views;
	uint32_t n_pages;
	uint32_t chunk;         // pages per block per round, <= viewsChunkBound(n_views)
	uint32_t plane_masking; // 1 unless some sphere has a negative / NaN radius
	uint32_t id_stride;     // words between two views' id buffers
	uint32_t mask_stride;   // words between two views' masks
	uint32_t type_base[256];
};

enum { CLS_SKIP = 0, CLS_COPY = 1, CLS_TEST = 2 };

struct ViewItem { // 32 B
	uint32_t page;
	uint32_t meta; // count | type << 8 | cls << 16 | view << 18 | planes needed << 24
	float rd[6];   // the view's plane offsets relative to the cell origin (TEST items)
};
static_assert(sizeof(ViewItem) == 32, "");

__device__ __forceinline__ float4 ldg_stream_v(const float4* p) {
	float4 r;
	asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
	return r;
}

__device__ __forceinline__ int ldg_stream_i32_v(const int* p) {
	int r;
	asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r) : "l"(p));
	return r;
}

__global__ void __launch_bounds__(VIEW_THREADS, 4) cull_views_kernel(const __grid_constant__ ViewsParams P,
	const lb200_page_desc* __restrict__ desc, const float4* __restrict__ spheres, const int* __restrict__ entities,
	uint32_t* __restrict__ out_ids, uint32_t* __restrict__ counters, uint32_t* __restrict__ next_counters, uint32_t* __restrict__ mask_out)
{
	__shared__ ViewItem s_item[MAX_ITEMS];
	__shared__ __align__(16) uint32_t s_bal[MAX_ITEMS][ROWS + 1]; // the 256-bit visibility row of a TEST item ([ROWS] = 0)
	__shared__ uint32_t s_off[MAX_ITEMS];  // visible ids of the item, then its offset inside its view's id buffer
	__shared__ uint32_t s_tpage[MAX_CHUNK]; // a page some view tests: its first TEST item | item count << 16
	__shared__ uint16_t s_cand[MAX_CHUNK];  // classify threads whose page some view kept in the cheap pass
	__shared__ uint8_t s_keep[MAX_CHUNK];   // views that kept the page in the cheap pass
	__shared__ uint8_t s_zero[MAX_CHUNK];   // views whose mask row of the page is zero (the page ends without work for them)
	__shared__ uint32_t s_stats[MAX_VIEWS][N_STATS];
	__shared__ uint32_t s_ntest, s_ncopy, s_ncand, s_ntpage, s_streamed;

	cudaTriggerProgrammaticLaunchCompletion();

	const int tid = threadIdx.x;
	const int lane = tid & 31;
	const int warp = tid >> 5;
	const uint32_t lt_mask = (1u << lane) - 1u;
	const uint32_t n_views = P.n_views;
	const uint32_t all_views = (1u << n_views) - 1u;

	if (tid < MAX_VIEWS * N_STATS) (&s_stats[0][0])[tid] = 0;
	if (tid == 0) { s_ntest = 0; s_ncopy = 0; s_ncand = 0; s_ntpage = 0; s_streamed = 0; }
	__syncthreads();

	for (uint32_t round = 0; round * P.chunk * gridDim.x < P.n_pages; ++round) {
		// ---------------- A1. cheap pass: one thread per page, one descriptor read, "definitely outside" per view ----------------
		{
			uint32_t keep = 0, zero = 0;
			if ((uint32_t)tid < P.chunk) {
				const uint32_t page = (round * P.chunk + tid) * gridDim.x + blockIdx.x;
				if (page < P.n_pages) {
					zero = all_views;
					const int4* dp = reinterpret_cast<const int4*>(desc + page);
					const int4 a = __ldg(dp);
					const int4 b = __ldg(dp + 1);
					const uint32_t count = (uint32_t)b.z;
					const uint32_t type = (uint32_t)b.w & 0xffu;
					const bool is_big = (((uint32_t)b.w >> 8) & 0xffu) != 0;
					if (count != 0) {
						const double org_x = __hiloint2double(a.y, a.x);
						const double org_y = __hiloint2double(a.w, a.z);
						const double org_z = __hiloint2double(b.y, b.x);
						const float cs = LB200_CELL_SIZE;
						const float cs2 = 2 * LB200_CELL_SIZE;
						const D3 lo = d3(LB_DSUB(org_x, (double)cs), LB_DSUB(org_y, (double)cs), LB_DSUB(org_z, (double)cs));
						#pragma unroll 1
						for (uint32_t v = 0; v < n_views; ++v) {
							if (P.type_filter[v] != 0xffu && type != P.type_filter[v]) { atomicAdd(&s_stats[v][lbcull::ST_PAGES_FILTERED], 1u); continue; }
							bool outside = false;
							if (!is_big) {
								const V3 rel_i = tofloat(sub(lo, d3(P.ox[v], P.oy[v], P.oz[v])));
								const V3 max_i = add(rel_i, v3(cs2, cs2, cs2));
#pragma unroll
								for (int p = 0; p < 6; ++p) {
									const float nx = P.nx[v][p], ny = P.ny[v][p], nz = P.nz[v][p], nd = -P.d[v][p];
									const float tx = LB_FMUL(nx, nx > 0.0f ? max_i.x : rel_i.x);
									const float ty = LB_FMUL(ny, ny > 0.0f ? max_i.y : rel_i.y);
									const float tz = LB_FMUL(nz, nz > 0.0f ? max_i.z : rel_i.z);
									const float dp_i = LB_FADD(LB_FADD(tx, ty), tz);
									const float margin = 1e-4f * (fabsf(nd) + fabsf(tx) + fabsf(ty) + fabsf(tz)) + 0.05f;
									if (dp_i + margin < nd) outside = true; // NaN anywhere: false, the page stays a candidate
								}
							}
							if (outside) atomicAdd(&s_stats[v][lbcull::ST_PAGES_OUTSIDE], 1u);
							else keep |= 1u << v;
						}
					}
					zero &= ~keep;
				}
			}
			const bool cand = keep != 0;
			const uint32_t bal = __ballot_sync(0xffffffffu, cand);
			uint32_t base = 0;
			if (lane == 0 && bal) base = atomicAdd(&s_ncand, (uint32_t)__popc(bal));
			base = __shfl_sync(0xffffffffu, base, 0);
			if (cand) s_cand[base + __popc(bal & lt_mask)] = (uint16_t)tid;
			s_keep[tid] = (uint8_t)keep;
			s_zero[tid] = (uint8_t)zero;
		}
		__syncthreads();

		// ---------------- A2. exact classification of every (candidate page, view that kept it) ----------------
		if ((uint32_t)tid < s_ncand) {
			const uint32_t t0 = s_cand[tid];
			const uint32_t page = (round * P.chunk + t0) * gridDim.x + blockIdx.x;
			const int4* dp = reinterpret_cast<const int4*>(desc + page); // read by the cheap pass a moment ago: an L1 hit
			const int4 a = __ldg(dp);
			const int4 b = __ldg(dp + 1);
			const double org_x = __hiloint2double(a.y, a.x);
			const double org_y = __hiloint2double(a.w, a.z);
			const double org_z = __hiloint2double(b.y, b.x);
			const uint32_t count = (uint32_t)b.z;
			const uint32_t type = (uint32_t)b.w & 0xffu;
			const bool is_big = (((uint32_t)b.w >> 8) & 0xffu) != 0;
			const uint32_t keep = s_keep[t0];
			const float cs = LB200_CELL_SIZE;
			const float cs2 = 2 * LB200_CELL_SIZE;
			// pass 1: the class per view and the statistics
			uint32_t cls_of = 0;   // 2 bits per view
			uint64_t need_of = 0;  // 6 bits per view
			uint32_t n_t = 0, n_c = 0, zero = 0;
			#pragma unroll 1
			for (uint32_t v = 0; v < n_views; ++v) {
				if (!((keep >> v) & 1u)) continue;
				int cls = CLS_SKIP;
				{
					// containsAABB(cell.origin + Vec3(cs), Vec3(cs)) and intersectsAABB(cell.origin - Vec3(cs), Vec3(2cs)) of view v
					const V3 rel_c = tofloat(sub(d3(LB_DADD(org_x, (double)cs), LB_DADD(org_y, (double)cs), LB_DADD(org_z, (double)cs)), d3(P.ox[v], P.oy[v], P.oz[v])));
					const V3 max_c = add(rel_c, v3(cs, cs, cs));
					const V3 rel_i = tofloat(sub(d3(LB_DSUB(org_x, (double)cs), LB_DSUB(org_y, (double)cs), LB_DSUB(org_z, (double)cs)), d3(P.ox[v], P.oy[v], P.oz[v])));
					const V3 max_i = add(rel_i, v3(cs2, cs2, cs2));
					bool contains = true, intersects = true;
#pragma unroll
					for (int p = 0; p < 6; ++p) {
						const float nx = P.nx[v][p], ny = P.ny[v][p], nz = P.nz[v][p], nd = -P.d[v][p];
						const float cbx = nx < 0.0f ? max_c.x : rel_c.x;
						const float cby = ny < 0.0f ? max_c.y : rel_c.y;
						const float cbz = nz < 0.0f ? max_c.z : rel_c.z;
						const float dp_c = LB_FADD(LB_FADD(LB_FMUL(nx, cbx), LB_FMUL(ny, cby)), LB_FMUL(nz, cbz));
						if (dp_c < nd) contains = false;
						const float ibx = nx > 0.0f ? max_i.x : rel_i.x;
						const float iby = ny > 0.0f ? max_i.y : rel_i.y;
						const float ibz = nz > 0.0f ? max_i.z : rel_i.z;
						const float dp_i = LB_FADD(LB_FADD(LB_FMUL(nx, ibx), LB_FMUL(ny, iby)), LB_FMUL(nz, ibz));
						if (dp_i < nd) intersects = false;
					}
					if (is_big) cls = CLS_TEST;
					else if (contains) cls = CLS_COPY;
					else if (intersects) cls = CLS_TEST;
					else atomicAdd(&s_stats[v][lbcull::ST_PAGES_OUTSIDE], 1u);
				}
				if (cls == CLS_SKIP) { zero |= 1u << v; continue; }
				if (cls == CLS_TEST) { atomicAdd(&s_stats[v][lbcull::ST_PAGES_TESTED], 1u); atomicAdd(&s_stats[v][lbcull::ST_ENT_TESTED], count); }
				else { atomicAdd(&s_stats[v][lbcull::ST_PAGES_INSIDE], 1u); atomicAdd(&s_stats[v][lbcull::ST_ENT_INSIDE], count); }
				cls_of |= (uint32_t)cls << (2 * v);
			}
			// pass 2: the plane mask of every TEST view (a loop of its own: the planes of the classification are not kept live across it)
			#pragma unroll 1
			for (uint32_t v = 0; v < n_views; ++v) {
				uint32_t cls = (cls_of >> (2 * v)) & 3u;
				if (cls == CLS_SKIP) continue;
				uint32_t need = 0x3fu;
				if (cls == CLS_TEST && P.plane_masking) {
					// ShiftedFrustum::getRelative(cell.origin) and the plane mask, as cull_pages_kernel computes them
					const V3 offset = tofloat(sub(d3(P.ox[v], P.oy[v], P.oz[v]), d3(org_x, org_y, org_z)));
					const float e = 1.0f + 1e-6f * fmaxf(fmaxf(fabsf((float)org_x), fabsf((float)org_y)), fabsf((float)org_z));
					const float lox = (org_x > 0.0 ? 0.0f : -cs) - e, hix = (org_x < 0.0 ? 0.0f : cs) + e;
					const float loy = (org_y > 0.0 ? 0.0f : -cs) - e, hiy = (org_y < 0.0 ? 0.0f : cs) + e;
					const float loz = (org_z > 0.0 ? 0.0f : -cs) - e, hiz = (org_z < 0.0 ? 0.0f : cs) + e;
					need = 0;
#pragma unroll
					for (int p = 0; p < 6; ++p) {
						const float nx = P.nx[v][p], ny = P.ny[v][p], nz = P.nz[v][p];
						const float dp = -dot(add(v3(P.px[v][p], P.py[v][p], P.pz[v][p]), offset), v3(nx, ny, nz));
						const float low = dp + fminf(nx * lox, nx * hix) + fminf(ny * loy, ny * hiy) + fminf(nz * loz, nz * hiz);
						const float margin = 1e-5f * (fabsf(dp) + 1000.0f * (fabsf(nx) + fabsf(ny) + fabsf(nz))) + 1e-3f;
						if (!(low > margin)) need |= 1u << p; // NaN keeps the plane
					}
					if (need == 0) cls = CLS_COPY; // every sphere of the page is visible to this view: ids only
				}
				if (cls == CLS_TEST) { atomicAdd(&s_stats[v][lbcull::ST_ENT_STREAMED], count); ++n_t; }
				else ++n_c;
				cls_of = (cls_of & ~(3u << (2 * v))) | (cls << (2 * v));
				need_of |= (uint64_t)need << (6 * v);
			}
			uint32_t t_slot = 0, c_slot = 0;
			if (n_t) {
				t_slot = atomicAdd(&s_ntest, n_t);
				s_tpage[atomicAdd(&s_ntpage, 1u)] = t_slot | (n_t << 16);
				atomicAdd(&s_streamed, count); // the page's rows are read once, whichever views test them
			}
			if (n_c) c_slot = atomicAdd(&s_ncopy, n_c);
			// pass 3: the items; the TEST items of the page take consecutive slots from the front, COPY items slots from the back
			#pragma unroll 1
			for (uint32_t v = 0; v < n_views; ++v) {
				const uint32_t cls = (cls_of >> (2 * v)) & 3u;
				if (cls == CLS_SKIP) continue;
				const uint32_t need = (uint32_t)(need_of >> (6 * v)) & 0x3fu;
				float rd[6];
#pragma unroll
				for (int p = 0; p < 6; ++p) rd[p] = 0.0f;
				uint32_t slot;
				if (cls == CLS_TEST) {
					const V3 offset = tofloat(sub(d3(P.ox[v], P.oy[v], P.oz[v]), d3(org_x, org_y, org_z)));
#pragma unroll
					for (int p = 0; p < 6; ++p) rd[p] = -dot(add(v3(P.px[v][p], P.py[v][p], P.pz[v][p]), offset), v3(P.nx[v][p], P.ny[v][p], P.nz[v][p]));
					slot = t_slot++;
				}
				else {
					slot = (uint32_t)MAX_ITEMS - 1u - c_slot++;
					s_off[slot] = count; // every entity of the page is visible to this view
				}
				uint4* it = reinterpret_cast<uint4*>(&s_item[slot]);
				it[0] = make_uint4(page, count | (type << 8) | (cls << 16) | (v << 18) | (need << 24), __float_as_uint(rd[0]), __float_as_uint(rd[1]));
				it[1] = make_uint4(__float_as_uint(rd[2]), __float_as_uint(rd[3]), __float_as_uint(rd[4]), __float_as_uint(rd[5]));
			}
			s_zero[t0] |= (uint8_t)zero;
		}
		__syncthreads();
		const uint32_t n_test = s_ntest;
		const uint32_t n_work = n_test + s_ncopy;
#define LB_VITEM(w) ((w) < n_test ? (w) : (uint32_t)MAX_ITEMS - 1u - ((w) - n_test))

		// ---------------- B. sphere tests: one warp per page some view tests, rows loaded once for all of its TEST items ----------------
		for (uint32_t jt = warp; jt < s_ntpage; jt += VIEW_WARPS) {
			const uint32_t tp = s_tpage[jt];
			const uint32_t first = tp & 0xffffu, n_items = tp >> 16;
			const uint32_t page = s_item[first].page;
			const uint32_t count = s_item[first].meta & 0xffu;
			const bool upper = count > 128u;
			float4 s[ROWS];
			const float4* sp = spheres + (size_t)page * LB200_PAGE_SLOTS;
			const uint32_t last = count - 1u;
#pragma unroll
			for (int k = 0; k < 4; ++k) { const uint32_t slot = k * 32 + lane; s[k] = ldg_stream_v(sp + (slot < last ? slot : last)); }
			if (upper) {
#pragma unroll
				for (int k = 4; k < ROWS; ++k) { const uint32_t slot = k * 32 + lane; s[k] = ldg_stream_v(sp + (slot < last ? slot : last)); }
			}
			if (!upper) {
#pragma unroll
				for (int k = 4; k < ROWS; ++k) s[k] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
			}
			#pragma unroll 1
			for (uint32_t iw = first; iw < first + n_items; ++iw) {
				const uint4 ia = *reinterpret_cast<const uint4*>(&s_item[iw]);
				const uint4 ib = *(reinterpret_cast<const uint4*>(&s_item[iw]) + 1);
				const uint32_t need = ia.y >> 24;
				const uint32_t v = (ia.y >> 18) & 7u;
				uint32_t acc[ROWS];
#pragma unroll
				for (int k = 0; k < ROWS; ++k) acc[k] = 0;
				// doCulling, culling_system.cpp:260-308, with view v's planes: t = cx*px + cy*py + cz*pz + pd ; t = t - r ; sign bits
#define LB_VROWS(pd, k0, k1)                                                                                                     \
				_Pragma("unroll") for (int k = k0; k < k1; ++k) {                                                                \
					float t = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(s[k].x, nx), LB_FMUL(s[k].y, ny)), LB_FMUL(s[k].z, nz)), pd);      \
					t = LB_FSUB(t, -s[k].w);                                                                                     \
					acc[k] |= __float_as_uint(t);                                                                                \
				}
#define LB_VPLANE(p, pd)                                                                                                         \
				if (need & (1u << p)) {                                                                                          \
					const float nx = P.nx[v][p], ny = P.ny[v][p], nz = P.nz[v][p];                                                \
					LB_VROWS(pd, 0, 4)                                                                                           \
					if (upper) { LB_VROWS(pd, 4, ROWS) }                                                                         \
				}
				LB_VPLANE(0, __uint_as_float(ia.z))
				LB_VPLANE(1, __uint_as_float(ia.w))
				LB_VPLANE(2, __uint_as_float(ib.x))
				LB_VPLANE(3, __uint_as_float(ib.y))
				LB_VPLANE(4, __uint_as_float(ib.z))
				LB_VPLANE(5, __uint_as_float(ib.w))
#undef LB_VPLANE
#undef LB_VROWS
				// a NaN radius: the sign of the radius decides, as in cull_pages_kernel (only scenes with a negative / NaN radius get here)
				if (!P.plane_masking) {
#pragma unroll
					for (int k = 0; k < ROWS; ++k) {
						const uint32_t rbits = __float_as_uint(s[k].w);
						uint32_t flipped;
						asm volatile("not.b32 %0, %1;" : "=r"(flipped) : "r"(rbits));
						if ((rbits & 0x7fffffffu) > 0x7f800000u && need) acc[k] = flipped & 0x80000000u;
					}
				}
				uint32_t bal[ROWS];
				uint32_t page_visible = 0;
#pragma unroll
				for (int k = 0; k < 4; ++k) {
					const bool visible = (acc[k] >> 31) == 0 && (uint32_t)(k * 32 + lane) < count;
					bal[k] = __ballot_sync(0xffffffffu, visible);
					page_visible += __popc(bal[k]);
				}
#pragma unroll
				for (int k = 4; k < ROWS; ++k) bal[k] = 0;
				if (upper) {
#pragma unroll
					for (int k = 4; k < ROWS; ++k) {
						const bool visible = (acc[k] >> 31) == 0 && (uint32_t)(k * 32 + lane) < count;
						bal[k] = __ballot_sync(0xffffffffu, visible);
						page_visible += __popc(bal[k]);
					}
				}
				if (lane == 0) {
					*reinterpret_cast<uint4*>(&s_bal[iw][0]) = make_uint4(bal[0], bal[1], bal[2], bal[3]);
					*reinterpret_cast<uint4*>(&s_bal[iw][4]) = make_uint4(bal[4], bal[5], bal[6], 0u);
					s_off[iw] = page_visible;
				}
			}
		}
		// nothing above wrote global memory; everything below does and has to wait for the previous kernel of the stream
		if (round == 0) cudaGridDependencySynchronize();
		// rows of pages that ended without work, per view
		if ((uint32_t)tid < P.chunk && s_zero[tid]) {
			const uint32_t page = (round * P.chunk + tid) * gridDim.x + blockIdx.x;
			for (uint32_t z = s_zero[tid]; z; z &= z - 1u) {
				uint4* row = reinterpret_cast<uint4*>(mask_out + (size_t)(__ffs((int)z) - 1) * P.mask_stride + (size_t)page * 8);
				row[0] = make_uint4(0u, 0u, 0u, 0u);
				row[1] = make_uint4(0u, 0u, 0u, 0u);
			}
		}
		// ---------------- C. claim: one global atomic per (warp, view, type), 32 items of the warp at a time ----------------
		// phase B dealt pages to the warps, C and D deal items: every ballot and visible count has to be in place first
		__syncthreads();
		{
			const uint32_t n_mine = (n_work + VIEW_WARPS - 1 - warp) / VIEW_WARPS; // items of this warp (warp-uniform)
			#pragma unroll 1
			for (uint32_t b0 = 0; b0 < n_mine; b0 += 32) {
				const uint32_t n_batch = n_mine - b0 < 32u ? n_mine - b0 : 32u;
				const bool has = (uint32_t)lane < n_batch;
				const uint32_t iwi = has ? LB_VITEM(warp + (b0 + (uint32_t)lane) * VIEW_WARPS) : 0u;
				const uint32_t meta = has ? s_item[iwi].meta : 0u;
				const uint32_t my_key = has ? ((meta >> 8) & 0xffu) | (((meta >> 18) & 7u) << 8) : 0xffffu; // type | view << 8
				const uint32_t my_count = has ? s_off[iwi] : 0u;
				const uint32_t packed = (my_key << 16) | my_count; // count <= 200
				uint32_t prefix = 0, total = 0;
				for (uint32_t l = 0; l < n_batch; ++l) {
					const uint32_t o = __shfl_sync(0xffffffffu, packed, (int)l);
					if ((o >> 16) == my_key) { total += o & 0xffffu; if (l < (uint32_t)lane) prefix += o & 0xffffu; }
				}
				const unsigned grp = __match_any_sync(0xffffffffu, my_key);
				const int leader = __ffs((int)grp) - 1;
				uint32_t base = 0;
				if (has && lane == leader && total) base = atomicAdd(&counters[(my_key >> 8) * COUNTER_WORDS + (my_key & 0xffu)], total);
				base = __shfl_sync(0xffffffffu, base, leader);
				if (has) s_off[iwi] = P.type_base[my_key & 0xffu] + base + prefix; // where the item's ids go in its view's buffer
			}
		}
		__syncwarp();

		// ---------------- D. write: gather the visible ids of each item into its view's buffer, and its mask row ----------------
		for (uint32_t w = warp; w < n_work; w += VIEW_WARPS) {
			const uint32_t iw = LB_VITEM(w);
			const uint32_t page = s_item[iw].page;
			const uint32_t meta = s_item[iw].meta;
			const uint32_t count = meta & 0xffu;
			const uint32_t v = (meta >> 18) & 7u;
			uint32_t* dst = out_ids + (size_t)v * P.id_stride + s_off[iw];
			const int* ep = entities + (size_t)page * LB200_PAGE_SLOTS;
			uint32_t row_word;
			if (((meta >> 16) & 3u) == CLS_COPY) {
				const int* src = ep + lane;
				uint32_t* d = dst + lane;
				int id[ROWS] = {};
#pragma unroll
				for (int k = 0; k < ROWS; ++k) if ((uint32_t)(k * 32 + lane) < count) id[k] = ldg_stream_i32_v(src + k * 32);
#pragma unroll
				for (int k = 0; k < ROWS; ++k) if ((uint32_t)(k * 32 + lane) < count) d[k * 32] = (uint32_t)id[k];
				const int rem = (int)count - (lane & 7) * 32;
				row_word = rem >= 32 ? 0xffffffffu : (rem > 0 ? ((1u << rem) - 1u) : 0u);
			}
			else {
				uint32_t bal[ROWS];
#pragma unroll
				for (int k = 0; k < ROWS; ++k) bal[k] = s_bal[iw][k];
				int id[ROWS] = {};
#pragma unroll
				for (int k = 0; k < ROWS; ++k) if ((bal[k] >> lane) & 1u) id[k] = ldg_stream_i32_v(ep + k * 32 + lane);
				uint32_t prefix = 0;
#pragma unroll
				for (int k = 0; k < ROWS; ++k) {
					if ((bal[k] >> lane) & 1u) dst[prefix + __popc(bal[k] & lt_mask)] = (uint32_t)id[k];
					prefix += __popc(bal[k]);
				}
				row_word = s_bal[iw][lane & 7];
			}
			if (lane < 8) mask_out[(size_t)v * P.mask_stride + (size_t)page * 8 + lane] = row_word;
		}
#undef LB_VITEM
		__syncthreads(); // every warp is done with s_item / s_bal / s_tpage / s_zero
		if (tid == 0) { s_ntest = 0; s_ncopy = 0; s_ncand = 0; s_ntpage = 0; }
		__syncthreads();
	}

	if ((uint32_t)tid < n_views * N_STATS) {
		const uint32_t v = (uint32_t)tid / N_STATS, i = (uint32_t)tid % N_STATS;
		if (s_stats[v][i]) atomicAdd(&counters[v * COUNTER_WORDS + 256 + i], s_stats[v][i]);
	}
	if (tid == 0 && s_streamed) atomicAdd(&counters[MAX_VIEWS * COUNTER_WORDS + CALL_STREAMED], s_streamed);
	// the other counter block is the next call's: zero it now so no memset sits between two calls
	if (blockIdx.x == 0) {
		for (int i = tid; i < CALL_COUNTER_WORDS; i += VIEW_THREADS) next_counters[i] = 0;
	}
}

} // namespace lbviews
