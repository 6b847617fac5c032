// cull_pages_kernel — CullingSystemImpl::cullInternal + doCulling (src/renderer/culling_system.cpp:260-369) on the GPU, ONE kernel per cull.
//
// Pages are dealt to the blocks round-robin; per round a block runs:
//   A1  cheap pass, one THREAD per page: coalesced 32-byte descriptors; free pages, the type filter and "definitely outside" — the
//       reference's intersectsAABB expression (geometry.cpp:159-178, bit-identical dp) failing by a safe margin, which also rules out the
//       shifted containsAABB box.  ~3/4 of the pages of a typical view end here.
//   A2  exact pass on the compacted survivors (dense threads): the cell tests of culling_system.cpp:342-363 (is_big -> test;
//       containsAABB(origin + cs, cs) -> copy every id; intersectsAABB(origin - cs, 2cs) -> test; else nothing) with
//       ShiftedFrustum::containsAABB / intersectsAABB arithmetic (geometry.cpp:99-118,159-178), the plane mask, and for pages that need
//       sphere tests the plane offsets re-based to the cell origin (ShiftedFrustum::getRelative, geometry.cpp:121-149 — only d
//       changes); pages with work go to a block-local list in shared memory.
//   B   test, one WARP per listed page: the <=200 spheres as 7 x 128-bit streaming loads per lane; the planes of the mask are walked by a
//       warp-uniform loop with the rows unrolled inside (no branch per sphere; rows 4-6 only for pages with more than 128 spheres), the
//       reference's op order and sign-bit test (culling_system.cpp:284-295, simd.h:119); ballots kept in shared memory.
//   C   claim: one global atomic per (warp, renderable type) reserves the output range of the warp's pages.
//   D   write: visible ids gathered (4 B) and written compacted, grouped by type; the id rows of the next page are loaded while the
//       current one is written.  The 32-byte visibility row of every worked page goes to the mask (row = page id; classify threads
//       zero the rows of skipped pages) or — exchange mode — as a {page id, row} record straight into every rank's slab over NVLink:
//       only rows that can be non-zero cross the links (SURVEY 8e: the bitmask is the exchanged product).
// One block barrier per round after A1 and A2 each; B, C and D run warp-autonomously, so a warp with cheap pages never waits for one
// with expensive pages.  No per-page global atomics; skipped pages never reach a warp.
// Everything before cudaGridDependencySynchronize() (launch, descriptor reads, classification, the sphere tests of phase B whose
// results sit in shared memory) only READS scene data: when culls are issued back to back with programmatic stream serialization it
// overlaps the tail of the previous cull.
// HBM-bound: 32 B descriptor per page + 16 B per tested sphere + 4 B read + 4 B write per visible id + 32 B mask row per page.
#pragma once

#include "culling_internal.h" // counter and slab layout
#include "lb200_internal.h"
#include "lb200_math.cuh"

namespace lbcull {

using namespace lb;

constexpr int ROWS = 7;                 // ceil(200 / 32)
constexpr int CULL_THREADS = 256;       // 4 blocks/SM at 64 registers; pages per block per round <= one classify thread each
constexpr int CULL_WARPS = CULL_THREADS / 32;
constexpr int MAX_CHUNK = CULL_THREADS;

struct CullParams {
	// planes NEAR, FAR, LEFT, RIGHT, TOP, BOTTOM of the ShiftedFrustum (relative to `origin`)
	float nx[6], ny[6], nz[6], d[6];
	// the frustum point each plane is re-anchored on by getRelative (geometry.cpp:134-142): points[0,4,1,0,0,2]
	float px[6], py[6], pz[6];
	double ox, oy, oz;
	uint32_t n_pages;
	uint32_t type_filter;   // 0xff = all
	uint32_t chunk;         // pages per block per round, <= MAX_CHUNK
	uint32_t plane_masking; // 1 unless some sphere has a negative / NaN radius
	uint32_t item_cap;      // record capacity of an exchange slab (>= n_pages)
	// exchange mode (n_ranks > 0): {page, row} records go straight into every rank's slab (peer memory)
	uint32_t n_ranks;
	uint32_t* xdst[LB200_MAX_RANKS]; // rank r's exchange buffer of this epoch, already offset to MY slab inside it
	// fused exchange steps (one kernel per step, lb200_culling_cull_exchange_n on two or more lanes): this cull also publishes the lane's
	// PREVIOUS epoch (pub_epoch != 0) and holds its record stores back until every rank has published wait_epoch (!= 0)
	uint32_t pub_epoch, wait_epoch, n_buffers, rank;
	uint32_t* xprev[LB200_MAX_RANKS];  // rank r's exchange buffer of pub_epoch, offset to MY slab
	uint32_t* xflags[LB200_MAX_RANKS]; // rank r's flag block: [n_buffers][LB200_MAX_RANKS]
	uint32_t type_base[256];
};

__device__ __forceinline__ int ldg_stream_i32(const int* p) {
	int r;
	asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r) : "l"(p));
	return r;
}

enum { CLS_SKIP = 0, CLS_COPY = 1, CLS_TEST = 2 };

struct WorkItem { // 32 B
	uint32_t page;
	uint32_t meta; // count | type << 8 | cls << 16 | planes needed << 24
	float rd[6];   // plane offsets relative to the cell origin (TEST pages)
};
static_assert(sizeof(WorkItem) == 32, "");

__device__ __forceinline__ float4 ldg_stream(const float4* p) {
	float4 r;
	asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
	return r;
}

__global__ void __launch_bounds__(CULL_THREADS, 4) cull_pages_kernel(const __grid_constant__ CullParams P,
	const lb200_page_desc* __restrict__ desc, const float4* __restrict__ spheres, const int* __restrict__ entities,
	uint32_t* __restrict__ out_ids, uint32_t* __restrict__ counters, uint32_t* __restrict__ next_counters, uint32_t* __restrict__ mask_out)
{
	__shared__ WorkItem s_item[MAX_CHUNK];
	__shared__ __align__(16) uint32_t s_bal[MAX_CHUNK][ROWS + 1]; // the 256-bit visibility row of a tested page ([ROWS] = 0)
	__shared__ uint32_t s_off[MAX_CHUNK];                         // visible ids of the page, then its offset inside out_ids
	__shared__ uint16_t s_cand[MAX_CHUNK]; // classify threads whose page survived the cheap pass
	__shared__ uint32_t s_stats[N_STATS];
	__shared__ uint32_t s_zpage[MAX_CHUNK]; // page whose mask row is zero (ends without work), or ~0
	__shared__ uint32_t s_ntest, s_ncopy, s_ncand;

	// let the next cull of the stream start its read-only prologue as soon as SM resources free up
	cudaTriggerProgrammaticLaunchCompletion();

	const int tid = threadIdx.x;
	const int lane = tid & 31;
	const int warp = tid >> 5;
	const uint32_t lt_mask = (1u << lane) - 1u;

	if (tid < N_STATS) s_stats[tid] = 0;
	if (tid == 0) { s_ntest = 0; s_ncopy = 0; s_ncand = 0; }
	__syncthreads();

	// Pages are dealt to blocks round-robin (page = j * gridDim + block): pages that always need sphere tests (is_big cells) and
	// frustum-boundary cells cluster in page-id space, and contiguous chunks left a few blocks with twice the work of the rest.
	for (uint32_t round = 0; round * P.chunk * gridDim.x < P.n_pages; ++round) {
		// ---------------- A1. cheap pass: one thread per page, "definitely outside" only ----------------
		{
			bool cand = false;
			uint32_t zpage = 0xffffffffu; // a page that ends here has an all-zero mask row
			if ((uint32_t)tid < P.chunk) {
				const uint32_t page = (round * P.chunk + tid) * gridDim.x + blockIdx.x;
				if (page < P.n_pages) {
					zpage = page;
					const int4* dp = reinterpret_cast<const int4*>(desc + page);
					const int4 a = __ldg(dp);
					const int4 b = __ldg(dp + 1);
					const uint32_t count = (uint32_t)b.z;
					const uint32_t type = (uint32_t)b.w & 0xffu;
					const bool is_big = (((uint32_t)b.w >> 8) & 0xffu) != 0;
					if (count != 0) {
						if (P.type_filter != 0xffu && type != P.type_filter) atomicAdd(&s_stats[ST_PAGES_FILTERED], 1u);
						else {
							bool outside = false;
							if (!is_big) {
								const double org_x = __hiloint2double(a.y, a.x);
								const double org_y = __hiloint2double(a.w, a.z);
								const double org_z = __hiloint2double(b.y, b.x);
								const float cs = LB200_CELL_SIZE;
								const float cs2 = 2 * LB200_CELL_SIZE;
								const V3 rel_i = tofloat(sub(d3(LB_DSUB(org_x, (double)cs), LB_DSUB(org_y, (double)cs), LB_DSUB(org_z, (double)cs)), d3(P.ox, P.oy, P.oz)));
								const V3 max_i = add(rel_i, v3(cs2, cs2, cs2));
#pragma unroll
								for (int p = 0; p < 6; ++p) {
									const float nx = P.nx[p], ny = P.ny[p], nz = P.nz[p], nd = -P.d[p];
									const float tx = LB_FMUL(nx, nx > 0.0f ? max_i.x : rel_i.x);
									const float ty = LB_FMUL(ny, ny > 0.0f ? max_i.y : rel_i.y);
									const float tz = LB_FMUL(nz, nz > 0.0f ? max_i.z : rel_i.z);
									const float dp_i = LB_FADD(LB_FADD(tx, ty), tz); // the exact pass computes the same value
									const float margin = 1e-4f * (fabsf(nd) + fabsf(tx) + fabsf(ty) + fabsf(tz)) + 0.05f;
									if (dp_i + margin < nd) outside = true; // NaN anywhere: false, the page stays a candidate
								}
							}
							if (outside) atomicAdd(&s_stats[ST_PAGES_OUTSIDE], 1u);
							else cand = true;
						}
					}
				}
			}
			// warp-aggregated append to the candidate list
			const uint32_t bal = __ballot_sync(0xffffffffu, cand);
			uint32_t base = 0;
			if (lane == 0 && bal) base = atomicAdd(&s_ncand, (uint32_t)__popc(bal));
			base = __shfl_sync(0xffffffffu, base, 0);
			if (cand) { s_cand[base + __popc(bal & lt_mask)] = (uint16_t)tid; zpage = 0xffffffffu; }
			s_zpage[tid] = zpage;
		}
		__syncthreads();

		// ---------------- A2. exact classification of the candidates (dense threads) ----------------
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
			int cls = CLS_SKIP;
			{
				// containsAABB(cell.origin + Vec3(cs), Vec3(cs)), geometry.cpp:99-118 (DVec3 + Vec3: math.cpp:512)
				const float cs = LB200_CELL_SIZE;
				const V3 rel_c = tofloat(sub(d3(LB_DADD(org_x, (double)cs), LB_DADD(org_y, (double)cs), LB_DADD(org_z, (double)cs)), d3(P.ox, P.oy, P.oz)));
				const V3 max_c = add(rel_c, v3(cs, cs, cs));
				// intersectsAABB(cell.origin - Vec3(cs), Vec3(2cs)), geometry.cpp:159-178 (DVec3 - Vec3: math.cpp:510)
				const float cs2 = 2 * LB200_CELL_SIZE;
				const V3 rel_i = tofloat(sub(d3(LB_DSUB(org_x, (double)cs), LB_DSUB(org_y, (double)cs), LB_DSUB(org_z, (double)cs)), d3(P.ox, P.oy, P.oz)));
				const V3 max_i = add(rel_i, v3(cs2, cs2, cs2));
				bool contains = true, intersects = true;
#pragma unroll
				for (int p = 0; p < 6; ++p) {
					const float nx = P.nx[p], ny = P.ny[p], nz = P.nz[p], nd = -P.d[p];
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
				// culling_system.cpp:342-363
				if (is_big) cls = CLS_TEST;
				else if (contains) cls = CLS_COPY;
				else if (intersects) cls = CLS_TEST;
				else atomicAdd(&s_stats[ST_PAGES_OUTSIDE], 1u);
			}
			uint32_t need = 0x3fu;
			float rd[6];
#pragma unroll
			for (int p = 0; p < 6; ++p) rd[p] = 0.0f;
			// statistics follow the reference's classification (culling_system.cpp:342-363), not the masking shortcut below
			if (cls == CLS_TEST) { atomicAdd(&s_stats[ST_PAGES_TESTED], 1u); atomicAdd(&s_stats[ST_ENT_TESTED], count); }
			else if (cls == CLS_COPY) { atomicAdd(&s_stats[ST_PAGES_INSIDE], 1u); atomicAdd(&s_stats[ST_ENT_INSIDE], count); }
			if (cls == CLS_TEST) {
				// ShiftedFrustum::getRelative(cell.origin), geometry.cpp:121-149: offset = Vec3(this->origin - origin);
				// d = -dot(point + offset, normal) (setPlane, geometry.cpp:412-418)
				const V3 offset = tofloat(sub(d3(P.ox, P.oy, P.oz), d3(org_x, org_y, org_z)));
#pragma unroll
				for (int p = 0; p < 6; ++p) rd[p] = -dot(add(v3(P.px[p], P.py[p], P.pz[p]), offset), v3(P.nx[p], P.ny[p], P.nz[p]));
				if (P.plane_masking) {
					// Plane masking: a plane cannot cull any sphere of this cell when its signed distance is positive over the whole cell box
					// by more than every rounding error of the reference's expression — then sign(t - r) is 0 for every sphere (radius >= 0)
					// and evaluating the plane changes nothing.  Cell box relative to the cell origin: [0,300] for positive cell indices,
					// [-300,0] for negative ones, [-300,300] for index 0 (truncation toward zero, math.cpp:133-138), widened by `e` because
					// the cell index comes from pos * float(1/300) and may put a sphere marginally outside its nominal cell.
					const float cs = LB200_CELL_SIZE;
					const float e = 1.0f + 1e-6f * fmaxf(fmaxf(fabsf((float)org_x), fabsf((float)org_y)), fabsf((float)org_z));
					const float lox = (org_x > 0.0 ? 0.0f : -cs) - e, hix = (org_x < 0.0 ? 0.0f : cs) + e;
					const float loy = (org_y > 0.0 ? 0.0f : -cs) - e, hiy = (org_y < 0.0 ? 0.0f : cs) + e;
					const float loz = (org_z > 0.0 ? 0.0f : -cs) - e, hiz = (org_z < 0.0 ? 0.0f : cs) + e;
					need = 0;
#pragma unroll
					for (int p = 0; p < 6; ++p) {
						const float nx = P.nx[p], ny = P.ny[p], nz = P.nz[p];
						const float dp = rd[p];
						const float low = dp + fminf(nx * lox, nx * hix) + fminf(ny * loy, ny * hiy) + fminf(nz * loz, nz * hiz);
						const float margin = 1e-5f * (fabsf(dp) + 1000.0f * (fabsf(nx) + fabsf(ny) + fabsf(nz))) + 1e-3f;
						if (!(low > margin)) need |= 1u << p; // NaN keeps the plane
					}
					if (need == 0) cls = CLS_COPY; // every sphere of the page is visible: ids only, no sphere traffic
				}
				if (cls == CLS_TEST) atomicAdd(&s_stats[ST_ENT_STREAMED], count);
			}
			if (cls != CLS_SKIP) {
				// TEST pages fill the list from the front, COPY pages from the back (compacted below): the warps take the list in strides, so
				// every warp gets the same number of sphere-test pages (+-1)
				const uint32_t slot = cls == CLS_TEST ? atomicAdd(&s_ntest, 1u) : (uint32_t)MAX_CHUNK - 1u - atomicAdd(&s_ncopy, 1u);
				uint4* it = reinterpret_cast<uint4*>(&s_item[slot]);
				it[0] = make_uint4(page, count | (type << 8) | ((uint32_t)cls << 16) | (need << 24), __float_as_uint(rd[0]), __float_as_uint(rd[1]));
				it[1] = make_uint4(__float_as_uint(rd[2]), __float_as_uint(rd[3]), __float_as_uint(rd[4]), __float_as_uint(rd[5]));
				if (cls == CLS_COPY) s_off[slot] = count; // culling_system.cpp:345-360: every entity of the page is visible
			}
			else s_zpage[t0] = page;
		}
		__syncthreads();
		const uint32_t n_test = s_ntest;
		const uint32_t n_work = n_test + s_ncopy;
		// listed page w: s_item[item_index(w)] — the COPY pages sit at the back of the array
#define LB_ITEM(w) ((w) < n_test ? (w) : (uint32_t)MAX_CHUNK - 1u - ((w) - n_test))

		// ---------------- B. sphere tests: one warp per listed TEST page (w = warp, warp + CULL_WARPS, ... < n_test) ----------------
		{
			for (uint32_t iw = warp; iw < n_test; iw += CULL_WARPS) {
				const uint4 ia = *reinterpret_cast<const uint4*>(&s_item[iw]);
				const uint32_t count = ia.y & 0xffu;
				const uint4 ib = *(reinterpret_cast<const uint4*>(&s_item[iw]) + 1);
				const uint32_t need = ia.y >> 24;
				const bool upper = count > 128u; // rows 4-6 exist (warp-uniform): half of the tested pages of a typical scene stop before
				float4 s[ROWS];
				const float4* sp = spheres + (size_t)ia.x * LB200_PAGE_SLOTS;
				const uint32_t last = count - 1u; // count >= 1 for listed pages
#pragma unroll
				for (int k = 0; k < 4; ++k) { const uint32_t slot = k * 32 + lane; s[k] = ldg_stream(sp + (slot < last ? slot : last)); } // lanes past the page re-read its last sphere
				if (upper) {
#pragma unroll
					for (int k = 4; k < ROWS; ++k) { const uint32_t slot = k * 32 + lane; s[k] = ldg_stream(sp + (slot < last ? slot : last)); }
				}
				if (!upper) {
#pragma unroll
					for (int k = 4; k < ROWS; ++k) s[k] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
				}
				// doCulling, culling_system.cpp:260-308, plane-outer: per sphere and plane exactly :284,291
				//   t = cx*px + cy*py + cz*pz + pd ;  t = t - r (r = -radius) ;  movemask = sign bits
				uint32_t acc[ROWS];
#pragma unroll
				for (int k = 0; k < ROWS; ++k) acc[k] = 0;
#define LB_ROWS(pd, k0, k1)                                                                                                      \
					_Pragma("unroll") for (int k = k0; k < k1; ++k) {                                                             \
						float t = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(s[k].x, nx), LB_FMUL(s[k].y, ny)), LB_FMUL(s[k].z, nz)), pd);   \
						t = LB_FSUB(t, -s[k].w); /* :282 f4Splat(-sphere->radius) */                                              \
						acc[k] |= __float_as_uint(t);                                                                             \
					}
#define LB_PLANE(p, pd)                                                                                                          \
				if (need & (1u << p)) {                                                                                           \
					const float nx = P.nx[p], ny = P.ny[p], nz = P.nz[p];                                                         \
					LB_ROWS(pd, 0, 4)                                                                                             \
					if (upper) { LB_ROWS(pd, 4, ROWS) }                                                                           \
				}
				LB_PLANE(0, __uint_as_float(ia.z))
				LB_PLANE(1, __uint_as_float(ia.w))
				LB_PLANE(2, __uint_as_float(ib.x))
				LB_PLANE(3, __uint_as_float(ib.y))
				LB_PLANE(4, __uint_as_float(ib.z))
				LB_PLANE(5, __uint_as_float(ib.w))
#undef LB_PLANE
#undef LB_ROWS
				// A NaN radius: on the reference's SSE path t - (-radius) hands the NaN through with the sign of -radius, and that sign is
				// what movemask reads (+NaN radius: culled by every plane; -NaN radius: passes every plane).  The GPU's subtraction returns
				// the canonical positive NaN instead, so the sign is taken from the radius directly (tests/golden/cull_kat.npz: special_*).
				// The complement goes through inline PTX: the compiler otherwise rewrites "sign of ~bits" as neg.f32 + a sign test, and
				// neg.f32 of a NaN does not keep the sign.  Only scenes that hold a negative / NaN radius get here (the host tracks them
				// and switches plane masking off with them): one warp-uniform branch per page otherwise.
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
		// nothing above wrote global memory (A and B read scene data, results sit in shared memory); everything below does
		// (counters, ids, mask rows) and has to wait for the previous kernel of the stream
		if (round == 0) cudaGridDependencySynchronize();
		if (round == 0 && P.n_ranks && (P.pub_epoch | P.wait_epoch)) {
			// Fused exchange step.  Behind the grid dependency the lane's previous cull is complete: its records lie in the peers' slabs, its
			// counters still in `next_counters` (zeroed at the end of THIS kernel, behind the round barrier every warp of block 0 passes).
			if (P.pub_epoch && blockIdx.x == 0 && warp == 0) { // publish that epoch: header to every rank, one system fence, the flags
				for (uint32_t i = (uint32_t)lane; i < XHEADER_WORDS; i += 32u) {
					uint32_t v = 0;
					if (i < 256u) v = __ldcg(next_counters + i);
					else if (i == 256u) v = P.n_pages;
					else if (i == 257u) v = __ldcg(next_counters + CNT_N_REC);
					else if (i == 259u) v = P.item_cap;
					for (uint32_t r = 0; r < P.n_ranks; ++r) P.xprev[r][i] = v;
				}
				__threadfence_system();
				__syncwarp();
				if ((uint32_t)lane < P.n_ranks) {
					__threadfence_system();
					volatile uint32_t* f = P.xflags[lane] + (P.pub_epoch % P.n_buffers) * LB200_MAX_RANKS + P.rank;
					*f = P.pub_epoch;
				}
				__syncwarp();
			}
			if (P.wait_epoch) { // flow control: nobody stores records of this epoch before every rank has published wait_epoch (= epoch - 2 x lanes)
				if ((uint32_t)lane < P.n_ranks) {
					const volatile uint32_t* f = P.xflags[P.rank] + (P.wait_epoch % P.n_buffers) * LB200_MAX_RANKS + lane;
					const long long t0 = clock64();
					while ((int)(*f - P.wait_epoch) < 0) { if (clock64() - t0 > 8000000000ll) break; } // a lost peer is reported by the batch's closing wait
				}
				__syncwarp();
			}
		}
		// rows of pages that ended without work
		if (mask_out && (uint32_t)tid < P.chunk && s_zpage[tid] != 0xffffffffu) {
			uint4* row = reinterpret_cast<uint4*>(mask_out + (size_t)s_zpage[tid] * 8);
			row[0] = make_uint4(0u, 0u, 0u, 0u);
			row[1] = make_uint4(0u, 0u, 0u, 0u);
		}
		// ---------------- C. claim: one global atomic per (warp, type) — no block barrier between B, C and D ----------------
		// lane i stands for the warp's i-th page (w = warp + i * CULL_WARPS; at most 32 per warp since chunk <= CULL_THREADS)
		__syncwarp();
		uint32_t rec_base = 0;
		{
			const uint32_t wi = warp + (uint32_t)lane * CULL_WARPS;
			const bool has = wi < n_work;
			const uint32_t iwi = LB_ITEM(wi);
			const uint32_t my_type = has ? ((s_item[iwi].meta >> 8) & 0xffu) : 0xffffu;
			const uint32_t my_count = has ? s_off[iwi] : 0u;
			const uint32_t n_mine = (n_work + CULL_WARPS - 1 - warp) / CULL_WARPS; // pages of this warp (warp-uniform)
			const uint32_t packed = (my_type << 16) | my_count; // count <= 200
			uint32_t prefix = 0, total = 0;
			for (uint32_t l = 0; l < n_mine; ++l) {
				const uint32_t o = __shfl_sync(0xffffffffu, packed, (int)l);
				if ((o >> 16) == my_type) { total += o & 0xffffu; if (l < (uint32_t)lane) prefix += o & 0xffffu; }
			}
			const unsigned grp = __match_any_sync(0xffffffffu, my_type);
			const int leader = __ffs((int)grp) - 1;
			uint32_t base = 0;
			if (has && lane == leader && total) base = atomicAdd(&counters[my_type], total);
			// exchange mode: the warp's pages also take n_mine consecutive record slots of this rank's slab
			if (P.n_ranks && lane == 31 && n_mine) rec_base = atomicAdd(&counters[CNT_N_REC], n_mine);
			base = __shfl_sync(0xffffffffu, base, leader);
			rec_base = __shfl_sync(0xffffffffu, rec_base, 31);
			if (has) s_off[iwi] = P.type_base[my_type] + base + prefix; // where the page's ids go in out_ids
		}
		__syncwarp();

		// ---------------- D. write: gather the visible ids of each listed page ----------------
		{
			uint32_t rec = rec_base;
			for (uint32_t w = warp; w < n_work; w += CULL_WARPS, ++rec) {
				const uint32_t iw = LB_ITEM(w);
				const uint32_t page = s_item[iw].page;
				const uint32_t meta = s_item[iw].meta;
				const uint32_t count = meta & 0xffu;
				uint32_t* dst = out_ids + s_off[iw];
				const int* ep = entities + (size_t)page * LB200_PAGE_SLOTS;
				uint32_t row_word; // lane k < 8 (and its images in the other 8-lane groups): word k of the page's visibility row
				if (((meta >> 16) & 3u) == CLS_COPY) {
					// every id of the page is visible (culling_system.cpp:345-360, or an empty plane mask): a straight copy, one base address per
					// lane and immediate offsets per row — no ballots, no ranks
					const int* src = ep + lane;
					uint32_t* d = dst + lane;
					int id[ROWS] = {}; // zeroed per page: unassigned elements were otherwise kept live across pages, and spilled
#pragma unroll
					for (int k = 0; k < ROWS; ++k) if ((uint32_t)(k * 32 + lane) < count) id[k] = ldg_stream_i32(src + k * 32);
#pragma unroll
					for (int k = 0; k < ROWS; ++k) if ((uint32_t)(k * 32 + lane) < count) d[k * 32] = (uint32_t)id[k];
					const int rem = (int)count - (lane & 7) * 32;
					row_word = rem >= 32 ? 0xffffffffu : (rem > 0 ? ((1u << rem) - 1u) : 0u);
				}
				else {
					uint32_t bal[ROWS];
#pragma unroll
					for (int k = 0; k < ROWS; ++k) bal[k] = s_bal[iw][k];
					int id[ROWS] = {}; // zeroed per page: unassigned elements were otherwise kept live across pages, and spilled
#pragma unroll
					for (int k = 0; k < ROWS; ++k) if ((bal[k] >> lane) & 1u) id[k] = ldg_stream_i32(ep + k * 32 + lane);
					uint32_t prefix = 0;
#pragma unroll
					for (int k = 0; k < ROWS; ++k) {
						if ((bal[k] >> lane) & 1u) dst[prefix + __popc(bal[k] & lt_mask)] = (uint32_t)id[k];
						prefix += __popc(bal[k]);
					}
					row_word = s_bal[iw][lane & 7];
				}
				if (mask_out && lane < 8) mask_out[(size_t)page * 8 + lane] = row_word;
				if (P.n_ranks) {
					for (uint32_t r = (uint32_t)lane >> 3; r < P.n_ranks; r += 4) { // 8 lanes per destination rank
						uint32_t* slab = P.xdst[r];
						slab[XHEADER_WORDS + P.item_cap + (size_t)rec * 8 + (lane & 7)] = row_word;
						if ((lane & 7) == 0) slab[XHEADER_WORDS + rec] = page;
					}
				}
			}
		}
#undef LB_ITEM
		__syncthreads(); // every warp is done with s_item / s_bal / s_zpage
		if (tid == 0) { s_ntest = 0; s_ncopy = 0; s_ncand = 0; }
		__syncthreads();
	}

	if (tid < N_STATS && s_stats[tid]) atomicAdd(&counters[256 + tid], s_stats[tid]);
	// the other counter buffer is the next cull's: zero it now so no memset sits between two culls
	if (blockIdx.x == 0) {
		for (int i = tid; i < COUNTER_WORDS; i += CULL_THREADS) next_counters[i] = 0;
	}
	// exchange mode: nothing more to do here.  The records were stored without a fence; publish_wait_kernel (culling_exchange.cu), which runs
	// after this grid has completed, sends the header, fences once at system scope and raises the epoch flags.
}

} // namespace lbcull
