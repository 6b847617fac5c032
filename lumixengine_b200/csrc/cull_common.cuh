// The culling core that cull_pages_kernel (cull_kernel.cuh) and cull_views_kernel (cull_views_kernel.cuh) share: the reference's
// cell tests and sphere test (CullingSystemImpl::cullInternal + doCulling, src/renderer/culling_system.cpp:260-369) and the claim and
// write of visible ids.  Each function is one phase piece of a kernel; what differs between the kernels (a view's frustum, its statistics
// row, its output buffers) comes in as arguments.  The expressions are the reference's, op for op: keep them as they are.
#pragma once

#include "culling_internal.h" // statistics
#include "lb200_internal.h"
#include "lb200_math.cuh"

namespace lbcull {

using namespace lb;

constexpr int ROWS = 7; // ceil(200 / 32)

enum { CLS_SKIP = 0, CLS_COPY = 1, CLS_TEST = 2 };

// One view's frustum as the kernels read it from their parameter block
struct CullFrustum {
	// planes NEAR, FAR, LEFT, RIGHT, TOP, BOTTOM of the ShiftedFrustum (relative to `origin`)
	float nx[6], ny[6], nz[6], d[6];
	// the frustum point each plane is re-anchored on by getRelative (geometry.cpp:134-142): points[0,4,1,0,0,2]
	float px[6], py[6], pz[6];
	double ox, oy, oz;
};
static_assert(sizeof(CullFrustum) == 192, "168 B of floats, then the origin");

__device__ __forceinline__ float4 ldg_stream(const float4* p) {
	float4 r;
	asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
	return r;
}

__device__ __forceinline__ int ldg_stream_i32(const int* p) {
	int r;
	asm volatile("ld.global.nc.L1::no_allocate.s32 %0, [%1];" : "=r"(r) : "l"(p));
	return r;
}

// a page descriptor: cell origin, entity count, renderable type, is_big cell
struct PageInfo {
	D3 org;
	uint32_t count, type;
	bool is_big;
};

__device__ __forceinline__ PageInfo load_page(const lb200_page_desc* desc, uint32_t page) {
	const int4* dp = reinterpret_cast<const int4*>(desc + page);
	const int4 a = __ldg(dp);
	const int4 b = __ldg(dp + 1);
	PageInfo pi;
	pi.org = d3(__hiloint2double(a.y, a.x), __hiloint2double(a.w, a.z), __hiloint2double(b.y, b.x));
	pi.count = (uint32_t)b.z;
	pi.type = (uint32_t)b.w & 0xffu;
	pi.is_big = (((uint32_t)b.w >> 8) & 0xffu) != 0;
	return pi;
}

// the low corner of the box the reference's intersectsAABB tests: cell.origin - Vec3(cs) (DVec3 - Vec3: math.cpp:510)
__device__ __forceinline__ D3 cell_lo(D3 org) {
	const float cs = LB200_CELL_SIZE;
	return d3(LB_DSUB(org.x, (double)cs), LB_DSUB(org.y, (double)cs), LB_DSUB(org.z, (double)cs));
}

// "Definitely outside" (not is_big cells): the reference's intersectsAABB expression (geometry.cpp:159-178, bit-identical dp) failing
// by a safe margin, which also rules out the shifted containsAABB box.  lo = cell_lo(cell origin).
__device__ __forceinline__ bool outside_by_margin(const CullFrustum& f, D3 lo) {
	const float cs2 = 2 * LB200_CELL_SIZE;
	const V3 rel_i = tofloat(sub(lo, d3(f.ox, f.oy, f.oz)));
	const V3 max_i = add(rel_i, v3(cs2, cs2, cs2));
	bool outside = false;
#pragma unroll
	for (int p = 0; p < 6; ++p) {
		const float nx = f.nx[p], ny = f.ny[p], nz = f.nz[p], nd = -f.d[p];
		const float tx = LB_FMUL(nx, nx > 0.0f ? max_i.x : rel_i.x);
		const float ty = LB_FMUL(ny, ny > 0.0f ? max_i.y : rel_i.y);
		const float tz = LB_FMUL(nz, nz > 0.0f ? max_i.z : rel_i.z);
		const float dp_i = LB_FADD(LB_FADD(tx, ty), tz); // the exact pass computes the same value
		const float margin = 1e-4f * (fabsf(nd) + fabsf(tx) + fabsf(ty) + fabsf(tz)) + 0.05f;
		if (dp_i + margin < nd) outside = true; // NaN anywhere: false, the page stays a candidate
	}
	return outside;
}

// The exact cell tests of culling_system.cpp:342-363 (is_big -> test; containsAABB(origin + cs, cs) -> copy every id;
// intersectsAABB(origin - cs, 2cs) -> test; else nothing) with ShiftedFrustum::containsAABB / intersectsAABB arithmetic
// (geometry.cpp:99-118,159-178), counted into the statistics row `stats` as the reference counts them.
__device__ __forceinline__ int classify_cell(const CullFrustum& f, const PageInfo& pi, uint32_t* stats) {
	const double org_x = pi.org.x, org_y = pi.org.y, org_z = pi.org.z;
	int cls = CLS_SKIP;
	{
		// containsAABB(cell.origin + Vec3(cs), Vec3(cs)), geometry.cpp:99-118 (DVec3 + Vec3: math.cpp:512)
		const float cs = LB200_CELL_SIZE;
		const V3 rel_c = tofloat(sub(d3(LB_DADD(org_x, (double)cs), LB_DADD(org_y, (double)cs), LB_DADD(org_z, (double)cs)), d3(f.ox, f.oy, f.oz)));
		const V3 max_c = add(rel_c, v3(cs, cs, cs));
		// intersectsAABB(cell.origin - Vec3(cs), Vec3(2cs)), geometry.cpp:159-178 (DVec3 - Vec3: math.cpp:510)
		const float cs2 = 2 * LB200_CELL_SIZE;
		const V3 rel_i = tofloat(sub(cell_lo(pi.org), d3(f.ox, f.oy, f.oz)));
		const V3 max_i = add(rel_i, v3(cs2, cs2, cs2));
		bool contains = true, intersects = true;
#pragma unroll
		for (int p = 0; p < 6; ++p) {
			const float nx = f.nx[p], ny = f.ny[p], nz = f.nz[p], nd = -f.d[p];
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
		if (pi.is_big) cls = CLS_TEST;
		else if (contains) cls = CLS_COPY;
		else if (intersects) cls = CLS_TEST;
		else atomicAdd(&stats[ST_PAGES_OUTSIDE], 1u);
	}
	// statistics follow the reference's classification, not the plane-masking shortcut (plane_mask)
	if (cls == CLS_TEST) { atomicAdd(&stats[ST_PAGES_TESTED], 1u); atomicAdd(&stats[ST_ENT_TESTED], pi.count); }
	else if (cls == CLS_COPY) { atomicAdd(&stats[ST_PAGES_INSIDE], 1u); atomicAdd(&stats[ST_ENT_INSIDE], pi.count); }
	return cls;
}

// ShiftedFrustum::getRelative(cell.origin), geometry.cpp:121-149: offset = Vec3(this->origin - origin);
// d = -dot(point + offset, normal) (setPlane, geometry.cpp:412-418).  Only d changes.
__device__ __forceinline__ void relative_offsets(const CullFrustum& f, D3 org, float rd[6]) {
	const V3 offset = tofloat(sub(d3(f.ox, f.oy, f.oz), org));
#pragma unroll
	for (int p = 0; p < 6; ++p) rd[p] = -dot(add(v3(f.px[p], f.py[p], f.pz[p]), offset), v3(f.nx[p], f.ny[p], f.nz[p]));
}

// Plane masking: a plane cannot cull any sphere of this cell when its signed distance is positive over the whole cell box by more than
// every rounding error of the reference's expression — then sign(t - r) is 0 for every sphere (radius >= 0) and evaluating the plane
// changes nothing.  Cell box relative to the cell origin: [0,300] for positive cell indices, [-300,0] for negative ones, [-300,300] for
// index 0 (truncation toward zero, math.cpp:133-138), widened by `e` because the cell index comes from pos * float(1/300) and may put a
// sphere marginally outside its nominal cell.  Returns the planes that are needed (bit p = plane p); rd from relative_offsets.
__device__ __forceinline__ uint32_t plane_mask(const CullFrustum& f, D3 org, const float rd[6]) {
	const double org_x = org.x, org_y = org.y, org_z = org.z;
	const float cs = LB200_CELL_SIZE;
	const float e = 1.0f + 1e-6f * fmaxf(fmaxf(fabsf((float)org_x), fabsf((float)org_y)), fabsf((float)org_z));
	const float lox = (org_x > 0.0 ? 0.0f : -cs) - e, hix = (org_x < 0.0 ? 0.0f : cs) + e;
	const float loy = (org_y > 0.0 ? 0.0f : -cs) - e, hiy = (org_y < 0.0 ? 0.0f : cs) + e;
	const float loz = (org_z > 0.0 ? 0.0f : -cs) - e, hiz = (org_z < 0.0 ? 0.0f : cs) + e;
	uint32_t need = 0;
#pragma unroll
	for (int p = 0; p < 6; ++p) {
		const float nx = f.nx[p], ny = f.ny[p], nz = f.nz[p];
		const float dp = rd[p];
		const float low = dp + fminf(nx * lox, nx * hix) + fminf(ny * loy, ny * hiy) + fminf(nz * loz, nz * hiz);
		const float margin = 1e-5f * (fabsf(dp) + 1000.0f * (fabsf(nx) + fabsf(ny) + fabsf(nz))) + 1e-3f;
		if (!(low > margin)) need |= 1u << p; // NaN keeps the plane
	}
	return need;
}

// A warp loads the <= 200 spheres of `page` as 7 x 128-bit streaming loads per lane; rows 4-6 only when `upper` (count > 128, warp-uniform).
// Lanes past the page re-read its last sphere (count >= 1).
__device__ __forceinline__ void load_rows(const float4* spheres, uint32_t page, uint32_t count, bool upper, int lane, float4 s[ROWS]) {
	const float4* sp = spheres + (size_t)page * LB200_PAGE_SLOTS;
	const uint32_t last = count - 1u;
#pragma unroll
	for (int k = 0; k < 4; ++k) { const uint32_t slot = k * 32 + lane; s[k] = ldg_stream(sp + (slot < last ? slot : last)); }
	if (upper) {
#pragma unroll
		for (int k = 4; k < ROWS; ++k) { const uint32_t slot = k * 32 + lane; s[k] = ldg_stream(sp + (slot < last ? slot : last)); }
	}
	if (!upper) {
#pragma unroll
		for (int k = 4; k < ROWS; ++k) s[k] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
	}
}

// The sphere test of one page against the needed planes of `f` (bit p of `need`), over the rows of load_rows.  The plane offsets rd[0..5]
// (relative_offsets) are the last six words of the page's 32-byte work item: ia.z, ia.w, ib.x .. ib.w.  The planes of the mask are walked
// by a warp-uniform loop with the rows unrolled inside (no branch per sphere).  Returns the page's visible count and its 7 ballot words.
__device__ __forceinline__ uint32_t test_rows(const CullFrustum& f, const float4 s[ROWS], uint4 ia, uint4 ib, uint32_t need, bool upper,
	uint32_t count, uint32_t plane_masking, int lane, uint32_t bal[ROWS])
{
	// doCulling, culling_system.cpp:260-308, plane-outer: per sphere and plane exactly :284,291
	//   t = cx*px + cy*py + cz*pz + pd ;  t = t - r (r = -radius) ;  movemask = sign bits
	uint32_t acc[ROWS];
#pragma unroll
	for (int k = 0; k < ROWS; ++k) acc[k] = 0;
#define LB_ROWS(pd, k0, k1)                                                                                                      \
	_Pragma("unroll") for (int k = k0; k < k1; ++k) {                                                                             \
		float t = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(s[k].x, nx), LB_FMUL(s[k].y, ny)), LB_FMUL(s[k].z, nz)), pd);                   \
		t = LB_FSUB(t, -s[k].w); /* :282 f4Splat(-sphere->radius) */                                                              \
		acc[k] |= __float_as_uint(t);                                                                                             \
	}
#define LB_PLANE(p, pd)                                                                                                          \
	if (need & (1u << p)) {                                                                                                       \
		const float nx = f.nx[p], ny = f.ny[p], nz = f.nz[p];                                                                     \
		LB_ROWS(pd, 0, 4)                                                                                                         \
		if (upper) { LB_ROWS(pd, 4, ROWS) }                                                                                       \
	}
	LB_PLANE(0, __uint_as_float(ia.z))
	LB_PLANE(1, __uint_as_float(ia.w))
	LB_PLANE(2, __uint_as_float(ib.x))
	LB_PLANE(3, __uint_as_float(ib.y))
	LB_PLANE(4, __uint_as_float(ib.z))
	LB_PLANE(5, __uint_as_float(ib.w))
#undef LB_PLANE
#undef LB_ROWS
	// A NaN radius: on the reference's SSE path t - (-radius) hands the NaN through with the sign of -radius, and that sign is what
	// movemask reads (+NaN radius: culled by every plane; -NaN radius: passes every plane).  The GPU's subtraction returns the canonical
	// positive NaN instead, so the sign is taken from the radius directly (tests/golden/cull_kat.npz: special_*).  The complement goes
	// through inline PTX: the compiler otherwise rewrites "sign of ~bits" as neg.f32 + a sign test, and neg.f32 of a NaN does not keep the
	// sign.  Only scenes that hold a negative / NaN radius get here (the host tracks them and switches plane masking off with them): one
	// warp-uniform branch per page otherwise.
	if (!plane_masking) {
#pragma unroll
		for (int k = 0; k < ROWS; ++k) {
			const uint32_t rbits = __float_as_uint(s[k].w);
			uint32_t flipped;
			asm volatile("not.b32 %0, %1;" : "=r"(flipped) : "r"(rbits));
			if ((rbits & 0x7fffffffu) > 0x7f800000u && need) acc[k] = flipped & 0x80000000u;
		}
	}
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
	return page_visible;
}

// A warp's claim over its lanes' pages (lanes < n, warp-uniform n <= 32): lane i holds the output key and the visible count of its page.
// prefix = visible ids of the same key in lower lanes, total = those of every lane, leader = the lowest lane of the key (whose one
// atomic reserves the key's range).
struct WarpClaim { uint32_t prefix, total; int leader; };

__device__ __forceinline__ WarpClaim warp_claim(uint32_t key, uint32_t count, uint32_t n, int lane) {
	const uint32_t packed = (key << 16) | count; // count <= 200
	WarpClaim c = {0, 0, 0};
	for (uint32_t l = 0; l < n; ++l) {
		const uint32_t o = __shfl_sync(0xffffffffu, packed, (int)l);
		if ((o >> 16) == key) { c.total += o & 0xffffu; if (l < (uint32_t)lane) c.prefix += o & 0xffffu; }
	}
	const unsigned grp = __match_any_sync(0xffffffffu, key);
	c.leader = __ffs((int)grp) - 1;
	return c;
}

// A warp writes the visible ids of one worked page (entity ids `ep`) to `dst`, compacted: a straight copy for a COPY page, a gather by
// the ballot row `bal_row` for a TEST page.  Returns the word (lane & 7) of the page's 32-byte visibility row.
__device__ __forceinline__ uint32_t write_ids(const int* ep, uint32_t* dst, bool copy, uint32_t count, const uint32_t* bal_row, int lane) {
	const uint32_t lt_mask = (1u << lane) - 1u;
	uint32_t row_word; // lane k < 8 (and its images in the other 8-lane groups): word k of the page's visibility row
	if (copy) {
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
		for (int k = 0; k < ROWS; ++k) bal[k] = bal_row[k];
		int id[ROWS] = {}; // zeroed per page: unassigned elements were otherwise kept live across pages, and spilled
#pragma unroll
		for (int k = 0; k < ROWS; ++k) if ((bal[k] >> lane) & 1u) id[k] = ldg_stream_i32(ep + k * 32 + lane);
		uint32_t prefix = 0;
#pragma unroll
		for (int k = 0; k < ROWS; ++k) {
			if ((bal[k] >> lane) & 1u) dst[prefix + __popc(bal[k] & lt_mask)] = (uint32_t)id[k];
			prefix += __popc(bal[k]);
		}
		row_word = bal_row[lane & 7];
	}
	return row_word;
}

// the all-zero 32-byte mask row of a page that ends without work
__device__ __forceinline__ void zero_row(uint32_t* mask, uint32_t page) {
	uint4* row = reinterpret_cast<uint4*>(mask + (size_t)page * 8);
	row[0] = make_uint4(0u, 0u, 0u, 0u);
	row[1] = make_uint4(0u, 0u, 0u, 0u);
}

} // namespace lbcull
