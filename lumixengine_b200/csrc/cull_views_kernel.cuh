// cull_views_kernel — several views of one scene (a frame's main camera and shadow cascades) culled in ONE pass over the pages.
//
// The phases are cull_pages_kernel's (cull_kernel.cuh) over the same culling core (cull_common.cuh), with each page's work split into
// (page, view) items:
//   A1  one THREAD per page: the 32-byte descriptor is read once; the type filter and outside_by_margin run per view.  A page is a
//       candidate if any view keeps it; per-view pages_filtered / pages_outside count as a lone cull of that view counts them.
//   A2  one THREAD per candidate page: classify_cell, relative_offsets and plane_mask per view that kept the page.  Every view that works
//       the page gets an item; the TEST items of one page take consecutive slots, so that phase B finds them together.
//   B   one WARP per page that some view must TEST: load_rows once, then test_rows for each TEST view over the rows held in registers;
//       ballots go to shared memory per item.
//   C   claim: one global atomic per (warp, view, renderable type) reserves the output range in that view's id buffer.
//   D   write: per item, write_ids into that view's buffer and the page's 32-byte row into that view's mask.  Pages that end without work
//       for a view get a zero row in that view's mask.
// Shared memory per (page, view) item bounds a round: chunk <= MAX_ITEMS / n_views pages (viewsChunkBound).  B deals pages to the warps
// and C / D deal items, so a block barrier separates B from C (the single cull's warps run B, C and D without one).
// Like the single cull, everything before cudaGridDependencySynchronize() only READS scene data, so the kernel may be launched with
// programmatic stream serialization behind another cull.
// Bytes: 32 B descriptor per page + 16 B per sphere of a page some view tests (each page's rows once) + per view 4 B read + 4 B write per
// visible id and a 32 B mask row per page.
#pragma once

#include "cull_common.cuh"
#include "culling_internal.h" // counter layout, statistics
#include "lb200_internal.h"
#include "lb200_math.cuh"

namespace lbviews {

using namespace lb;
using namespace lbcull;

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
	CullFrustum f[MAX_VIEWS];
	uint32_t type_filter[MAX_VIEWS]; // 0xff = all
	uint32_t n_views;
	uint32_t n_pages;
	uint32_t chunk;         // pages per block per round, <= viewsChunkBound(n_views)
	uint32_t plane_masking; // 1 unless some sphere has a negative / NaN radius
	uint32_t id_stride;     // words between two views' id buffers
	uint32_t mask_stride;   // words between two views' masks
	uint32_t type_base[256];
};

struct ViewItem { // 32 B
	uint32_t page;
	uint32_t meta; // count | type << 8 | cls << 16 | view << 18 | planes needed << 24
	float rd[6];   // the view's plane offsets relative to the cell origin (TEST items)
};
static_assert(sizeof(ViewItem) == 32, "");

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
					const PageInfo pi = load_page(desc, page);
					if (pi.count != 0) {
						const D3 lo = cell_lo(pi.org);
						#pragma unroll 1
						for (uint32_t v = 0; v < n_views; ++v) {
							if (P.type_filter[v] != 0xffu && pi.type != P.type_filter[v]) { atomicAdd(&s_stats[v][lbcull::ST_PAGES_FILTERED], 1u); continue; }
							const bool outside = !pi.is_big && outside_by_margin(P.f[v], lo);
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
			const PageInfo pi = load_page(desc, page); // read by the cheap pass a moment ago: an L1 hit
			const uint32_t count = pi.count;
			const uint32_t type = pi.type;
			const uint32_t keep = s_keep[t0];
			// pass 1: the class per view and the statistics
			uint32_t cls_of = 0;   // 2 bits per view
			uint64_t need_of = 0;  // 6 bits per view
			uint32_t n_t = 0, n_c = 0, zero = 0;
			#pragma unroll 1
			for (uint32_t v = 0; v < n_views; ++v) {
				if (!((keep >> v) & 1u)) continue;
				const int cls = classify_cell(P.f[v], pi, s_stats[v]);
				if (cls == CLS_SKIP) { zero |= 1u << v; continue; }
				cls_of |= (uint32_t)cls << (2 * v);
			}
			// pass 2: the plane mask of every TEST view (a loop of its own: the planes of the classification are not kept live across it)
			#pragma unroll 1
			for (uint32_t v = 0; v < n_views; ++v) {
				uint32_t cls = (cls_of >> (2 * v)) & 3u;
				if (cls == CLS_SKIP) continue;
				uint32_t need = 0x3fu;
				if (cls == CLS_TEST && P.plane_masking) {
					float rd[6];
					relative_offsets(P.f[v], pi.org, rd);
					need = plane_mask(P.f[v], pi.org, rd);
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
					relative_offsets(P.f[v], pi.org, rd);
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
#define LB_ITEM(w) ((w) < n_test ? (w) : (uint32_t)MAX_ITEMS - 1u - ((w) - n_test))

		// ---------------- B. sphere tests: one warp per page some view tests, rows loaded once for all of its TEST items ----------------
		for (uint32_t jt = warp; jt < s_ntpage; jt += VIEW_WARPS) {
			const uint32_t tp = s_tpage[jt];
			const uint32_t first = tp & 0xffffu, n_items = tp >> 16;
			const uint32_t page = s_item[first].page;
			const uint32_t count = s_item[first].meta & 0xffu;
			const bool upper = count > 128u;
			float4 s[ROWS];
			load_rows(spheres, page, count, upper, lane, s);
			#pragma unroll 1
			for (uint32_t iw = first; iw < first + n_items; ++iw) {
				const uint4 ia = *reinterpret_cast<const uint4*>(&s_item[iw]);
				const uint4 ib = *(reinterpret_cast<const uint4*>(&s_item[iw]) + 1);
				const uint32_t need = ia.y >> 24;
				const uint32_t v = (ia.y >> 18) & 7u;
				uint32_t bal[ROWS];
				const uint32_t page_visible = test_rows(P.f[v], s, ia, ib, need, upper, count, P.plane_masking, lane, bal);
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
			for (uint32_t z = s_zero[tid]; z; z &= z - 1u) zero_row(mask_out + (size_t)(__ffs((int)z) - 1) * P.mask_stride, page);
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
				const uint32_t iwi = has ? LB_ITEM(warp + (b0 + (uint32_t)lane) * VIEW_WARPS) : 0u;
				const uint32_t meta = has ? s_item[iwi].meta : 0u;
				const uint32_t my_key = has ? ((meta >> 8) & 0xffu) | (((meta >> 18) & 7u) << 8) : 0xffffu; // type | view << 8
				const uint32_t my_count = has ? s_off[iwi] : 0u;
				const WarpClaim c = warp_claim(my_key, my_count, n_batch, lane);
				uint32_t base = 0;
				if (has && lane == c.leader && c.total) base = atomicAdd(&counters[(my_key >> 8) * COUNTER_WORDS + (my_key & 0xffu)], c.total);
				base = __shfl_sync(0xffffffffu, base, c.leader);
				if (has) s_off[iwi] = P.type_base[my_key & 0xffu] + base + c.prefix; // where the item's ids go in its view's buffer
			}
		}
		__syncwarp();

		// ---------------- D. write: gather the visible ids of each item into its view's buffer, and its mask row ----------------
		for (uint32_t w = warp; w < n_work; w += VIEW_WARPS) {
			const uint32_t iw = LB_ITEM(w);
			const uint32_t page = s_item[iw].page;
			const uint32_t meta = s_item[iw].meta;
			const uint32_t count = meta & 0xffu;
			const uint32_t v = (meta >> 18) & 7u;
			const int* ep = entities + (size_t)page * LB200_PAGE_SLOTS;
			const uint32_t row_word = write_ids(ep, out_ids + (size_t)v * P.id_stride + s_off[iw], ((meta >> 16) & 3u) == CLS_COPY, count, s_bal[iw], lane);
			if (lane < 8) mask_out[(size_t)v * P.mask_stride + (size_t)page * 8 + lane] = row_word;
		}
#undef LB_ITEM
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
