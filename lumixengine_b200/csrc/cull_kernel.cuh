// cull_pages_kernel — CullingSystemImpl::cullInternal + doCulling (src/renderer/culling_system.cpp:260-369) on the GPU, ONE kernel per cull.
// The culling core (cell tests, plane mask, sphere test, claim, id write) is cull_common.cuh's, shared with cull_views_kernel.
//
// Pages are dealt to the blocks round-robin; per round a block runs:
//   A1  cheap pass, one THREAD per page: coalesced 32-byte descriptors; free pages, the type filter and outside_by_margin.  ~3/4 of the
//       pages of a typical view end here.
//   A2  exact pass on the compacted survivors (dense threads): classify_cell, and for TEST pages relative_offsets and plane_mask; pages
//       with work go to a block-local list in shared memory.
//   B   test, one WARP per listed TEST page: load_rows, test_rows; ballots kept in shared memory.
//   C   claim: one global atomic per (warp, renderable type) reserves the output range of the warp's pages (warp_claim).
//   D   write: write_ids, grouped by type.  The 32-byte visibility row of every worked page goes to the mask (row = page id; classify
//       threads zero the rows of skipped pages) or — exchange mode — as a {page id, row} record straight into every rank's slab over
//       NVLink: only rows that can be non-zero cross the links (SURVEY 8e: the bitmask is the exchanged product).
// One block barrier per round after A1 and A2 each; B, C and D run warp-autonomously, so a warp with cheap pages never waits for one
// with expensive pages.  No per-page global atomics; skipped pages never reach a warp.
// Everything before cudaGridDependencySynchronize() (launch, descriptor reads, classification, the sphere tests of phase B whose
// results sit in shared memory) only READS scene data: when culls are issued back to back with programmatic stream serialization it
// overlaps the tail of the previous cull.
// HBM-bound: 32 B descriptor per page + 16 B per tested sphere + 4 B read + 4 B write per visible id + 32 B mask row per page.
#pragma once

#include "cull_common.cuh"
#include "culling_internal.h" // counter and slab layout
#include "lb200_internal.h"
#include "lb200_math.cuh"

namespace lbcull {

using namespace lb;

constexpr int CULL_THREADS = 256;       // 4 blocks/SM at 64 registers; pages per block per round <= one classify thread each
constexpr int CULL_WARPS = CULL_THREADS / 32;
constexpr int MAX_CHUNK = CULL_THREADS;

struct CullParams {
	CullFrustum f;
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

struct WorkItem { // 32 B
	uint32_t page;
	uint32_t meta; // count | type << 8 | cls << 16 | planes needed << 24
	float rd[6];   // plane offsets relative to the cell origin (TEST pages)
};
static_assert(sizeof(WorkItem) == 32, "");

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
					const PageInfo pi = load_page(desc, page);
					if (pi.count != 0) {
						if (P.type_filter != 0xffu && pi.type != P.type_filter) atomicAdd(&s_stats[ST_PAGES_FILTERED], 1u);
						else {
							const bool outside = !pi.is_big && outside_by_margin(P.f, cell_lo(pi.org));
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
			const PageInfo pi = load_page(desc, page); // read by the cheap pass a moment ago: an L1 hit
			const uint32_t count = pi.count;
			const uint32_t type = pi.type;
			int cls = classify_cell(P.f, pi, s_stats);
			uint32_t need = 0x3fu;
			float rd[6];
#pragma unroll
			for (int p = 0; p < 6; ++p) rd[p] = 0.0f;
			if (cls == CLS_TEST) {
				relative_offsets(P.f, pi.org, rd);
				if (P.plane_masking) {
					need = plane_mask(P.f, pi.org, rd);
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
				load_rows(spheres, ia.x, count, upper, lane, s);
				uint32_t bal[ROWS];
				const uint32_t page_visible = test_rows(P.f, s, ia, ib, need, upper, count, P.plane_masking, lane, bal);
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
		if (mask_out && (uint32_t)tid < P.chunk && s_zpage[tid] != 0xffffffffu) zero_row(mask_out, s_zpage[tid]);
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
			const WarpClaim c = warp_claim(my_type, my_count, n_mine, lane);
			uint32_t base = 0;
			if (has && lane == c.leader && c.total) base = atomicAdd(&counters[my_type], c.total);
			// exchange mode: the warp's pages also take n_mine consecutive record slots of this rank's slab
			if (P.n_ranks && lane == 31 && n_mine) rec_base = atomicAdd(&counters[CNT_N_REC], n_mine);
			base = __shfl_sync(0xffffffffu, base, c.leader);
			rec_base = __shfl_sync(0xffffffffu, rec_base, 31);
			if (has) s_off[iwi] = P.type_base[my_type] + base + c.prefix; // where the page's ids go in out_ids
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
				const int* ep = entities + (size_t)page * LB200_PAGE_SLOTS;
				const uint32_t row_word = write_ids(ep, out_ids + s_off[iw], ((meta >> 16) & 3u) == CLS_COPY, count, s_bal[iw], lane);
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
