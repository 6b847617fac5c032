// =====================================================================================================================================
// Device-side re-binning (SURVEY.md 8f N3): CullingSystem::set (src/renderer/culling_system.cpp:222-240) for a batch of DISTINCT entities
// whose new world spheres already lie in HBM (the sphere refresh behind a hierarchy propagate, render_module.cpp:1544-1554), without the
// host hash map in the loop:
//   1. classify   one thread per mover: new cell = IVec3(pos * (1 / 300.f)) (culling_system.cpp:25-31), is_big = radius > 300; same cell
//                 and same big-ness -> the sphere is overwritten in its slot (:228-233); otherwise the mover joins the changer list;
//   2. remove     changers leave their pages (:160-187): the slot is tombstoned, the page marked dirty; one warp per dirty page then
//                 compacts the survivors (the reference swaps the last sphere into the hole: same set, slots differ), pages that run empty
//                 go to the free list (:169-176);
//   3. add        changers sorted by target chain (cell, type, is_big) with the device radix sort; the head of every run fills the chain's
//                 open page (the reference's map head, :110-127) and opens new pages from the free list as it overflows (:143-156).
// Results of a cull afterwards are the reference's: every entity sits in the chain of its cell with the sphere relative to the cell
// origin computed exactly as culling_system.cpp:100 does, pages hold <= 200 spheres, empty pages are skipped.  Which slot / which page of
// its chain an entity occupies differs from the sequential host order (as it does between two edit orders on the host); the per-page
// statistics of a cull can therefore differ from a host-side replay, visible sets cannot.
// Device adds and removes (CullingSystem::add / remove, culling_system.cpp:131-187, for batches whose data lies in HBM) use the same steps:
//   add      one thread per new entity claims its id in entity -> slot (a refused batch releases its claims and changes nothing else) and
//            builds its chain key; after one read-back the keys go through step 3 exactly as re-binned changers do;
//   remove   one thread per id takes the entity's slot out of entity -> slot and tombstones it; step 2's compaction follows.
// Both keep per-type count deltas, which the batch's last read-back applies to the host's type counts (the cull's output layout).
// The chain hash map counts its keys and is rehashed on the device into a larger table before a batch could fill it past half.
// The pull-back of the host mirror (syncHostFromDevice) lives here too: it undoes what these kernels leave ahead of the host.
// The device keys a chain by 18 bits per cell axis, so it holds only cells in [-131 072, 131 071] (about +-39 321 km).  A batch that
// computes a cell outside that range, and any batch while the host mirror holds such a chain, is applied by the host bookkeeping instead:
// the device never holds two chains whose packed keys alias.
// =====================================================================================================================================
#include "culling_internal.h"

#include <algorithm>

using namespace lb;
using namespace lbcull;

namespace {

// counter words: [0, RB_WORDS) the state every batch reads back (RB_OVERFLOW holds OVERFLOW_PAGES | OVERFLOW_HASH | OVERFLOW_RANGE), then the words of an
// add batch's first read-back, then RB_TYPE_DELTA: 256 per-type count deltas of an add / remove batch (two's complement).  The batch
// words are zeroed by the batch that uses them.
enum { RB_HIGH_WATER = 0, RB_N_FREE, RB_N_CHANGERS, RB_N_DIRTY, RB_OVERFLOW, RB_BAD_RADIUS, RB_N_KEYS, RB_NEW_PAGES, RB_WORDS,
	RB_REFUSED = RB_WORDS, RB_MAX_ID, RB_ADD_WORDS = RB_WORDS + 8 };
constexpr uint32_t RB_TYPE_DELTA = RB_ADD_WORDS, RB_ALL_WORDS = RB_ADD_WORDS + 256;
// OVERFLOW_RANGE: a batch computed a cell the packed key cannot hold; it is applied on the host, and the next batch rebuilds the counters
constexpr uint32_t OVERFLOW_PAGES = 1u, OVERFLOW_HASH = 2u, OVERFLOW_RANGE = 4u;
constexpr unsigned long long HASH_EMPTY = ~0ull;
constexpr uint32_t NO_OPEN_PAGE = 0xffffffffu;
constexpr uint32_t CLAIMED = 0xfffffffeu; // entity -> slot of an id an add batch has claimed and not placed yet (no page reaches it)

__host__ __device__ __forceinline__ unsigned long long packCellKey(int x, int y, int z, uint32_t type, uint32_t is_big) {
	// 18 bits per axis (+-131 071 cells of 300 m), 8 bits type, 1 bit is_big
	return ((unsigned long long)((uint32_t)x & 0x3ffffu)) | ((unsigned long long)((uint32_t)y & 0x3ffffu) << 18) | ((unsigned long long)((uint32_t)z & 0x3ffffu) << 36)
		| ((unsigned long long)(type & 0xffu) << 54) | ((unsigned long long)(is_big & 1u) << 62);
}
// the cells packCellKey keeps apart: [-131 072, 131 071] on every axis
__host__ __device__ __forceinline__ bool cellInKeyRange(int x, int y, int z) {
	return (uint32_t)(x + 0x20000) < 0x40000u && (uint32_t)(y + 0x20000) < 0x40000u && (uint32_t)(z + 0x20000) < 0x40000u;
}
__host__ __device__ __forceinline__ uint32_t hashCellKey(unsigned long long k) {
	k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
	return (uint32_t)k;
}

__device__ __forceinline__ uint32_t hashFind(const unsigned long long* keys, const uint32_t* vals, uint32_t cap, unsigned long long key, uint32_t* slot_out) {
	uint32_t i = hashCellKey(key) & (cap - 1);
	for (uint32_t probe = 0; probe < cap; ++probe) {
		const unsigned long long k = keys[i];
		if (k == key) { *slot_out = i; return vals[i]; }
		if (k == HASH_EMPTY) { *slot_out = i; return NO_OPEN_PAGE; }
		i = (i + 1) & (cap - 1);
	}
	*slot_out = 0; // a full table without the key: the key has no open page
	return NO_OPEN_PAGE;
}

// find or claim `key`'s slot (linear probing, at most `cap` probes); false: the table is full
__device__ __forceinline__ bool hashClaim(unsigned long long* keys, uint32_t cap, unsigned long long key, uint32_t* slot_out, bool* inserted) {
	uint32_t i = hashCellKey(key) & (cap - 1);
	for (uint32_t probe = 0; probe < cap; ++probe) {
		const unsigned long long prev = atomicCAS(&keys[i], HASH_EMPTY, key);
		if (prev == HASH_EMPTY || prev == key) { *slot_out = i; *inserted = prev == HASH_EMPTY; return true; }
		i = (i + 1) & (cap - 1);
	}
	return false;
}

// chain of an entity: cell = IVec3(pos * (1 / 300.f)) (culling_system.cpp:25-31), is_big = radius > 300
__device__ __forceinline__ unsigned long long chainKey(const double* __restrict__ pos3, uint32_t i, uint32_t type, float radius, int* ix_out) {
	const double inv = (double)(1 / LB200_CELL_SIZE);
	const int ix = (int)__dmul_rn(pos3[3 * (size_t)i], inv), iy = (int)__dmul_rn(pos3[3 * (size_t)i + 1], inv), iz = (int)__dmul_rn(pos3[3 * (size_t)i + 2], inv);
	*ix_out = ix;
	return packCellKey(ix, iy, iz, type, radius > LB200_CELL_SIZE ? 1u : 0u);
}

// 1. classify + in-place overwrite
__global__ void __launch_bounds__(256) rebin_classify_kernel(uint32_t n, const int32_t* __restrict__ ents, const double* __restrict__ pos3, const float* __restrict__ radius,
	const uint32_t* __restrict__ entity_to_slot, uint32_t entity_cap, const lb200_page_desc* __restrict__ desc, const int4* __restrict__ page_cell,
	float4* __restrict__ spheres, uint32_t* __restrict__ changers, uint32_t* __restrict__ counters)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	bool changer = false;
	if (i < n) {
		const int32_t e = ents ? ents[i] : (int32_t)i;
		const uint32_t slot = (uint32_t)e < entity_cap ? entity_to_slot[e] : NO_SLOT;
		if (slot != NO_SLOT) {
			const uint32_t page = slot / PAGE_SLOTS;
			const double px = pos3[3 * (size_t)i], py = pos3[3 * (size_t)i + 1], pz = pos3[3 * (size_t)i + 2];
			const float r = radius[i];
			const double inv = (double)(1 / LB200_CELL_SIZE); // culling_system.cpp:25-31: IVec3(pos * (1 / cell_size)), DVec3 * float
			const int ix = (int)__dmul_rn(px, inv), iy = (int)__dmul_rn(py, inv), iz = (int)__dmul_rn(pz, inv);
			if (!cellInKeyRange(ix, iy, iz)) atomicOr(&counters[RB_OVERFLOW], OVERFLOW_RANGE); // the batch goes to the host after the read-back
			const int4 c = page_cell[page];
			const bool was_big = ((uint32_t)c.w >> 8) != 0, is_big = r > LB200_CELL_SIZE;
			if (was_big == is_big && ix == c.x && iy == c.y && iz == c.z) { // :228-233
				const lb200_page_desc d = desc[page];
				const float old_r = spheres[slot].w;
				spheres[slot] = make_float4((float)__dsub_rn(px, d.origin[0]), (float)__dsub_rn(py, d.origin[1]), (float)__dsub_rn(pz, d.origin[2]), r);
				const int delta = (!(r >= 0.0f) ? 1 : 0) - (!(old_r >= 0.0f) ? 1 : 0);
				if (delta) atomicAdd(&counters[RB_BAD_RADIUS], (uint32_t)delta);
			}
			else changer = true;
		}
	}
	const uint32_t bal = __ballot_sync(0xffffffffu, changer);
	if (bal) {
		const uint32_t lane = threadIdx.x & 31u;
		uint32_t base = 0;
		if (lane == 0) base = atomicAdd(&counters[RB_N_CHANGERS], (uint32_t)__popc(bal));
		base = __shfl_sync(0xffffffffu, base, 0);
		if (changer) changers[base + __popc(bal & ((1u << lane) - 1u))] = i;
	}
}

// 2a. changers leave their slots; the sort keys of step 3 are built on the way
__global__ void __launch_bounds__(256) rebin_remove_kernel(const uint32_t* __restrict__ changers, const int32_t* __restrict__ ents,
	const double* __restrict__ pos3, const float* __restrict__ radius, uint32_t* __restrict__ entity_to_slot, const int4* __restrict__ page_cell, float4* __restrict__ spheres,
	int* __restrict__ entities, uint32_t* __restrict__ page_dirty, uint32_t* __restrict__ dirty_pages, uint32_t* wcounters, uint64_t* __restrict__ keys, uint64_t* __restrict__ vals)
{
	const uint32_t n = wcounters[RB_N_CHANGERS];
	for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
		const uint32_t i = changers[k];
		const int32_t e = ents ? ents[i] : (int32_t)i;
		const uint32_t slot = entity_to_slot[e];
		const uint32_t page = slot / PAGE_SLOTS;
		const float old_r = spheres[slot].w;
		if (!(old_r >= 0.0f)) atomicAdd(&wcounters[RB_BAD_RADIUS], 0xffffffffu);
		entities[slot] = -1 - e; // tombstone
		if (atomicExch(&page_dirty[page], 1u) == 0u) dirty_pages[atomicAdd(&wcounters[RB_N_DIRTY], 1u)] = page;
		int ix;
		const uint32_t type = (uint32_t)page_cell[page].w & 0xffu; // set() keeps the renderable type (:236-239)
		keys[k] = chainKey(pos3, i, type, radius[i], &ix);
		vals[k] = ((uint64_t)(uint32_t)ix) | ((uint64_t)i << 32); // mover index; the cell indices are recomputed by the add kernel
		if (!(radius[i] >= 0.0f)) atomicAdd(&wcounters[RB_BAD_RADIUS], 1u);
	}
}

// 2b. one warp per dirty page: survivors move up, the count drops, empty pages are freed
__global__ void __launch_bounds__(256) rebin_compact_kernel(const uint32_t* __restrict__ dirty_pages, uint32_t* __restrict__ counters, lb200_page_desc* __restrict__ desc,
	const int4* __restrict__ page_cell, float4* __restrict__ spheres, int* __restrict__ entities, uint32_t* __restrict__ entity_to_slot, uint32_t* __restrict__ page_dirty,
	uint32_t* __restrict__ free_pages, unsigned long long* __restrict__ hash_keys, uint32_t* __restrict__ hash_vals, uint32_t hash_cap)
{
	const uint32_t n = counters[RB_N_DIRTY];
	const uint32_t lane = threadIdx.x & 31u;
	for (uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5; w < n; w += (gridDim.x * blockDim.x) >> 5) {
		const uint32_t page = dirty_pages[w];
		const uint32_t count = desc[page].count;
		const size_t base = (size_t)page * PAGE_SLOTS;
		float4 sp[7]; int en[7]; uint32_t bal[7];
#pragma unroll
		for (int k = 0; k < 7; ++k) {
			const uint32_t s = k * 32 + lane;
			const bool in = s < count;
			if (in) { sp[k] = spheres[base + s]; en[k] = entities[base + s]; }
			bal[k] = __ballot_sync(0xffffffffu, in && en[k] >= 0);
		}
		__syncwarp();
		uint32_t at = 0;
#pragma unroll
		for (int k = 0; k < 7; ++k) {
			if ((bal[k] >> lane) & 1u) {
				const uint32_t dst = at + __popc(bal[k] & ((1u << lane) - 1u));
				spheres[base + dst] = sp[k];
				entities[base + dst] = en[k];
				entity_to_slot[en[k]] = (uint32_t)(base + dst);
			}
			at += __popc(bal[k]);
		}
		if (lane == 0) {
			desc[page].count = at;
			page_dirty[page] = 0;
			if (at == 0) { // culling_system.cpp:169-176: the page leaves its chain; if it was the chain's open page the chain has none now
				free_pages[atomicAdd(&counters[RB_N_FREE], 1u)] = page;
				const int4 c = page_cell[page];
				uint32_t slot;
				const uint32_t open = hashFind(hash_keys, hash_vals, hash_cap, packCellKey(c.x, c.y, c.z, (uint32_t)c.w & 0xffu, (uint32_t)c.w >> 8), &slot);
				if (open == page) hash_vals[slot] = NO_OPEN_PAGE;
			}
		}
	}
}

// Device add, before step 3: every id is claimed (atomicCAS NO_SLOT -> CLAIMED, so an added id or one listed twice fails), ids outside
// [0, max_entity] and the reserved type are refused, the batch's types and its largest id are counted, and every entity's chain key is
// built for step 3.  Nothing but this batch's claims and its zeroed batch words is written: rebin_add_release_kernel undoes a refusal.
__global__ void __launch_bounds__(256) rebin_add_claim_kernel(uint32_t n, const int32_t* __restrict__ ents, const uint8_t* __restrict__ types,
	const double* __restrict__ pos3, const float* __restrict__ radius, uint32_t max_entity, uint32_t* __restrict__ entity_to_slot, uint32_t* __restrict__ counters,
	uint64_t* __restrict__ keys, uint64_t* __restrict__ vals)
{
	__shared__ uint32_t s_types[256];
	__shared__ uint32_t s_max, s_refused;
	s_types[threadIdx.x] = 0;
	if (threadIdx.x == 0) { s_max = 0; s_refused = 0; }
	__syncthreads();
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) {
		const int32_t e = ents ? ents[i] : (int32_t)i;
		const uint32_t type = types[i];
		bool ok = e >= 0 && (uint32_t)e <= max_entity && type != LB200_TYPE_ALL;
		if (ok) ok = atomicCAS(&entity_to_slot[e], NO_SLOT, CLAIMED) == NO_SLOT;
		if (ok) { atomicAdd(&s_types[type], 1u); atomicMax(&s_max, (uint32_t)e); }
		else atomicAdd(&s_refused, 1u);
		int ix;
		keys[i] = chainKey(pos3, i, type, radius[i], &ix);
		vals[i] = ((uint64_t)(uint32_t)ix) | ((uint64_t)i << 32);
		const double inv = (double)(1 / LB200_CELL_SIZE);
		if (!cellInKeyRange(ix, (int)__dmul_rn(pos3[3 * (size_t)i + 1], inv), (int)__dmul_rn(pos3[3 * (size_t)i + 2], inv)))
			atomicOr(&counters[RB_OVERFLOW], OVERFLOW_RANGE); // the batch releases its claims and goes to the host
	}
	if (i == 0) counters[RB_N_CHANGERS] = n; // step 3 places every entity of an accepted batch
	__syncthreads();
	if (s_types[threadIdx.x]) atomicAdd(&counters[RB_TYPE_DELTA + threadIdx.x], s_types[threadIdx.x]);
	if (threadIdx.x == 0) {
		if (s_refused) atomicAdd(&counters[RB_REFUSED], s_refused);
		atomicMax(&counters[RB_MAX_ID], s_max);
	}
}

// a refused add batch: the ids it claimed go back to NO_SLOT
__global__ void __launch_bounds__(256) rebin_add_release_kernel(uint32_t n, const int32_t* __restrict__ ents, uint32_t max_entity, uint32_t* __restrict__ entity_to_slot) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const int32_t e = ents ? ents[i] : (int32_t)i;
	if (e >= 0 && (uint32_t)e <= max_entity && entity_to_slot[e] == CLAIMED) entity_to_slot[e] = NO_SLOT;
}

// Device remove: each id takes its slot out of entity -> slot (atomicExch, so an id listed twice finds NO_SLOT the second time; ids that
// are not added are skipped, culling_system.cpp:160-163) and tombstones it as step 2a does; rebin_compact_kernel then compacts the pages.
__global__ void __launch_bounds__(256) rebin_remove_ids_kernel(uint32_t n, const int32_t* __restrict__ ents, uint32_t* __restrict__ entity_to_slot, uint32_t entity_cap,
	const int4* __restrict__ page_cell, const float4* __restrict__ spheres, int* __restrict__ entities, uint32_t* __restrict__ page_dirty, uint32_t* __restrict__ dirty_pages,
	uint32_t* __restrict__ counters)
{
	__shared__ uint32_t s_types[256];
	__shared__ uint32_t s_bad;
	s_types[threadIdx.x] = 0;
	if (threadIdx.x == 0) s_bad = 0;
	__syncthreads();
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i < n) {
		const int32_t e = ents[i];
		const uint32_t slot = e >= 0 && (uint32_t)e < entity_cap ? atomicExch(&entity_to_slot[e], NO_SLOT) : NO_SLOT;
		if (slot != NO_SLOT) {
			const uint32_t page = slot / PAGE_SLOTS;
			atomicAdd(&s_types[(uint32_t)page_cell[page].w & 0xffu], 1u);
			if (!(spheres[slot].w >= 0.0f)) atomicAdd(&s_bad, 1u);
			entities[slot] = -1 - e; // tombstone
			if (atomicExch(&page_dirty[page], 1u) == 0u) dirty_pages[atomicAdd(&counters[RB_N_DIRTY], 1u)] = page;
		}
	}
	__syncthreads();
	if (s_types[threadIdx.x]) atomicSub(&counters[RB_TYPE_DELTA + threadIdx.x], s_types[threadIdx.x]);
	if (threadIdx.x == 0 && s_bad) atomicSub(&counters[RB_BAD_RADIUS], s_bad);
}

// the chain hash map moved into a larger, emptied table; entries without an open page are dropped (a missing key reads the same)
__global__ void __launch_bounds__(256) rebin_rehash_kernel(const unsigned long long* __restrict__ old_keys, const uint32_t* __restrict__ old_vals, uint32_t old_cap,
	unsigned long long* __restrict__ keys, uint32_t* __restrict__ vals, uint32_t cap, uint32_t* __restrict__ counters)
{
	for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < old_cap; j += gridDim.x * blockDim.x) {
		const unsigned long long k = old_keys[j];
		const uint32_t v = old_vals[j];
		if (k == HASH_EMPTY || v == NO_OPEN_PAGE) continue;
		uint32_t slot; bool inserted;
		if (!hashClaim(keys, cap, k, &slot, &inserted)) { atomicOr(&counters[RB_OVERFLOW], OVERFLOW_HASH); continue; }
		vals[slot] = v;
		atomicAdd(&counters[RB_N_KEYS], 1u);
	}
}

// 3a. adds, sorted by chain: the head of every run of equal keys plans the run — how many go into the chain's open page, how many new
// pages the rest needs (taken from the free list / the high-water mark), the pages' descriptors and final counts, the chain's new open
// page.  Work per run is proportional to its PAGES, not its entities: a crowd that moves into one cell is placed in parallel by 3b.
struct RunPlan { uint32_t open_page, open_count, free_in_open, new_base; }; // stored at the run's first index
__global__ void __launch_bounds__(128) rebin_plan_kernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ vals, uint32_t* counters,
	const double* __restrict__ pos3, lb200_page_desc* __restrict__ desc, int4* __restrict__ page_cell, const uint32_t* __restrict__ free_pages,
	unsigned long long* __restrict__ hash_keys, uint32_t* __restrict__ hash_vals, uint32_t hash_cap, uint32_t page_cap, RunPlan* __restrict__ plans,
	uint32_t* __restrict__ new_pages, uint32_t* __restrict__ n_new_pages)
{
	const uint32_t n = counters[RB_N_CHANGERS];
	for (uint32_t k = blockIdx.x * blockDim.x + threadIdx.x; k < n; k += gridDim.x * blockDim.x) {
		const uint64_t key = keys[k];
		if (k != 0 && keys[k - 1] == key) continue; // not the head of its run
		uint32_t lo = k, hi = n; // end of the run: first index whose key differs (the keys are sorted)
		while (hi - lo > 1) { const uint32_t mid = lo + (hi - lo) / 2; if (keys[mid] == key) lo = mid; else hi = mid; }
		const uint32_t run = hi - k;
		// find or claim the key's hash slot (runs have distinct keys: no two threads insert the same one); the host keeps the table at most
		// half full before a batch, so a full one is an error, not a wait
		uint32_t hslot = 0;
		bool inserted = false;
		uint32_t page = NO_OPEN_PAGE;
		const bool have_slot = hashClaim(hash_keys, hash_cap, key, &hslot, &inserted);
		if (!have_slot) atomicOr(&counters[RB_OVERFLOW], OVERFLOW_HASH);
		else if (inserted) { hash_vals[hslot] = NO_OPEN_PAGE; atomicAdd(&counters[RB_N_KEYS], 1u); }
		else page = hash_vals[hslot];
		RunPlan plan;
		plan.open_page = page;
		plan.open_count = page != NO_OPEN_PAGE ? desc[page].count : PAGE_SLOTS;
		plan.free_in_open = PAGE_SLOTS - plan.open_count;
		const uint32_t into_open = run < plan.free_in_open ? run : plan.free_in_open;
		const uint32_t rest = run - into_open;
		const uint32_t m = (rest + PAGE_SLOTS - 1) / PAGE_SLOTS; // culling_system.cpp:110-127 / :143-156: new pages in front of the chain
		plan.new_base = m ? atomicAdd(n_new_pages, m) : 0u;
		if (page != NO_OPEN_PAGE) desc[page].count = plan.open_count + into_open;
		if (m) {
			const uint32_t i0 = (uint32_t)(vals[k] >> 32); // any member of the run gives the cell
			const double inv = (double)(1 / LB200_CELL_SIZE);
			const int ix = (int)__dmul_rn(pos3[3 * (size_t)i0], inv), iy = (int)__dmul_rn(pos3[3 * (size_t)i0 + 1], inv), iz = (int)__dmul_rn(pos3[3 * (size_t)i0 + 2], inv);
			const uint32_t type = (uint32_t)(key >> 54) & 0xffu, is_big = (uint32_t)(key >> 62) & 1u;
			lb200_page_desc d;
			d.origin[0] = __dmul_rn((double)LB200_CELL_SIZE, (double)ix); // :146
			d.origin[1] = __dmul_rn((double)LB200_CELL_SIZE, (double)iy);
			d.origin[2] = __dmul_rn((double)LB200_CELL_SIZE, (double)iz);
			d.type = (uint8_t)type; d.is_big = (uint8_t)is_big; d.pad = 0;
			for (uint32_t q = 0; q < m; ++q) {
				uint32_t np;
				const uint32_t nf = atomicSub(&counters[RB_N_FREE], 1u);
				if (nf != 0u && nf < 0x80000000u) np = free_pages[nf - 1];
				else { atomicAdd(&counters[RB_N_FREE], 1u); np = atomicAdd(&counters[RB_HIGH_WATER], 1u); }
				if (np >= page_cap) { atomicOr(&counters[RB_OVERFLOW], OVERFLOW_PAGES); np = 0; }
				d.count = q + 1 < m ? PAGE_SLOTS : rest - q * PAGE_SLOTS;
				desc[np] = d;
				page_cell[np] = make_int4(ix, iy, iz, (int)(type | (is_big << 8)));
				new_pages[plan.new_base + q] = np;
				page = np;
			}
		}
		plans[k] = plan;
		if (have_slot && page != NO_OPEN_PAGE) hash_vals[hslot] = page; // the last page opened (or the old open page) takes the chain's next adds
	}
}

// 3b. every changer finds its run (binary search on the sorted keys), its rank in it, and from the run's plan its page and slot.
// bad_radius: the counter new spheres with radius < 0 or NaN are counted into (device adds; re-binned changers were counted by step 2a)
__global__ void __launch_bounds__(256) rebin_place_kernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ vals, const uint32_t* counters,
	const int32_t* __restrict__ ents, const double* __restrict__ pos3, const float* __restrict__ radius, uint32_t* __restrict__ entity_to_slot,
	const lb200_page_desc* __restrict__ desc, float4* __restrict__ spheres, int* __restrict__ entities, const RunPlan* __restrict__ plans, const uint32_t* __restrict__ new_pages,
	uint32_t* bad_radius)
{
	const uint32_t n = counters[RB_N_CHANGERS];
	for (uint32_t j = blockIdx.x * blockDim.x + threadIdx.x; j < n; j += gridDim.x * blockDim.x) {
		const uint64_t key = keys[j];
		uint32_t lo = 0, hi = j; // first index of the run: smallest index with this key
		while (lo < hi) { const uint32_t mid = lo + (hi - lo) / 2; if (keys[mid] < key) lo = mid + 1; else hi = mid; }
		const RunPlan plan = plans[lo];
		const uint32_t r = j - lo;
		uint32_t page, idx;
		if (r < plan.free_in_open) { page = plan.open_page; idx = plan.open_count + r; }
		else { const uint32_t q = r - plan.free_in_open; page = new_pages[plan.new_base + q / PAGE_SLOTS]; idx = q % PAGE_SLOTS; }
		const uint32_t i = (uint32_t)(vals[j] >> 32);
		const int32_t e = ents ? ents[i] : (int32_t)i;
		const lb200_page_desc d = desc[page];
		const uint32_t slot = page * PAGE_SLOTS + idx;
		spheres[slot] = make_float4((float)__dsub_rn(pos3[3 * (size_t)i], d.origin[0]), (float)__dsub_rn(pos3[3 * (size_t)i + 1], d.origin[1]),
			(float)__dsub_rn(pos3[3 * (size_t)i + 2], d.origin[2]), radius[i]); // :100
		entities[slot] = e;
		entity_to_slot[e] = slot;
		if (bad_radius && !(radius[i] >= 0.0f)) atomicAdd(bad_radius, 1u);
	}
}

// ensureRebinState's answer when the host mirror holds a chain whose cell packCellKey cannot hold: the batch goes to the host bookkeeping
constexpr int REBIN_ON_HOST = 1;

// device-side tables for the re-binning, (re)built from the host mirror whenever it was edited since; REBIN_ON_HOST instead of a build
// from a mirror with a chain outside the packed key's range (the device never holds one)
int ensureRebinState(lb200_culling* cs, uint32_t max_entity) {
	lb200_ctx* ctx = cs->ctx;
	lb::CullingHost& h = cs->host;
	if (cs->replicas != 1) { lb200_set_error(ctx, "device re-binning works on the live page arrays: set_replicas(1)"); return LB200_ERR_STATE; }
	int rc = flushPages(cs);
	if (rc) return rc;
	if (!cs->d_rebin_counters || !cs->h_rebin_counters || !cs->rb_radix_scratch.state) {
		DeviceArray<uint32_t> d_counters; PinnedArray<uint32_t> h_counters; RadixSortScratch sort;
		LB200_CUDA(ctx, d_counters.alloc(RB_ALL_WORDS));
		LB200_CUDA(ctx, h_counters.alloc(RB_ALL_WORDS));
		rc = lb200_radix_sort_alloc_scratch(ctx, (uint32_t)ctx->sm_count * 2, sort);
		if (rc) return rc;
		cs->d_rebin_counters = std::move(d_counters); cs->h_rebin_counters = std::move(h_counters); cs->rb_radix_scratch = std::move(sort);
	}
	if (!cs->d_page_cell) { // the per-page side arrays: none yet, or released by a discarding resizePages, which also reset rebin_built_gen
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		const uint32_t cap = cs->dev_cap;
		DeviceArray<int4> page_cell; DeviceArray<uint32_t> free_pages, page_dirty, dirty_pages;
		LB200_CUDA(ctx, page_cell.alloc(cap));
		LB200_CUDA(ctx, free_pages.alloc(cap));
		LB200_CUDA(ctx, page_dirty.alloc(cap));
		LB200_CUDA(ctx, dirty_pages.alloc(cap));
		LB200_CUDA(ctx, cudaMemsetAsync(page_dirty, 0, sizeof(uint32_t) * (size_t)cap, ctx->stream));
		cs->d_page_cell = std::move(page_cell); cs->d_free_pages = std::move(free_pages); cs->d_page_dirty = std::move(page_dirty); cs->d_dirty_pages = std::move(dirty_pages);
	}
	const uint32_t need_entities = std::max((uint32_t)h.entity_to_slot.size(), max_entity + 1);
	if (cs->d_entity_to_slot.size() < need_entities) {
		// grown with its contents: while the device is authoritative the table is live and nothing rebuilds it from the host
		const size_t old = cs->d_entity_to_slot.size();
		const size_t cap = grownCapacity(old, 4096, need_entities);
		DeviceArray<uint32_t> grown;
		LB200_CUDA(ctx, grown.alloc(cap));
		if (old) LB200_CUDA(ctx, cudaMemcpyAsync(grown, cs->d_entity_to_slot, sizeof(uint32_t) * old, cudaMemcpyDeviceToDevice, ctx->stream));
		LB200_CUDA(ctx, cudaMemsetAsync(grown + old, 0xff, sizeof(uint32_t) * (cap - old), ctx->stream)); // NO_SLOT
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_entity_to_slot = std::move(grown);
	}
	if (cs->rebin_built_gen == h.edit_gen && !cs->device_authoritative) return LB200_OK;
	if (cs->device_authoritative) return LB200_OK; // the tables are live on the device
	// ---- build from the host mirror ----
	for (const auto& kv : h.cell_map) if (!cellInKeyRange(kv.first.x, kv.first.y, kv.first.z)) return REBIN_ON_HOST;
	const uint32_t n_pages = h.high_water;
	std::vector<int4> cells(n_pages);
	for (uint32_t p = 0; p < n_pages; ++p) cells[p] = make_int4(h.keys[p].x, h.keys[p].y, h.keys[p].z, (int)(h.keys[p].type | ((uint32_t)h.keys[p].is_big << 8)));
	uint32_t hcap = 1024;
	while (hcap < 4 * std::max<uint32_t>(n_pages, 256)) hcap *= 2;
	if (std::min(cs->d_hash_keys.size(), cs->d_hash_vals.size()) < hcap) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_hash_keys.reset(); cs->d_hash_vals.reset(); // before the new ones are allocated
		DeviceArray<unsigned long long> keys; DeviceArray<uint32_t> vals;
		LB200_CUDA(ctx, keys.alloc(hcap));
		LB200_CUDA(ctx, vals.alloc(hcap));
		cs->d_hash_keys = std::move(keys); cs->d_hash_vals = std::move(vals);
	}
	hcap = (uint32_t)cs->d_hash_keys.size();
	std::vector<unsigned long long> hk(hcap, HASH_EMPTY);
	std::vector<uint32_t> hv(hcap, NO_OPEN_PAGE);
	for (const auto& kv : h.cell_map) { // key -> head page of the chain (the page adds go to, culling_system.cpp:110-127)
		const unsigned long long key = packCellKey(kv.first.x, kv.first.y, kv.first.z, kv.first.type, kv.first.is_big);
		uint32_t i = hashCellKey(key) & (hcap - 1);
		while (hk[i] != HASH_EMPTY) i = (i + 1) & (hcap - 1);
		hk[i] = key; hv[i] = kv.second;
	}
	std::vector<uint32_t> e2s(cs->d_entity_to_slot.size(), NO_SLOT);
	std::copy(h.entity_to_slot.begin(), h.entity_to_slot.end(), e2s.begin());
	uint32_t counters[RB_WORDS] = {};
	counters[RB_HIGH_WATER] = n_pages;
	counters[RB_N_FREE] = (uint32_t)h.free_pages.size();
	counters[RB_BAD_RADIUS] = h.n_bad_radius;
	counters[RB_N_KEYS] = (uint32_t)h.cell_map.size();
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_page_cell, cells.data(), sizeof(int4) * n_pages, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_hash_keys, hk.data(), sizeof(unsigned long long) * hcap, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_hash_vals, hv.data(), sizeof(uint32_t) * hcap, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_entity_to_slot, e2s.data(), sizeof(uint32_t) * e2s.size(), cudaMemcpyHostToDevice, ctx->stream));
	if (!h.free_pages.empty()) LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_free_pages, h.free_pages.data(), sizeof(uint32_t) * h.free_pages.size(), cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_rebin_counters, counters, sizeof(counters), cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // the staging vectors go out of scope
	cs->dev_high_water = n_pages;
	cs->rebin_built_gen = h.edit_gen;
	return LB200_OK;
}

// the per-changer buffers (changer list, run plans, sort keys / values and their alternates) for n changers
int ensureChangerBuffers(lb200_culling* cs, uint32_t n) {
	lb200_ctx* ctx = cs->ctx;
	if (cs->d_changers.size() >= n) return LB200_OK;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	const size_t cap = grownCapacity(cs->d_changers.size(), 4096, n);
	// the old buffers go before the new ones are allocated
	cs->d_changers.reset(); cs->d_rb_plans.reset();
	for (int b = 0; b < 2; ++b) { cs->d_rb_keys[b].reset(); cs->d_rb_vals[b].reset(); }
	DeviceArray<uint32_t> changers; DeviceArray<uint4> plans; DeviceArray<uint64_t> keys[2], vals[2];
	LB200_CUDA(ctx, changers.alloc(cap));
	LB200_CUDA(ctx, plans.alloc(cap));
	for (int b = 0; b < 2; ++b) {
		LB200_CUDA(ctx, keys[b].alloc(cap));
		LB200_CUDA(ctx, vals[b].alloc(cap));
	}
	cs->d_changers = std::move(changers); cs->d_rb_plans = std::move(plans);
	for (int b = 0; b < 2; ++b) { cs->d_rb_keys[b] = std::move(keys[b]); cs->d_rb_vals[b] = std::move(vals[b]); }
	return LB200_OK;
}

// Keys are never removed from the chain hash map, so before a batch that may insert `adding` keys into a table holding `keys` (RB_N_KEYS
// of the last read-back) the table is rehashed on the device into one at least twice that size: it stays at most half full.
int growCellMap(lb200_culling* cs, uint32_t keys, uint32_t adding) {
	lb200_ctx* ctx = cs->ctx;
	const uint32_t old_cap = (uint32_t)cs->d_hash_keys.size();
	const uint64_t need = 2 * ((uint64_t)keys + adding);
	if (need <= old_cap) return LB200_OK;
	uint64_t cap = old_cap;
	while (cap < need) cap *= 2;
	if (cap > 0x80000000ull) { lb200_set_error(ctx, "the chain hash map would need %llu slots", (unsigned long long)cap); return LB200_ERR_CAPACITY; }
	cudaStream_t s = ctx->stream;
	DeviceArray<unsigned long long> hk; DeviceArray<uint32_t> hv;
	LB200_CUDA(ctx, hk.alloc(cap));
	LB200_CUDA(ctx, hv.alloc(cap));
	LB200_CUDA(ctx, cudaMemsetAsync(hk, 0xff, sizeof(unsigned long long) * cap, s)); // HASH_EMPTY
	LB200_CUDA(ctx, cudaMemsetAsync(hv, 0xff, sizeof(uint32_t) * cap, s));           // NO_OPEN_PAGE
	LB200_CUDA(ctx, cudaMemsetAsync(cs->d_rebin_counters + RB_N_KEYS, 0, sizeof(uint32_t), s));
	rebin_rehash_kernel<<<std::max(1u, std::min((uint32_t)ctx->sm_count * 4u, (old_cap + 255) / 256)), 256, 0, s>>>(cs->d_hash_keys, cs->d_hash_vals, old_cap, hk, hv,
		(uint32_t)cap, cs->d_rebin_counters);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaStreamSynchronize(s)); // the old table is read up to here
	cs->d_hash_keys = std::move(hk); cs->d_hash_vals = std::move(hv);
	return LB200_OK;
}

// step 3 for the n_changers keys / values in d_rb_keys[0] / d_rb_vals[0] (their count in RB_N_CHANGERS): sort by chain, plan every
// run, place every changer.  count_bad: the new spheres' bad radii are counted here (device adds) rather than by step 2a.
int placeChangers(lb200_culling* cs, const int32_t* ents, const double* pos3, const float* radius, uint32_t n_changers, bool count_bad) {
	lb200_ctx* ctx = cs->ctx;
	cudaStream_t s = ctx->stream;
	uint32_t* C = cs->d_rebin_counters;
	int rc = lb200_radix_sort_pairs(ctx, s, cs->d_rb_keys[0], cs->d_rb_keys[1], cs->d_rb_vals[0], cs->d_rb_vals[1], C + RB_N_CHANGERS, (uint32_t)cs->d_changers.size(),
		cs->rb_radix_scratch, 0, false, nullptr);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaMemsetAsync(C + RB_NEW_PAGES, 0, sizeof(uint32_t), s)); // the new-page cursor of this batch
	rebin_plan_kernel<<<std::max(1u, std::min((uint32_t)ctx->sm_count * 8u, (n_changers + 127) / 128)), 128, 0, s>>>(cs->d_rb_keys[0], cs->d_rb_vals[0], C, pos3, cs->d_desc,
		cs->d_page_cell, cs->d_free_pages, cs->d_hash_keys, cs->d_hash_vals, (uint32_t)cs->d_hash_keys.size(), cs->dev_cap, (RunPlan*)cs->d_rb_plans.get(),
		(uint32_t*)cs->d_rb_vals[1].get(), C + RB_NEW_PAGES);
	LB200_CHECK_LAUNCH(ctx);
	rebin_place_kernel<<<std::max(1u, std::min((uint32_t)ctx->sm_count * 4u, (n_changers + 255) / 256)), 256, 0, s>>>(cs->d_rb_keys[0], cs->d_rb_vals[0], C, ents, pos3,
		radius, cs->d_entity_to_slot, cs->d_desc, cs->d_spheres, cs->d_entities, (const RunPlan*)cs->d_rb_plans.get(), (const uint32_t*)cs->d_rb_vals[1].get(),
		count_bad ? C + RB_BAD_RADIUS : nullptr);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

// the read-back of a batch's end, in h_rebin_counters: the error of a full page array or hash map, if any
int checkOverflow(lb200_culling* cs) {
	const uint32_t of = cs->h_rebin_counters[RB_OVERFLOW];
	if (of & OVERFLOW_PAGES) { lb200_set_error(cs->ctx, "device re-binning ran out of pages (capacity %u)", cs->dev_cap); return LB200_ERR_CAPACITY; }
	if (of & OVERFLOW_HASH) { lb200_set_error(cs->ctx, "device re-binning found the chain hash map full (%zu slots)", cs->d_hash_keys.size()); return LB200_ERR_CAPACITY; }
	return LB200_OK;
}

// the read-back of an add / remove batch's end (RB_ALL_WORDS) -> the host's counts, which the cull's output layout, its output capacity
// and its plane-masking switch come from
void applyBatchCounts(lb200_culling* cs) {
	lb::CullingHost& h = cs->host;
	const uint32_t* delta = cs->h_rebin_counters + RB_TYPE_DELTA;
	for (int t = 0; t < 256; ++t) { h.type_counts[t] += delta[t]; h.n_entities += delta[t]; } // two's complement: removals wrap back
	h.n_bad_radius = cs->h_rebin_counters[RB_BAD_RADIUS];
	cs->dev_high_water = cs->h_rebin_counters[RB_HIGH_WATER];
}

// ---- batches with a cell outside the packed key's range: the host bookkeeping applies them ----

// the range flag belongs to the batch that raised it (the page and hash flags stay: their batch failed)
int clearRangeOverflow(lb200_culling* cs) {
	cs->h_rebin_counters[RB_OVERFLOW] &= ~OVERFLOW_RANGE;
	LB200_CUDA(cs->ctx, cudaMemcpyAsync(cs->d_rebin_counters + RB_OVERFLOW, cs->h_rebin_counters + RB_OVERFLOW, sizeof(uint32_t), cudaMemcpyHostToDevice, cs->ctx->stream));
	return LB200_OK;
}

template <class T> int copyBatch(lb200_ctx* ctx, std::vector<T>& out, const T* dev, size_t n) {
	out.resize(n);
	LB200_CUDA(ctx, cudaMemcpyAsync(out.data(), dev, sizeof(T) * n, cudaMemcpyDeviceToHost, ctx->stream));
	return LB200_OK;
}

// set_many_device: CullingHost::set for every added mover (ids that are not added are skipped, as the classify kernel skips them), after
// the pull-back (which brings the classify kernel's in-place writes home; set() writes them again).  The changer count
// lb200_culling_last_rebin_changers reports is the classify kernel's: movers whose cell or big-ness changes.
int setOnHost(lb200_culling* cs, const int32_t* dev_entities, const double* dev_pos3, const float* dev_radius, uint32_t n) {
	lb200_ctx* ctx = cs->ctx;
	int rc = syncHostFromDevice(cs);
	std::vector<int32_t> ents; std::vector<double> pos; std::vector<float> rad;
	if (!rc && dev_entities) rc = copyBatch(ctx, ents, dev_entities, n);
	if (!rc) rc = copyBatch(ctx, pos, dev_pos3, 3 * (size_t)n);
	if (!rc) rc = copyBatch(ctx, rad, dev_radius, n);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	lb::CullingHost& h = cs->host;
	uint32_t changers = 0;
	for (uint32_t i = 0; i < n; ++i) {
		const int32_t e = dev_entities ? ents[i] : (int32_t)i;
		if (!h.isAdded(e)) continue;
		const uint32_t page = h.entity_to_slot[e] / PAGE_SLOTS;
		const double* p = pos.data() + 3 * (size_t)i;
		if (!lb::CullingHost::sameCell(lb::CullingHost::makeKey(p, 0, false), h.keys[page]) || (h.desc[page].is_big != 0) != (rad[i] > LB200_CELL_SIZE)) ++changers;
		rc = h.set(e, p, rad[i]);
		if (rc) return rc;
	}
	cs->h_rebin_counters[RB_N_CHANGERS] = changers;
	return LB200_OK;
}

// add_many_device: the batch is refused whole for the same ids and types the claim kernel refuses; otherwise CullingHost::add for each
int addOnHost(lb200_culling* cs, const int32_t* dev_entities, const uint8_t* dev_types, const double* dev_pos3, const float* dev_radius, uint32_t n,
	uint32_t max_entity)
{
	lb200_ctx* ctx = cs->ctx;
	int rc = syncHostFromDevice(cs);
	std::vector<int32_t> ents; std::vector<uint8_t> types; std::vector<double> pos; std::vector<float> rad;
	if (!rc && dev_entities) rc = copyBatch(ctx, ents, dev_entities, n);
	if (!rc) rc = copyBatch(ctx, types, dev_types, n);
	if (!rc) rc = copyBatch(ctx, pos, dev_pos3, 3 * (size_t)n);
	if (!rc) rc = copyBatch(ctx, rad, dev_radius, n);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	lb::CullingHost& h = cs->host;
	if (!dev_entities) { ents.resize(n); for (uint32_t i = 0; i < n; ++i) ents[i] = (int32_t)i; }
	std::vector<int32_t> sorted(ents);
	std::sort(sorted.begin(), sorted.end());
	uint32_t refused = 0;
	for (uint32_t i = 0; i < n; ++i) {
		const int32_t e = ents[i];
		if (e < 0 || (uint32_t)e > max_entity || types[i] == LB200_TYPE_ALL || h.isAdded(e) || (i && sorted[i] == sorted[i - 1])) ++refused;
	}
	if (refused) {
		lb200_set_error(ctx, "add_many_device: %u of %u entities refused (an id added already, listed twice or outside [0, %u], or type 0xff)", refused, n, max_entity);
		return LB200_ERR_INVALID;
	}
	for (uint32_t i = 0; i < n; ++i) {
		rc = h.add(ents[i], types[i], pos.data() + 3 * (size_t)i, rad[i]);
		if (rc) return rc;
	}
	return LB200_OK;
}

// remove_many_device: CullingHost::remove for every id (ids that are not added, and repeats, are skipped there)
int removeOnHost(lb200_culling* cs, const int32_t* dev_entities, uint32_t n) {
	lb200_ctx* ctx = cs->ctx;
	int rc = syncHostFromDevice(cs);
	std::vector<int32_t> ents;
	if (!rc) rc = copyBatch(ctx, ents, dev_entities, n);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	for (uint32_t i = 0; i < n; ++i) cs->host.remove(ents[i]);
	return LB200_OK;
}

} // namespace

// pull the device state back into the host mirror (page arrays, counts, entity -> slot, chains regrouped by key with the open page as head)
int lbcull::syncHostFromDevice(lb200_culling* cs) {
	if (!cs->device_authoritative) return LB200_OK;
	lb200_ctx* ctx = cs->ctx;
	lb::CullingHost& h = cs->host;
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_rebin_counters, cs->d_rebin_counters, sizeof(uint32_t) * RB_WORDS, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	const uint32_t n_pages = cs->h_rebin_counters[RB_HIGH_WATER];
	if (h.cap < n_pages && !h.grow(n_pages)) return LB200_ERR_CUDA;
	std::vector<int4> cells(n_pages);
	const uint32_t hash_cap = (uint32_t)cs->d_hash_keys.size();
	std::vector<unsigned long long> hk(hash_cap);
	std::vector<uint32_t> hv(hash_cap);
	LB200_CUDA(ctx, cudaMemcpyAsync(h.spheres, cs->d_spheres, sizeof(float4) * PAGE_SLOTS * (size_t)n_pages, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(h.entities, cs->d_entities, sizeof(int) * PAGE_SLOTS * (size_t)n_pages, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(h.desc, cs->d_desc, sizeof(lb200_page_desc) * (size_t)n_pages, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(cells.data(), cs->d_page_cell, sizeof(int4) * (size_t)n_pages, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(hk.data(), cs->d_hash_keys, sizeof(unsigned long long) * hash_cap, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(hv.data(), cs->d_hash_vals, sizeof(uint32_t) * hash_cap, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(h.entity_to_slot.data(), cs->d_entity_to_slot, sizeof(uint32_t) * h.entity_to_slot.size(), cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	h.high_water = n_pages;
	h.cells.clear(); h.cell_map.clear(); h.free_pages.clear();
	h.n_bad_radius = 0;
	std::unordered_map<lb::CellKey, uint32_t, lb::CellKeyHasher> tail; // last page linked so far of each chain
	for (uint32_t i = 0; i < hash_cap; ++i) { // the open page of every chain is its head (culling_system.cpp:110-127)
		if (hk[i] == HASH_EMPTY || hv[i] == NO_OPEN_PAGE || hv[i] >= n_pages || h.desc[hv[i]].count == 0) continue;
		const uint32_t p = hv[i];
		lb::CellKey k; k.x = cells[p].x; k.y = cells[p].y; k.z = cells[p].z; k.type = (uint8_t)(cells[p].w & 0xff); k.is_big = (uint8_t)((uint32_t)cells[p].w >> 8);
		h.cell_map[k] = p;
	}
	for (uint32_t p = 0; p < n_pages; ++p) {
		h.next[p] = h.prev[p] = lb::NO_PAGE;
		if (h.desc[p].count == 0) { h.free_pages.push_back(p); continue; }
		lb::CellKey k; k.x = cells[p].x; k.y = cells[p].y; k.z = cells[p].z; k.type = (uint8_t)(cells[p].w & 0xff); k.is_big = (uint8_t)((uint32_t)cells[p].w >> 8);
		h.keys[p] = k;
		h.cellsPush(p);
		for (uint32_t s = 0; s < h.desc[p].count; ++s) if (lb::CullingHost::badRadius(h.spheres[4 * ((size_t)p * PAGE_SLOTS + s) + 3])) ++h.n_bad_radius;
		if (h.cell_map.find(k) == h.cell_map.end()) h.cell_map[k] = p; // a chain whose open page ran empty: any of its pages heads it
	}
	for (uint32_t p = 0; p < n_pages; ++p) { // link the other pages of every chain behind its head
		if (h.desc[p].count == 0) continue;
		const uint32_t head = h.cell_map[h.keys[p]];
		if (p == head) continue;
		auto it = tail.find(h.keys[p]);
		const uint32_t last = it == tail.end() ? head : it->second;
		h.next[last] = (int32_t)p; h.prev[p] = (int32_t)last;
		tail[h.keys[p]] = p;
	}
	h.clearDirty();
	++h.edit_gen;
	cs->device_authoritative = false;
	cs->membership_on_device = false;
	cs->rebin_built_gen = ~0ull;
	return LB200_OK;
}

extern "C" {

int lb200_culling_set_many_device(lb200_culling* cs, const int32_t* dev_entities, const double* dev_pos3, const float* dev_radius, uint32_t n, uint32_t max_entity) {
	if (!cs || !dev_pos3 || !dev_radius) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (n == 0) return LB200_OK;
	lb200_ctx* ctx = cs->ctx;
	lb200_range range("culling set many");
	int rc = ensureRebinState(cs, max_entity);
	if (rc == REBIN_ON_HOST) return setOnHost(cs, dev_entities, dev_pos3, dev_radius, n);
	if (rc) return rc;
	rc = ensureChangerBuffers(cs, n);
	if (rc) return rc;
	cudaStream_t s = ctx->stream;
	uint32_t* C = cs->d_rebin_counters;
	LB200_CUDA(ctx, cudaMemsetAsync(C + RB_N_CHANGERS, 0, sizeof(uint32_t) * 2, s)); // changers, dirty pages
	rebin_classify_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, dev_entities, dev_pos3, dev_radius, cs->d_entity_to_slot, (uint32_t)cs->d_entity_to_slot.size(), cs->d_desc, cs->d_page_cell, cs->d_spheres, cs->d_changers, C);
	LB200_CHECK_LAUNCH(ctx);
	// how many entities change their chain decides how many new pages the adds may need: one small read-back
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_rebin_counters, C, sizeof(uint32_t) * RB_WORDS, cudaMemcpyDeviceToHost, s));
	LB200_CUDA(ctx, cudaStreamSynchronize(s));
	const uint32_t n_changers = cs->h_rebin_counters[RB_N_CHANGERS];
	cs->device_authoritative = true;
	cs->uploaded_since_last_cull = true; // the page arrays changed: the next cull must not overlap these kernels
	if (cs->h_rebin_counters[RB_OVERFLOW] & OVERFLOW_RANGE) { // a mover's cell lies outside the packed key's range
		rc = clearRangeOverflow(cs);
		return rc ? rc : setOnHost(cs, dev_entities, dev_pos3, dev_radius, n);
	}
	if (n_changers) {
		rc = resizePages(cs, cs->h_rebin_counters[RB_HIGH_WATER] + n_changers, true); // worst case: every changer opens a page
		if (rc) return rc;
		rc = growCellMap(cs, cs->h_rebin_counters[RB_N_KEYS], n_changers); // worst case: every changer starts a chain
		if (rc) return rc;
		const uint32_t grid = std::max(1u, std::min((uint32_t)ctx->sm_count * 4u, (n_changers + 255) / 256));
		rebin_remove_kernel<<<grid, 256, 0, s>>>(cs->d_changers, dev_entities, dev_pos3, dev_radius, cs->d_entity_to_slot, cs->d_page_cell, cs->d_spheres, cs->d_entities,
			cs->d_page_dirty, cs->d_dirty_pages, C, cs->d_rb_keys[0], cs->d_rb_vals[0]);
		LB200_CHECK_LAUNCH(ctx);
		rebin_compact_kernel<<<grid, 256, 0, s>>>(cs->d_dirty_pages, C, cs->d_desc, cs->d_page_cell, cs->d_spheres, cs->d_entities, cs->d_entity_to_slot, cs->d_page_dirty,
			cs->d_free_pages, cs->d_hash_keys, cs->d_hash_vals, (uint32_t)cs->d_hash_keys.size());
		LB200_CHECK_LAUNCH(ctx);
		rc = placeChangers(cs, dev_entities, dev_pos3, dev_radius, n_changers, false);
		if (rc) return rc;
		LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_rebin_counters, C, sizeof(uint32_t) * RB_WORDS, cudaMemcpyDeviceToHost, s));
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		rc = checkOverflow(cs);
		if (rc) return rc;
	}
	cs->dev_high_water = cs->h_rebin_counters[RB_HIGH_WATER];
	cs->host.n_bad_radius = cs->h_rebin_counters[RB_BAD_RADIUS]; // plane masking of the cull kernel needs radius >= 0 everywhere
	return LB200_OK;
}

int lb200_culling_add_many_device(lb200_culling* cs, const int32_t* dev_entities, const uint8_t* dev_types, const double* dev_pos3, const float* dev_radius,
	uint32_t n, uint32_t max_entity)
{
	if (!cs || !dev_types || !dev_pos3 || !dev_radius) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (n == 0) return LB200_OK;
	lb200_ctx* ctx = cs->ctx;
	if (max_entity > (uint32_t)INT32_MAX) { lb200_set_error(ctx, "add_many_device: max_entity %u is not an entity id", max_entity); return LB200_ERR_INVALID; }
	lb200_range range("culling add many");
	int rc = ensureRebinState(cs, max_entity);
	if (rc == REBIN_ON_HOST) return addOnHost(cs, dev_entities, dev_types, dev_pos3, dev_radius, n, max_entity);
	if (rc) return rc;
	rc = ensureChangerBuffers(cs, n);
	if (rc) return rc;
	cudaStream_t s = ctx->stream;
	uint32_t* C = cs->d_rebin_counters;
	const uint32_t blocks = (n + 255) / 256;
	LB200_CUDA(ctx, cudaMemsetAsync(C + RB_REFUSED, 0, sizeof(uint32_t) * 2, s)); // refused, largest id
	LB200_CUDA(ctx, cudaMemsetAsync(C + RB_TYPE_DELTA, 0, sizeof(uint32_t) * 256, s));
	rebin_add_claim_kernel<<<blocks, 256, 0, s>>>(n, dev_entities, dev_types, dev_pos3, dev_radius, max_entity, cs->d_entity_to_slot, C, cs->d_rb_keys[0], cs->d_rb_vals[0]);
	LB200_CHECK_LAUNCH(ctx);
	// the one read-back before placement: whether the batch is refused, and the page and key counts its placement is sized by
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_rebin_counters, C, sizeof(uint32_t) * RB_ADD_WORDS, cudaMemcpyDeviceToHost, s));
	LB200_CUDA(ctx, cudaStreamSynchronize(s));
	const uint32_t refused = cs->h_rebin_counters[RB_REFUSED];
	const bool out_of_range = (cs->h_rebin_counters[RB_OVERFLOW] & OVERFLOW_RANGE) != 0; // a cell the packed key cannot hold
	if (!refused && !out_of_range) {
		rc = resizePages(cs, cs->h_rebin_counters[RB_HIGH_WATER] + n, true); // worst case: every entity opens a page
		if (!rc) rc = growCellMap(cs, cs->h_rebin_counters[RB_N_KEYS], n); // worst case: every entity starts a chain
	}
	if (refused || out_of_range || rc) { // the device changes nothing: the batch's claims are released
		rebin_add_release_kernel<<<blocks, 256, 0, s>>>(n, dev_entities, max_entity, cs->d_entity_to_slot);
		LB200_CHECK_LAUNCH(ctx);
		if (rc) return rc;
		if (out_of_range) rc = clearRangeOverflow(cs);
		if (rc) return rc;
		if (out_of_range && !refused) return addOnHost(cs, dev_entities, dev_types, dev_pos3, dev_radius, n, max_entity);
		lb200_set_error(ctx, "add_many_device: %u of %u entities refused (an id added already, listed twice or outside [0, %u], or type 0xff)", refused, n, max_entity);
		return LB200_ERR_INVALID;
	}
	cs->device_authoritative = true;
	cs->membership_on_device = true;
	cs->uploaded_since_last_cull = true; // the page arrays change: the next cull must not overlap these kernels
	rc = placeChangers(cs, dev_entities, dev_pos3, dev_radius, n, true);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_rebin_counters, C, sizeof(uint32_t) * RB_ALL_WORDS, cudaMemcpyDeviceToHost, s));
	LB200_CUDA(ctx, cudaStreamSynchronize(s));
	rc = checkOverflow(cs);
	if (rc) return rc;
	lb::CullingHost& h = cs->host;
	const uint32_t max_id = cs->h_rebin_counters[RB_MAX_ID];
	// the pull-back brings the new ids home, and the ids a cull can emit stay inside entity_range (createSortKeys checks it)
	if (h.entity_to_slot.size() <= max_id) h.entity_to_slot.resize((size_t)max_id + 1, NO_SLOT);
	applyBatchCounts(cs);
	return LB200_OK;
}

int lb200_culling_remove_many_device(lb200_culling* cs, const int32_t* dev_entities, uint32_t n) {
	if (!cs || !dev_entities) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (n == 0) return LB200_OK;
	lb200_ctx* ctx = cs->ctx;
	lb200_range range("culling remove many");
	int rc = ensureRebinState(cs, 0);
	if (rc == REBIN_ON_HOST) return removeOnHost(cs, dev_entities, n);
	if (rc) return rc;
	cudaStream_t s = ctx->stream;
	uint32_t* C = cs->d_rebin_counters;
	LB200_CUDA(ctx, cudaMemsetAsync(C + RB_N_DIRTY, 0, sizeof(uint32_t), s));
	LB200_CUDA(ctx, cudaMemsetAsync(C + RB_TYPE_DELTA, 0, sizeof(uint32_t) * 256, s));
	rebin_remove_ids_kernel<<<(n + 255) / 256, 256, 0, s>>>(n, dev_entities, cs->d_entity_to_slot, (uint32_t)cs->d_entity_to_slot.size(), cs->d_page_cell, cs->d_spheres,
		cs->d_entities, cs->d_page_dirty, cs->d_dirty_pages, C);
	LB200_CHECK_LAUNCH(ctx);
	rebin_compact_kernel<<<std::max(1u, std::min((uint32_t)ctx->sm_count * 4u, (n + 255) / 256)), 256, 0, s>>>(cs->d_dirty_pages, C, cs->d_desc, cs->d_page_cell, cs->d_spheres,
		cs->d_entities, cs->d_entity_to_slot, cs->d_page_dirty, cs->d_free_pages, cs->d_hash_keys, cs->d_hash_vals, (uint32_t)cs->d_hash_keys.size());
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_rebin_counters, C, sizeof(uint32_t) * RB_ALL_WORDS, cudaMemcpyDeviceToHost, s));
	LB200_CUDA(ctx, cudaStreamSynchronize(s));
	const uint32_t before = cs->host.n_entities;
	applyBatchCounts(cs);
	if (cs->host.n_entities != before) { // something was removed: the pages in HBM are ahead of the mirror now
		cs->device_authoritative = true;
		cs->membership_on_device = true;
		cs->uploaded_since_last_cull = true;
	}
	return LB200_OK;
}

int lb200_culling_sync_host(lb200_culling* cs) {
	if (!cs) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_OK;
	return syncHostFromDevice(cs);
}

uint32_t lb200_culling_last_rebin_changers(const lb200_culling* cs) { return cs && cs->h_rebin_counters ? cs->h_rebin_counters[RB_N_CHANGERS] : 0; }

} // extern "C"
