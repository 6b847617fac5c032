// GPU CullingSystem: host side + C-ABI (include/lumix_b200.h "CullingSystem").
//
// Replaces CullingSystemImpl::cullInternal + doCulling (src/renderer/culling_system.cpp:260-369).  The cull itself is one kernel,
// cull_pages_kernel (cull_kernel.cuh, which describes its phases, included here and nowhere else; its culling core, cull_common.cuh, is
// shared with cull_views_kernel).  The culling system's sources:
//   culling.cu           the host-edit C API, the page upload (ensureDevice, resizePages, flushPages), the cull launch and its lanes,
//                        the delivery of results to the caller (cull, begin / poll / end, cull_device[_n], read_bitmask, time_lone_cull)
//   culling_exchange.cu  the multi-GPU exchange: all-gather of visible ids, NVLink push, bitmask exchange steps
//   culling_rebin.cu     device re-binning (set_many_device), device adds / removes (add_many_device, remove_many_device) and the
//                        pull-back of the host mirror
//   culling_views.cu     several views in one pass (cull_views, select_view): cull_views_kernel.cuh, or this file's launchCull for one view
//   culling_internal.h   struct lb200_culling, the counter and slab layout, and the functions the four share
#include "cull_kernel.cuh"
#include "culling_internal.h"
#include "lb200_math.cuh"

#include <algorithm>
#include <new>

namespace {

using namespace lb;

using namespace lbcull;

// scatter packed dirty pages from a staging buffer into the page arrays (one block per page)
__global__ void __launch_bounds__(256) scatter_pages_kernel(const uint32_t* __restrict__ page_idx, const lb200_page_desc* __restrict__ st_desc,
	const float4* __restrict__ st_spheres, const int* __restrict__ st_entities, lb200_page_desc* __restrict__ desc, float4* __restrict__ spheres,
	int* __restrict__ entities)
{
	const uint32_t i = blockIdx.x;
	const uint32_t p = page_idx[i];
	if (threadIdx.x < PAGE_SLOTS) {
		spheres[(size_t)p * PAGE_SLOTS + threadIdx.x] = st_spheres[(size_t)i * PAGE_SLOTS + threadIdx.x];
		entities[(size_t)p * PAGE_SLOTS + threadIdx.x] = st_entities[(size_t)i * PAGE_SLOTS + threadIdx.x];
	}
	if (threadIdx.x < 2) reinterpret_cast<int4*>(desc + p)[threadIdx.x] = reinterpret_cast<const int4*>(st_desc + i)[threadIdx.x];
}

// Visible ids of one cull packed type after type, and its counters, read on the device: into page-locked HOST memory (posted writes over
// PCIe, no count round trip) or into the NCCL send slab.  Ids beyond `capacity` are dropped; the counts show it (LB200_ERR_CAPACITY).
struct PackParams { uint32_t type_base[256]; uint32_t capacity; };

__global__ void __launch_bounds__(256) pack_kernel(const __grid_constant__ PackParams P, const uint32_t* __restrict__ counters,
	const uint32_t* __restrict__ out_ids, uint32_t* __restrict__ ids_dst, uint32_t* __restrict__ counters_dst, uint32_t counter_words)
{
	__shared__ uint32_t s_cnt[256];
	__shared__ uint32_t s_off[257];
	__shared__ uint32_t s_list[256];
	__shared__ uint32_t s_nnz;
	scan_types(counters, s_cnt, s_off, s_list, &s_nnz);
	if (blockIdx.x == 0) for (uint32_t i = threadIdx.x; i < counter_words; i += blockDim.x) counters_dst[i] = counters[i];
	const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, gsize = gridDim.x * blockDim.x;
	for (uint32_t k = 0; k < s_nnz; ++k) {
		const uint32_t t = s_list[k];
		const uint32_t c = s_cnt[t];
		const uint32_t* src = out_ids + P.type_base[t];
		const uint32_t off = s_off[t];
		for (uint32_t i = gtid; i < c; i += gsize) if (off + i < P.capacity) ids_dst[off + i] = src[i];
	}
}

// holds the stream for a while, so that whatever the host enqueues behind it is already queued when the device gets there
__global__ void delay_kernel(long long cycles) {
	const long long t0 = clock64();
	while (clock64() - t0 < cycles) {}
}

// allocators of culling_host.hpp's host arrays, raw: without a context the same arrays come from malloc
void* pinnedAlloc(size_t n) {
	void* p = nullptr;
	if (cudaHostAlloc(&p, n ? n : 1, cudaHostAllocDefault) != cudaSuccess) { cudaGetLastError(); return nullptr; }
	return p;
}
void pinnedFree(void* p) { if (p) cudaFreeHost(p); }
void* plainAlloc(size_t n) { return malloc(n ? n : 1); }
void plainFree(void* p) { free(p); }

} // namespace

lb200_culling::lb200_culling(lb200_ctx* c) : ctx(c), host(c ? pinnedAlloc : plainAlloc, c ? pinnedFree : plainFree) {}

namespace lbcull {

int ensureDevice(lb200_culling* cs) {
	lb200_ctx* ctx = cs->ctx;
	lb::CullingHost& h = cs->host;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!cs->d_counters || !cs->h_counters) { // the launch shape comes first: once the counters exist, it is set
		cs->lanes = lb200_cull_lanes();
		int per_sm = 0;
		LB200_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, cull_pages_kernel, CULL_THREADS, 0));
		if (per_sm < 1) per_sm = 1;
		cs->grid = ctx->sm_count * per_sm;
		// cull_device_n runs independent culls concurrently: half-occupancy grids let two of them share every SM, so one cull's
		// classify / test phases fill the memory pipeline while another is in its claim / write phases (measured: profiles/, DESIGN 4.1)
		int lane_per_sm = std::min(per_sm, 2);
		if (const char* e = getenv("LB200_CULL_BLOCKS_PER_SM")) lane_per_sm = std::max(1, std::min(per_sm, atoi(e))); // tuning knob
		cs->grid_lanes = ctx->sm_count * lane_per_sm;
		DeviceArray<uint32_t> d_counters;
		PinnedArray<uint32_t, cudaHostAllocMapped> h_counters;
		LB200_CUDA(ctx, d_counters.alloc(2 * cs->lanes * COUNTER_WORDS));
		LB200_CUDA(ctx, cudaMemsetAsync(d_counters, 0, sizeof(uint32_t) * 2 * cs->lanes * COUNTER_WORDS, ctx->stream));
		LB200_CUDA(ctx, h_counters.alloc(COUNTER_WORDS));
		const cudaError_t me = cudaHostGetDevicePointer((void**)&cs->h_counters_dev, h_counters, 0);
		if (me != cudaSuccess) {
			cudaGetLastError();
			cs->h_counters_dev = nullptr;
			cudaPointerAttributes pa = {}; // unified addressing: page-locked memory has a device address whether or not it was asked to be "mapped"
			if (cudaPointerGetAttributes(&pa, h_counters) == cudaSuccess && pa.devicePointer) cs->h_counters_dev = (uint32_t*)pa.devicePointer;
			else { cudaGetLastError(); lb200_set_error(ctx, "page-locked counters have no device address: %s", cudaGetErrorString(me)); }
		}
		cs->d_counters = std::move(d_counters); cs->h_counters = std::move(h_counters);
	}
	if (cs->dev_cap < h.high_water) {
		const int rc = resizePages(cs, h.high_water, false);
		if (rc) return rc;
	}
	const size_t out_cap = cs->d_out_ids.size() / cs->lanes;
	if (out_cap < h.n_entities || !cs->d_out_ids) {
		const size_t cap = grownCapacity(out_cap, 4096, h.n_entities);
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_out_ids.reset();
		LB200_CUDA(ctx, cs->d_out_ids.alloc(cap * cs->lanes));
	}
	return LB200_OK;
}

// Grows the page arrays and the per-page re-binning arrays to hold min_pages pages; sets dev_cap and item_cap.
//   keep = false  free first (peak memory = the new arrays), zero the descriptors, upload the host mirror in full at the next flush; the
//                 per-page arrays are released for ensureRebinState to re-create.  Only while the host mirror is authoritative: while
//                 the device is ahead, the host's high-water mark is stale and never exceeds dev_cap, and set_replicas syncs the mirror.
//   keep = true   allocate, copy, synchronise, swap, so that a failure leaves the old arrays in place (device re-binning, replicas == 1).
int resizePages(lb200_culling* cs, uint32_t min_pages, bool keep) {
	lb200_ctx* ctx = cs->ctx;
	if (min_pages <= cs->dev_cap) return LB200_OK;
	const uint32_t cap = (uint32_t)grownCapacity(cs->dev_cap, 1024, min_pages);
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	releaseViews(cs);
	if (!keep) {
		cs->d_spheres.reset(); cs->d_entities.reset(); cs->d_desc.reset(); cs->d_mask.reset(); // before the new ones are allocated
		cs->d_page_cell.reset(); cs->d_free_pages.reset(); cs->d_page_dirty.reset(); cs->d_dirty_pages.reset();
		cs->rebin_built_gen = ~0ull;
		cs->dev_cap = 0; // until the four arrays are back
	}
	const size_t R = cs->replicas;
	DeviceArray<float4> spheres; DeviceArray<int> entities; DeviceArray<lb200_page_desc> desc; DeviceArray<uint32_t> mask;
	LB200_CUDA(ctx, spheres.alloc(PAGE_SLOTS * (size_t)cap * R));
	LB200_CUDA(ctx, entities.alloc(PAGE_SLOTS * (size_t)cap * R));
	LB200_CUDA(ctx, desc.alloc((size_t)cap * R));
	LB200_CUDA(ctx, mask.alloc(8 * (size_t)cap * cs->lanes));
	DeviceArray<int4> page_cell; DeviceArray<uint32_t> free_pages, page_dirty, dirty_pages;
	if (keep) {
		LB200_CUDA(ctx, page_cell.alloc(cap));
		LB200_CUDA(ctx, free_pages.alloc(cap));
		LB200_CUDA(ctx, page_dirty.alloc(cap));
		LB200_CUDA(ctx, dirty_pages.alloc(cap));
	}
	// free / never-used pages must read count == 0
	LB200_CUDA(ctx, cudaMemsetAsync(desc, 0, sizeof(lb200_page_desc) * (size_t)cap * R, ctx->stream));
	if (keep) {
		LB200_CUDA(ctx, cudaMemsetAsync(page_dirty, 0, sizeof(uint32_t) * (size_t)cap, ctx->stream));
		const size_t old = cs->dev_cap;
		if (old) {
			LB200_CUDA(ctx, cudaMemcpyAsync(spheres, cs->d_spheres, sizeof(float4) * PAGE_SLOTS * old, cudaMemcpyDeviceToDevice, ctx->stream));
			LB200_CUDA(ctx, cudaMemcpyAsync(entities, cs->d_entities, sizeof(int) * PAGE_SLOTS * old, cudaMemcpyDeviceToDevice, ctx->stream));
			LB200_CUDA(ctx, cudaMemcpyAsync(desc, cs->d_desc, sizeof(lb200_page_desc) * old, cudaMemcpyDeviceToDevice, ctx->stream));
			if (cs->d_page_cell) LB200_CUDA(ctx, cudaMemcpyAsync(page_cell, cs->d_page_cell, sizeof(int4) * old, cudaMemcpyDeviceToDevice, ctx->stream));
			if (cs->d_free_pages) LB200_CUDA(ctx, cudaMemcpyAsync(free_pages, cs->d_free_pages, sizeof(uint32_t) * old, cudaMemcpyDeviceToDevice, ctx->stream));
		}
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_page_cell = std::move(page_cell); cs->d_free_pages = std::move(free_pages); cs->d_page_dirty = std::move(page_dirty); cs->d_dirty_pages = std::move(dirty_pages);
	}
	cs->d_spheres = std::move(spheres); cs->d_entities = std::move(entities); cs->d_desc = std::move(desc); cs->d_mask = std::move(mask);
	cs->item_cap = cap; // every page can end up with a record
	cs->dev_cap = cap;
	if (!keep) cs->host.all_dirty = true;
	return LB200_OK;
}

int flushPages(lb200_culling* cs) {
	lb200_ctx* ctx = cs->ctx;
	lb::CullingHost& h = cs->host;
	int rc = ensureDevice(cs);
	if (rc) return rc;
	if (!h.all_dirty && h.dirty_list.empty()) return LB200_OK;
	const uint32_t n = h.high_water;
	const bool full = h.all_dirty || h.dirty_list.size() * 8 > n;
	if (full) {
		LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_spheres, h.spheres, sizeof(float4) * PAGE_SLOTS * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
		LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_entities, h.entities, sizeof(int) * PAGE_SLOTS * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
		LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_desc, h.desc, sizeof(lb200_page_desc) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
		for (uint32_t r = 1; r < cs->replicas; ++r) { // bench replicas: copy inside HBM
			const size_t off = (size_t)r * cs->dev_cap;
			LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_spheres + off * PAGE_SLOTS, cs->d_spheres, sizeof(float4) * PAGE_SLOTS * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
			LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_entities + off * PAGE_SLOTS, cs->d_entities, sizeof(int) * PAGE_SLOTS * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
			LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_desc + off, cs->d_desc, sizeof(lb200_page_desc) * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
		}
	}
	else {
		const size_t m = h.dirty_list.size();
		const size_t per_page = sizeof(float4) * PAGE_SLOTS + sizeof(int) * PAGE_SLOTS + sizeof(lb200_page_desc) + sizeof(uint32_t);
		const size_t stage_pages = std::min(cs->h_stage.size(), cs->d_stage.size()) / per_page;
		if (stage_pages < m) {
			const size_t cap = grownCapacity(stage_pages, 256, m);
			LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
			cs->h_stage.reset(); cs->d_stage.reset(); // before the new ones are allocated
			PinnedArray<uint8_t> h_stage; DeviceArray<uint8_t> d_stage;
			LB200_CUDA(ctx, h_stage.alloc(per_page * cap));
			LB200_CUDA(ctx, d_stage.alloc(per_page * cap));
			cs->h_stage = std::move(h_stage); cs->d_stage = std::move(d_stage);
		}
		else {
			// the previous scatter may still be reading the staging buffer
			LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		}
		// staging layout: [spheres cap][entities cap][desc cap][idx cap], of which the first m entries of each are used
		const size_t cap = cs->h_stage.size() / per_page;
		float* st_s = reinterpret_cast<float*>(cs->h_stage.get());
		int* st_e = reinterpret_cast<int*>(cs->h_stage + sizeof(float4) * PAGE_SLOTS * cap);
		lb200_page_desc* st_d = reinterpret_cast<lb200_page_desc*>(cs->h_stage + (sizeof(float4) + sizeof(int)) * PAGE_SLOTS * cap);
		uint32_t* st_i = reinterpret_cast<uint32_t*>(cs->h_stage + (sizeof(float4) + sizeof(int)) * PAGE_SLOTS * cap + sizeof(lb200_page_desc) * cap);
		for (size_t i = 0; i < m; ++i) {
			const uint32_t p = h.dirty_list[i];
			memcpy(st_s + 4 * PAGE_SLOTS * i, h.spheres + 4 * PAGE_SLOTS * (size_t)p, sizeof(float4) * PAGE_SLOTS);
			memcpy(st_e + PAGE_SLOTS * i, h.entities + PAGE_SLOTS * (size_t)p, sizeof(int) * PAGE_SLOTS);
			st_d[i] = h.desc[p];
			st_i[i] = p;
		}
		// only the m used entries of each of the four sections travel
		const size_t sec[5] = {0, sizeof(float4) * PAGE_SLOTS * cap, (sizeof(float4) + sizeof(int)) * PAGE_SLOTS * cap,
			(sizeof(float4) + sizeof(int)) * PAGE_SLOTS * cap + sizeof(lb200_page_desc) * cap, 0};
		const size_t used[4] = {sizeof(float4) * PAGE_SLOTS * m, sizeof(int) * PAGE_SLOTS * m, sizeof(lb200_page_desc) * m, sizeof(uint32_t) * m};
		for (int k = 0; k < 4; ++k)
			LB200_CUDA(ctx, cudaMemcpyAsync(cs->d_stage + sec[k], cs->h_stage + sec[k], used[k], cudaMemcpyHostToDevice, ctx->stream));
		const float4* d_s = reinterpret_cast<const float4*>(cs->d_stage.get());
		const int* d_e = reinterpret_cast<const int*>(cs->d_stage + sizeof(float4) * PAGE_SLOTS * cap);
		const lb200_page_desc* d_d = reinterpret_cast<const lb200_page_desc*>(cs->d_stage + (sizeof(float4) + sizeof(int)) * PAGE_SLOTS * cap);
		const uint32_t* d_i = reinterpret_cast<const uint32_t*>(cs->d_stage + (sizeof(float4) + sizeof(int)) * PAGE_SLOTS * cap + sizeof(lb200_page_desc) * cap);
		for (uint32_t r = 0; r < cs->replicas; ++r) {
			const size_t off = (size_t)r * cs->dev_cap;
			scatter_pages_kernel<<<(unsigned)m, 256, 0, ctx->stream>>>(d_i, d_d, d_s, d_e, cs->d_desc + off, cs->d_spheres + off * PAGE_SLOTS, cs->d_entities + off * PAGE_SLOTS);
			LB200_CHECK_LAUNCH(ctx);
		}
	}
	h.clearDirty();
	cs->uploaded_since_last_cull = true;
	return LB200_OK;
}

void fillFrustum(CullFrustum* F, const lb200_shifted_frustum* f) {
	static const int point_of_plane[6] = {0, 4, 1, 0, 0, 2}; // geometry.cpp:134-142
	for (int i = 0; i < 6; ++i) {
		F->nx[i] = f->xs[i]; F->ny[i] = f->ys[i]; F->nz[i] = f->zs[i]; F->d[i] = f->ds[i];
		F->px[i] = f->points[point_of_plane[i]][0];
		F->py[i] = f->points[point_of_plane[i]][1];
		F->pz[i] = f->points[point_of_plane[i]][2];
	}
	F->ox = f->origin[0]; F->oy = f->origin[1]; F->oz = f->origin[2];
}

CullLaunch prepareLaunch(lb200_culling* cs, uint32_t* type_base, uint32_t resident, uint32_t chunk_bound) {
	const lb::CullingHost& h = cs->host;
	CullLaunch L;
	const uint32_t n_pages = livePages(cs);
	L.n_pages = n_pages;
	uint32_t acc = 0;
	for (int t = 0; t < 256; ++t) { type_base[t] = acc; acc += h.type_counts[t]; }
	const uint32_t r = cs->next_replica;
	cs->next_replica = (cs->next_replica + 1) % cs->replicas;
	L.off = (size_t)r * cs->dev_cap;
	static const bool no_mask = getenv("LB200_NO_PLANE_MASKING") != nullptr;
	L.plane_masking = (h.n_bad_radius == 0 && !no_mask && cs->launch_plane_masking != 0) ? 1u : 0u;
	// Programmatic stream serialization: the kernel's prologue (up to cudaGridDependencySynchronize: descriptor reads, classification, the
	// sphere tests of round 0, whose results sit in shared memory) only READS scene data.  Those arrays are written by flushPages alone, so
	// unless something was uploaded since the last cull the prologue may overlap the tail of whatever kernel precedes it on the stream —
	// for back-to-back views (main, shadow cascades, lights) that is the previous cull, which releases its dependents at its first
	// instruction.  The flag is sticky: whichever call uploaded (flush, set_many, ...), the first cull after it is launched plain.
	static const bool no_pdl = getenv("LB200_NO_PDL") != nullptr;
	L.pdl = !no_pdl && !cs->uploaded_since_last_cull;
	cs->uploaded_since_last_cull = false;
	// chunk = pages per block per round: spread the pages over every resident block, at most one classify thread per page.
	// lb200_culling_set_launch may force either: the kernels are correct for any grid (no co-residency, no grid barrier) and any chunk in
	// 1..chunk_bound, so a forced block count is capped by neither residency nor the work; the floor of 32 pages is a speed choice.
	const uint32_t spread = cs->launch_blocks > 0 ? (uint32_t)cs->launch_blocks : cs->launch_blocks < 0 ? (uint32_t)cs->grid : resident;
	uint32_t chunk = (n_pages + spread - 1) / spread;
	chunk = std::max(32u, std::min(chunk_bound, chunk));
	if (cs->launch_chunk) chunk = std::min((uint32_t)cs->launch_chunk, chunk_bound);
	L.chunk = chunk;
	L.blocks = cs->launch_blocks ? spread : std::max(1u, std::min(resident, (n_pages + chunk - 1) / chunk));
	return L;
}

void recordLaunch(lb200_culling* cs, const CullLaunch& L) {
	cs->last_blocks = L.blocks; cs->last_chunk = L.chunk;
	cs->last_rounds = (uint32_t)((L.n_pages + (uint64_t)L.blocks * L.chunk - 1) / ((uint64_t)L.blocks * L.chunk));
	cs->last_pdl = L.pdl ? 1 : 0; cs->last_plane_masking = (int)L.plane_masking;
}

int launchCull(lb200_culling* cs, const lb200_shifted_frustum* f, uint8_t type, const Exchange* xchg, cudaStream_t stream, const CullOutput* dest) {
	lb200_range range("culling"); // culling_system.cpp:330
	lb200_ctx* ctx = cs->ctx;
	int rc = flushPages(cs);
	if (rc) return rc;

	CullParams P = {}; // outside exchange mode the exchange fields stay zero / null
	fillFrustum(&P.f, f);
	const CullLaunch L = prepareLaunch(cs, P.type_base, (uint32_t)(stream || xchg ? cs->grid_lanes : cs->grid), MAX_CHUNK);
	memcpy(dest ? dest->type_base : cs->last_type_base, P.type_base, sizeof(P.type_base));
	P.n_pages = L.n_pages;
	P.type_filter = type;
	P.chunk = L.chunk;
	P.plane_masking = L.plane_masking;
	P.item_cap = cs->item_cap;
	const uint32_t lane = (uint32_t)((xchg ? (uint64_t)xchg->epoch : cs->seq) % cs->lanes);
	uint32_t* cur = cs->d_counters + ((size_t)lane * 2 + cs->lane_parity[lane]) * COUNTER_WORDS;
	uint32_t* nxt = cs->d_counters + ((size_t)lane * 2 + (cs->lane_parity[lane] ^ 1u)) * COUNTER_WORDS;
	uint32_t* out = cs->d_out_ids + (size_t)lane * (cs->d_out_ids.size() / cs->lanes);
	uint32_t* mask = cs->d_mask + (size_t)lane * (cs->d_mask.size() / cs->lanes);
	if (dest) { cur = dest->counters; nxt = dest->next_counters; out = dest->ids; mask = dest->mask; }
	P.n_buffers = 1;
	if (xchg) {
		P.n_ranks = (uint32_t)ctx->n_ranks;
		peerTargets(ctx, xchg->epoch, P.xdst, P.xflags);
		P.pub_epoch = xchg->pub_epoch; P.wait_epoch = xchg->wait_epoch; P.n_buffers = ctx->peer.n_buffers; P.rank = (uint32_t)ctx->rank;
		if (xchg->pub_epoch) for (int r = 0; r < ctx->n_ranks; ++r) P.xprev[r] = peerSlab(ctx, xchg->pub_epoch, r);
	}
	cudaLaunchAttribute attr;
	const cudaLaunchConfig_t cfg = launchConfig(L.blocks, CULL_THREADS, stream ? stream : ctx->stream, &attr, L.pdl);
	uint32_t* mask_arg = xchg ? (uint32_t*)nullptr : mask;
	LB200_CUDA(ctx, cudaLaunchKernelEx(&cfg, cull_pages_kernel, P, (const lb200_page_desc*)(cs->d_desc + L.off), (const float4*)(cs->d_spheres + L.off * PAGE_SLOTS),
		(const int*)(cs->d_entities + L.off * PAGE_SLOTS), out, cur, nxt, mask_arg));
	LB200_CHECK_LAUNCH(ctx);
	if (!dest) {
		cs->last_counters = cur; cs->last_out = out; cs->last_mask = mask_arg; // exchange culls keep their rows in the slabs
		cs->last_is_view = false;
		cs->lane_parity[lane] ^= 1u;
		if (!xchg) ++cs->seq;
		cs->last_pages = L.n_pages;
	}
	recordLaunch(cs, L);
	return LB200_OK;
}

int forkLanes(lb200_culling* cs) {
	lb200_ctx* ctx = cs->ctx;
	if (!cs->fork_event) {
		Stream streams[lb200_culling::MAX_LANES]; Event events[lb200_culling::MAX_LANES], fork;
		for (uint32_t l = 0; l < cs->lanes; ++l) {
			LB200_CUDA(ctx, cudaStreamCreateWithFlags(streams[l].create(), cudaStreamNonBlocking));
			LB200_CUDA(ctx, cudaEventCreateWithFlags(events[l].create(), cudaEventDisableTiming));
		}
		LB200_CUDA(ctx, cudaEventCreateWithFlags(fork.create(), cudaEventDisableTiming));
		for (uint32_t l = 0; l < cs->lanes; ++l) { cs->lane_stream[l] = std::move(streams[l]); cs->lane_event[l] = std::move(events[l]); }
		cs->fork_event = std::move(fork); // marks the lanes complete
	}
	LB200_CUDA(ctx, cudaEventRecord(cs->fork_event, ctx->stream));
	for (uint32_t l = 0; l < cs->lanes; ++l) LB200_CUDA(ctx, cudaStreamWaitEvent(cs->lane_stream[l], cs->fork_event, 0));
	return LB200_OK;
}

int joinLanes(lb200_culling* cs) {
	lb200_ctx* ctx = cs->ctx;
	for (uint32_t l = 0; l < cs->lanes; ++l) {
		LB200_CUDA(ctx, cudaEventRecord(cs->lane_event[l], cs->lane_stream[l]));
		LB200_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, cs->lane_event[l], 0));
	}
	return LB200_OK;
}

void fillResult(const lb200_culling* cs, const uint32_t* counters, const uint32_t* type_base, lb200_cull_result* res) {
	memset(res, 0, sizeof(*res));
	for (int t = 0; t < 256; ++t) {
		res->type_count[t] = counters[t];
		res->type_offset[t] = type_base[t];
		res->total += res->type_count[t];
		if (cs->host.type_counts[t]) res->n_types = t + 1;
	}
	res->pages_tested = counters[256 + ST_PAGES_TESTED];
	res->pages_inside = counters[256 + ST_PAGES_INSIDE];
	res->pages_outside = counters[256 + ST_PAGES_OUTSIDE];
	res->pages_filtered = counters[256 + ST_PAGES_FILTERED];
	res->entities_tested = counters[256 + ST_ENT_TESTED];
	res->entities_inside = counters[256 + ST_ENT_INSIDE];
}

int launchPack(lb200_culling* cs, const uint32_t* counters, uint32_t capacity, uint32_t* ids_dst, uint32_t* counters_dst, uint32_t counter_words, int blocks) {
	lb200_ctx* ctx = cs->ctx;
	PackParams PP;
	memcpy(PP.type_base, cs->last_type_base, sizeof(PP.type_base));
	PP.capacity = capacity;
	pack_kernel<<<blocks, 256, 0, ctx->stream>>>(PP, counters, cs->last_out, ids_dst, counters_dst, counter_words);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

} // namespace lbcull

namespace {

// h_counters (already on the host) -> cs->last / *result
void parseCounts(lb200_culling* cs, lb200_cull_result* result) {
	lb200_cull_result& res = cs->last;
	fillResult(cs, cs->h_counters, cs->last_type_base, &res);
	cs->has_last = true;
	// DESIGN.md §4.1: descriptor per page + 16 B per sphere the kernel reads (pages left to test after plane masking) + (4 B id read +
	// 4 B id write) per visible + 32 B mask per page
	const uint64_t streamed = cs->h_counters[256 + ST_ENT_STREAMED];
	cs->last_bytes = (uint64_t)cs->last_pages * 32 + streamed * 16 + (uint64_t)res.total * 8 + (uint64_t)cs->last_pages * 32;
	if (result) *result = res;
}

int readCounts(lb200_culling* cs, lb200_cull_result* result) {
	lb200_ctx* ctx = cs->ctx;
	const uint32_t* cur = cs->last_counters;
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_counters, cur, sizeof(uint32_t) * COUNTER_WORDS, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	parseCounts(cs, result);
	return LB200_OK;
}

// ids delivered to the host are dense, type after type (the pack kernel's layout, and the copies of the pageable path)
void denseOffsets(lb200_cull_result* result) {
	uint32_t off = 0;
	for (int t = 0; t < 256; ++t) { result->type_offset[t] = off; off += result->type_count[t]; }
}

// device address of a page-locked destination (lb200_host_alloc / cudaHostRegister) or null; *attr and *pe keep the query for an error text
uint32_t* pinnedDestination(const lb200_culling* cs, const uint32_t* out_ids, cudaPointerAttributes* attr, cudaError_t* pe) {
	*pe = cudaPointerGetAttributes(attr, out_ids);
	if (!cs->h_counters_dev || *pe != cudaSuccess || attr->type != cudaMemoryTypeHost || !attr->devicePointer) {
		cudaGetLastError(); // unregistered host memory makes cudaPointerGetAttributes fail on old drivers
		return nullptr;
	}
	return (uint32_t*)attr->devicePointer;
}

// the cull, then its counters and ids packed straight into page-locked host memory (dst: pinnedDestination)
int cullIntoPinned(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t* dst, uint32_t capacity) {
	const int rc = launchCull(cs, frustum, type);
	if (rc) return rc;
	return launchPack(cs, cs->last_counters, capacity, dst, cs->h_counters_dev, COUNTER_WORDS, cs->ctx->sm_count * 2);
}

// the counters cullIntoPinned delivered -> the caller's result
int pinnedResult(lb200_culling* cs, lb200_cull_result* result, uint32_t capacity) {
	parseCounts(cs, result);
	denseOffsets(result);
	return result->total > capacity ? LB200_ERR_CAPACITY : LB200_OK;
}

} // namespace

int lb200_culling_internal_last(lb200_culling* cs, const uint32_t** out_ids, const uint32_t** counters, const uint32_t** type_base, const uint32_t** type_counts) {
	if (!cs || !cs->ctx) return LB200_ERR_INVALID;
	if (!cs->last_counters) { lb200_set_error(cs->ctx, "no cull has been issued on this culling system yet"); return LB200_ERR_STATE; }
	*out_ids = cs->last_out; *counters = cs->last_counters; *type_base = cs->last_type_base; *type_counts = cs->host.type_counts;
	return LB200_OK;
}

// the device re-binning only moves entities the host mirror added, and a device add grows the host's entity -> slot table to its largest
// id (lb200_culling_add_many_device), so the table spans every id a cull can emit
uint32_t lb200_culling_internal_entity_range(const lb200_culling* cs) { return (uint32_t)cs->host.entity_to_slot.size(); }
lb200_ctx* lb200_culling_internal_ctx(const lb200_culling* cs) { return cs->ctx; }

extern "C" {

int lb200_culling_create(lb200_ctx* ctx, lb200_culling** out) {
	if (!out) return LB200_ERR_INVALID;
	if (ctx && cudaSetDevice(ctx->device) != cudaSuccess) { cudaGetLastError(); return LB200_ERR_CUDA; }
	*out = new (std::nothrow) lb200_culling(ctx);
	return *out ? LB200_OK : LB200_ERR_CUDA;
}

void lb200_culling_destroy(lb200_culling* cs) {
	if (!cs) return;
	if (cs->ctx) {
		cudaSetDevice(cs->ctx->device);
		cudaStreamSynchronize(cs->ctx->stream);
		for (uint32_t l = 0; l < lb200_culling::MAX_LANES; ++l) if (cs->lane_stream[l]) cudaStreamSynchronize(cs->lane_stream[l]);
	}
	delete cs;
}

int lb200_culling_add(lb200_culling* cs, int32_t entity, uint8_t type, const double pos[3], float radius) {
	LB200_HOST_VIEW(cs);
	if (!cs || !pos || type == LB200_TYPE_ALL) return LB200_ERR_INVALID;
	return cs->host.add(entity, type, pos, radius);
}
int lb200_culling_remove(lb200_culling* cs, int32_t entity) { LB200_HOST_VIEW(cs); return cs ? cs->host.remove(entity) : LB200_ERR_INVALID; }
int lb200_culling_set_position(lb200_culling* cs, int32_t entity, const double pos[3]) { LB200_HOST_VIEW(cs); return cs && pos ? cs->host.setPosition(entity, pos) : LB200_ERR_INVALID; }
int lb200_culling_set_radius(lb200_culling* cs, int32_t entity, float radius) { LB200_HOST_VIEW(cs); return cs ? cs->host.setRadius(entity, radius) : LB200_ERR_INVALID; }
int lb200_culling_set(lb200_culling* cs, int32_t entity, const double pos[3], float radius) { LB200_HOST_VIEW(cs); return cs && pos ? cs->host.set(entity, pos, radius) : LB200_ERR_INVALID; }
float lb200_culling_get_radius(const lb200_culling* cs, int32_t entity) {
	if (hostView(cs)) return 0.0f;
	return cs && cs->host.isAdded(entity) ? cs->host.getRadius(entity) : 0.0f;
}
int lb200_culling_is_added(const lb200_culling* cs, int32_t entity) {
	// device re-binning alone moves entities but keeps the set the mirror holds; device adds / removes change it, and then it is pulled back
	if (cs && cs->membership_on_device && hostView(cs)) return 0;
	return cs && cs->host.isAdded(entity) ? 1 : 0;
}

int lb200_culling_add_many(lb200_culling* cs, const int32_t* entities, const uint8_t* types, const double* pos3, const float* radius, uint32_t n) {
	LB200_HOST_VIEW(cs);
	if (!cs || (n && (!entities || !types || !pos3 || !radius))) return LB200_ERR_INVALID;
	for (uint32_t i = 0; i < n; ++i) {
		if (types[i] == LB200_TYPE_ALL) return LB200_ERR_INVALID;
		const int rc = cs->host.add(entities[i], types[i], pos3 + 3 * (size_t)i, radius[i]);
		if (rc) return rc;
	}
	return LB200_OK;
}
int lb200_culling_set_many(lb200_culling* cs, const int32_t* entities, const double* pos3, const float* radius, uint32_t n) {
	LB200_HOST_VIEW(cs);
	if (!cs || (n && (!entities || !pos3 || !radius))) return LB200_ERR_INVALID;
	for (uint32_t i = 0; i < n; ++i) {
		const int rc = cs->host.set(entities[i], pos3 + 3 * (size_t)i, radius[i]);
		if (rc) return rc;
	}
	return LB200_OK;
}
int lb200_culling_set_many_unique(lb200_culling* cs, const int32_t* entities, const double* pos3, const float* radius, uint32_t n) {
	LB200_HOST_VIEW(cs);
	if (!cs || (n && (!entities || !pos3 || !radius))) return LB200_ERR_INVALID;
	return cs->host.setManyUnique(entities, pos3, radius, n);
}

int lb200_culling_set_position_many(lb200_culling* cs, const int32_t* entities, const double* pos3, uint32_t n) {
	LB200_HOST_VIEW(cs);
	if (!cs || (n && (!entities || !pos3))) return LB200_ERR_INVALID;
	for (uint32_t i = 0; i < n; ++i) {
		const int rc = cs->host.setPosition(entities[i], pos3 + 3 * (size_t)i);
		if (rc) return rc;
	}
	return LB200_OK;
}
int lb200_culling_set_radius_many(lb200_culling* cs, const int32_t* entities, const float* radius, uint32_t n) {
	LB200_HOST_VIEW(cs);
	if (!cs || (n && (!entities || !radius))) return LB200_ERR_INVALID;
	for (uint32_t i = 0; i < n; ++i) {
		const int rc = cs->host.setRadius(entities[i], radius[i]);
		if (rc) return rc;
	}
	return LB200_OK;
}
int lb200_culling_remove_many(lb200_culling* cs, const int32_t* entities, uint32_t n) {
	LB200_HOST_VIEW(cs);
	if (!cs || (n && !entities)) return LB200_ERR_INVALID;
	for (uint32_t i = 0; i < n; ++i) cs->host.remove(entities[i]);
	return LB200_OK;
}

uint32_t lb200_culling_page_count(const lb200_culling* cs) {
	if (hostView(cs)) return 0;
	return cs ? (uint32_t)cs->host.cells.size() : 0;
}
uint32_t lb200_culling_entity_count(const lb200_culling* cs) { return cs ? cs->host.n_entities : 0; }

int lb200_culling_get_page(const lb200_culling* cs, uint32_t page, double origin[3], int32_t indices[3], uint8_t* type, uint8_t* is_big,
	uint32_t* count, float* spheres4, int32_t* entities)
{
	LB200_HOST_VIEW(cs);
	if (!cs || page >= cs->host.cells.size()) return LB200_ERR_INVALID;
	const lb::CullingHost& h = cs->host;
	const uint32_t p = h.cells[page];
	if (origin) memcpy(origin, h.desc[p].origin, sizeof(double) * 3);
	if (indices) { indices[0] = h.keys[p].x; indices[1] = h.keys[p].y; indices[2] = h.keys[p].z; }
	if (type) *type = h.desc[p].type;
	if (is_big) *is_big = h.desc[p].is_big;
	if (count) *count = h.desc[p].count;
	if (spheres4) memcpy(spheres4, h.spheres + 4 * PAGE_SLOTS * (size_t)p, sizeof(float) * 4 * h.desc[p].count);
	if (entities) memcpy(entities, h.entities + PAGE_SLOTS * (size_t)p, sizeof(int32_t) * h.desc[p].count);
	return LB200_OK;
}

int32_t lb200_culling_page_id(const lb200_culling* cs, uint32_t page) {
	if (hostView(cs)) return -1;
	return cs && page < cs->host.cells.size() ? (int32_t)cs->host.cells[page] : -1;
}

int lb200_culling_flush(lb200_culling* cs) {
	LB200_HOST_VIEW(cs);
	if (!cs) return LB200_ERR_INVALID;
	if (!cs->ctx) { return LB200_ERR_NO_DEVICE; }
	return flushPages(cs);
}

int lb200_culling_set_replicas(lb200_culling* cs, uint32_t replicas) {
	LB200_HOST_VIEW(cs);
	if (!cs || replicas < 1 || replicas > 64) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (replicas == cs->replicas) return LB200_OK;
	LB200_CUDA(cs->ctx, cudaStreamSynchronize(cs->ctx->stream));
	releaseViews(cs);
	cs->replicas = replicas;
	cs->next_replica = 0;
	cs->dev_cap = 0; // forces reallocation + full upload at the next flush (resizePages, discarding)
	return LB200_OK;
}

int lb200_culling_cull_device(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, const uint32_t** out_dev_ids,
	lb200_cull_result* result, int want_counts)
{
	if (!cs || !frustum) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (noEntities(cs)) { // culling_system.cpp:322
		if (result) memset(result, 0, sizeof(*result));
		if (out_dev_ids) *out_dev_ids = nullptr;
		memset(&cs->last, 0, sizeof(cs->last));
		return LB200_OK;
	}
	int rc = launchCull(cs, frustum, type);
	if (rc) return rc;
	if (out_dev_ids) *out_dev_ids = cs->last_out;
	if (want_counts) rc = readCounts(cs, result);
	else cs->has_last = false;
	return rc;
}

int lb200_culling_cull_device_n(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t n) {
	if (!cs || !frustum) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (noEntities(cs)) return LB200_OK;
	cs->has_last = false;
	int rc = flushPages(cs); // uploads (if any) go to the context stream before the lanes fork from it
	if (rc) return rc;
	const uint32_t L = std::min(cs->lanes, n);
	if (L < 2) {
		for (uint32_t i = 0; i < n; ++i) {
			rc = launchCull(cs, frustum, type);
			if (rc) return rc;
		}
		return LB200_OK;
	}
	// independent views: consecutive culls go to different streams and different output lanes, so the device overlaps them freely;
	// culls of one lane share buffers and stay ordered on their stream.  Fork from / join into the context stream.
	rc = forkLanes(cs);
	if (rc) return rc;
	for (uint32_t i = 0; i < n; ++i) {
		rc = launchCull(cs, frustum, type, nullptr, cs->lane_stream[cs->seq % cs->lanes]);
		if (rc) return rc;
	}
	return joinLanes(cs);
}

// ---- asynchronous form of lb200_culling_cull for callers that must not block their thread (the engine calls cull from job-system
// fibers, src/renderer/pipeline.cpp:1036-1041: begin, then jobs::yield() while poll says "running", then end) ----
int lb200_culling_cull_begin(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t* out_ids, uint32_t capacity) {
	if (!cs || !frustum || !out_ids || !capacity) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	if (cs->pending) { lb200_set_error(ctx, "cull_begin: the previous cull_begin has not been ended"); return LB200_ERR_STATE; }
	if (noEntities(cs)) { lb200_set_error(ctx, "cull_begin on an empty culling system (cull() handles that case)"); return LB200_ERR_STATE; }
	int rc = ensureDevice(cs);
	if (rc) return rc;
	cudaPointerAttributes attr = {};
	cudaError_t pe;
	uint32_t* dst = pinnedDestination(cs, out_ids, &attr, &pe);
	if (!dst) {
		lb200_set_error(ctx, "cull_begin needs a page-locked destination (lb200_host_alloc): cudaPointerGetAttributes -> %s, memory type %d, device pointer %p, counters mapped %d",
			cudaGetErrorString(pe), (int)attr.type, attr.devicePointer, cs->h_counters_dev ? 1 : 0);
		return LB200_ERR_INVALID;
	}
	if (!cs->done_event) LB200_CUDA(ctx, cudaEventCreateWithFlags(cs->done_event.create(), cudaEventDisableTiming));
	rc = cullIntoPinned(cs, frustum, type, dst, capacity);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaEventRecord(cs->done_event, ctx->stream));
	cs->pending = true;
	cs->pending_capacity = capacity;
	cs->has_last = false;
	return LB200_OK;
}

int lb200_culling_cull_poll(lb200_culling* cs) {
	if (!cs || !cs->ctx) return LB200_ERR_INVALID;
	if (!cs->pending) return 1;
	const cudaError_t e = cudaEventQuery(cs->done_event);
	if (e == cudaSuccess) return 1;
	if (e == cudaErrorNotReady) { cudaGetLastError(); return 0; }
	lb200_set_error(cs->ctx, "cudaEventQuery failed: %s", cudaGetErrorString(e));
	return LB200_ERR_CUDA;
}

int lb200_culling_cull_end(lb200_culling* cs, lb200_cull_result* result) {
	if (!cs || !result) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	if (!cs->pending) { lb200_set_error(ctx, "cull_end without cull_begin"); return LB200_ERR_STATE; }
	cs->pending = false;
	LB200_CUDA(ctx, cudaEventSynchronize(cs->done_event));
	return pinnedResult(cs, result, cs->pending_capacity);
}

int lb200_culling_last_result(lb200_culling* cs, const uint32_t** out_dev_ids, lb200_cull_result* result) {
	if (!cs) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (!cs->last_counters) { lb200_set_error(cs->ctx, "last_result needs a preceding cull"); return LB200_ERR_STATE; }
	if (out_dev_ids) *out_dev_ids = cs->last_out;
	return readCounts(cs, result);
}

int lb200_culling_cull(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t* out_ids, uint32_t capacity,
	lb200_cull_result* result)
{
	if (!cs || !frustum || !result) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	// Destination in page-locked host memory (lb200_host_alloc / cudaHostAlloc / cudaHostRegister): the device writes the result there
	// itself — one launch behind the cull, one synchronisation, no count round trip.  Pageable destinations take the copy path below.
	static const bool no_direct = getenv("LB200_CULL_HOST_MEMCPY") != nullptr;
	if (!no_direct && out_ids && capacity && !noEntities(cs) && ensureDevice(cs) == LB200_OK && cs->h_counters_dev) {
		cudaPointerAttributes attr = {};
		cudaError_t pe;
		if (uint32_t* dst = pinnedDestination(cs, out_ids, &attr, &pe)) {
			const int rc = cullIntoPinned(cs, frustum, type, dst, capacity);
			if (rc) return rc;
			LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
			return pinnedResult(cs, result, capacity);
		}
	}
	lb200_cull_result dev;
	const uint32_t* d_ids = nullptr;
	int rc = lb200_culling_cull_device(cs, frustum, type, &d_ids, &dev, 1);
	if (rc) return rc;
	*result = dev;
	denseOffsets(result);
	if (dev.total > capacity || (dev.total && !out_ids)) return LB200_ERR_CAPACITY;
	for (int t = 0; t < 256; ++t) {
		if (!dev.type_count[t]) continue;
		LB200_CUDA(ctx, cudaMemcpyAsync(out_ids + result->type_offset[t], d_ids + dev.type_offset[t], sizeof(uint32_t) * dev.type_count[t], cudaMemcpyDeviceToHost, ctx->stream));
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

int lb200_culling_read_bitmask(lb200_culling* cs, uint32_t* out_words, uint32_t capacity_words) {
	LB200_HOST_VIEW(cs);
	if (!cs || !out_words) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	// bitmask is indexed by page id; report it in m_cells order like lb200_culling_get_page
	const lb::CullingHost& h = cs->host;
	const size_t n = h.cells.size();
	if (capacity_words < n * 8) return LB200_ERR_CAPACITY;
	if (!cs->last_pages) { lb200_set_error(cs->ctx, "read_bitmask needs a preceding cull"); return LB200_ERR_STATE; }
	if (!cs->last_mask) { lb200_set_error(cs->ctx, "the last cull was an exchange step: its visibility rows are in the exchanged slabs"); return LB200_ERR_STATE; }
	std::vector<uint32_t> tmp((size_t)cs->last_pages * 8);
	LB200_CUDA(cs->ctx, cudaMemcpyAsync(tmp.data(), cs->last_mask, sizeof(uint32_t) * tmp.size(), cudaMemcpyDeviceToHost, cs->ctx->stream));
	LB200_CUDA(cs->ctx, cudaStreamSynchronize(cs->ctx->stream));
	for (size_t i = 0; i < n; ++i) {
		const uint32_t p = h.cells[i];
		if (p >= cs->last_pages) { memset(out_words + 8 * i, 0, sizeof(uint32_t) * 8); continue; } // page created after the last cull
		memcpy(out_words + 8 * i, tmp.data() + 8 * (size_t)p, sizeof(uint32_t) * 8);
	}
	return LB200_OK;
}

// Device time of ONE cull that has the device to itself (the latency of a lone view): per iteration a short delay kernel, then
// event / cull / event enqueued while it runs, so the interval holds no host launch latency and nothing overlaps the cull.
// mode 0: the cull; 1: nothing between the events (what the two event records cost by themselves); 2: one empty kernel of the cull's
// grid (the fixed cost of any kernel launch).  CUDA events tick in ~1 us steps.
int lb200_culling_time_lone_cull(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t iters, int mode, float* out_ms) {
	if (!cs || !frustum || !out_ms || !iters || mode < 0 || mode > 2) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	if (noEntities(cs)) return LB200_ERR_STATE;
	int rc = flushPages(cs);
	if (rc) return rc;
	Event e0, e1;
	LB200_CUDA(ctx, cudaEventCreate(e0.create()));
	LB200_CUDA(ctx, cudaEventCreate(e1.create()));
	for (uint32_t i = 0; i < iters; ++i) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		delay_kernel<<<1, 32, 0, ctx->stream>>>(200000); // ~100 us
		LB200_CHECK_LAUNCH(ctx);
		LB200_CUDA(ctx, cudaEventRecord(e0, ctx->stream));
		if (mode == 2) delay_kernel<<<cs->grid, CULL_THREADS, 0, ctx->stream>>>(0);
		else if (mode == 0) rc = launchCull(cs, frustum, type);
		if (rc) break;
		LB200_CUDA(ctx, cudaEventRecord(e1, ctx->stream));
		LB200_CUDA(ctx, cudaEventSynchronize(e1));
		LB200_CUDA(ctx, cudaEventElapsedTime(&out_ms[i], e0, e1));
	}
	cs->has_last = false;
	return rc;
}

uint64_t lb200_culling_last_algorithmic_bytes(const lb200_culling* cs) { return cs && cs->has_last ? cs->last_bytes : 0; }

int lb200_culling_set_launch(lb200_culling* cs, int blocks, int chunk, int plane_masking) {
	if (!cs) return LB200_ERR_INVALID;
	if (blocks < -1 || blocks > LB200_CULL_MAX_BLOCKS) { lb200_set_error(cs->ctx, "set_launch: blocks %d is not -1, 0 or a block count up to %d", blocks, LB200_CULL_MAX_BLOCKS); return LB200_ERR_INVALID; }
	if (chunk < 0 || chunk > MAX_CHUNK) { lb200_set_error(cs->ctx, "set_launch: chunk %d is not 0 or 1..%d", chunk, MAX_CHUNK); return LB200_ERR_INVALID; }
	if (plane_masking != -1 && plane_masking != 0) { lb200_set_error(cs->ctx, "set_launch: plane_masking %d is not -1 or 0", plane_masking); return LB200_ERR_INVALID; }
	cs->launch_blocks = blocks;
	cs->launch_chunk = chunk;
	cs->launch_plane_masking = plane_masking;
	return LB200_OK;
}

int lb200_culling_get_launch(lb200_culling* cs, uint32_t* blocks, uint32_t* chunk, uint32_t* rounds, int* pdl, int* plane_masking) {
	if (!cs) return LB200_ERR_INVALID;
	if (blocks) *blocks = cs->last_blocks;
	if (chunk) *chunk = cs->last_chunk;
	if (rounds) *rounds = cs->last_rounds;
	if (pdl) *pdl = cs->last_pdl;
	if (plane_masking) *plane_masking = cs->last_plane_masking;
	return LB200_OK;
}

} // extern "C"
