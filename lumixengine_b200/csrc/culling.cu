// GPU CullingSystem: host side + C-ABI (include/lumix_b200.h "CullingSystem").
//
// Replaces CullingSystemImpl::cullInternal + doCulling (src/renderer/culling_system.cpp:260-369).  The cull itself is one kernel,
// cull_pages_kernel (cull_kernel.cuh, which describes its phases); this file holds the page upload, the launches, the result delivery
// and the multi-GPU exchange kernels around it.
#include "cull_kernel.cuh"
#include "culling_host.hpp"
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

// 256 per-type counts -> exclusive offsets + compact list of the non-empty types (block of 256 threads)
__device__ __forceinline__ void scan_types(const uint32_t* __restrict__ counters, uint32_t* s_cnt, uint32_t* s_off, uint32_t* s_list, uint32_t* s_nnz) {
	__shared__ uint32_t s_warp[8];
	const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
	const uint32_t c = counters[tid];
	uint32_t x = c;
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
		if (lane >= (uint32_t)d) x += y;
	}
	if (lane == 31) s_warp[warp] = x;
	if (tid == 0) *s_nnz = 0;
	__syncthreads();
	uint32_t base = 0;
	for (uint32_t w = 0; w < warp; ++w) base += s_warp[w];
	s_cnt[tid] = c;
	s_off[tid] = base + x - c;
	if (tid == 255) s_off[256] = base + x;
	if (c) s_list[atomicAdd(s_nnz, 1u)] = tid;
	__syncthreads();
}

// Pack this rank's visible ids (per-type segments of out_ids) behind a 256-word header of per-type counts: the send slab of the
// multi-GPU exchange.  Reads the counters on the device: no host round trip between the cull and the all-gather.
struct PackParams { uint32_t type_base[256]; uint32_t slab_ids; };

__global__ void __launch_bounds__(256) pack_slab_kernel(const __grid_constant__ PackParams P, const uint32_t* __restrict__ counters,
	const uint32_t* __restrict__ out_ids, uint32_t* __restrict__ slab)
{
	__shared__ uint32_t s_cnt[256];
	__shared__ uint32_t s_off[257];
	__shared__ uint32_t s_list[256];
	__shared__ uint32_t s_nnz;
	scan_types(counters, s_cnt, s_off, s_list, &s_nnz);
	if (blockIdx.x == 0) slab[threadIdx.x] = s_cnt[threadIdx.x];
	const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, gsize = gridDim.x * blockDim.x;
	for (uint32_t k = 0; k < s_nnz; ++k) {
		const uint32_t t = s_list[k];
		const uint32_t c = s_cnt[t];
		const uint32_t* src = out_ids + P.type_base[t];
		const uint32_t off = s_off[t];
		for (uint32_t i = gtid; i < c; i += gsize) if (off + i < P.slab_ids) slab[256 + off + i] = src[i];
	}
}

// Result of one cull straight into page-locked HOST memory (lb200_culling_cull with a pinned destination): all counters into
// host_counters, the visible ids packed type after type into host_ids — posted writes over PCIe while the copy engine stays idle, and no
// count round trip between the cull and the transfer.  Ids beyond `slab_ids` (the caller's capacity) are dropped; the host sees the
// counts and reports LB200_ERR_CAPACITY.
__global__ void __launch_bounds__(256) pack_host_kernel(const __grid_constant__ PackParams P, const uint32_t* __restrict__ counters,
	const uint32_t* __restrict__ out_ids, uint32_t* __restrict__ host_ids, uint32_t* __restrict__ host_counters)
{
	__shared__ uint32_t s_cnt[256];
	__shared__ uint32_t s_off[257];
	__shared__ uint32_t s_list[256];
	__shared__ uint32_t s_nnz;
	scan_types(counters, s_cnt, s_off, s_list, &s_nnz);
	if (blockIdx.x == 0) for (uint32_t i = threadIdx.x; i < (uint32_t)COUNTER_WORDS; i += blockDim.x) host_counters[i] = counters[i];
	const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, gsize = gridDim.x * blockDim.x;
	for (uint32_t k = 0; k < s_nnz; ++k) {
		const uint32_t t = s_list[k];
		const uint32_t c = s_cnt[t];
		const uint32_t* src = out_ids + P.type_base[t];
		const uint32_t off = s_off[t];
		for (uint32_t i = gtid; i < c; i += gsize) if (off + i < P.slab_ids) host_ids[off + i] = src[i];
	}
}

// Fused pack + NVLink push: the slab is written straight into every rank's gather buffer through peer-mapped pointers (P2P stores
// over NVSwitch), then the last block publishes this rank's epoch in every rank's flag block.  No NCCL call on the per-frame path.
struct PushParams {
	uint32_t type_base[256];
	uint32_t slab_ids;
	uint32_t n_ranks, rank, epoch, n_buffers;
	uint32_t* dst[LB200_MAX_RANKS];   // rank r's gather buffer of this epoch, already offset to MY slab inside it
	uint32_t* flags[LB200_MAX_RANKS]; // rank r's flag block: [2][LB200_MAX_RANKS]
};

__global__ void __launch_bounds__(256) pack_push_kernel(const __grid_constant__ PushParams P, const uint32_t* __restrict__ counters,
	const uint32_t* __restrict__ out_ids, uint32_t* __restrict__ done_counter)
{
	__shared__ uint32_t s_cnt[256];
	__shared__ uint32_t s_off[257];
	__shared__ uint32_t s_list[256];
	__shared__ uint32_t s_nnz;
	__shared__ bool s_last;
	scan_types(counters, s_cnt, s_off, s_list, &s_nnz);
	if (blockIdx.x == 0) for (uint32_t r = 0; r < P.n_ranks; ++r) P.dst[r][threadIdx.x] = s_cnt[threadIdx.x];
	const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x, gsize = gridDim.x * blockDim.x;
	for (uint32_t k = 0; k < s_nnz; ++k) {
		const uint32_t t = s_list[k];
		const uint32_t c = s_cnt[t];
		const uint32_t* src = out_ids + P.type_base[t];
		const uint32_t off = s_off[t];
		const uint32_t lim = min(c, P.slab_ids > off ? P.slab_ids - off : 0u);
		if (((P.type_base[t] ^ off) & 3u) == 0) {
			// source and destination share their 16-byte phase: scalar head, 128-bit body, scalar tail
			const uint32_t head = min(lim, (4u - (off & 3u)) & 3u);
			if (gtid < head) { const uint32_t v = src[gtid]; for (uint32_t r = 0; r < P.n_ranks; ++r) P.dst[r][256 + off + gtid] = v; }
			const uint32_t n4 = (lim - head) / 4;
			const uint4* src4 = reinterpret_cast<const uint4*>(src + head);
			// four 128-bit loads in flight per thread before the peer stores: the stores are posted, the loads are what a thread waits for
			for (uint32_t i0 = gtid; i0 < n4; i0 += 4 * gsize) {
				uint4 v[4];
#pragma unroll
				for (int u = 0; u < 4; ++u) { const uint32_t i = i0 + u * gsize; if (i < n4) v[u] = src4[i]; }
#pragma unroll
				for (int u = 0; u < 4; ++u) {
					const uint32_t i = i0 + u * gsize;
					if (i < n4) for (uint32_t r = 0; r < P.n_ranks; ++r) reinterpret_cast<uint4*>(P.dst[r] + 256 + off + head)[i] = v[u];
				}
			}
			const uint32_t done = head + 4 * n4;
			if (gtid < lim - done) { const uint32_t v = src[done + gtid]; for (uint32_t r = 0; r < P.n_ranks; ++r) P.dst[r][256 + off + done + gtid] = v; }
		}
		else {
			for (uint32_t i = gtid; i < lim; i += gsize) {
				const uint32_t v = src[i];
				for (uint32_t r = 0; r < P.n_ranks; ++r) P.dst[r][256 + off + i] = v;
			}
		}
	}
	// publish: all stores of all blocks must be visible system-wide before the flag
	__threadfence_system();
	__syncthreads();
	if (threadIdx.x == 0) s_last = atomicAdd(done_counter, 1u) == gridDim.x - 1;
	__syncthreads();
	if (s_last) {
		__threadfence_system();
		if (threadIdx.x < P.n_ranks) {
			volatile uint32_t* f = P.flags[threadIdx.x] + (P.epoch % P.n_buffers) * LB200_MAX_RANKS + P.rank;
			*f = P.epoch;
		}
		if (threadIdx.x == 0) *done_counter = 0;
	}
}

// Wait until every rank's slab of `epoch` has landed in this rank's gather buffer.  Spins on local memory; gives up after ~4 s.
__global__ void wait_peers_kernel(const uint32_t* flags, uint32_t n_ranks, uint32_t epoch, uint32_t n_buffers, uint32_t* timed_out) {
	// Launched with programmatic stream serialization behind the kernel that publishes this rank's flag, and releasing its own
	// dependents at once: the next cull's read-only prologue runs while this block spins.  Its own flag is among the awaited ones,
	// so the wait cannot end before the local producer has published; the grid dependency below covers that kernel's last stores.
	cudaTriggerProgrammaticLaunchCompletion();
	if (threadIdx.x < n_ranks) {
		const volatile uint32_t* f = flags + (epoch % n_buffers) * LB200_MAX_RANKS + threadIdx.x;
		const long long t0 = clock64();
		while ((int)(*f - epoch) < 0) {
			if (clock64() - t0 > 8000000000ll) { *timed_out = 1; break; }
		}
	}
	cudaGridDependencySynchronize();
	__threadfence_system();
}

// Second half of an exchange step (lb200_culling_cull_exchange): runs behind the cull kernel that stored this rank's mask rows into
// every rank's slab.  Once that grid has completed (its peer stores are performed, its counters final) one block sends the slab
// header, fences ONCE at system scope and raises this rank's epoch flag everywhere, then holds the stream until every rank's flag of
// this epoch is here.  Launched with programmatic stream serialization and releasing its own dependents at once: the next cull of
// the stream runs its read-only prologue meanwhile.
struct PublishParams {
	uint32_t n_ranks, rank, epoch, n_buffers;
	uint32_t n_pages, item_cap;
	uint32_t* dst[LB200_MAX_RANKS];   // rank r's exchange buffer of this epoch, already offset to MY slab inside it
	uint32_t* flags[LB200_MAX_RANKS]; // rank r's flag block: [n_buffers][LB200_MAX_RANKS]
};

__global__ void __launch_bounds__(288) publish_wait_kernel(const __grid_constant__ PublishParams P, const uint32_t* counters, uint32_t* timed_out) {
	cudaTriggerProgrammaticLaunchCompletion();
	cudaGridDependencySynchronize();
	const uint32_t i = threadIdx.x;
	if (i < XHEADER_WORDS) {
		uint32_t v = 0;
		if (i < 256) v = __ldcg(counters + i);
		else if (i == 256) v = P.n_pages;
		else if (i == 257) v = __ldcg(counters + CNT_N_REC);
		else if (i == 259) v = P.item_cap;
		for (uint32_t r = 0; r < P.n_ranks; ++r) P.dst[r][i] = v;
	}
	// release: everything that happened before the flag store — the work grid's records (ordered before us by the grid dependency) and
	// the header just written by all threads of this block (barrier, then a system-scope fence by the storing threads) — is visible to
	// whoever observes the flag
	__threadfence_system();
	__syncthreads();
	if (i < P.n_ranks) {
		__threadfence_system();
		volatile uint32_t* f = P.flags[i] + (P.epoch % P.n_buffers) * LB200_MAX_RANKS + P.rank;
		*f = P.epoch;
		const volatile uint32_t* mine = P.flags[P.rank] + (P.epoch % P.n_buffers) * LB200_MAX_RANKS + i;
		const long long t0 = clock64();
		while ((int)(*mine - P.epoch) < 0) {
			if (clock64() - t0 > 8000000000ll) { *timed_out = 1; break; }
		}
	}
	__threadfence_system();
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

struct lb200_culling {
	lb200_culling(lb200_ctx* c) : ctx(c), host(c ? pinnedAlloc : plainAlloc, c ? pinnedFree : plainFree) {}
	lb200_ctx* ctx;
	lb::CullingHost host;

	// HBM mirror
	uint32_t dev_cap = 0; // pages per replica: d_spheres, d_entities and d_desc hold replicas x dev_cap pages, d_mask lanes x dev_cap rows
	uint32_t replicas = 1;
	uint32_t next_replica = 0;
	DeviceArray<float4> d_spheres;
	DeviceArray<int> d_entities;
	DeviceArray<lb200_page_desc> d_desc;
	// Output lanes: a cull on lane l writes ids to d_out_ids[l], mask rows to d_mask[l], counts to one of lane l's two counter buffers
	// and zeroes the other one for the lane's next cull.  Plain culls take lane seq % lanes, exchange culls lane epoch % lanes.  Culls
	// of one lane are always ordered (same stream inside a batch; batches fork from / join into the context stream, single culls run
	// on it); culls of different lanes share nothing they write and may run concurrently (cull_device_n, cull_exchange_n).
	static constexpr uint32_t MAX_LANES = LB200_MAX_LANES;
	uint32_t lanes = 3;
	uint8_t lane_parity[MAX_LANES] = {};
	Stream lane_stream[MAX_LANES];
	Event lane_event[MAX_LANES];
	Event fork_event; // created with the lanes' streams and events (forkLanes)
	// fused exchange steps (lb200_culling_cull_exchange_n): the epoch of the lane's previous step, whose publish has not been issued yet
	// (0 = none), and the counters of the lane's last cull (the closing publish reads them)
	uint32_t lane_owed[MAX_LANES] = {};
	uint32_t* lane_last_counters[MAX_LANES] = {};
	uint64_t seq = 0;
	DeviceArray<uint32_t> d_out_ids; // lanes equal parts
	DeviceArray<uint32_t> d_mask;    // lanes equal parts; row of page p = words [8p, 8p + 8) of a part
	uint32_t item_cap = 0; // record capacity of an exchange slab
	bool uploaded_since_last_cull = true; // the next cull's kernels are launched plain (no programmatic overlap with the upload)
	DeviceArray<uint32_t> d_counters; // lanes * 2 * COUNTER_WORDS: [lane][parity]
	// asynchronous host delivery (lb200_culling_cull_begin / _poll / _end)
	Event done_event;
	bool pending = false;
	uint32_t pending_capacity = 0;
	// the cull issued last
	uint32_t* last_counters = nullptr;
	uint32_t* last_out = nullptr;
	uint32_t* last_mask = nullptr;
	PinnedArray<uint32_t, cudaHostAllocMapped> h_counters; // COUNTER_WORDS, allocated and released with d_counters
	uint32_t* h_counters_dev = nullptr; // the same memory as the device addresses it (null: no direct host writes)
	int grid = 0;       // resident blocks of a cull that has the device to itself
	int grid_lanes = 0; // resident blocks of a cull issued by cull_device_n (runs next to its neighbours)
	int threads = 256;
	// staging for sparse dirty uploads, the same size on both sides, allocated and released together
	PinnedArray<uint8_t> h_stage;
	DeviceArray<uint8_t> d_stage;
	// multi-GPU gather buffers
	DeviceArray<uint32_t> d_gather_ids;
	DeviceArray<uint32_t> d_slab;

	// ---- device-side re-binning (lb200_culling_set_many_device, SURVEY 8f N3) ----
	// While `device_authoritative`, the page arrays in HBM are ahead of the host mirror (entities were re-binned by kernels); any host-side
	// accessor or mutator first pulls the device state back (syncHostFromDevice).
	bool device_authoritative = false;
	uint64_t rebin_built_gen = ~0ull;   // host.edit_gen the device-side tables were built from
	// Each group below is allocated and released as a whole (ensureRebinState, lb200_culling_set_many_device).
	DeviceArray<uint32_t> d_entity_to_slot;
	// per-page side arrays, dev_cap pages each
	DeviceArray<int4> d_page_cell;          // per page: cell indices x, y, z, type | is_big << 8
	DeviceArray<uint32_t> d_free_pages;     // stack of free page ids
	DeviceArray<uint32_t> d_page_dirty, d_dirty_pages;
	DeviceArray<unsigned long long> d_hash_keys; DeviceArray<uint32_t> d_hash_vals; // packed cell key -> open page of its chain
	DeviceArray<uint32_t> d_rebin_counters; PinnedArray<uint32_t> h_rebin_counters; // RB_* below; pinned mirror
	DeviceArray<uint8_t> d_rb_sort_state; DeviceArray<uint32_t> d_rb_block_hist; uint32_t rb_sort_blocks = 0;
	// per changer slot
	DeviceArray<uint32_t> d_changers;       // mover indices that change cell / chain
	DeviceArray<uint4> d_rb_plans;          // one RunPlan per changer slot (used at the first index of every run)
	DeviceArray<uint64_t> d_rb_keys[2], d_rb_vals[2];
	uint32_t dev_high_water = 0;        // pages [0, dev_high_water) may be in use on the device

	uint32_t last_type_base[256];
	lb200_cull_result last = {};
	bool has_last = false;
	uint64_t last_bytes = 0;
	uint32_t last_pages = 0;
};

namespace {

int syncHostFromDevice(lb200_culling* cs);
// pages the kernels have to look at: the host's high-water mark, or the device's own while it is ahead of the host mirror
inline uint32_t livePages(const lb200_culling* cs) { return cs->device_authoritative ? cs->dev_high_water : cs->host.high_water; }
#define LB200_HOST_VIEW(cs)                                               \
	do {                                                                  \
		if ((cs) && (cs)->device_authoritative) {                         \
			const int rc__ = syncHostFromDevice(cs);                      \
			if (rc__) return rc__;                                        \
		}                                                                 \
	} while (0)

int ensureDevice(lb200_culling* cs) {
	lb200_ctx* ctx = cs->ctx;
	lb::CullingHost& h = cs->host;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!cs->d_counters || !cs->h_counters) { // the launch shape comes first: once the counters exist, it is set
		cs->lanes = lb200_cull_lanes();
		cs->threads = CULL_THREADS;
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
		uint32_t cap = cs->dev_cap ? cs->dev_cap : 1024;
		while (cap < h.high_water) cap *= 2;
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_spheres.reset(); cs->d_entities.reset(); cs->d_desc.reset(); cs->d_mask.reset(); // before the new ones are allocated
		cs->dev_cap = 0; // until the four arrays are back
		const size_t R = cs->replicas;
		DeviceArray<float4> spheres; DeviceArray<int> entities; DeviceArray<lb200_page_desc> desc; DeviceArray<uint32_t> mask;
		LB200_CUDA(ctx, spheres.alloc(PAGE_SLOTS * (size_t)cap * R));
		LB200_CUDA(ctx, entities.alloc(PAGE_SLOTS * (size_t)cap * R));
		LB200_CUDA(ctx, desc.alloc((size_t)cap * R));
		LB200_CUDA(ctx, mask.alloc(8 * (size_t)cap * cs->lanes));
		// free / never-used pages must read count == 0
		LB200_CUDA(ctx, cudaMemsetAsync(desc, 0, sizeof(lb200_page_desc) * (size_t)cap * R, ctx->stream));
		cs->d_spheres = std::move(spheres); cs->d_entities = std::move(entities); cs->d_desc = std::move(desc); cs->d_mask = std::move(mask);
		cs->item_cap = cap; // every page can end up with a record
		cs->dev_cap = cap;
		h.all_dirty = true;
	}
	const size_t out_cap = cs->d_out_ids.size() / cs->lanes;
	if (out_cap < h.n_entities || !cs->d_out_ids) {
		uint32_t cap = out_cap ? (uint32_t)out_cap : 4096;
		while (cap < h.n_entities) cap *= 2;
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_out_ids.reset();
		LB200_CUDA(ctx, cs->d_out_ids.alloc((size_t)cap * cs->lanes));
	}
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
			size_t cap = stage_pages ? stage_pages : 256;
			while (cap < m) cap *= 2;
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

struct Exchange { uint32_t epoch; uint32_t pub_epoch = 0, wait_epoch = 0; }; // non-null: store {page, row} records + counts into every rank's slab (peer memory); lane = epoch % lanes; pub / wait: fused steps (cull_kernel.cuh)

// words one rank contributes to a bitmask exchange step: header + page ids + rows (cull_kernel.cuh)
size_t exchangeSlabWords(const lb200_culling* cs) { return XHEADER_WORDS + 9 * (size_t)cs->item_cap; }

int launchCull(lb200_culling* cs, const lb200_shifted_frustum* f, uint8_t type, const Exchange* xchg = nullptr, cudaStream_t stream = nullptr) {
	lb200_range range("culling"); // culling_system.cpp:330
	lb200_ctx* ctx = cs->ctx;
	lb::CullingHost& h = cs->host;
	int rc = flushPages(cs);
	if (rc) return rc;

	CullParams P;
	static const int point_of_plane[6] = {0, 4, 1, 0, 0, 2}; // geometry.cpp:134-142
	for (int i = 0; i < 6; ++i) {
		P.nx[i] = f->xs[i]; P.ny[i] = f->ys[i]; P.nz[i] = f->zs[i]; P.d[i] = f->ds[i];
		P.px[i] = f->points[point_of_plane[i]][0];
		P.py[i] = f->points[point_of_plane[i]][1];
		P.pz[i] = f->points[point_of_plane[i]][2];
	}
	P.ox = f->origin[0]; P.oy = f->origin[1]; P.oz = f->origin[2];
	const uint32_t n_pages = livePages(cs);
	P.n_pages = n_pages;
	P.type_filter = type;
	P.item_cap = cs->item_cap;
	uint32_t acc = 0;
	for (int t = 0; t < 256; ++t) { P.type_base[t] = acc; acc += h.type_counts[t]; }
	memcpy(cs->last_type_base, P.type_base, sizeof(P.type_base));

	const uint32_t r = cs->next_replica;
	cs->next_replica = (cs->next_replica + 1) % cs->replicas;
	const size_t off = (size_t)r * cs->dev_cap;
	const uint32_t lane = (uint32_t)((xchg ? (uint64_t)xchg->epoch : cs->seq) % cs->lanes);
	uint32_t* cur = cs->d_counters + ((size_t)lane * 2 + cs->lane_parity[lane]) * COUNTER_WORDS;
	uint32_t* nxt = cs->d_counters + ((size_t)lane * 2 + (cs->lane_parity[lane] ^ 1u)) * COUNTER_WORDS;
	uint32_t* out = cs->d_out_ids + (size_t)lane * (cs->d_out_ids.size() / cs->lanes);
	uint32_t* mask = cs->d_mask + (size_t)lane * (cs->d_mask.size() / cs->lanes);
	P.n_ranks = 0;
	for (int r = 0; r < LB200_MAX_RANKS; ++r) P.xdst[r] = nullptr;
	P.pub_epoch = 0; P.wait_epoch = 0; P.n_buffers = 1; P.rank = 0;
	for (int r = 0; r < LB200_MAX_RANKS; ++r) { P.xprev[r] = nullptr; P.xflags[r] = nullptr; }
	if (xchg) {
		lb200_ctx::Peer& peer = ctx->peer;
		P.n_ranks = (uint32_t)ctx->n_ranks;
		for (int r = 0; r < ctx->n_ranks; ++r) P.xdst[r] = peer.gather[xchg->epoch % peer.n_buffers][r] + peer.slab_words * (size_t)ctx->rank;
		P.pub_epoch = xchg->pub_epoch; P.wait_epoch = xchg->wait_epoch; P.n_buffers = peer.n_buffers; P.rank = (uint32_t)ctx->rank;
		for (int r = 0; r < ctx->n_ranks; ++r) {
			P.xflags[r] = peer.flags[r];
			P.xprev[r] = xchg->pub_epoch ? peer.gather[xchg->pub_epoch % peer.n_buffers][r] + peer.slab_words * (size_t)ctx->rank : nullptr;
		}
	}
	static const bool no_mask = getenv("LB200_NO_PLANE_MASKING") != nullptr;
	P.plane_masking = (h.n_bad_radius == 0 && !no_mask) ? 1u : 0u;
	// Programmatic stream serialization: the kernel's prologue (up to cudaGridDependencySynchronize: descriptor reads, classification, the
	// sphere tests of round 0, whose results sit in shared memory) only READS scene data.  Those arrays are written by flushPages alone, so
	// unless something was uploaded since the last cull the prologue may overlap the tail of whatever kernel precedes it on the stream —
	// for back-to-back views (main, shadow cascades, lights) that is the previous cull, which releases its dependents at its first
	// instruction.  The flag is sticky: whichever call uploaded (flush, set_many, ...), the first cull after it is launched plain.
	static const bool no_pdl = getenv("LB200_NO_PDL") != nullptr;
	const bool pdl = !no_pdl && !cs->uploaded_since_last_cull;
	cs->uploaded_since_last_cull = false;
	// chunk = pages per block per round: spread the pages over every resident block, at most one classify thread per page
	const uint32_t resident = (uint32_t)(stream || xchg ? cs->grid_lanes : cs->grid);
	uint32_t chunk = (n_pages + resident - 1) / resident;
	chunk = std::max(32u, std::min((uint32_t)MAX_CHUNK, chunk));
	const uint32_t blocks = std::max(1u, std::min(resident, (n_pages + chunk - 1) / chunk));
	P.chunk = chunk;
	cudaLaunchAttribute attr[1];
	attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
	attr[0].val.programmaticStreamSerializationAllowed = 1;
	cudaLaunchConfig_t cfg = {};
	cfg.gridDim = dim3(blocks);
	cfg.blockDim = dim3(CULL_THREADS);
	cfg.stream = stream ? stream : ctx->stream;
	cfg.attrs = attr;
	cfg.numAttrs = pdl ? 1 : 0;
	uint32_t* mask_arg = xchg ? (uint32_t*)nullptr : mask;
	LB200_CUDA(ctx, cudaLaunchKernelEx(&cfg, cull_pages_kernel, P, (const lb200_page_desc*)(cs->d_desc + off), (const float4*)(cs->d_spheres + off * PAGE_SLOTS),
		(const int*)(cs->d_entities + off * PAGE_SLOTS), out, cur, nxt, mask_arg));
	LB200_CHECK_LAUNCH(ctx);
	cs->last_counters = cur; cs->last_out = out; cs->last_mask = mask_arg; // exchange culls keep their rows in the slabs
	cs->lane_parity[lane] ^= 1u;
	if (!xchg) ++cs->seq;
	cs->last_pages = n_pages;
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

void parseCounts(lb200_culling* cs, lb200_cull_result* result);

int readCounts(lb200_culling* cs, lb200_cull_result* result) {
	lb200_ctx* ctx = cs->ctx;
	const uint32_t* cur = cs->last_counters;
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_counters, cur, sizeof(uint32_t) * COUNTER_WORDS, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	parseCounts(cs, result);
	return LB200_OK;
}

// h_counters (already on the host) -> cs->last / *result
void parseCounts(lb200_culling* cs, lb200_cull_result* result) {
	lb200_cull_result& res = cs->last;
	memset(&res, 0, sizeof(res));
	for (int t = 0; t < 256; ++t) {
		res.type_count[t] = cs->h_counters[t];
		res.type_offset[t] = cs->last_type_base[t];
		res.total += res.type_count[t];
		if (cs->host.type_counts[t]) res.n_types = t + 1;
	}
	res.pages_tested = cs->h_counters[256 + ST_PAGES_TESTED];
	res.pages_inside = cs->h_counters[256 + ST_PAGES_INSIDE];
	res.pages_outside = cs->h_counters[256 + ST_PAGES_OUTSIDE];
	res.pages_filtered = cs->h_counters[256 + ST_PAGES_FILTERED];
	res.entities_tested = cs->h_counters[256 + ST_ENT_TESTED];
	res.entities_inside = cs->h_counters[256 + ST_ENT_INSIDE];
	cs->has_last = true;
	// DESIGN.md §4.1: descriptor per page + 16 B per sphere the kernel reads (pages left to test after plane masking) + (4 B id read +
	// 4 B id write) per visible + 32 B mask per page
	const uint64_t streamed = cs->h_counters[256 + ST_ENT_STREAMED];
	cs->last_bytes = (uint64_t)cs->last_pages * 32 + streamed * 16 + (uint64_t)res.total * 8 + (uint64_t)cs->last_pages * 32;
	if (result) *result = res;
}

} // namespace

int lb200_culling_internal_last(lb200_culling* cs, const uint32_t** out_ids, const uint32_t** counters, const uint32_t** type_base, const uint32_t** type_counts) {
	if (!cs || !cs->ctx) return LB200_ERR_INVALID;
	if (!cs->last_counters) { lb200_set_error(cs->ctx, "no cull has been issued on this culling system yet"); return LB200_ERR_STATE; }
	*out_ids = cs->last_out; *counters = cs->last_counters; *type_base = cs->last_type_base; *type_counts = cs->host.type_counts;
	return LB200_OK;
}

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
	if (cs && cs->device_authoritative && syncHostFromDevice(const_cast<lb200_culling*>(cs))) return 0.0f;
	return cs && cs->host.isAdded(entity) ? cs->host.getRadius(entity) : 0.0f;
}
int lb200_culling_is_added(const lb200_culling* cs, int32_t entity) { return cs && cs->host.isAdded(entity) ? 1 : 0; } // re-binning never adds or removes entities

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
	if (cs && cs->device_authoritative && syncHostFromDevice(const_cast<lb200_culling*>(cs))) return 0;
	return cs ? (uint32_t)cs->host.cells.size() : 0;
}
uint32_t lb200_culling_entity_count(const lb200_culling* cs) { return cs ? cs->host.n_entities : 0; }

int lb200_culling_get_page(const lb200_culling* cs, uint32_t page, double origin[3], int32_t indices[3], uint8_t* type, uint8_t* is_big,
	uint32_t* count, float* spheres4, int32_t* entities)
{
	if (cs && cs->device_authoritative) { const int rc = syncHostFromDevice(const_cast<lb200_culling*>(cs)); if (rc) return rc; }
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
	if (cs && cs->device_authoritative && syncHostFromDevice(const_cast<lb200_culling*>(cs))) return -1;
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
	cs->replicas = replicas;
	cs->next_replica = 0;
	cs->dev_cap = 0; // forces reallocation + full upload at the next flush
	return LB200_OK;
}

int lb200_culling_cull_device(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, const uint32_t** out_dev_ids,
	lb200_cull_result* result, int want_counts)
{
	if (!cs || !frustum) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (cs->host.cells.empty()) { // culling_system.cpp:322
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
	if (cs->host.cells.empty()) return LB200_OK;
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
	if (cs->host.cells.empty()) { lb200_set_error(ctx, "cull_begin on an empty culling system (cull() handles that case)"); return LB200_ERR_STATE; }
	int rc = ensureDevice(cs);
	if (rc) return rc;
	cudaPointerAttributes attr = {};
	const cudaError_t pe = cudaPointerGetAttributes(&attr, out_ids);
	if (!cs->h_counters_dev || pe != cudaSuccess || attr.type != cudaMemoryTypeHost || !attr.devicePointer) {
		cudaGetLastError();
		lb200_set_error(ctx, "cull_begin needs a page-locked destination (lb200_host_alloc): cudaPointerGetAttributes -> %s, memory type %d, device pointer %p, counters mapped %d",
			cudaGetErrorString(pe), (int)attr.type, attr.devicePointer, cs->h_counters_dev ? 1 : 0);
		return LB200_ERR_INVALID;
	}
	if (!cs->done_event) LB200_CUDA(ctx, cudaEventCreateWithFlags(cs->done_event.create(), cudaEventDisableTiming));
	rc = launchCull(cs, frustum, type);
	if (rc) return rc;
	PackParams PP;
	memcpy(PP.type_base, cs->last_type_base, sizeof(PP.type_base));
	PP.slab_ids = capacity;
	pack_host_kernel<<<ctx->sm_count * 2, 256, 0, ctx->stream>>>(PP, cs->last_counters, cs->last_out, (uint32_t*)attr.devicePointer, cs->h_counters_dev);
	LB200_CHECK_LAUNCH(ctx);
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
	parseCounts(cs, result);
	uint32_t off = 0;
	for (int t = 0; t < 256; ++t) { result->type_offset[t] = off; off += result->type_count[t]; }
	return result->total > cs->pending_capacity ? LB200_ERR_CAPACITY : LB200_OK;
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
	if (!no_direct && out_ids && capacity && !cs->host.cells.empty() && ensureDevice(cs) == LB200_OK && cs->h_counters_dev) {
		cudaPointerAttributes attr = {};
		if (cudaPointerGetAttributes(&attr, out_ids) == cudaSuccess && attr.type == cudaMemoryTypeHost && attr.devicePointer) {
			int rc = launchCull(cs, frustum, type);
			if (rc) return rc;
			PackParams PP;
			memcpy(PP.type_base, cs->last_type_base, sizeof(PP.type_base));
			PP.slab_ids = capacity;
			pack_host_kernel<<<ctx->sm_count * 2, 256, 0, ctx->stream>>>(PP, cs->last_counters, cs->last_out, (uint32_t*)attr.devicePointer, cs->h_counters_dev);
			LB200_CHECK_LAUNCH(ctx);
			LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
			parseCounts(cs, result);
			uint32_t off = 0;
			for (int t = 0; t < 256; ++t) { result->type_offset[t] = off; off += result->type_count[t]; }
			return result->total > capacity ? LB200_ERR_CAPACITY : LB200_OK;
		}
		cudaGetLastError(); // unregistered host memory makes cudaPointerGetAttributes fail on old drivers: not an error here
	}
	lb200_cull_result dev;
	const uint32_t* d_ids = nullptr;
	int rc = lb200_culling_cull_device(cs, frustum, type, &d_ids, &dev, 1);
	if (rc) return rc;
	*result = dev;
	uint32_t off = 0;
	for (int t = 0; t < 256; ++t) { result->type_offset[t] = off; off += dev.type_count[t]; }
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
	if (cs->host.cells.empty()) return LB200_ERR_STATE;
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

} // extern "C"

// ---- multi-GPU exchange (SURVEY.md §8e) ----
int lb200_comm_allgather_u32(lb200_ctx* ctx, const uint32_t* send, uint32_t* recv, size_t words); // comm.cu

namespace {

int pushGridMul() {
	static int mul = [] { const char* e = getenv("LB200_PUSH_GRID"); const int v = e ? atoi(e) : 2; return v < 1 ? 1 : (v > 16 ? 16 : v); }();
	return mul;
}

int ensureGather(lb200_culling* cs, uint32_t slab_ids) {
	lb200_ctx* ctx = cs->ctx;
	const size_t words = 256 + (size_t)slab_ids;
	const size_t R = (size_t)ctx->n_ranks;
	if (cs->d_slab.size() < words) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		LB200_CUDA(ctx, cs->d_slab.alloc(words));
	}
	if (cs->d_gather_ids.size() < words * R) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		LB200_CUDA(ctx, cs->d_gather_ids.alloc(words * R));
	}
	return LB200_OK;
}

// pack the counters + ids of the cull whose counters live in `cur`, then all-gather the slabs
int packAndGather(lb200_culling* cs, const uint32_t* cur, uint32_t slab_ids) {
	lb200_ctx* ctx = cs->ctx;
	int rc = ensureGather(cs, slab_ids);
	if (rc) return rc;
	PackParams PP;
	memcpy(PP.type_base, cs->last_type_base, sizeof(PP.type_base));
	PP.slab_ids = slab_ids;
	pack_slab_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(PP, cur, cs->last_out, cs->d_slab);
	LB200_CHECK_LAUNCH(ctx);
	return lb200_comm_allgather_u32(ctx, cs->d_slab, cs->d_gather_ids, 256 + (size_t)slab_ids);
}

} // namespace

extern "C" {

int lb200_culling_cull_gather(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t slab_ids, const uint32_t** out_dev_slabs) {
	if (!cs || !frustum) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	if (cs->host.cells.empty()) { lb200_set_error(ctx, "cull_gather on an empty culling system"); return LB200_ERR_STATE; }
	int rc = lb200_comm_check(ctx);
	if (rc) return rc;
	rc = launchCull(cs, frustum, type);
	if (rc) return rc;
	const uint32_t* cur = cs->last_counters;
	cs->has_last = false;
	lb200_ctx::Peer& peer = ctx->peer;
	if (peer.ready && 256 + (size_t)slab_ids <= peer.slab_words) {
		// NVLink peer path: fused pack + push, then wait for the peers' slabs.  Slabs are peer.slab_words apart.
		const uint32_t epoch = ++peer.epoch;
		PushParams PP;
		memcpy(PP.type_base, cs->last_type_base, sizeof(PP.type_base));
		PP.slab_ids = slab_ids;
		PP.n_ranks = (uint32_t)ctx->n_ranks; PP.rank = (uint32_t)ctx->rank; PP.epoch = epoch; PP.n_buffers = peer.n_buffers;
		for (int r = 0; r < LB200_MAX_RANKS; ++r) {
			PP.dst[r] = r < ctx->n_ranks ? peer.gather[epoch % peer.n_buffers][r] + peer.slab_words * (size_t)ctx->rank : nullptr;
			PP.flags[r] = r < ctx->n_ranks ? peer.flags[r] : nullptr;
		}
		pack_push_kernel<<<ctx->sm_count * pushGridMul(), 256, 0, ctx->stream>>>(PP, cur, cs->last_out, peer.done_counter);
		LB200_CHECK_LAUNCH(ctx);
		wait_peers_kernel<<<1, 32, 0, ctx->stream>>>(peer.flags[ctx->rank], (uint32_t)ctx->n_ranks, epoch, peer.n_buffers, peer.d_timeout);
		LB200_CHECK_LAUNCH(ctx);
		if (out_dev_slabs) *out_dev_slabs = peer.gather[epoch % peer.n_buffers][ctx->rank];
		return LB200_OK;
	}
	rc = packAndGather(cs, cur, slab_ids);
	if (rc) return rc;
	if (out_dev_slabs) *out_dev_slabs = cs->d_gather_ids;
	return LB200_OK;
}

uint32_t lb200_culling_gather_stride_words(const lb200_culling* cs, uint32_t slab_ids) {
	if (!cs || !cs->ctx) return 0;
	const lb200_ctx::Peer& peer = cs->ctx->peer;
	return (peer.ready && 256 + (size_t)slab_ids <= peer.slab_words) ? (uint32_t)peer.slab_words : 256 + slab_ids;
}

static int prepareExchange(lb200_culling* cs, const lb200_shifted_frustum* frustum) {
	if (!cs || !frustum) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	lb200_ctx::Peer& peer = ctx->peer;
	if (!peer.ready) { lb200_set_error(ctx, "cull_exchange needs lb200_comm_enable_p2p"); return LB200_ERR_STATE; }
	if (cs->host.cells.empty()) { lb200_set_error(ctx, "cull_exchange on an empty culling system"); return LB200_ERR_STATE; }
	int rc = flushPages(cs); // uploads (if any) go to the context stream, before any lane forks from it
	if (rc) return rc;
	if (peer.lanes != cs->lanes) { lb200_set_error(ctx, "exchange lanes (%u) differ from cull lanes (%u)", peer.lanes, cs->lanes); return LB200_ERR_STATE; }
	if (exchangeSlabWords(cs) > peer.slab_words) {
		lb200_set_error(ctx, "exchange slab too small: %zu words needed, %zu mapped", exchangeSlabWords(cs), peer.slab_words);
		return LB200_ERR_CAPACITY;
	}
	return lb200_comm_check(ctx);
}

// publish + wait of one epoch as a kernel of its own behind the cull that stored the epoch's records: the second kernel of a two-kernel
// step, and the closing step of every lane of a fused batch
static int publishAndWait(lb200_culling* cs, uint32_t epoch, const uint32_t* counters, cudaStream_t stream) {
	lb200_ctx* ctx = cs->ctx;
	lb200_ctx::Peer& peer = ctx->peer;
	PublishParams PP;
	PP.n_ranks = (uint32_t)ctx->n_ranks; PP.rank = (uint32_t)ctx->rank; PP.epoch = epoch; PP.n_buffers = peer.n_buffers;
	PP.n_pages = cs->last_pages; PP.item_cap = cs->item_cap;
	for (int r = 0; r < LB200_MAX_RANKS; ++r) {
		PP.dst[r] = r < ctx->n_ranks ? peer.gather[epoch % peer.n_buffers][r] + peer.slab_words * (size_t)ctx->rank : nullptr;
		PP.flags[r] = r < ctx->n_ranks ? peer.flags[r] : nullptr;
	}
	cudaLaunchConfig_t cfg = {};
	cfg.gridDim = dim3(1);
	cfg.blockDim = dim3(288);
	cfg.stream = stream;
	cudaLaunchAttribute attr[1];
	attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
	attr[0].val.programmaticStreamSerializationAllowed = 1;
	cfg.attrs = attr;
	cfg.numAttrs = 1;
	LB200_CUDA(ctx, cudaLaunchKernelEx(&cfg, publish_wait_kernel, PP, counters, peer.d_timeout));
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

// one two-kernel exchange step on the context stream: the cull kernel stores rows + counts into every rank, publish_wait_kernel then
// raises this rank's epoch flag everywhere and holds the stream until every rank's flag of this epoch is here
static int exchangeStep(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type) {
	Exchange x;
	x.epoch = ++cs->ctx->peer.epoch;
	const int rc = launchCull(cs, frustum, type, &x);
	if (rc) return rc;
	return publishAndWait(cs, x.epoch, cs->last_counters, cs->ctx->stream);
}

// One fused step on lane l = epoch % lanes: ONE kernel.  The cull of epoch e publishes the lane's previous epoch from its own prologue and
// holds its record stores back until every rank has published e - 2 x lanes (cull_kernel.cuh); the batch closes with publishAndWait per lane.
static int exchangeStepFused(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type) {
	lb200_ctx::Peer& peer = cs->ctx->peer;
	Exchange x;
	x.epoch = ++peer.epoch;
	const uint32_t l = x.epoch % cs->lanes;
	x.pub_epoch = cs->lane_owed[l];
	x.wait_epoch = x.epoch > 2 * cs->lanes ? x.epoch - 2 * cs->lanes : 0u;
	int rc = launchCull(cs, frustum, type, &x, cs->lane_stream[l]);
	if (rc) return rc;
	cs->lane_owed[l] = x.epoch;
	cs->lane_last_counters[l] = cs->last_counters;
	return LB200_OK;
}

static void lastExchange(lb200_culling* cs, const uint32_t** out_dev_ids, const uint32_t** out_dev_slabs, uint32_t* out_slab_stride_words) {
	const lb200_ctx::Peer& peer = cs->ctx->peer;
	if (out_dev_ids) *out_dev_ids = cs->last_out;
	if (out_dev_slabs) *out_dev_slabs = peer.gather[peer.epoch % peer.n_buffers][cs->ctx->rank];
	if (out_slab_stride_words) *out_slab_stride_words = (uint32_t)peer.slab_words;
}

int lb200_culling_cull_exchange(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, const uint32_t** out_dev_ids,
	const uint32_t** out_dev_slabs, uint32_t* out_slab_stride_words)
{
	int rc = prepareExchange(cs, frustum);
	if (rc) return rc;
	rc = exchangeStep(cs, frustum, type);
	if (rc) return rc;
	cs->has_last = false;
	lastExchange(cs, out_dev_ids, out_dev_slabs, out_slab_stride_words);
	return LB200_OK;
}

int lb200_culling_cull_exchange_n(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t n, const uint32_t** out_dev_ids,
	const uint32_t** out_dev_slabs, uint32_t* out_slab_stride_words)
{
	if (n == 0) return LB200_ERR_INVALID;
	int rc = prepareExchange(cs, frustum);
	if (rc) return rc;
	cs->has_last = false;
	if (cs->lanes < 2 || n < 2) {
		for (uint32_t i = 0; i < n; ++i) {
			rc = exchangeStep(cs, frustum, type);
			if (rc) return rc;
		}
		lastExchange(cs, out_dev_ids, out_dev_slabs, out_slab_stride_words);
		return LB200_OK;
	}
	// independent steps: epoch e runs on stream e % lanes (every rank makes the same choice), so one step's remote stores, fences and
	// flag round trip overlap the neighbouring steps' culls; see lb200_ctx::Peer for why 3 x lanes exchange buffers make that safe.
	// ONE kernel per step (exchangeStepFused); the batch closes with publish + wait of every lane's last epoch.
	rc = forkLanes(cs);
	if (rc) return rc;
	for (uint32_t i = 0; i < n; ++i) {
		rc = exchangeStepFused(cs, frustum, type);
		if (rc) return rc;
	}
	for (uint32_t l = 0; l < cs->lanes; ++l) {
		if (!cs->lane_owed[l]) continue;
		rc = publishAndWait(cs, cs->lane_owed[l], cs->lane_last_counters[l], cs->lane_stream[l]);
		if (rc) return rc;
		cs->lane_owed[l] = 0;
	}
	lastExchange(cs, out_dev_ids, out_dev_slabs, out_slab_stride_words);
	return joinLanes(cs);
}

uint32_t lb200_culling_exchange_slab_words(lb200_culling* cs) {
	if (!cs || !cs->ctx || ensureDevice(cs) != LB200_OK) return 0;
	return (uint32_t)exchangeSlabWords(cs);
}

int lb200_culling_allgather(lb200_culling* cs, uint32_t slab_ids, const uint32_t** out_dev_ids, uint32_t* out_counts) {
	if (!cs) return LB200_ERR_INVALID;
	lb200_ctx* ctx = cs->ctx;
	if (!ctx) return LB200_ERR_NO_DEVICE;
	if (!cs->last_pages) { lb200_set_error(ctx, "allgather needs a preceding cull"); return LB200_ERR_STATE; }
	const uint32_t* cur = cs->last_counters; // the preceding cull's
	int rc = packAndGather(cs, cur, slab_ids);
	if (rc) return rc;
	const size_t words = 256 + (size_t)slab_ids;
	if (out_counts) {
		for (int r = 0; r < ctx->n_ranks; ++r)
			LB200_CUDA(ctx, cudaMemcpyAsync(out_counts + 256 * (size_t)r, cs->d_gather_ids + words * r, sizeof(uint32_t) * 256, cudaMemcpyDeviceToHost, ctx->stream));
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (out_dev_ids) *out_dev_ids = cs->d_gather_ids;
	return LB200_OK;
}

} // extern "C"

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
// =====================================================================================================================================
namespace {

enum { RB_HIGH_WATER = 0, RB_N_FREE, RB_N_CHANGERS, RB_N_DIRTY, RB_OVERFLOW, RB_BAD_RADIUS, RB_WORDS = 8 };
constexpr unsigned long long HASH_EMPTY = ~0ull;
constexpr uint32_t NO_OPEN_PAGE = 0xffffffffu;

__host__ __device__ __forceinline__ unsigned long long packCellKey(int x, int y, int z, uint32_t type, uint32_t is_big) {
	// 18 bits per axis (+-131 071 cells of 300 m), 8 bits type, 1 bit is_big
	return ((unsigned long long)((uint32_t)x & 0x3ffffu)) | ((unsigned long long)((uint32_t)y & 0x3ffffu) << 18) | ((unsigned long long)((uint32_t)z & 0x3ffffu) << 36)
		| ((unsigned long long)(type & 0xffu) << 54) | ((unsigned long long)(is_big & 1u) << 62);
}
__host__ __device__ __forceinline__ uint32_t hashCellKey(unsigned long long k) {
	k ^= k >> 33; k *= 0xff51afd7ed558ccdull; k ^= k >> 33; k *= 0xc4ceb9fe1a85ec53ull; k ^= k >> 33;
	return (uint32_t)k;
}

__device__ __forceinline__ uint32_t hashFind(const unsigned long long* keys, const uint32_t* vals, uint32_t cap, unsigned long long key, uint32_t* slot_out) {
	uint32_t i = hashCellKey(key) & (cap - 1);
	for (;;) {
		const unsigned long long k = keys[i];
		if (k == key) { *slot_out = i; return vals[i]; }
		if (k == HASH_EMPTY) { *slot_out = i; return NO_OPEN_PAGE; }
		i = (i + 1) & (cap - 1);
	}
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
		const double inv = (double)(1 / LB200_CELL_SIZE);
		const int ix = (int)__dmul_rn(pos3[3 * (size_t)i], inv), iy = (int)__dmul_rn(pos3[3 * (size_t)i + 1], inv), iz = (int)__dmul_rn(pos3[3 * (size_t)i + 2], inv);
		const uint32_t type = (uint32_t)page_cell[page].w & 0xffu; // set() keeps the renderable type (:236-239)
		keys[k] = packCellKey(ix, iy, iz, type, radius[i] > LB200_CELL_SIZE ? 1u : 0u);
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
		uint32_t hslot = hashCellKey(key) & (hash_cap - 1);
		uint32_t page = NO_OPEN_PAGE;
		for (;;) { // find or claim the key's hash slot (runs have distinct keys: no two threads insert the same one)
			const unsigned long long prev = atomicCAS(&hash_keys[hslot], HASH_EMPTY, (unsigned long long)key);
			if (prev == HASH_EMPTY) { hash_vals[hslot] = NO_OPEN_PAGE; break; }
			if (prev == key) { page = hash_vals[hslot]; break; }
			hslot = (hslot + 1) & (hash_cap - 1);
		}
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
				if (np >= page_cap) { atomicExch(&counters[RB_OVERFLOW], 1u); np = 0; }
				d.count = q + 1 < m ? PAGE_SLOTS : rest - q * PAGE_SLOTS;
				desc[np] = d;
				page_cell[np] = make_int4(ix, iy, iz, (int)(type | (is_big << 8)));
				new_pages[plan.new_base + q] = np;
				page = np;
			}
		}
		plans[k] = plan;
		if (page != NO_OPEN_PAGE) hash_vals[hslot] = page; // the last page opened (or the old open page) takes the chain's next adds
	}
}

// 3b. every changer finds its run (binary search on the sorted keys), its rank in it, and from the run's plan its page and slot
__global__ void __launch_bounds__(256) rebin_place_kernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ vals, const uint32_t* __restrict__ counters,
	const int32_t* __restrict__ ents, const double* __restrict__ pos3, const float* __restrict__ radius, uint32_t* __restrict__ entity_to_slot,
	const lb200_page_desc* __restrict__ desc, float4* __restrict__ spheres, int* __restrict__ entities, const RunPlan* __restrict__ plans, const uint32_t* __restrict__ new_pages)
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
	}
}

int growDevicePages(lb200_culling* cs, uint32_t min_cap) {
	lb200_ctx* ctx = cs->ctx;
	if (min_cap <= cs->dev_cap) return LB200_OK;
	uint32_t cap = cs->dev_cap ? cs->dev_cap : 1024;
	while (cap < min_cap) cap *= 2;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	// allocate, copy, swap: the page arrays keep their contents, and a failure leaves the old ones in place
	DeviceArray<float4> ns; DeviceArray<int> ne; DeviceArray<lb200_page_desc> nd; DeviceArray<uint32_t> nm; DeviceArray<int4> nc; DeviceArray<uint32_t> nf, npd, ndp;
	LB200_CUDA(ctx, ns.alloc(PAGE_SLOTS * (size_t)cap));
	LB200_CUDA(ctx, ne.alloc(PAGE_SLOTS * (size_t)cap));
	LB200_CUDA(ctx, nd.alloc(cap));
	LB200_CUDA(ctx, nm.alloc(8 * (size_t)cap * cs->lanes));
	LB200_CUDA(ctx, nc.alloc(cap));
	LB200_CUDA(ctx, nf.alloc(cap));
	LB200_CUDA(ctx, npd.alloc(cap));
	LB200_CUDA(ctx, ndp.alloc(cap));
	LB200_CUDA(ctx, cudaMemsetAsync(nd, 0, sizeof(lb200_page_desc) * (size_t)cap, ctx->stream));
	LB200_CUDA(ctx, cudaMemsetAsync(npd, 0, sizeof(uint32_t) * (size_t)cap, ctx->stream));
	const size_t old = cs->dev_cap;
	if (old) {
		LB200_CUDA(ctx, cudaMemcpyAsync(ns, cs->d_spheres, sizeof(float4) * PAGE_SLOTS * old, cudaMemcpyDeviceToDevice, ctx->stream));
		LB200_CUDA(ctx, cudaMemcpyAsync(ne, cs->d_entities, sizeof(int) * PAGE_SLOTS * old, cudaMemcpyDeviceToDevice, ctx->stream));
		LB200_CUDA(ctx, cudaMemcpyAsync(nd, cs->d_desc, sizeof(lb200_page_desc) * old, cudaMemcpyDeviceToDevice, ctx->stream));
		if (cs->d_page_cell) LB200_CUDA(ctx, cudaMemcpyAsync(nc, cs->d_page_cell, sizeof(int4) * old, cudaMemcpyDeviceToDevice, ctx->stream));
		if (cs->d_free_pages) LB200_CUDA(ctx, cudaMemcpyAsync(nf, cs->d_free_pages, sizeof(uint32_t) * old, cudaMemcpyDeviceToDevice, ctx->stream));
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	cs->d_spheres = std::move(ns); cs->d_entities = std::move(ne); cs->d_desc = std::move(nd); cs->d_mask = std::move(nm);
	cs->d_page_cell = std::move(nc); cs->d_free_pages = std::move(nf); cs->d_page_dirty = std::move(npd); cs->d_dirty_pages = std::move(ndp);
	cs->item_cap = cap;
	cs->dev_cap = cap;
	return LB200_OK;
}

// device-side tables for the re-binning, (re)built from the host mirror whenever it was edited since
int ensureRebinState(lb200_culling* cs, uint32_t max_entity) {
	lb200_ctx* ctx = cs->ctx;
	lb::CullingHost& h = cs->host;
	if (cs->replicas != 1) { lb200_set_error(ctx, "device re-binning works on the live page arrays: set_replicas(1)"); return LB200_ERR_STATE; }
	int rc = flushPages(cs);
	if (rc) return rc;
	if (!cs->d_rebin_counters || !cs->h_rebin_counters || !cs->d_rb_sort_state || !cs->d_rb_block_hist) {
		cs->rb_sort_blocks = (uint32_t)ctx->sm_count * 2;
		DeviceArray<uint32_t> d_counters; PinnedArray<uint32_t> h_counters; DeviceArray<uint8_t> sort_state; DeviceArray<uint32_t> block_hist;
		LB200_CUDA(ctx, d_counters.alloc(RB_WORDS));
		LB200_CUDA(ctx, h_counters.alloc(RB_WORDS));
		LB200_CUDA(ctx, sort_state.alloc(lb200_radix_sort_state_bytes()));
		LB200_CUDA(ctx, block_hist.alloc(256 * (size_t)cs->rb_sort_blocks));
		cs->d_rebin_counters = std::move(d_counters); cs->h_rebin_counters = std::move(h_counters);
		cs->d_rb_sort_state = std::move(sort_state); cs->d_rb_block_hist = std::move(block_hist);
	}
	if (!cs->d_page_cell || cs->d_page_cell.size() != cs->dev_cap) { // the per-page side arrays follow dev_cap
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_page_cell.reset(); cs->d_free_pages.reset(); cs->d_page_dirty.reset(); cs->d_dirty_pages.reset(); // before the new ones are allocated
		cs->rebin_built_gen = ~0ull;
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
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		uint32_t cap = cs->d_entity_to_slot.size() ? (uint32_t)cs->d_entity_to_slot.size() : 4096;
		while (cap < need_entities) cap *= 2;
		cs->d_entity_to_slot.reset();
		cs->rebin_built_gen = ~0ull;
		LB200_CUDA(ctx, cs->d_entity_to_slot.alloc(cap));
	}
	if (cs->rebin_built_gen == h.edit_gen && !cs->device_authoritative) return LB200_OK;
	if (cs->device_authoritative) return LB200_OK; // the tables are live on the device
	// ---- build from the host mirror ----
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

// pull the device state back into the host mirror (page arrays, counts, entity -> slot, chains regrouped by key with the open page as head)
int syncHostFromDevice(lb200_culling* cs) {
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
	cs->rebin_built_gen = ~0ull;
	return LB200_OK;
}

} // namespace

extern "C" {

int lb200_culling_set_many_device(lb200_culling* cs, const int32_t* dev_entities, const double* dev_pos3, const float* dev_radius, uint32_t n, uint32_t max_entity) {
	if (!cs || !dev_pos3 || !dev_radius) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (n == 0) return LB200_OK;
	lb200_ctx* ctx = cs->ctx;
	lb200_range range("culling set many");
	int rc = ensureRebinState(cs, max_entity);
	if (rc) return rc;
	cudaStream_t s = ctx->stream;
	if (cs->d_changers.size() < n) {
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		uint32_t cap = cs->d_changers.size() ? (uint32_t)cs->d_changers.size() : 4096;
		while (cap < n) cap *= 2;
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
	}
	const uint32_t changers_cap = (uint32_t)cs->d_changers.size(), hash_cap = (uint32_t)cs->d_hash_keys.size();
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
	if (n_changers) {
		rc = growDevicePages(cs, cs->h_rebin_counters[RB_HIGH_WATER] + n_changers); // worst case: every changer opens a page
		if (rc) return rc;
		const uint32_t grid = std::max(1u, std::min((uint32_t)ctx->sm_count * 4u, (n_changers + 255) / 256));
		rebin_remove_kernel<<<grid, 256, 0, s>>>(cs->d_changers, dev_entities, dev_pos3, dev_radius, cs->d_entity_to_slot, cs->d_page_cell, cs->d_spheres, cs->d_entities,
			cs->d_page_dirty, cs->d_dirty_pages, C, cs->d_rb_keys[0], cs->d_rb_vals[0]);
		LB200_CHECK_LAUNCH(ctx);
		rebin_compact_kernel<<<grid, 256, 0, s>>>(cs->d_dirty_pages, C, cs->d_desc, cs->d_page_cell, cs->d_spheres, cs->d_entities, cs->d_entity_to_slot, cs->d_page_dirty,
			cs->d_free_pages, cs->d_hash_keys, cs->d_hash_vals, hash_cap);
		LB200_CHECK_LAUNCH(ctx);
		rc = lb200_radix_sort_pairs(ctx, s, cs->d_rb_keys[0], cs->d_rb_keys[1], cs->d_rb_vals[0], cs->d_rb_vals[1], C + RB_N_CHANGERS, changers_cap, cs->d_rb_sort_state,
			cs->d_rb_block_hist, cs->rb_sort_blocks, false, nullptr);
		if (rc) return rc;
		LB200_CUDA(ctx, cudaMemsetAsync(C + RB_WORDS - 1, 0, sizeof(uint32_t), s)); // the new-page cursor of this batch
		rebin_plan_kernel<<<std::max(1u, std::min((uint32_t)ctx->sm_count * 8u, (n_changers + 127) / 128)), 128, 0, s>>>(cs->d_rb_keys[0], cs->d_rb_vals[0], C, dev_pos3, cs->d_desc,
			cs->d_page_cell, cs->d_free_pages, cs->d_hash_keys, cs->d_hash_vals, hash_cap, cs->dev_cap, (RunPlan*)cs->d_rb_plans.get(), (uint32_t*)cs->d_rb_vals[1].get(), C + RB_WORDS - 1);
		LB200_CHECK_LAUNCH(ctx);
		rebin_place_kernel<<<grid, 256, 0, s>>>(cs->d_rb_keys[0], cs->d_rb_vals[0], C, dev_entities, dev_pos3, dev_radius, cs->d_entity_to_slot, cs->d_desc, cs->d_spheres,
			cs->d_entities, (const RunPlan*)cs->d_rb_plans.get(), (const uint32_t*)cs->d_rb_vals[1].get());
		LB200_CHECK_LAUNCH(ctx);
		LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_rebin_counters, C, sizeof(uint32_t) * RB_WORDS, cudaMemcpyDeviceToHost, s));
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		if (cs->h_rebin_counters[RB_OVERFLOW]) { lb200_set_error(ctx, "device re-binning ran out of pages (capacity %u)", cs->dev_cap); return LB200_ERR_CAPACITY; }
	}
	cs->dev_high_water = cs->h_rebin_counters[RB_HIGH_WATER];
	cs->host.n_bad_radius = cs->h_rebin_counters[RB_BAD_RADIUS]; // plane masking of the cull kernel needs radius >= 0 everywhere
	return LB200_OK;
}

int lb200_culling_sync_host(lb200_culling* cs) {
	if (!cs) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_OK;
	return syncHostFromDevice(cs);
}

uint32_t lb200_culling_last_rebin_changers(const lb200_culling* cs) { return cs && cs->h_rebin_counters ? cs->h_rebin_counters[RB_N_CHANGERS] : 0; }

} // extern "C"
