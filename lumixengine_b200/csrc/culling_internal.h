// Private to the culling sources: culling.cu (host edits, page upload, the cull launch, result delivery), culling_exchange.cu (the
// multi-GPU exchange) and culling_rebin.cu (device re-binning).  The cull kernel is cull_kernel.cuh, which culling.cu alone includes.
#pragma once

#include "culling_host.hpp"
#include "lb200_internal.h"

namespace lbcull {

constexpr int N_STATS = 8;
enum { ST_PAGES_TESTED = 0, ST_PAGES_INSIDE, ST_PAGES_OUTSIDE, ST_PAGES_FILTERED, ST_ENT_TESTED, ST_ENT_INSIDE, ST_ENT_STREAMED };
// counters of one cull: [0,256) visible per type, [256,264) statistics, [264] exchange records written
constexpr int CNT_N_REC = 256 + N_STATS;
constexpr int COUNTER_WORDS = 256 + N_STATS + 8;
// exchange slab = [256 per-type counts][n_pages, n_records, 0, item_cap, 0, 0, 0, 0][page ids: item_cap][rows: item_cap x 8]
constexpr uint32_t XHEADER_WORDS = 264;

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

} // namespace lbcull

struct lb200_culling {
	explicit lb200_culling(lb200_ctx* c); // culling.cu: the host mirror's arrays are page-locked when there is a context
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
	// lb200_culling_set_launch (0, 0, -1: the default rule) and what the last cull launched (lb200_culling_get_launch)
	int launch_blocks = 0, launch_chunk = 0, launch_plane_masking = -1;
	uint32_t last_blocks = 0, last_chunk = 0, last_rounds = 0;
	int last_pdl = 0, last_plane_masking = 0;
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
	// Device adds / removes (lb200_culling_add_many_device, _remove_many_device) changed which entities are added since the last pull-back:
	// is_added has to pull back first.  Type counts, entity count and bad-radius count stay current on the host either way.
	bool membership_on_device = false;
	uint64_t rebin_built_gen = ~0ull;   // host.edit_gen the device-side tables were built from
	// Each group below is allocated and released as a whole (ensureRebinState, lb200_culling_set_many_device).
	DeviceArray<uint32_t> d_entity_to_slot;
	// per-page side arrays: absent, or dev_cap pages each (resizePages).  set_replicas zeroes dev_cap and leaves them as they are; the
	// next flush with pages in use, which ensureRebinState runs before it uses them, resizes the page arrays and releases these.
	DeviceArray<int4> d_page_cell;          // per page: cell indices x, y, z, type | is_big << 8
	DeviceArray<uint32_t> d_free_pages;     // stack of free page ids
	DeviceArray<uint32_t> d_page_dirty, d_dirty_pages;
	DeviceArray<unsigned long long> d_hash_keys; DeviceArray<uint32_t> d_hash_vals; // packed cell key -> open page of its chain
	DeviceArray<uint32_t> d_rebin_counters; PinnedArray<uint32_t> h_rebin_counters; // RB_* and per-type deltas (culling_rebin.cu); pinned mirror
	RadixSortScratch rb_radix_scratch; // the changer sort, with d_rb_keys[1] / d_rb_vals[1] as its alternate buffers
	// per changer slot
	DeviceArray<uint32_t> d_changers;       // mover indices that change cell / chain
	DeviceArray<uint4> d_rb_plans;          // one RunPlan per changer slot (used at the first index of every run)
	DeviceArray<uint64_t> d_rb_keys[2], d_rb_vals[2];
	uint32_t dev_high_water = 0;        // pages [0, dev_high_water) may be in use on the device

	// ---- several views in one pass (lb200_culling_cull_views, culling_views.cu) ----
	// The latest call's results: view v's ids at d_view_ids + v * view_id_cap, its rows at d_view_mask + v * 8 * dev_cap, its counters in
	// one of two counter blocks (a call zeroes the other one for the next call).  The fused kernel and the single kernel (n_views = 1)
	// keep separate counter blocks, each with its own parity, because each zeroes only the layout it writes.
	DeviceArray<uint32_t> d_view_ids;
	DeviceArray<uint32_t> d_view_mask;       // released with the page arrays (resizePages) and by set_replicas
	DeviceArray<uint32_t> d_view_counters;   // [2][CALL_COUNTER_WORDS] for the fused kernel, then [2][COUNTER_WORDS] for n_views = 1
	PinnedArray<uint32_t> h_view_counters;   // CALL_COUNTER_WORDS
	uint32_t view_id_cap = 0;
	uint8_t view_parity[2] = {};             // fused, single
	uint32_t views_n = 0;                    // n_views of the latest call, 0 = none issued
	bool views_live = false;                 // the view buffers hold that call's results
	uint32_t* views_counters = nullptr;      // counters of that call's view 0; view v's at + v * COUNTER_WORDS
	uint32_t views_pages = 0;
	uint32_t views_type_base[256];
	bool last_is_view = false;               // the "last cull" below is a view selected by lb200_culling_select_view

	uint32_t last_type_base[256];
	lb200_cull_result last = {};
	bool has_last = false;
	uint64_t last_bytes = 0;
	uint32_t last_pages = 0;
};

namespace lbcull {

// non-null: store {page, row} records + counts into every rank's slab (peer memory); lane = epoch % lanes; pub / wait: fused steps (cull_kernel.cuh)
struct Exchange { uint32_t epoch; uint32_t pub_epoch = 0, wait_epoch = 0; };

// non-null: the cull writes here instead of into a lane, and leaves the lanes, the sequence and "the last cull" as they are
struct CullOutput { uint32_t* ids; uint32_t* counters; uint32_t* next_counters; uint32_t* mask; uint32_t* type_base; };

// What a launch of cull_pages_kernel and one of cull_views_kernel decide the same way (prepareLaunch)
struct CullLaunch {
	uint32_t n_pages;       // pages the kernel looks at
	size_t off;             // first page of the replica it reads
	uint32_t plane_masking; // 1 unless a negative / NaN radius, LB200_NO_PLANE_MASKING or set_launch switches it off
	bool pdl;               // programmatic stream serialization behind the previous kernel of the stream
	uint32_t blocks, chunk; // grid, pages per block per round
};
struct CullFrustum; // cull_common.cuh

// culling.cu
int ensureDevice(lb200_culling* cs);
int flushPages(lb200_culling* cs);
int resizePages(lb200_culling* cs, uint32_t min_pages, bool keep); // the one owner of the page arrays' size
// a frustum as the cull kernels read it
void fillFrustum(CullFrustum* F, const lb200_shifted_frustum* f);
// type bases into type_base[256], the next replica, plane masking, PDL, and the launch shape: spread over `resident` blocks (or the
// set_launch override), at most chunk_bound pages per block and round
CullLaunch prepareLaunch(lb200_culling* cs, uint32_t* type_base, uint32_t resident, uint32_t chunk_bound);
// the launch as lb200_culling_get_launch reports it
void recordLaunch(lb200_culling* cs, const CullLaunch& L);
int launchCull(lb200_culling* cs, const lb200_shifted_frustum* f, uint8_t type, const Exchange* xchg = nullptr, cudaStream_t stream = nullptr,
	const CullOutput* out = nullptr);
// counters of one cull (on the host) and the type bases it was culled with -> *res
void fillResult(const lb200_culling* cs, const uint32_t* counters, const uint32_t* type_base, lb200_cull_result* res);
// culling_views.cu: drop the results of the latest cull_views call (their masks are sized by the page arrays); the stream is idle
void releaseViews(lb200_culling* cs);
int forkLanes(lb200_culling* cs);
int joinLanes(lb200_culling* cs);
// pack_kernel on the context stream: ids of the cull with these counters into ids_dst (at most `capacity`), counters[0, counter_words) into counters_dst
int launchPack(lb200_culling* cs, const uint32_t* counters, uint32_t capacity, uint32_t* ids_dst, uint32_t* counters_dst, uint32_t counter_words, int blocks);
// culling_rebin.cu: pull the device state back into the host mirror (no-op unless the device is ahead of it)
int syncHostFromDevice(lb200_culling* cs);

// pages the kernels have to look at: the host's high-water mark, or the device's own while it is ahead of the host mirror
inline uint32_t livePages(const lb200_culling* cs) { return cs->device_authoritative ? cs->dev_high_water : cs->host.high_water; }
// no entity is added (the reference's empty m_cells, culling_system.cpp:322): the host's chains are stale after device adds / removes,
// its entity count is not
inline bool noEntities(const lb200_culling* cs) { return cs->device_authoritative ? cs->host.n_entities == 0 : cs->host.cells.empty(); }

// the host mirror made current before it is read or edited, by const accessors too: LB200_OK or the error of the pull-back
inline int hostView(const lb200_culling* cs) { return cs && cs->device_authoritative ? syncHostFromDevice(const_cast<lb200_culling*>(cs)) : LB200_OK; }
#define LB200_HOST_VIEW(cs)                                               \
	do {                                                                  \
		if (const int rc__ = lbcull::hostView(cs)) return rc__;           \
	} while (0)

// rank r's exchange buffer of epoch `epoch` as this process addresses it, and in it the slab this rank writes
inline uint32_t* peerBuffer(const lb200_ctx* ctx, uint32_t epoch, int r) { return ctx->peer.gather[epoch % ctx->peer.n_buffers][r]; }
inline uint32_t* peerSlab(const lb200_ctx* ctx, uint32_t epoch, int r) { return peerBuffer(ctx, epoch, r) + ctx->peer.slab_words * (size_t)ctx->rank; }
// every rank's slab of `epoch` and flag block, null beyond the ranks: where a kernel that publishes an epoch stores
inline void peerTargets(const lb200_ctx* ctx, uint32_t epoch, uint32_t** dst, uint32_t** flags) {
	for (int r = 0; r < LB200_MAX_RANKS; ++r) {
		dst[r] = r < ctx->n_ranks ? peerSlab(ctx, epoch, r) : nullptr;
		flags[r] = r < ctx->n_ranks ? ctx->peer.flags[r] : nullptr;
	}
}

// launch on `stream`, with programmatic stream serialization when `pdl`; *attr holds the attribute for as long as the config is used
inline cudaLaunchConfig_t launchConfig(unsigned grid, unsigned block, cudaStream_t stream, cudaLaunchAttribute* attr, bool pdl) {
	attr->id = cudaLaunchAttributeProgrammaticStreamSerialization;
	attr->val.programmaticStreamSerializationAllowed = 1;
	cudaLaunchConfig_t cfg = {};
	cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.stream = stream; cfg.attrs = attr; cfg.numAttrs = pdl ? 1 : 0;
	return cfg;
}

} // namespace lbcull
