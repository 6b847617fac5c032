// Internal declarations shared by the translation units of liblumix_b200.so.
#pragma once

#include "../../include/lumix_b200.h"

#include <cuda_runtime.h>
#include <nvtx3/nvToolsExt.h> // header-only; a no-op unless a tool (ncu, nsys) injects itself

#include <atomic>
#include <stdarg.h>
#include <stdio.h>
#include <string.h>
#include <utility>

// ---- Owning handles of the CUDA resources the library allocates for itself ----
// A handle frees its resource when it is destroyed or re-allocated, so an object's destructor releases everything it owns.  An
// empty handle makes no CUDA call at all: a culling system without a context never touches the runtime.  Arrays record their
// element count, so no separate capacity can disagree with the pointer.  Handles convert to the raw pointer or handle, which is
// what kernels, their parameter structs and the runtime calls take.
struct lb200_device_mem {
	static cudaError_t alloc(void** p, size_t bytes) { return cudaMalloc(p, bytes); }
	static void release(void* p) { cudaFree(p); }
};
template <unsigned Flags> struct lb200_pinned_mem {
	static cudaError_t alloc(void** p, size_t bytes) { return cudaHostAlloc(p, bytes, Flags); }
	static void release(void* p) { cudaFreeHost(p); }
};

template <class T, class Mem> class lb200_array {
public:
	lb200_array() = default;
	lb200_array(lb200_array&& o) noexcept : p_(std::exchange(o.p_, nullptr)), n_(std::exchange(o.n_, 0)) {}
	lb200_array& operator=(lb200_array&& o) noexcept {
		if (this != &o) { reset(); p_ = std::exchange(o.p_, nullptr); n_ = std::exchange(o.n_, 0); }
		return *this;
	}
	~lb200_array() { reset(); }
	void reset() {
		if (p_) Mem::release(p_);
		p_ = nullptr;
		n_ = 0;
	}
	// Frees what the handle holds, then allocates n elements (bytes_if_empty bytes when n is 0, so that an empty table can still have
	// an address).  Returns the runtime's error for LB200_CUDA to report; a failed allocation leaves the handle empty with size 0.
	cudaError_t alloc(size_t n, size_t bytes_if_empty = 0) {
		reset();
		void* p = nullptr;
		const cudaError_t e = Mem::alloc(&p, n ? sizeof(T) * n : bytes_if_empty);
		if (e != cudaSuccess) {
			cudaGetLastError(); // an allocation failure is reported here, not by the next kernel launch check
			return e;
		}
		p_ = static_cast<T*>(p);
		n_ = p ? n : 0;
		return cudaSuccess;
	}
	size_t size() const { return n_; }
	T* get() const { return p_; }
	operator T*() const { return p_; }

private:
	T* p_ = nullptr;
	size_t n_ = 0;
};
template <class T> using DeviceArray = lb200_array<T, lb200_device_mem>;
template <class T, unsigned Flags = cudaHostAllocDefault> using PinnedArray = lb200_array<T, lb200_pinned_mem<Flags>>;

template <class H, cudaError_t (*Destroy)(H)> class lb200_handle {
public:
	lb200_handle() = default;
	lb200_handle(lb200_handle&& o) noexcept : h_(std::exchange(o.h_, nullptr)) {}
	lb200_handle& operator=(lb200_handle&& o) noexcept {
		if (this != &o) { reset(); h_ = std::exchange(o.h_, nullptr); }
		return *this;
	}
	~lb200_handle() { reset(); }
	void reset() {
		if (h_) Destroy(h_);
		h_ = nullptr;
	}
	// destroys what the handle holds and returns where a cudaEventCreate* / cudaStreamCreate* call stores the new one
	H* create() {
		reset();
		return &h_;
	}
	operator H() const { return h_; }

private:
	H h_ = nullptr;
};
using Event = lb200_handle<cudaEvent_t, cudaEventDestroy>;
using Stream = lb200_handle<cudaStream_t, cudaStreamDestroy>;

// Scratch of one caller of the device radix sort (radix_sort.cu): the sort's state, a type private to radix_sort.cu, and one 256-digit
// histogram row per block a sort with it may launch.  lb200_radix_sort_alloc_scratch sizes it; the alternate key / value buffers stay
// with the caller.
struct RadixSortScratch {
	DeviceArray<uint8_t> state;
	DeviceArray<uint32_t> block_hist; // [blocks()][256]
	uint32_t blocks() const { return (uint32_t)(block_hist.size() / 256); }
};

#define LB200_MAX_RANKS 8
#define LB200_MAX_LANES 8  // concurrent culls (streams / output lanes); exchange buffers = 3 x lanes

struct lb200_ctx {
	int device = -1;
	Stream stream;
	Stream copy_stream;
	int sm_count = 0;
	uint32_t radix_sort_grid = 0; // blocks of radix_sort_kernel that can be co-resident (radix_sort.cu), 0 until the first scratch is sized
	std::atomic<uint64_t> launches{0};
	char error[512] = {0};
	// scratch of lb200_radix_sort_device (radix_sort.cu): the alternate key / value buffers, grown to the largest cap asked for (their size is
	// the capacity), and the sort's own scratch for every co-resident block
	DeviceArray<uint64_t> radix_keys1, radix_values1;
	RadixSortScratch radix_scratch;
	// NCCL (dlopen) state, see comm.cu
	void* nccl_lib = nullptr;
	void* nccl_comm = nullptr;
	int n_ranks = 1;
	int rank = 0;
	// NVLink peer exchange (comm.cu lb200_comm_enable_p2p): every rank's gather buffers mapped into every process
	struct Peer {
		bool ready = false;
		size_t slab_words = 0;            // capacity of one rank's slab (header + ids)
		// Exchange epoch e uses buffer e % n_buffers, n_buffers = 3 x lanes.  A batch of lb200_culling_cull_exchange_n with lanes > 1 and
		// n > 1 issues epoch e on stream e % lanes as ONE kernel: the cull of e publishes the lane's previous epoch (e - lanes) from its
		// prologue and holds its record stores back until every rank has published e - 2 x lanes.  So a rank overwrites buffer b for epoch
		// e only after every rank published e - 2 x lanes, which a rank does from its cull of e - lanes — issued behind whatever consumed
		// e - 3 x lanes, the previous owner of b.  Every other step (lb200_culling_cull_exchange, and batches with one lane or one step)
		// runs on the context stream as the cull followed by publish_wait_kernel, after everything issued before it has finished waiting.
		// tests/test_exchange_protocol_model.py replays both kinds, mixed as callers issue them, under a random scheduler, and shows that
		// fewer buffers or no flow control would not do.
		uint32_t lanes = 1, n_buffers = 3;
		DeviceArray<char> local_block;    // this rank's allocation: [flags n_buffers x 8 x u32 in 512 B][gather 0] .. [gather n_buffers-1]
		uint32_t* gather[3 * LB200_MAX_LANES][LB200_MAX_RANKS] = {}; // gather[b][r] = rank r's buffer b as seen from this process
		uint32_t* flags[LB200_MAX_RANKS] = {};     // flags[r] = rank r's flag block
		// cudaIpcOpenMemHandle results, raw: comm.cu closes them before local_block is freed, an order the peer protocol depends on
		void* opened[LB200_MAX_RANKS] = {};
		DeviceArray<uint32_t> done_counter; // local, one per lane, for the last-block election
		uint32_t epoch = 0;
		// a wait kernel that gave up on a peer (~4 s) raises this word; page-locked + mapped so the host sees it without a copy.
		// lb200_comm_check() turns it into LB200_ERR_NCCL and resets it (called by lb200_synchronize and every exchange entry point)
		PinnedArray<uint32_t, cudaHostAllocMapped> h_timeout;
		uint32_t* d_timeout = nullptr; // h_timeout as the device addresses it
	} peer;
};

void lb200_set_error(lb200_ctx* ctx, const char* fmt, ...);

// NVTX range named like the reference's PROFILE_BLOCK / PROFILE_FUNCTION scopes (SURVEY.md §5: culling_system.cpp:330 "culling",
// animation_module.cpp:743 "update animables"), so that a timeline of the engine with this library reads like the reference's own.
struct lb200_range {
	explicit lb200_range(const char* name) { nvtxRangePushA(name); }
	~lb200_range() { nvtxRangePop(); }
	lb200_range(const lb200_range&) = delete;
	lb200_range& operator=(const lb200_range&) = delete;
};
// culling.cu: where the last cull left its result (device: ids, counters; host: per-type segment bases and entity counts, 256 each)
int lb200_culling_internal_last(lb200_culling* cs, const uint32_t** out_ids, const uint32_t** counters, const uint32_t** type_base, const uint32_t** type_counts);
// culling.cu: 1 + the largest entity id ever added (0 if none): every id a cull of cs can emit is below it
uint32_t lb200_culling_internal_entity_range(const lb200_culling* cs);
// context.cu: *out = blocks of a cooperative kernel that can be co-resident on the context's device (threads per block, dynamic smem)
int lb200_coop_grid_limit(lb200_ctx* ctx, const void* kernel, int threads, size_t smem, uint32_t* out);
// radix_sort.cu: scratch for sorts of up to min(blocks, co-resident blocks) blocks; on failure `out` is left as it was
int lb200_radix_sort_alloc_scratch(lb200_ctx* ctx, uint32_t blocks, RadixSortScratch& out);
// radix_sort.cu: stable LSD radix sort of n = min(*count_dev, cap) (u64 key, u64 value) pairs, one cooperative launch on `stream`, n read on
// the device; the result ends in buffer 0.  Launches max(1, min(scratch.blocks(), max_blocks unless 0, ceil(cap / 2048))) blocks.
// force_tiled: the tiled path at any n (the register path is taken iff !force_tiled && n <= grid * 512 * 16); *out_grid (may be null) = blocks launched
int lb200_radix_sort_pairs(lb200_ctx* ctx, cudaStream_t stream, uint64_t* keys0, uint64_t* keys1, uint64_t* values0, uint64_t* values1, const uint32_t* count_dev, uint32_t cap,
	const RadixSortScratch& scratch, uint32_t max_blocks, bool force_tiled, uint32_t* out_grid);
int lb200_comm_check(lb200_ctx* ctx); // comm.cu: LB200_ERR_NCCL (and reset) if a peer wait timed out since the last check
int lb200_comm_allgather_u32(lb200_ctx* ctx, const uint32_t* send, uint32_t* recv, size_t words); // comm.cu, asynchronous on the context stream
uint32_t lb200_cull_lanes(); // LB200_CULL_LANES, default 2, 1..LB200_MAX_LANES (context.cu)

#define LB200_CUDA(ctx, expr)                                                                        \
	do {                                                                                             \
		cudaError_t e__ = (expr);                                                                    \
		if (e__ != cudaSuccess) {                                                                    \
			lb200_set_error((ctx), "%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
			return LB200_ERR_CUDA;                                                                   \
		}                                                                                            \
	} while (0)

#define LB200_CHECK_LAUNCH(ctx)                                                                      \
	do {                                                                                             \
		(ctx)->launches.fetch_add(1, std::memory_order_relaxed);                                     \
		cudaError_t e__ = cudaGetLastError();                                                        \
		if (e__ != cudaSuccess) {                                                                    \
			lb200_set_error((ctx), "kernel launch failed: %s (%s:%d)", cudaGetErrorString(e__), __FILE__, __LINE__); \
			return LB200_ERR_CUDA;                                                                   \
		}                                                                                            \
	} while (0)

// Device page layout (DESIGN.md §3): page p owns slots [p*200, p*200+200) of the sphere / entity arrays.
struct alignas(32) lb200_page_desc {
	double origin[3]; // CellPage::header.origin, culling_system.cpp:55
	uint32_t count;   // header.count (0 = free page, skipped by the kernel)
	uint8_t type;     // header.indices.type
	uint8_t is_big;   // header.indices.is_big
	uint16_t pad;
};
static_assert(sizeof(lb200_page_desc) == 32, "page descriptor is one 32-byte sector");
static_assert(sizeof(lb200_shifted_frustum) == 256, "ShiftedFrustum image, geometry.h:99-149");
static_assert(sizeof(lb200_transform) == 56, "Transform image, math.h:306-327");
static_assert(sizeof(lb200_track) == 32, "track descriptor");
static_assert(sizeof(lb200_sk_model) == 64 && sizeof(lb200_sk_mesh) == 16 && sizeof(lb200_sk_view) == 1352, "sort-key tables");
