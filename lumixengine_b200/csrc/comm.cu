// Multi-GPU exchange of the visible lists (include/lumix_b200.h "Multi-GPU"; SURVEY.md §8e).
//
// The reference has no distributed code at all; the path shards by whole cell pages (each rank owns a subset of the
// entities and runs the same cull), and the only exchange step is the all-gather of the compacted visible lists.
// NCCL is resolved with dlopen so that single-GPU users never need it; inside a torch process the already-loaded
// libnccl.so.2 (torch's bundled copy) is the one that gets picked up.
#include "lb200_internal.h"

#include <dlfcn.h>

// minimal NCCL ABI (nccl.h): only what is called here
typedef struct ncclComm* ncclComm_t;
typedef struct { char internal[128]; } ncclUniqueId;
typedef int ncclResult_t;
enum { ncclUint8_dt = 1, ncclUint32_dt = 3 };

typedef ncclResult_t (*PFN_ncclGetUniqueId)(ncclUniqueId*);
typedef ncclResult_t (*PFN_ncclCommInitRank)(ncclComm_t*, int, ncclUniqueId, int);
typedef ncclResult_t (*PFN_ncclCommDestroy)(ncclComm_t);
typedef ncclResult_t (*PFN_ncclAllGather)(const void*, void*, size_t, int, ncclComm_t, cudaStream_t);
typedef const char* (*PFN_ncclGetErrorString)(ncclResult_t);

static PFN_ncclGetUniqueId p_ncclGetUniqueId;
static PFN_ncclCommInitRank p_ncclCommInitRank;
static PFN_ncclCommDestroy p_ncclCommDestroy;
static PFN_ncclAllGather p_ncclAllGather;
static PFN_ncclGetErrorString p_ncclGetErrorString;


static int loadNccl(lb200_ctx* ctx) {
	if (ctx->nccl_lib) return LB200_OK;
	void* lib = dlopen("libnccl.so.2", RTLD_NOW | RTLD_GLOBAL);
	if (!lib) lib = dlopen("libnccl.so", RTLD_NOW | RTLD_GLOBAL);
	if (!lib) {
		lb200_set_error(ctx, "cannot dlopen libnccl.so.2: %s", dlerror());
		return LB200_ERR_NCCL;
	}
	p_ncclGetUniqueId = (PFN_ncclGetUniqueId)dlsym(lib, "ncclGetUniqueId");
	p_ncclCommInitRank = (PFN_ncclCommInitRank)dlsym(lib, "ncclCommInitRank");
	p_ncclCommDestroy = (PFN_ncclCommDestroy)dlsym(lib, "ncclCommDestroy");
	p_ncclAllGather = (PFN_ncclAllGather)dlsym(lib, "ncclAllGather");
	p_ncclGetErrorString = (PFN_ncclGetErrorString)dlsym(lib, "ncclGetErrorString");
	if (!p_ncclGetUniqueId || !p_ncclCommInitRank || !p_ncclCommDestroy || !p_ncclAllGather) {
		lb200_set_error(ctx, "libnccl lacks a required symbol");
		dlclose(lib);
		return LB200_ERR_NCCL;
	}
	ctx->nccl_lib = lib;
	return LB200_OK;
}

#define LB200_NCCL(ctx, expr)                                                                                  \
	do {                                                                                                       \
		ncclResult_t r__ = (expr);                                                                             \
		if (r__ != 0) {                                                                                        \
			lb200_set_error((ctx), "%s failed: %s", #expr, p_ncclGetErrorString ? p_ncclGetErrorString(r__) : "?"); \
			return LB200_ERR_NCCL;                                                                             \
		}                                                                                                      \
	} while (0)

// used by culling_exchange.cu: all-gather `words` u32 per rank on the context stream (asynchronous)
int lb200_comm_allgather_u32(lb200_ctx* ctx, const uint32_t* send, uint32_t* recv, size_t words) {
	if (!ctx->nccl_comm) { lb200_set_error(ctx, "lb200_comm_init has not been called"); return LB200_ERR_STATE; }
	LB200_NCCL(ctx, p_ncclAllGather(send, recv, words, ncclUint32_dt, (ncclComm_t)ctx->nccl_comm, ctx->stream));
	ctx->launches.fetch_add(1, std::memory_order_relaxed);
	return LB200_OK;
}

int lb200_comm_check(lb200_ctx* ctx) {
	lb200_ctx::Peer& P = ctx->peer;
	volatile uint32_t* timeout = P.h_timeout;
	if (!timeout || !*timeout) return LB200_OK;
	*timeout = 0;
	lb200_set_error(ctx, "multi-GPU exchange: a peer's slab did not arrive within the wait limit (~4 s); the exchanged slabs of that step are incomplete");
	return LB200_ERR_NCCL;
}

extern "C" {

int lb200_comm_status(lb200_ctx* ctx) { return ctx ? lb200_comm_check(ctx) : LB200_ERR_INVALID; }

int lb200_comm_get_unique_id(lb200_ctx* ctx, uint8_t out_id[128]) {
	if (!ctx || !out_id) return LB200_ERR_INVALID;
	int rc = loadNccl(ctx);
	if (rc) return rc;
	ncclUniqueId id;
	LB200_NCCL(ctx, p_ncclGetUniqueId(&id));
	memcpy(out_id, &id, 128);
	return LB200_OK;
}

int lb200_comm_init(lb200_ctx* ctx, int n_ranks, int rank, const uint8_t unique_id[128]) {
	if (!ctx || !unique_id || n_ranks < 1 || rank < 0 || rank >= n_ranks) return LB200_ERR_INVALID;
	int rc = loadNccl(ctx);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	ncclUniqueId id;
	memcpy(&id, unique_id, 128);
	ncclComm_t comm = nullptr;
	LB200_NCCL(ctx, p_ncclCommInitRank(&comm, n_ranks, id, rank));
	ctx->nccl_comm = comm;
	ctx->n_ranks = n_ranks;
	ctx->rank = rank;
	return LB200_OK;
}

// Map every rank's gather buffers into every process (CUDA IPC over NVLink peer access).  Collective: all ranks call it with the same
// max_slab_ids.  The IPC handles travel through one ncclAllGather, so the caller needs no extra side channel.
static int enableP2p(lb200_ctx* ctx, uint32_t max_slab_ids) {
	const int R = ctx->n_ranks;
	lb200_ctx::Peer& P = ctx->peer;
	P.slab_words = (256 + (size_t)max_slab_ids + 63) & ~(size_t)63;
	const size_t flag_bytes = 1024;
	const size_t buf_bytes = sizeof(uint32_t) * P.slab_words * (size_t)R;
	P.lanes = lb200_cull_lanes(); // the same on every rank (same environment)
	P.n_buffers = 3 * P.lanes;
	static_assert(3 * LB200_MAX_LANES * LB200_MAX_RANKS * sizeof(uint32_t) <= 1024, "flag block");
	const size_t total = flag_bytes + P.n_buffers * buf_bytes;
	LB200_CUDA(ctx, P.local_block.alloc(total));
	LB200_CUDA(ctx, cudaMemsetAsync(P.local_block, 0, flag_bytes, ctx->stream));
	LB200_CUDA(ctx, P.done_counter.alloc(LB200_MAX_LANES));
	LB200_CUDA(ctx, cudaMemsetAsync(P.done_counter, 0, sizeof(uint32_t) * LB200_MAX_LANES, ctx->stream));
	LB200_CUDA(ctx, P.h_timeout.alloc(1));
	*P.h_timeout = 0;
	LB200_CUDA(ctx, cudaHostGetDevicePointer((void**)&P.d_timeout, P.h_timeout, 0));
	cudaIpcMemHandle_t mine;
	LB200_CUDA(ctx, cudaIpcGetMemHandle(&mine, P.local_block));
	// exchange the 64-byte handles with NCCL
	static_assert(sizeof(cudaIpcMemHandle_t) == 64, "");
	DeviceArray<uint32_t> d_h;
	LB200_CUDA(ctx, d_h.alloc(16 * (size_t)(R + 1)));
	LB200_CUDA(ctx, cudaMemcpyAsync(d_h + 16 * (size_t)R, &mine, 64, cudaMemcpyHostToDevice, ctx->stream));
	LB200_NCCL(ctx, p_ncclAllGather(d_h + 16 * (size_t)R, d_h, 16, ncclUint32_dt, (ncclComm_t)ctx->nccl_comm, ctx->stream));
	cudaIpcMemHandle_t all[LB200_MAX_RANKS];
	LB200_CUDA(ctx, cudaMemcpyAsync(all, d_h, 64 * (size_t)R, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	d_h.reset();
	for (int r = 0; r < R; ++r) {
		char* base;
		if (r == ctx->rank) base = P.local_block;
		else {
			void* p = nullptr;
			LB200_CUDA(ctx, cudaIpcOpenMemHandle(&p, all[r], cudaIpcMemLazyEnablePeerAccess));
			P.opened[r] = p;
			base = (char*)p;
		}
		P.flags[r] = (uint32_t*)base;
		for (uint32_t b = 0; b < P.n_buffers; ++b) P.gather[b][r] = (uint32_t*)(base + flag_bytes + b * buf_bytes);
	}
	// nobody may start pushing before every rank has mapped every buffer (and zeroed its flags): one more collective as a barrier
	DeviceArray<uint32_t> d_b;
	LB200_CUDA(ctx, d_b.alloc((size_t)(R + 1)));
	LB200_NCCL(ctx, p_ncclAllGather(d_b + R, d_b, 1, ncclUint32_dt, (ncclComm_t)ctx->nccl_comm, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	P.epoch = 0;
	P.ready = true;
	return LB200_OK;
}

static void releasePeer(lb200_ctx* ctx) {
	// the peers' mappings are closed before this rank's block is freed
	for (int r = 0; r < LB200_MAX_RANKS; ++r) if (ctx->peer.opened[r]) cudaIpcCloseMemHandle(ctx->peer.opened[r]);
	ctx->peer.local_block.reset();
	ctx->peer = lb200_ctx::Peer();
}

int lb200_comm_enable_p2p(lb200_ctx* ctx, uint32_t max_slab_ids) {
	if (!ctx) return LB200_ERR_INVALID;
	if (!ctx->nccl_comm) { lb200_set_error(ctx, "lb200_comm_init has not been called"); return LB200_ERR_STATE; }
	if (ctx->n_ranks > LB200_MAX_RANKS) { lb200_set_error(ctx, "peer exchange supports up to %d ranks (one NVSwitch box)", LB200_MAX_RANKS); return LB200_ERR_INVALID; }
	if (ctx->peer.ready) return LB200_OK;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const int rc = enableP2p(ctx, max_slab_ids);
	if (rc) { // a failed call leaves no peer state behind: a retry starts from scratch
		cudaStreamSynchronize(ctx->stream);
		releasePeer(ctx);
	}
	return rc;
}

void lb200_comm_destroy(lb200_ctx* ctx) {
	if (!ctx || !ctx->nccl_comm) return;
	cudaSetDevice(ctx->device);
	cudaStreamSynchronize(ctx->stream);
	releasePeer(ctx);
	// the NCCL communicator is a raw handle: it is created and destroyed here only, through the dlopen'ed library
	p_ncclCommDestroy((ncclComm_t)ctx->nccl_comm);
	ctx->nccl_comm = nullptr;
	ctx->n_ranks = 1;
	ctx->rank = 0;
}

} // extern "C"
