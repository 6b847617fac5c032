// Multi-GPU exchange of the culling system (SURVEY.md §8e): the all-gather of visible ids (NCCL, or the fused pack + NVLink push), and
// the bitmask exchange steps whose cull kernel stores its {page, row} records straight into every rank's slab.
#include "culling_internal.h"

namespace {

using namespace lbcull;

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

// words one rank contributes to a bitmask exchange step: header + page ids + rows (cull_kernel.cuh)
size_t exchangeSlabWords(const lb200_culling* cs) { return XHEADER_WORDS + 9 * (size_t)cs->item_cap; }

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
	rc = launchPack(cs, cur, slab_ids, cs->d_slab + 256, cs->d_slab, 256, ctx->sm_count * 8);
	if (rc) return rc;
	return lb200_comm_allgather_u32(ctx, cs->d_slab, cs->d_gather_ids, 256 + (size_t)slab_ids);
}

int prepareExchange(lb200_culling* cs, const lb200_shifted_frustum* frustum) {
	if (!cs || !frustum) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	lb200_ctx::Peer& peer = ctx->peer;
	if (!peer.ready) { lb200_set_error(ctx, "cull_exchange needs lb200_comm_enable_p2p"); return LB200_ERR_STATE; }
	if (noEntities(cs)) { lb200_set_error(ctx, "cull_exchange on an empty culling system"); return LB200_ERR_STATE; }
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
int publishAndWait(lb200_culling* cs, uint32_t epoch, const uint32_t* counters, cudaStream_t stream) {
	lb200_ctx* ctx = cs->ctx;
	lb200_ctx::Peer& peer = ctx->peer;
	PublishParams PP;
	PP.n_ranks = (uint32_t)ctx->n_ranks; PP.rank = (uint32_t)ctx->rank; PP.epoch = epoch; PP.n_buffers = peer.n_buffers;
	PP.n_pages = cs->last_pages; PP.item_cap = cs->item_cap;
	peerTargets(ctx, epoch, PP.dst, PP.flags);
	cudaLaunchAttribute attr;
	const cudaLaunchConfig_t cfg = launchConfig(1, 288, stream, &attr, true);
	LB200_CUDA(ctx, cudaLaunchKernelEx(&cfg, publish_wait_kernel, PP, counters, peer.d_timeout));
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

// one two-kernel exchange step on the context stream: the cull kernel stores rows + counts into every rank, publish_wait_kernel then
// raises this rank's epoch flag everywhere and holds the stream until every rank's flag of this epoch is here
int exchangeStep(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type) {
	Exchange x;
	x.epoch = ++cs->ctx->peer.epoch;
	const int rc = launchCull(cs, frustum, type, &x);
	if (rc) return rc;
	return publishAndWait(cs, x.epoch, cs->last_counters, cs->ctx->stream);
}

// One fused step on lane l = epoch % lanes: ONE kernel.  The cull of epoch e publishes the lane's previous epoch from its own prologue and
// holds its record stores back until every rank has published e - 2 x lanes (cull_kernel.cuh); the batch closes with publishAndWait per lane.
int exchangeStepFused(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type) {
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

void lastExchange(lb200_culling* cs, const uint32_t** out_dev_ids, const uint32_t** out_dev_slabs, uint32_t* out_slab_stride_words) {
	const lb200_ctx::Peer& peer = cs->ctx->peer;
	if (out_dev_ids) *out_dev_ids = cs->last_out;
	if (out_dev_slabs) *out_dev_slabs = peerBuffer(cs->ctx, peer.epoch, cs->ctx->rank);
	if (out_slab_stride_words) *out_slab_stride_words = (uint32_t)peer.slab_words;
}

} // namespace

extern "C" {

int lb200_culling_cull_gather(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t slab_ids, const uint32_t** out_dev_slabs) {
	if (!cs || !frustum) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	if (noEntities(cs)) { lb200_set_error(ctx, "cull_gather on an empty culling system"); return LB200_ERR_STATE; }
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
		peerTargets(ctx, epoch, PP.dst, PP.flags);
		pack_push_kernel<<<ctx->sm_count * pushGridMul(), 256, 0, ctx->stream>>>(PP, cur, cs->last_out, peer.done_counter);
		LB200_CHECK_LAUNCH(ctx);
		wait_peers_kernel<<<1, 32, 0, ctx->stream>>>(peer.flags[ctx->rank], (uint32_t)ctx->n_ranks, epoch, peer.n_buffers, peer.d_timeout);
		LB200_CHECK_LAUNCH(ctx);
		if (out_dev_slabs) *out_dev_slabs = peerBuffer(ctx, epoch, ctx->rank);
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
