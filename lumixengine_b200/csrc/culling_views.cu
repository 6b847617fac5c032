// Several views of one frame culled in one pass (lb200_culling_cull_views, lb200_culling_select_view): the fused kernel cull_views_kernel
// (cull_views_kernel.cuh) for two or more views, cull_pages_kernel through launchCull for one.  The results go to buffers of their own,
// apart from the output lanes, so that plain culls and calls of this kind never disturb each other's results.
#include "cull_views_kernel.cuh"
#include "culling_internal.h"

#include <algorithm>

using namespace lbcull;
using namespace lbviews;

namespace lbcull {

// a view selected as the last cull stops being one: no cull is the last cull until the next plain cull or select_view
static void forgetSelectedView(lb200_culling* cs) {
	if (!cs->last_is_view) return;
	cs->last_counters = nullptr; cs->last_out = nullptr; cs->last_mask = nullptr; cs->last_pages = 0;
	cs->last_is_view = false;
}

void releaseViews(lb200_culling* cs) {
	cs->d_view_mask.reset();
	cs->views_live = false;
	forgetSelectedView(cs);
}

} // namespace lbcull

namespace {

// Counter blocks (once), then ids and masks of n_views views sized for the current entity count and page arrays
int ensureViewBuffers(lb200_culling* cs, uint32_t n_views) {
	lb200_ctx* ctx = cs->ctx;
	if (!cs->d_view_counters) {
		DeviceArray<uint32_t> counters;
		PinnedArray<uint32_t> h_counters;
		const size_t words = 2 * (size_t)CALL_COUNTER_WORDS + 2 * (size_t)COUNTER_WORDS;
		LB200_CUDA(ctx, counters.alloc(words));
		LB200_CUDA(ctx, cudaMemsetAsync(counters, 0, sizeof(uint32_t) * words, ctx->stream));
		LB200_CUDA(ctx, h_counters.alloc(CALL_COUNTER_WORDS));
		cs->d_view_counters = std::move(counters); cs->h_view_counters = std::move(h_counters);
	}
	const size_t id_cap = grownCapacity(cs->view_id_cap, 4096, cs->host.n_entities);
	if (id_cap != cs->view_id_cap || cs->d_view_ids.size() < id_cap * n_views) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_view_ids.reset();
		cs->view_id_cap = 0;
		LB200_CUDA(ctx, cs->d_view_ids.alloc(id_cap * n_views));
		cs->view_id_cap = (uint32_t)id_cap;
	}
	const size_t mask_words = (size_t)8 * cs->dev_cap * n_views;
	if (cs->d_view_mask.size() < mask_words) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		cs->d_view_mask.reset();
		LB200_CUDA(ctx, cs->d_view_mask.alloc(mask_words));
	}
	return LB200_OK;
}

// the fused kernel for n_views >= 2 views on the context stream; launch shape and programmatic launch decided as for launchCull (prepareLaunch)
int launchViews(lb200_culling* cs, const lb200_shifted_frustum* frusta, const uint8_t* types, uint32_t n_views, uint32_t* counters, uint32_t* next_counters) {
	lb200_range range("culling views");
	lb200_ctx* ctx = cs->ctx;
	ViewsParams P = {};
	for (uint32_t v = 0; v < n_views; ++v) {
		fillFrustum(&P.f[v], frusta + v);
		P.type_filter[v] = types[v];
	}
	// the chunk bounded by the items a round holds: min(256, 512 / n_views) pages
	const CullLaunch L = prepareLaunch(cs, P.type_base, (uint32_t)cs->grid, viewsChunkBound(n_views));
	memcpy(cs->views_type_base, P.type_base, sizeof(P.type_base));
	P.n_views = n_views;
	P.n_pages = L.n_pages;
	P.chunk = L.chunk;
	P.plane_masking = L.plane_masking;
	P.id_stride = cs->view_id_cap;
	P.mask_stride = 8 * cs->dev_cap;
	cudaLaunchAttribute attr;
	const cudaLaunchConfig_t cfg = launchConfig(L.blocks, VIEW_THREADS, ctx->stream, &attr, L.pdl);
	LB200_CUDA(ctx, cudaLaunchKernelEx(&cfg, cull_views_kernel, P, (const lb200_page_desc*)(cs->d_desc + L.off), (const float4*)(cs->d_spheres + L.off * LB200_PAGE_SLOTS),
		(const int*)(cs->d_entities + L.off * LB200_PAGE_SLOTS), cs->d_view_ids.get(), counters, next_counters, cs->d_view_mask.get()));
	LB200_CHECK_LAUNCH(ctx);
	recordLaunch(cs, L);
	return LB200_OK;
}

} // namespace

int lb200_culling_internal_views(lb200_culling* cs, CullViewsResult* out) {
	if (!cs || !cs->ctx || !out) return LB200_ERR_INVALID;
	if (!cs->views_n) { lb200_set_error(cs->ctx, "no cull_views has been issued on this culling system yet"); return LB200_ERR_STATE; }
	if (!cs->views_live) {
		lb200_set_error(cs->ctx, "the latest cull_views call has no results (an empty culling system, or the page arrays grew / set_replicas since)");
		return LB200_ERR_STATE;
	}
	out->n_views = cs->views_n; out->id_stride = cs->view_id_cap; out->counter_stride = COUNTER_WORDS;
	out->ids = cs->d_view_ids; out->counters = cs->views_counters; out->type_base = cs->views_type_base; out->type_counts = cs->host.type_counts;
	return LB200_OK;
}

extern "C" {

int lb200_culling_cull_views(lb200_culling* cs, const lb200_shifted_frustum* frusta, const uint8_t* types, uint32_t n_views,
	const uint32_t** dev_ids, lb200_cull_result* results, int want_counts)
{
	if (!cs || !frusta) return LB200_ERR_INVALID;
	if (n_views < 1 || n_views > LB200_CULL_MAX_VIEWS) { lb200_set_error(cs->ctx, "cull_views: n_views %u is not 1..%d", n_views, LB200_CULL_MAX_VIEWS); return LB200_ERR_INVALID; }
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	lb200_ctx* ctx = cs->ctx;
	forgetSelectedView(cs); // the previous call's results end here
	cs->views_n = n_views;
	cs->views_live = false;
	if (noEntities(cs)) { // culling_system.cpp:322
		if (results) memset(results, 0, sizeof(*results) * n_views);
		if (dev_ids) for (uint32_t v = 0; v < n_views; ++v) dev_ids[v] = nullptr;
		cs->has_last = false;
		return LB200_OK;
	}
	int rc = flushPages(cs);
	if (rc) return rc;
	rc = ensureViewBuffers(cs, n_views);
	if (rc) return rc;
	uint8_t tf[LB200_CULL_MAX_VIEWS];
	for (uint32_t v = 0; v < n_views; ++v) tf[v] = types ? types[v] : (uint8_t)LB200_TYPE_ALL;
	const bool single = n_views == 1;
	const size_t block_words = single ? COUNTER_WORDS : CALL_COUNTER_WORDS;
	uint32_t* blocks = single ? cs->d_view_counters + 2 * (size_t)CALL_COUNTER_WORDS : cs->d_view_counters.get();
	uint8_t& parity = cs->view_parity[single ? 1 : 0];
	uint32_t* cur = blocks + parity * block_words;
	uint32_t* nxt = blocks + (parity ^ 1u) * block_words;
	if (single) {
		const CullOutput dest = {cs->d_view_ids.get(), cur, nxt, cs->d_view_mask.get(), cs->views_type_base};
		rc = launchCull(cs, frusta, tf[0], nullptr, nullptr, &dest);
	}
	else rc = launchViews(cs, frusta, tf, n_views, cur, nxt);
	if (rc) return rc;
	parity ^= 1u;
	cs->views_counters = cur;
	cs->views_pages = livePages(cs);
	cs->views_live = true;
	if (dev_ids) for (uint32_t v = 0; v < n_views; ++v) dev_ids[v] = cs->d_view_ids + (size_t)v * cs->view_id_cap;
	if (!want_counts) { cs->has_last = false; return LB200_OK; }
	LB200_CUDA(ctx, cudaMemcpyAsync(cs->h_view_counters, cur, sizeof(uint32_t) * block_words, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	// DESIGN.md §4.1: descriptors once, each tested page's spheres once, then per view (4 B id read + 4 B id write) per visible + its mask
	const uint32_t* hc = cs->h_view_counters;
	const uint64_t streamed = single ? hc[256 + ST_ENT_STREAMED] : hc[MAX_VIEWS * COUNTER_WORDS + CALL_STREAMED];
	const uint64_t pages = cs->views_pages;
	uint64_t bytes = pages * 32 + streamed * 16;
	for (uint32_t v = 0; v < n_views; ++v) {
		lb200_cull_result res;
		fillResult(cs, hc + (size_t)v * COUNTER_WORDS, cs->views_type_base, &res);
		bytes += (uint64_t)res.total * 8 + pages * 32;
		if (results) results[v] = res;
	}
	cs->last_bytes = bytes;
	cs->has_last = true;
	return LB200_OK;
}

int lb200_culling_select_view(lb200_culling* cs, uint32_t k) {
	if (!cs) return LB200_ERR_INVALID;
	if (!cs->ctx) return LB200_ERR_NO_DEVICE;
	if (!cs->views_n) { lb200_set_error(cs->ctx, "select_view needs a preceding cull_views"); return LB200_ERR_STATE; }
	if (k >= cs->views_n) { lb200_set_error(cs->ctx, "select_view: view %u of a cull_views call of %u views", k, cs->views_n); return LB200_ERR_INVALID; }
	if (!cs->views_live) {
		lb200_set_error(cs->ctx, "select_view: the latest cull_views call has no results (an empty culling system, or the page arrays grew / set_replicas since)");
		return LB200_ERR_STATE;
	}
	cs->last_counters = cs->views_counters + (size_t)k * COUNTER_WORDS;
	cs->last_out = cs->d_view_ids + (size_t)k * cs->view_id_cap;
	cs->last_mask = cs->d_view_mask + (size_t)k * 8 * cs->dev_cap;
	cs->last_pages = cs->views_pages;
	memcpy(cs->last_type_base, cs->views_type_base, sizeof(cs->last_type_base));
	cs->last_is_view = true;
	return LB200_OK;
}

} // extern "C"
