// PipelineImpl::radixSort (src/renderer/pipeline.cpp:4020-4144) on the device: the stable sort of (u64 key, u64 value) pairs behind
// createSortKeys (sortkeys.cu), the sort of the chain changers of the device re-binning (culling_rebin.cu) and lb200_radix_sort_device.
//
//   radix_sort_kernel  LSD, 8 bits per pass over the 64-bit keys, stable, hand-written, ONE cooperative launch for all passes: only bits that
//             differ between keys are sorted on (OR of all keys / of all complements; the reference skips the all-in-bin-0 case, :4120);
//             per pass block histograms -> grid barrier -> every block sums the histograms of the blocks before it -> stable scatter
//             (warp match + per-warp digit counters) -> grid barrier.  No library sort.
// Its scratch (the SortState and one histogram row per block) is a RadixSortScratch, laid out here alone; the alternate key / value
// buffers belong to the callers.
#include "grid_barrier.cuh"
#include "lb200_internal.h"

#include <algorithm>

namespace {

using namespace lb;

constexpr int RS_THREADS = 512;
constexpr int RS_WARPS = RS_THREADS / 32;
constexpr int RS_ITEMS = 4;                         // keys per thread and tile
constexpr int RS_TILE = RS_THREADS * RS_ITEMS;      // 2048 keys
constexpr int RS_PASSES = 8;
struct SortState { // zero-initialised before every launch
	GridBar bar; uint32_t pad[2];
	unsigned long long key_or, key_or_not; // OR of all keys, OR of all complements
	uint32_t digit_total[RS_PASSES][256];    // per digit window: keys of every digit, summed by the blocks with one atomic each
};

constexpr int RS_REG_ITEMS = 16;                    // keys a thread can keep in registers over all passes

// Where this block's keys of digit d start: all keys of smaller digits + the keys of digit d in the blocks before this one.
// In: block_hist[b][d] of every block and digit_total[d] = their column sums (behind a grid barrier).  Out: s_hist[d].  All RS_THREADS threads.
// A block in the first half of the grid sums the rows before it, one in the second half subtracts the rows from itself on from the total:
// nobody reads more than half of the rows.
__device__ __forceinline__ void digit_starts(const uint32_t* block_hist, const uint32_t* digit_total, uint32_t* s_hist, uint32_t (*s_part)[256], uint32_t* s_wsum) {
	const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
	const uint32_t d = tid & 255u, part = tid >> 8;
	const bool front = 2u * blockIdx.x <= gridDim.x;
	const uint32_t row_begin = front ? 0u : blockIdx.x, row_end = front ? blockIdx.x : gridDim.x;
	uint32_t sum = 0;
	// 8 rows in flight per thread: the rows come from L2 and a row-at-a-time loop would pay one L2 round trip per row
	for (uint32_t b0 = row_begin + part; b0 < row_end; b0 += 8 * (RS_THREADS / 256)) {
		uint32_t c[8];
#pragma unroll
		for (int u = 0; u < 8; ++u) {
			const uint32_t b = b0 + u * (RS_THREADS / 256);
			c[u] = b < row_end ? __ldcg(block_hist + b * 256 + d) : 0u;
		}
#pragma unroll
		for (int u = 0; u < 8; ++u) sum += c[u];
	}
	s_part[part][d] = sum;
	__syncthreads();
	uint32_t x = 0, mine = 0, before = 0;
	if (tid < 256) { // exclusive scan of the 256 digit totals by the first 8 warps
		mine = __ldcg(digit_total + tid);
		const uint32_t rows = s_part[0][tid] + s_part[1][tid];
		before = front ? rows : mine - rows;
		x = mine;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (uint32_t)o) x += y; }
		if (lane == 31) s_wsum[warp] = x;
	}
	__syncthreads();
	if (tid < 256) {
		uint32_t start = x - mine;
		for (uint32_t w = 0; w < warp; ++w) start += s_wsum[w];
		s_hist[tid] = start + before;
	}
	__syncthreads();
}

// All passes in one cooperative launch, stable: the key order is "block, then position inside the block's contiguous run".
//   n <= gridDim * RS_THREADS * RS_REG_ITEMS (a frame's worth of draw keys): every block owns ONE run of `items` keys per thread that stays in
//   registers from the pass's ranking to its scatter — a pass reads every pair once and writes it once;
//   larger n: tiles of RS_TILE keys, dealt to the blocks in contiguous runs (block b: tiles [b*T/G, (b+1)*T/G)), counted, then re-read and scattered.
__global__ void __launch_bounds__(RS_THREADS, 1) radix_sort_kernel(uint64_t* kbuf0, uint64_t* kbuf1, uint64_t* vbuf0, uint64_t* vbuf1, const uint32_t* __restrict__ counts, uint32_t cap,
	SortState* st, uint32_t* block_hist /* [gridDim][256] */, uint32_t reg_items /* RS_REG_ITEMS; 0 forces the tiled path (tests) */)
{
	__shared__ uint32_t s_hist[256];              // count phase: this block's digit histogram; scatter phase: the block's running digit cursors
	__shared__ uint32_t s_part[2][256], s_wsum[8];
	__shared__ uint32_t s_wcnt[RS_WARPS][256];    // per warp: keys of digit d in the warp's part of the tile, then the warp's first destination of digit d
	__shared__ unsigned long long s_red[2][RS_WARPS];
	const uint32_t n = min(counts[0], cap);
	if (n < 2) return; // uniform over the grid: nothing to sort (buffer 0 already holds the result)
	uint32_t barriers_passed = 0;
	const uint32_t tid = threadIdx.x, lane = tid & 31u, warp = tid >> 5;
	const bool in_regs = n <= gridDim.x * (uint32_t)RS_THREADS * reg_items;
	uint32_t key_begin, key_end, tile_begin = 0, tile_end = 0, items = 0;
	if (in_regs) {
		items = (n + gridDim.x * RS_THREADS - 1) / (gridDim.x * RS_THREADS); // 1..RS_REG_ITEMS keys per thread
		key_begin = min(n, blockIdx.x * items * RS_THREADS);
		key_end = min(n, key_begin + items * RS_THREADS);
	}
	else {
		const uint32_t n_tiles = (n + RS_TILE - 1) / RS_TILE;
		tile_begin = (uint32_t)(((unsigned long long)blockIdx.x * n_tiles) / gridDim.x);
		tile_end = (uint32_t)(((unsigned long long)(blockIdx.x + 1) * n_tiles) / gridDim.x);
		key_begin = tile_begin * RS_TILE;
		key_end = min(n, tile_end * RS_TILE);
	}

	// which bits differ at all: OR of every key and OR of every complement
	{
		unsigned long long o = 0ull, a = 0ull;
		for (uint32_t i = key_begin + tid; i < key_end; i += RS_THREADS) { const unsigned long long k = kbuf0[i]; o |= k; a |= ~k; }
#pragma unroll
		for (int d = 16; d > 0; d >>= 1) { o |= __shfl_xor_sync(0xffffffffu, o, d); a |= __shfl_xor_sync(0xffffffffu, a, d); }
		if (lane == 0) { s_red[0][warp] = o; s_red[1][warp] = a; }
		__syncthreads();
		if (tid == 0) {
			for (int w = 1; w < RS_WARPS; ++w) { o |= s_red[0][w]; a |= s_red[1][w]; }
			if (key_begin < key_end) { atomicOr(&st->key_or, o); atomicOr(&st->key_or_not, a); }
		}
	}
	grid_barrier(&st->bar, barriers_passed);
	const unsigned long long varying = __ldcg(&st->key_or) & __ldcg(&st->key_or_not); // bits that are 1 in some key and 0 in another

	uint32_t cur = 0;
	int window = 0; // at most RS_PASSES digit windows: each takes at least one differing bit out of 64 and 8 bits wide windows cover them all
	if (in_regs) {
		// the warp's run: [key_begin + warp * items * 32, + items * 32); item j of lane l = run + j * 32 + l, so (j, lane) is the key order
		const uint32_t wbase = key_begin + warp * items * 32u;
		uint64_t k[RS_REG_ITEMS], v[RS_REG_ITEMS];
		uint16_t rk[RS_REG_ITEMS];
		// digit windows: 8 bits from the lowest bit that still differs between keys, then from the next such bit above the window, ...
		// (bytes in which every key agrees cost nothing, and a group of differing bits that straddles a byte border is one pass, not two)
#pragma unroll 1
		for (unsigned long long left = varying; left != 0ull; ++window) {
			const int shift = __ffsll((long long)left) - 1;
			left &= ~(0xffull << shift);
			const uint64_t* ksrc = cur ? kbuf1 : kbuf0;
			const uint64_t* vsrc = cur ? vbuf1 : vbuf0;
			uint64_t* kdst = cur ? kbuf0 : kbuf1;
			uint64_t* vdst = cur ? vbuf0 : vbuf1;
#pragma unroll
			for (int j = 0; j < RS_REG_ITEMS; ++j) {
				const uint32_t i = wbase + j * 32 + lane;
				const bool has = (uint32_t)j < items && i < key_end;
				k[j] = has ? __ldcg(ksrc + i) : 0;
				v[j] = has ? __ldcg(vsrc + i) : 0;
			}
			for (int d = lane; d < 256; d += 32) s_wcnt[warp][d] = 0;
			__syncwarp();
#pragma unroll
			for (int j = 0; j < RS_REG_ITEMS; ++j) {
				if ((uint32_t)j < items) { // uniform
					const bool has = wbase + j * 32 + lane < key_end;
					const uint32_t dg = has ? (uint32_t)(k[j] >> shift) & 0xffu : 0x100u; // lanes past the end match only each other
					const uint32_t peers = __match_any_sync(0xffffffffu, dg);
					const uint32_t below = __popc(peers & ((1u << lane) - 1u));
					uint32_t seen = 0;
					if (has) seen = s_wcnt[warp][dg];
					__syncwarp();
					if (has && below == 0) s_wcnt[warp][dg] = seen + __popc(peers);
					__syncwarp();
					rk[j] = (uint16_t)(seen + below);
				}
			}
			__syncthreads();
			if (tid < 256) { // digit tid: the warps' counts -> each warp's offset inside the block's slice; the sum is the block's histogram entry
				uint32_t acc = 0;
#pragma unroll
				for (int w = 0; w < RS_WARPS; ++w) { const uint32_t t = s_wcnt[w][tid]; s_wcnt[w][tid] = acc; acc += t; }
				block_hist[blockIdx.x * 256 + tid] = acc;
				if (acc) atomicAdd(&st->digit_total[window][tid], acc);
			}
			grid_barrier(&st->bar, barriers_passed);
			digit_starts(block_hist, st->digit_total[window], s_hist, s_part, s_wsum);
#pragma unroll
			for (int j = 0; j < RS_REG_ITEMS; ++j) {
				if ((uint32_t)j < items && wbase + j * 32 + lane < key_end) {
					const uint32_t dg = (uint32_t)(k[j] >> shift) & 0xffu;
					const uint32_t dest = s_hist[dg] + s_wcnt[warp][dg] + rk[j];
					kdst[dest] = k[j];
					vdst[dest] = v[j];
				}
			}
			grid_barrier(&st->bar, barriers_passed);
			cur ^= 1u;
		}
	}
	else {
#pragma unroll 1
		for (unsigned long long left = varying; left != 0ull; ++window) {
			const int shift = __ffsll((long long)left) - 1;
			left &= ~(0xffull << shift);
			const uint64_t* ksrc = cur ? kbuf1 : kbuf0;
			const uint64_t* vsrc = cur ? vbuf1 : vbuf0;
			uint64_t* kdst = cur ? kbuf0 : kbuf1;
			uint64_t* vdst = cur ? vbuf0 : vbuf1;
			// count
			if (tid < 256) s_hist[tid] = 0;
			__syncthreads();
			for (uint32_t i = key_begin + tid; i < key_end; i += RS_THREADS) atomicAdd(&s_hist[(uint32_t)(__ldcg(ksrc + i) >> shift) & 0xffu], 1u);
			__syncthreads();
			if (tid < 256) {
				block_hist[blockIdx.x * 256 + tid] = s_hist[tid];
				if (s_hist[tid]) atomicAdd(&st->digit_total[window][tid], s_hist[tid]);
			}
			grid_barrier(&st->bar, barriers_passed);
			digit_starts(block_hist, st->digit_total[window], s_hist, s_part, s_wsum);
			// stable scatter, tile by tile
			for (uint32_t tile = tile_begin; tile < tile_end; ++tile) {
				const uint32_t wbase = tile * RS_TILE + warp * (32 * RS_ITEMS);
				uint64_t k[RS_ITEMS], v[RS_ITEMS];
				uint32_t dg[RS_ITEMS], rk[RS_ITEMS];
#pragma unroll
				for (int j = 0; j < RS_ITEMS; ++j) {
					const uint32_t i = wbase + j * 32 + lane;
					const bool has = i < n;
					k[j] = has ? __ldcg(ksrc + i) : 0;
					v[j] = has ? __ldcg(vsrc + i) : 0;
					dg[j] = has ? (uint32_t)(k[j] >> shift) & 0xffu : 0x100u; // keys past the end match only each other
				}
				for (int d = lane; d < 256; d += 32) s_wcnt[warp][d] = 0;
				__syncwarp();
#pragma unroll
				for (int j = 0; j < RS_ITEMS; ++j) {
					const uint32_t peers = __match_any_sync(0xffffffffu, dg[j]);
					const uint32_t below = __popc(peers & ((1u << lane) - 1u));
					uint32_t seen = 0;
					if (dg[j] < 256) seen = s_wcnt[warp][dg[j]];
					__syncwarp();
					if (dg[j] < 256 && below == 0) s_wcnt[warp][dg[j]] = seen + __popc(peers);
					__syncwarp();
					rk[j] = seen + below;
				}
				__syncthreads();
				if (tid < 256) { // digit tid: the warps' slices in warp order, then advance the block's cursor past the tile
					uint32_t acc = s_hist[tid];
#pragma unroll
					for (int w = 0; w < RS_WARPS; ++w) { const uint32_t t = s_wcnt[w][tid]; s_wcnt[w][tid] = acc; acc += t; }
					s_hist[tid] = acc;
				}
				__syncthreads();
#pragma unroll
				for (int j = 0; j < RS_ITEMS; ++j) {
					if (dg[j] < 256) {
						const uint32_t dest = s_wcnt[warp][dg[j]] + rk[j];
						kdst[dest] = k[j];
						vdst[dest] = v[j];
					}
				}
				__syncthreads();
			}
			grid_barrier(&st->bar, barriers_passed);
			cur ^= 1u;
		}
	}
	if (cur) { // sorted data to buffer 0 if it ended up in buffer 1
		for (uint32_t i = key_begin + tid; i < key_end; i += RS_THREADS) { kbuf0[i] = __ldcg(kbuf1 + i); vbuf0[i] = __ldcg(vbuf1 + i); }
	}
}

} // namespace

int lb200_radix_sort_alloc_scratch(lb200_ctx* ctx, uint32_t blocks, RadixSortScratch& out) {
	if (!ctx->radix_sort_grid) {
		const int rc = lb200_coop_grid_limit(ctx, (const void*)radix_sort_kernel, RS_THREADS, 0, &ctx->radix_sort_grid);
		if (rc) return rc;
	}
	RadixSortScratch s;
	LB200_CUDA(ctx, s.state.alloc(sizeof(SortState)));
	LB200_CUDA(ctx, s.block_hist.alloc(256 * (size_t)std::min(blocks, ctx->radix_sort_grid)));
	out = std::move(s);
	return LB200_OK;
}

int lb200_radix_sort_pairs(lb200_ctx* ctx, cudaStream_t s, uint64_t* keys0, uint64_t* keys1, uint64_t* values0, uint64_t* values1, const uint32_t* count_dev, uint32_t cap,
	const RadixSortScratch& scratch, uint32_t max_blocks, bool force_tiled, uint32_t* out_grid)
{
	SortState* st = reinterpret_cast<SortState*>(scratch.state.get());
	uint32_t* block_hist = scratch.block_hist;
	LB200_CUDA(ctx, cudaMemsetAsync(st, 0, sizeof(SortState), s));
	uint32_t grid = std::max(1u, std::min(std::min(scratch.blocks(), max_blocks ? max_blocks : UINT32_MAX), (cap + RS_TILE - 1) / RS_TILE));
	uint32_t reg_items = force_tiled ? 0u : (uint32_t)RS_REG_ITEMS;
	void* args[] = {&keys0, &keys1, &values0, &values1, &count_dev, &cap, &st, &block_hist, &reg_items};
	LB200_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)radix_sort_kernel, dim3(grid), dim3(RS_THREADS), args, 0, s));
	LB200_CHECK_LAUNCH(ctx);
	if (out_grid) *out_grid = grid;
	return LB200_OK;
}

// On caller buffers, with the context's scratch: the alternate key / value buffers grow to the largest cap asked for, the SortState and
// histogram rows are sized once for every co-resident block.
extern "C" int lb200_radix_sort_device(lb200_ctx* ctx, uint64_t* dev_keys, uint64_t* dev_values, const uint32_t* dev_count, uint32_t cap, uint32_t max_blocks, int force_tiled,
	uint32_t* out_grid)
{
	if (!ctx || !dev_keys || !dev_values || !dev_count) return LB200_ERR_INVALID;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!ctx->radix_scratch.state) {
		const int rc = lb200_radix_sort_alloc_scratch(ctx, UINT32_MAX, ctx->radix_scratch);
		if (rc) return rc;
	}
	const uint32_t need = std::max(cap, 1u);
	if (need > ctx->radix_keys1.size()) { // the stream may still use the old buffers
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		ctx->radix_keys1.reset(); ctx->radix_values1.reset(); // both go before either is allocated again
		DeviceArray<uint64_t> keys1, values1;
		LB200_CUDA(ctx, keys1.alloc(need));
		LB200_CUDA(ctx, values1.alloc(need));
		ctx->radix_keys1 = std::move(keys1); ctx->radix_values1 = std::move(values1);
	}
	return lb200_radix_sort_pairs(ctx, ctx->stream, dev_keys, ctx->radix_keys1, dev_values, ctx->radix_values1, dev_count, cap, ctx->radix_scratch, max_blocks,
		force_tiled != 0, out_grid);
}
