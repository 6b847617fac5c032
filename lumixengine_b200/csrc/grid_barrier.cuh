// Grid-wide barrier of a cooperative launch (every block of the grid is resident), shared by create_keys_kernel (sortkeys.cu) and
// radix_sort_kernel (radix_sort.cu).  The host side, the number of blocks that can be co-resident, is lb200_coop_grid_limit (context.cu).
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace lb {

// One word that only counts up (zeroed before the launch): barrier number k of the launch is complete when it reads k * gridDim.  Per block:
// one release-add by thread 0 after the block barrier, then acquire-polls — no generation word, no reset by a last arriver.
struct GridBar { uint32_t count, pad; };
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
	uint32_t v;
	asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
	return v;
}
__device__ __forceinline__ void grid_barrier(GridBar* b, uint32_t& passed /* barriers this block has been through; starts at 0 */) {
	__syncthreads();
	++passed;
	if (threadIdx.x == 0) {
		__threadfence(); // the block's writes (ordered before this by the block barrier) before the arrival
		atomicAdd(&b->count, 1u);
		const uint32_t target = passed * gridDim.x;
		while (ld_acquire_gpu(&b->count) < target) {}
		__threadfence(); // gpu-scope fence: also drops this SM's L1 lines, the block's plain loads behind the barrier see the other blocks' writes
	}
	__syncthreads();
}

} // namespace lb
