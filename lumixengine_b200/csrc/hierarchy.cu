// GPU hierarchy propagation: kernels + C-ABI (include/lumix_b200.h "Hierarchy").
//
// Replaces the serial recursion World::transformEntity (src/engine/world.cpp:255-282):
//     child.global = parent.global.compose(child.local_transform)            (world.cpp:274-276)
// with a batched level-order pass: nodes are sorted by depth once (children of one parent adjacent), every depth level
// is one launch over a contiguous index range, and each thread evaluates Transform::compose (src/core/math.cpp:801-807)
// with the reference's op order — fp64 position (Quat::rotate(DVec3), math.cpp:177-188), fp32 rotation / scale.
// HBM layout is SoA (px,py,pz fp64; rot float4; sx,sy,sz fp32) so that every load/store instruction is fully coalesced;
// the 56-byte engine Transform (math.h:306-327) exists only at the API boundary.
// HBM-bound: 52 B local read + 4 B parent index + 52 B global write per node, + 52 B/fan-out for the parent gather.
#include "lb200_internal.h"
#include "lb200_math.cuh"

#include <memory>
#include <new>
#include <vector>

namespace {

using namespace lb;

struct SoaTransforms {
	double* px = nullptr; double* py = nullptr; double* pz = nullptr;
	float4* rot = nullptr;
	float* sx = nullptr; float* sy = nullptr; float* sz = nullptr;
};

constexpr int HT = 256;

// AoS (engine Transform, 56 B) in caller order -> SoA in level order.  only_roots: touch level-0 nodes only.
__global__ void __launch_bounds__(HT) aos_to_soa_kernel(const lb200_transform* __restrict__ in, const uint32_t* __restrict__ order, uint32_t n,
	SoaTransforms out)
{
	const uint32_t i = blockIdx.x * HT + threadIdx.x;
	if (i >= n) return;
	const lb200_transform t = in[order[i]];
	out.px[i] = t.pos[0]; out.py[i] = t.pos[1]; out.pz[i] = t.pos[2];
	out.rot[i] = make_float4(t.rot[0], t.rot[1], t.rot[2], t.rot[3]);
	out.sx[i] = t.scale[0]; out.sy[i] = t.scale[1]; out.sz[i] = t.scale[2];
}

// a few transforms (World::setTransform / setLocalTransform for some entities): node ids + values -> their level positions
__global__ void __launch_bounds__(HT) scatter_transforms_kernel(const uint32_t* __restrict__ nodes, const lb200_transform* __restrict__ values, uint32_t count,
	const uint32_t* __restrict__ pos_of_node, SoaTransforms out)
{
	const uint32_t k = blockIdx.x * HT + threadIdx.x;
	if (k >= count) return;
	const uint32_t i = pos_of_node[nodes[k]];
	const lb200_transform t = values[k];
	out.px[i] = t.pos[0]; out.py[i] = t.pos[1]; out.pz[i] = t.pos[2];
	out.rot[i] = make_float4(t.rot[0], t.rot[1], t.rot[2], t.rot[3]);
	out.sx[i] = t.scale[0]; out.sy[i] = t.scale[1]; out.sz[i] = t.scale[2];
}

__global__ void __launch_bounds__(HT) soa_to_aos_kernel(SoaTransforms in, const uint32_t* __restrict__ order, uint32_t n, lb200_transform* __restrict__ out) {
	const uint32_t i = blockIdx.x * HT + threadIdx.x;
	if (i >= n) return;
	lb200_transform t;
	t.pos[0] = in.px[i]; t.pos[1] = in.py[i]; t.pos[2] = in.pz[i];
	const float4 r = in.rot[i];
	t.rot[0] = r.x; t.rot[1] = r.y; t.rot[2] = r.z; t.rot[3] = r.w;
	t.scale[0] = in.sx[i]; t.scale[1] = in.sy[i]; t.scale[2] = in.sz[i];
	out[order[i]] = t;
}

// compose one node (level position i) from its parent's global: Transform::compose, math.cpp:801-807
__device__ __forceinline__ void compose_node(uint32_t i, const int* __restrict__ parent, const SoaTransforms& L, const SoaTransforms& G) {
	const int p = parent[i];
	// parent global (siblings are adjacent: these loads coalesce to a few sectors per warp)
	const D3 ppos = d3(G.px[p], G.py[p], G.pz[p]);
	const float4 pr = G.rot[p];
	const Q4 prot = q4(pr.x, pr.y, pr.z, pr.w);
	const V3 pscale = v3(G.sx[p], G.sy[p], G.sz[p]);
	// own local
	const D3 lpos = d3(L.px[i], L.py[i], L.pz[i]);
	const float4 lr = L.rot[i];
	const V3 lscale = v3(L.sx[i], L.sy[i], L.sz[i]);
	// { rot.rotate(rhs.pos * scale) + pos, rot * rhs.rot, scale * rhs.scale }
	const D3 scaled = d3(LB_DMUL(lpos.x, (double)pscale.x), LB_DMUL(lpos.y, (double)pscale.y), LB_DMUL(lpos.z, (double)pscale.z)); // DVec3 * Vec3, math.cpp:498
	const D3 gpos = add(rotate(prot, scaled), ppos);
	const Q4 grot = qmul(prot, q4(lr.x, lr.y, lr.z, lr.w));
	const V3 gscale = mul(pscale, lscale);
	G.px[i] = gpos.x; G.py[i] = gpos.y; G.pz[i] = gpos.z;
	G.rot[i] = make_float4(grot.x, grot.y, grot.z, grot.w);
	G.sx[i] = gscale.x; G.sy[i] = gscale.y; G.sz[i] = gscale.z;
}

// The update_local branch of World::transformEntity (world.cpp:267-270) for every non-root node at once:
// local = Transform::computeLocal(parent global, own global), math.cpp:809-816.  No dependency between nodes: one flat launch.
__global__ void __launch_bounds__(HT) compute_locals_kernel(uint32_t begin, uint32_t end, const int* __restrict__ parent, SoaTransforms G, SoaTransforms L) {
	const uint32_t i = begin + blockIdx.x * HT + threadIdx.x;
	if (i >= end) return;
	const int p = parent[i];
	const float4 pr = G.rot[p];
	const Q4 c = q4(pr.x, pr.y, pr.z, -pr.w); // Quat::conjugated() = (x, y, z, -w), math.cpp:664-667
	const double psx = (double)G.sx[p], psy = (double)G.sy[p], psz = (double)G.sz[p];
	// inv_parent_pos = conj.rotate(-parent.pos) / parent.scale      (DVec3 / Vec3: double / float per component, math.cpp:502)
	const D3 rp = rotate(c, d3(-G.px[p], -G.py[p], -G.pz[p]));
	const D3 inv_parent_pos = d3(LB_DDIV(rp.x, psx), LB_DDIV(rp.y, psy), LB_DDIV(rp.z, psz));
	// pos = conj.rotate(child.pos) / parent.scale + inv_parent_pos
	const D3 rc = rotate(c, d3(G.px[i], G.py[i], G.pz[i]));
	const D3 lpos = add(d3(LB_DDIV(rc.x, psx), LB_DDIV(rc.y, psy), LB_DDIV(rc.z, psz)), inv_parent_pos);
	const float4 cr = G.rot[i];
	const Q4 lrot = qmul(c, q4(cr.x, cr.y, cr.z, cr.w));
	L.px[i] = lpos.x; L.py[i] = lpos.y; L.pz[i] = lpos.z;
	L.rot[i] = make_float4(lrot.x, lrot.y, lrot.z, lrot.w);
	L.sx[i] = LB_FDIV(G.sx[i], G.sx[p]); L.sy[i] = LB_FDIV(G.sy[i], G.sy[p]); L.sz[i] = LB_FDIV(G.sz[i], G.sz[p]); // Vec3 / Vec3, math.cpp:468
}

// One depth level: nodes [begin, end) in level order; parents live in earlier levels.
// Launched with programmatic stream serialization: the block starts while the previous level is still draining, loads its
// own locals (independent of that level) and only then waits for the parents' globals.
__global__ void __launch_bounds__(HT) propagate_level_kernel(uint32_t begin, uint32_t end, const int* __restrict__ parent, SoaTransforms L, SoaTransforms G) {
	const uint32_t i = begin + blockIdx.x * HT + threadIdx.x;
	const bool active = i < end;
	int p = 0;
	D3 lpos = d3(0, 0, 0);
	float4 lr = make_float4(0, 0, 0, 1);
	V3 lscale = v3(1, 1, 1);
	if (active) {
		p = parent[i];
		lpos = d3(L.px[i], L.py[i], L.pz[i]);
		lr = L.rot[i];
		lscale = v3(L.sx[i], L.sy[i], L.sz[i]);
	}
	cudaGridDependencySynchronize();
	if (!active) return;
	const D3 ppos = d3(G.px[p], G.py[p], G.pz[p]);
	const float4 pr = G.rot[p];
	const Q4 prot = q4(pr.x, pr.y, pr.z, pr.w);
	const V3 pscale = v3(G.sx[p], G.sy[p], G.sz[p]);
	// math.cpp:801-807 { rot.rotate(rhs.pos * scale) + pos, rot * rhs.rot, scale * rhs.scale }
	const D3 scaled = d3(LB_DMUL(lpos.x, (double)pscale.x), LB_DMUL(lpos.y, (double)pscale.y), LB_DMUL(lpos.z, (double)pscale.z)); // DVec3 * Vec3, math.cpp:498
	const D3 gpos = add(rotate(prot, scaled), ppos);
	const Q4 grot = qmul(prot, q4(lr.x, lr.y, lr.z, lr.w));
	const V3 gscale = mul(pscale, lscale);
	G.px[i] = gpos.x; G.py[i] = gpos.y; G.pz[i] = gpos.z;
	G.rot[i] = make_float4(grot.x, grot.y, grot.z, grot.w);
	G.sx[i] = gscale.x; G.sy[i] = gscale.y; G.sz[i] = gscale.z;
}

// The narrow top of the hierarchy (levels of at most a few thousand nodes) in ONE block: a launch per tiny level would cost
// more than the level itself.  __syncthreads() orders a level's global writes before the next level's reads.
constexpr int SMALL_THREADS = 1024;
constexpr int MAX_SMALL_LEVELS = 30;
struct SmallLevels { uint32_t start[MAX_SMALL_LEVELS + 1]; uint32_t n; };

__global__ void __launch_bounds__(SMALL_THREADS) propagate_small_levels_kernel(const __grid_constant__ SmallLevels S, const int* __restrict__ parent, SoaTransforms L, SoaTransforms G) {
	for (uint32_t l = 0; l < S.n; ++l) {
		for (uint32_t i = S.start[l] + threadIdx.x; i < S.start[l + 1]; i += SMALL_THREADS) compose_node(i, parent, L, G);
		__syncthreads();
	}
}

// render_module.cpp:1544-1554: world bounding sphere of a moved model instance
__global__ void __launch_bounds__(HT) spheres_kernel(SoaTransforms G, const uint32_t* __restrict__ order, const float* __restrict__ bounding_radius, uint32_t n,
	double* __restrict__ out_pos3, float* __restrict__ out_radius)
{
	const uint32_t i = blockIdx.x * HT + threadIdx.x;
	if (i >= n) return;
	const uint32_t node = order[i];
	const float sx = G.sx[i], sy = G.sy[i], sz = G.sz[i];
	const float bc = sy > sz ? sy : sz; // maximum(a, b, c) = a > max(b, c) ? a : max(b, c), math.h:468-475
	const float m = sx > bc ? sx : bc;
	out_pos3[3 * (size_t)node + 0] = G.px[i];
	out_pos3[3 * (size_t)node + 1] = G.py[i];
	out_pos3[3 * (size_t)node + 2] = G.pz[i];
	out_radius[node] = LB_FMUL(bounding_radius[node], m);
}

// World::getRelativeMatrix, world.cpp:370-377: rot.toMatrix(), translation = Vec3(pos - base), multiply3x3(scale).
// One thread per node: 52 B of SoA globals in (coalesced), one 64-byte matrix out at the caller's node index (two full sectors).
__global__ void __launch_bounds__(HT) relative_matrices_kernel(SoaTransforms G, const uint32_t* __restrict__ order, uint32_t n,
	double bx, double by, double bz, float4* __restrict__ out)
{
	const uint32_t i = blockIdx.x * HT + threadIdx.x;
	if (i >= n) return;
	Rigid r;
	r.pos = v3((float)LB_DSUB(G.px[i], bx), (float)LB_DSUB(G.py[i], by), (float)LB_DSUB(G.pz[i], bz));
	const float4 q = G.rot[i];
	r.rot = q4(q.x, q.y, q.z, q.w);
	float m[16];
	to_matrix(r, m);
	const float sx = G.sx[i], sy = G.sy[i], sz = G.sz[i];
	m[0] = LB_FMUL(m[0], sx); m[1] = LB_FMUL(m[1], sx); m[2] = LB_FMUL(m[2], sx);   // math.cpp:1207-1217
	m[4] = LB_FMUL(m[4], sy); m[5] = LB_FMUL(m[5], sy); m[6] = LB_FMUL(m[6], sy);
	m[8] = LB_FMUL(m[8], sz); m[9] = LB_FMUL(m[9], sz); m[10] = LB_FMUL(m[10], sz);
	float4* dst = out + 4 * (size_t)order[i];
	dst[0] = make_float4(m[0], m[1], m[2], m[3]);
	dst[1] = make_float4(m[4], m[5], m[6], m[7]);
	dst[2] = make_float4(m[8], m[9], m[10], m[11]);
	dst[3] = make_float4(m[12], m[13], m[14], m[15]);
}

// the arrays of one SoaTransforms, which is what the kernels take
struct SoaArrays {
	DeviceArray<double> px, py, pz;
	DeviceArray<float4> rot;
	DeviceArray<float> sx, sy, sz;
	int alloc(lb200_ctx* ctx, uint32_t n) {
		LB200_CUDA(ctx, px.alloc(n));
		LB200_CUDA(ctx, py.alloc(n));
		LB200_CUDA(ctx, pz.alloc(n));
		LB200_CUDA(ctx, rot.alloc(n));
		LB200_CUDA(ctx, sx.alloc(n));
		LB200_CUDA(ctx, sy.alloc(n));
		LB200_CUDA(ctx, sz.alloc(n));
		return LB200_OK;
	}
	operator SoaTransforms() const { return SoaTransforms{px, py, pz, rot, sx, sy, sz}; }
};

} // namespace

struct lb200_hierarchy {
	lb200_ctx* ctx = nullptr;
	uint32_t n = 0;
	std::vector<uint32_t> level_start; // size depth + 1
	DeviceArray<uint32_t> d_order;       // level position -> caller node index
	DeviceArray<uint32_t> d_pos_of_node; // caller node index -> level position
	// staging of set_subset: [node ids][transforms], pinned + device, two of each used in turn: an upload waits only for the upload before last.
	// The four buffers are allocated and released together.
	DeviceArray<uint8_t> d_subset[2]; PinnedArray<uint8_t> h_subset[2]; Event subset_done[2]; uint32_t subset_turn = 0;
	DeviceArray<int> d_parent;           // level position -> parent's level position
	SoaArrays L, G;
	DeviceArray<lb200_transform> d_stage; // n Transforms (API boundary)
	DeviceArray<float4> d_matrices;       // n relative matrices, 4 float4 each (lb200_hierarchy_get_relative_matrices)
	// the inputs and outputs of spheres_kernel, allocated and released together
	DeviceArray<float> d_radius_in;
	DeviceArray<double> d_sphere_pos;
	DeviceArray<float> d_sphere_radius;
	uint64_t gather_bytes = 0;
};

namespace {

int upload(lb200_hierarchy* h, const lb200_transform* src, SoaTransforms dst, uint32_t count_levelorder) {
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_stage, src, sizeof(lb200_transform) * (size_t)h->n, cudaMemcpyHostToDevice, ctx->stream));
	aos_to_soa_kernel<<<(count_levelorder + HT - 1) / HT, HT, 0, ctx->stream>>>(h->d_stage, h->d_order, count_levelorder, dst);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

int allocSpheres(lb200_hierarchy* h) {
	if (h->d_radius_in && h->d_sphere_pos && h->d_sphere_radius) return LB200_OK;
	lb200_ctx* ctx = h->ctx;
	DeviceArray<float> radius_in, sphere_radius; DeviceArray<double> sphere_pos;
	LB200_CUDA(ctx, radius_in.alloc(h->n));
	LB200_CUDA(ctx, sphere_pos.alloc(3 * (size_t)h->n));
	LB200_CUDA(ctx, sphere_radius.alloc(h->n));
	h->d_radius_in = std::move(radius_in); h->d_sphere_pos = std::move(sphere_pos); h->d_sphere_radius = std::move(sphere_radius);
	return LB200_OK;
}

} // namespace

extern "C" {

int lb200_hierarchy_create(lb200_ctx* ctx, const int32_t* parents, uint32_t n, lb200_hierarchy** out) {
	if (!out || !parents || !n) return LB200_ERR_INVALID;
	if (!ctx) return LB200_ERR_NO_DEVICE;
	*out = nullptr;
	// level order: children lists (as World::setParent keeps them, world.cpp:619-701), then BFS from the roots
	std::vector<int32_t> first_child(n, -1), next_sibling(n, -1);
	std::vector<uint32_t> order;
	order.reserve(n);
	for (uint32_t i = n; i-- > 0;) {
		const int32_t p = parents[i];
		if (p >= (int32_t)n) { lb200_set_error(ctx, "parent index %d out of range", p); return LB200_ERR_INVALID; }
		if (p >= 0) { next_sibling[i] = first_child[p]; first_child[p] = (int32_t)i; }
	}
	std::vector<uint32_t> level_start;
	level_start.push_back(0);
	for (uint32_t i = 0; i < n; ++i) if (parents[i] < 0) order.push_back(i);
	std::vector<int> parent_pos(n, -1);
	std::vector<uint32_t> pos_of(n, 0);
	uint32_t begin = 0;
	while (begin < order.size()) {
		const uint32_t end = (uint32_t)order.size();
		level_start.push_back(end);
		for (uint32_t k = begin; k < end; ++k) {
			pos_of[order[k]] = k;
			for (int32_t c = first_child[order[k]]; c >= 0; c = next_sibling[c]) {
				parent_pos[order.size()] = (int)k;
				order.push_back((uint32_t)c);
			}
		}
		begin = end;
	}
	if (order.size() != n) { lb200_set_error(ctx, "hierarchy has a cycle (%zu of %u nodes reachable from roots)", order.size(), n); return LB200_ERR_INVALID; }

	std::unique_ptr<lb200_hierarchy, decltype(&lb200_hierarchy_destroy)> h(new (std::nothrow) lb200_hierarchy, lb200_hierarchy_destroy);
	if (!h) return LB200_ERR_CUDA;
	h->ctx = ctx;
	h->n = n;
	h->level_start = level_start;
	// distinct parents per level -> bytes of the parent-global gather
	uint64_t distinct = 0;
	for (size_t l = 1; l + 1 < level_start.size(); ++l) {
		int last = -1;
		for (uint32_t k = level_start[l]; k < level_start[l + 1]; ++k) if (parent_pos[k] != last) { ++distinct; last = parent_pos[k]; }
	}
	h->gather_bytes = distinct * 52;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, h->d_order.alloc(n));
	LB200_CUDA(ctx, h->d_parent.alloc(n));
	LB200_CUDA(ctx, h->d_stage.alloc(n));
	int rc = h->L.alloc(ctx, n);
	if (!rc) rc = h->G.alloc(ctx, n);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_order, order.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	std::vector<uint32_t> pos_of_node(n);
	for (uint32_t i = 0; i < n; ++i) pos_of_node[order[i]] = i;
	LB200_CUDA(ctx, h->d_pos_of_node.alloc(n));
	LB200_CUDA(ctx, cudaMemcpy(h->d_pos_of_node, pos_of_node.data(), sizeof(uint32_t) * n, cudaMemcpyHostToDevice));
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_parent, parent_pos.data(), sizeof(int) * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	*out = h.release();
	return LB200_OK;
}

void lb200_hierarchy_destroy(lb200_hierarchy* h) {
	if (!h) return;
	cudaSetDevice(h->ctx->device);
	cudaStreamSynchronize(h->ctx->stream);
	delete h;
}

uint32_t lb200_hierarchy_depth(const lb200_hierarchy* h) { return h ? (uint32_t)h->level_start.size() - 1 : 0; }

int lb200_hierarchy_set_locals(lb200_hierarchy* h, const lb200_transform* locals) {
	if (!h || !locals) return LB200_ERR_INVALID;
	return upload(h, locals, h->L, h->n);
}

int lb200_hierarchy_set_root_globals(lb200_hierarchy* h, const lb200_transform* globals) {
	if (!h || !globals) return LB200_ERR_INVALID;
	return upload(h, globals, h->G, h->level_start[1]); // level 0 only: everything else is produced by propagate
}

int lb200_hierarchy_propagate(lb200_hierarchy* h) {
	if (!h) return LB200_ERR_INVALID;
	lb200_range range("transform hierarchy"); // World::transformEntity, world.cpp:255
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const size_t n_levels = h->level_start.size() - 1;
	size_t l = 1;
	// levels up to SMALL_LEVEL_NODES nodes run inside one block (no launch per level)
	const uint32_t SMALL_LEVEL_NODES = 8192;
	SmallLevels S;
	S.n = 0;
	while (l < n_levels && S.n < MAX_SMALL_LEVELS && h->level_start[l + 1] - h->level_start[l] <= SMALL_LEVEL_NODES) {
		S.start[S.n] = h->level_start[l];
		S.start[S.n + 1] = h->level_start[l + 1];
		++S.n;
		++l;
	}
	if (S.n) {
		propagate_small_levels_kernel<<<1, SMALL_THREADS, 0, ctx->stream>>>(S, h->d_parent, h->L, h->G);
		LB200_CHECK_LAUNCH(ctx);
	}
	bool chained = S.n != 0; // the first kernel of a propagate is a plain launch: whatever precedes it has fully completed
	for (; l < n_levels; ++l) {
		const uint32_t begin = h->level_start[l], end = h->level_start[l + 1];
		if (end == begin) continue;
		cudaLaunchConfig_t cfg = {};
		cfg.gridDim = dim3((end - begin + HT - 1) / HT);
		cfg.blockDim = dim3(HT);
		cfg.stream = ctx->stream;
		cudaLaunchAttribute attr[1];
		attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
		attr[0].val.programmaticStreamSerializationAllowed = 1;
		cfg.attrs = attr;
		cfg.numAttrs = chained ? 1 : 0;
		chained = true;
		LB200_CUDA(ctx, cudaLaunchKernelEx(&cfg, propagate_level_kernel, begin, end, (const int*)h->d_parent, h->L, h->G));
		LB200_CHECK_LAUNCH(ctx);
	}
	return LB200_OK;
}

int lb200_hierarchy_get_globals(lb200_hierarchy* h, lb200_transform* out_globals) {
	if (!h || !out_globals) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	soa_to_aos_kernel<<<(h->n + HT - 1) / HT, HT, 0, ctx->stream>>>(h->G, h->d_order, h->n, h->d_stage);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaMemcpyAsync(out_globals, h->d_stage, sizeof(lb200_transform) * (size_t)h->n, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

int lb200_hierarchy_get_spheres(lb200_hierarchy* h, const float* bounding_radius, double* out_pos3, float* out_radius) {
	if (!h || !bounding_radius || !out_pos3 || !out_radius) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	int rc = allocSpheres(h);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_radius_in, bounding_radius, sizeof(float) * h->n, cudaMemcpyHostToDevice, ctx->stream));
	spheres_kernel<<<(h->n + HT - 1) / HT, HT, 0, ctx->stream>>>(h->G, h->d_order, h->d_radius_in, h->n, h->d_sphere_pos, h->d_sphere_radius);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaMemcpyAsync(out_pos3, h->d_sphere_pos, sizeof(double) * 3 * (size_t)h->n, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(out_radius, h->d_sphere_radius, sizeof(float) * h->n, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

int lb200_hierarchy_set_subset(lb200_hierarchy* h, const uint32_t* nodes, const lb200_transform* values, uint32_t count, int globals) {
	if (!h || (count && (!nodes || !values))) return LB200_ERR_INVALID;
	if (!count) return LB200_OK;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const size_t bytes = (sizeof(uint32_t) + sizeof(lb200_transform)) * (size_t)count + 16;
	if (h->d_subset[1].size() < bytes) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		size_t cap = h->d_subset[1].size() ? h->d_subset[1].size() : 4096;
		while (cap < bytes) cap *= 2;
		for (int b = 0; b < 2; ++b) { h->d_subset[b].reset(); h->h_subset[b].reset(); } // before the new ones are allocated
		DeviceArray<uint8_t> d_new[2]; PinnedArray<uint8_t> h_new[2];
		for (int b = 0; b < 2; ++b) {
			LB200_CUDA(ctx, d_new[b].alloc(cap));
			LB200_CUDA(ctx, h_new[b].alloc(cap));
			if (!h->subset_done[b]) LB200_CUDA(ctx, cudaEventCreateWithFlags(h->subset_done[b].create(), cudaEventDisableTiming));
			LB200_CUDA(ctx, cudaEventRecord(h->subset_done[b], ctx->stream));
		}
		for (int b = 0; b < 2; ++b) { h->d_subset[b] = std::move(d_new[b]); h->h_subset[b] = std::move(h_new[b]); }
	}
	const uint32_t turn = h->subset_turn++ & 1u;
	LB200_CUDA(ctx, cudaEventSynchronize(h->subset_done[turn])); // the upload before last has left this pair of buffers (no wait for the frame in flight)
	uint8_t* hs = h->h_subset[turn];
	uint8_t* ds = h->d_subset[turn];
	const size_t tr_off = (sizeof(uint32_t) * (size_t)count + 15) & ~(size_t)15;
	memcpy(hs, nodes, sizeof(uint32_t) * (size_t)count);
	memcpy(hs + tr_off, values, sizeof(lb200_transform) * (size_t)count);
	LB200_CUDA(ctx, cudaMemcpyAsync(ds, hs, tr_off + sizeof(lb200_transform) * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
	scatter_transforms_kernel<<<(count + HT - 1) / HT, HT, 0, ctx->stream>>>((const uint32_t*)ds, (const lb200_transform*)(ds + tr_off), count, h->d_pos_of_node, globals ? h->G : h->L);
	LB200_CUDA(ctx, cudaEventRecord(h->subset_done[turn], ctx->stream));
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

int lb200_hierarchy_refresh_spheres(lb200_hierarchy* h, const float* bounding_radius, const double** dev_pos3, const float** dev_radius) {
	if (!h || !dev_pos3 || !dev_radius) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!h->d_radius_in && !bounding_radius) { lb200_set_error(ctx, "refresh_spheres: the first call needs the bounding radii"); return LB200_ERR_INVALID; }
	int rc = allocSpheres(h);
	if (rc) return rc;
	if (bounding_radius) LB200_CUDA(ctx, cudaMemcpyAsync(h->d_radius_in, bounding_radius, sizeof(float) * h->n, cudaMemcpyHostToDevice, ctx->stream));
	spheres_kernel<<<(h->n + HT - 1) / HT, HT, 0, ctx->stream>>>(h->G, h->d_order, h->d_radius_in, h->n, h->d_sphere_pos, h->d_sphere_radius);
	LB200_CHECK_LAUNCH(ctx);
	*dev_pos3 = h->d_sphere_pos;
	*dev_radius = h->d_sphere_radius;
	return LB200_OK;
}

int lb200_hierarchy_set_globals(lb200_hierarchy* h, const lb200_transform* globals) {
	if (!h || !globals) return LB200_ERR_INVALID;
	return upload(h, globals, h->G, h->n);
}

int lb200_hierarchy_compute_locals(lb200_hierarchy* h) {
	if (!h) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const uint32_t begin = h->level_start[1], end = h->n; // level 0 = roots: no parent, local transform left alone
	if (end > begin) {
		compute_locals_kernel<<<(end - begin + HT - 1) / HT, HT, 0, ctx->stream>>>(begin, end, h->d_parent, h->G, h->L);
		LB200_CHECK_LAUNCH(ctx);
	}
	return LB200_OK;
}

int lb200_hierarchy_get_locals(lb200_hierarchy* h, lb200_transform* out_locals) {
	if (!h || !out_locals) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	soa_to_aos_kernel<<<(h->n + HT - 1) / HT, HT, 0, ctx->stream>>>(h->L, h->d_order, h->n, h->d_stage);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaMemcpyAsync(out_locals, h->d_stage, sizeof(lb200_transform) * (size_t)h->n, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

int lb200_hierarchy_get_relative_matrices(lb200_hierarchy* h, const double base_pos[3], float* out_matrices) {
	if (!h || !base_pos || !out_matrices) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!h->d_matrices) LB200_CUDA(ctx, h->d_matrices.alloc(4 * (size_t)h->n));
	relative_matrices_kernel<<<(h->n + HT - 1) / HT, HT, 0, ctx->stream>>>(h->G, h->d_order, h->n, base_pos[0], base_pos[1], base_pos[2], h->d_matrices);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaMemcpyAsync(out_matrices, h->d_matrices, sizeof(float) * 16 * (size_t)h->n, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

uint64_t lb200_hierarchy_algorithmic_bytes(const lb200_hierarchy* h) {
	if (!h) return 0;
	const uint64_t non_root = h->n - h->level_start[1];
	return non_root * (52 + 4 + 52) + h->gather_bytes;
}

} // extern "C"
