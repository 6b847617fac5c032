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
//
// The level order itself is built on the device (buildTopology, behind lb200_hierarchy_create and lb200_hierarchy_set_parents*): the stable
// radix sort of (parent, node) pairs gives every parent's children as one ascending run, and one cooperative kernel expands the levels
// from the roots.  A topology change keeps the object: transforms move with their nodes to the new level positions.
#include "grid_barrier.cuh"
#include "lb200_internal.h"
#include "lb200_math.cuh"

#include <algorithm>
#include <memory>
#include <new>
#include <utility>
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

// a few transforms (World::setTransform / setLocalTransform for some entities): node ids + values -> their level positions, which are
// marked as moved for the next propagate_moved
__global__ void __launch_bounds__(HT) scatter_transforms_kernel(const uint32_t* __restrict__ nodes, const lb200_transform* __restrict__ values, uint32_t count,
	const uint32_t* __restrict__ pos_of_node, SoaTransforms out, uint8_t* __restrict__ mark)
{
	const uint32_t k = blockIdx.x * HT + threadIdx.x;
	if (k >= count) return;
	const uint32_t i = pos_of_node[nodes[k]];
	const lb200_transform t = values[k];
	out.px[i] = t.pos[0]; out.py[i] = t.pos[1]; out.pz[i] = t.pos[2];
	out.rot[i] = make_float4(t.rot[0], t.rot[1], t.rot[2], t.rot[3]);
	out.sx[i] = t.scale[0]; out.sy[i] = t.scale[1]; out.sz[i] = t.scale[2];
	mark[i] = 1;
}

// lb200_hierarchy_mark_moved: node ids -> marks at their level positions
__global__ void __launch_bounds__(HT) mark_nodes_kernel(const uint32_t* __restrict__ nodes, uint32_t count, const uint32_t* __restrict__ pos_of_node,
	uint8_t* __restrict__ mark)
{
	const uint32_t k = blockIdx.x * HT + threadIdx.x;
	if (k < count) mark[pos_of_node[nodes[k]]] = 1;
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
__device__ __forceinline__ void compute_local_node(uint32_t i, int p, const SoaTransforms& G, const SoaTransforms& L) {
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

__global__ void __launch_bounds__(HT) compute_locals_kernel(uint32_t begin, uint32_t end, const int* __restrict__ parent, SoaTransforms G, SoaTransforms L) {
	const uint32_t i = begin + blockIdx.x * HT + threadIdx.x;
	if (i >= end) return;
	compute_local_node(i, parent[i], G, L);
}

// One depth level: nodes [begin, end) in level order; parents live in earlier levels.
// Launched with programmatic stream serialization: the block starts while the previous level is still draining, loads its
// own locals (independent of that level) and only then waits for the parents' globals.
// FLAGS (propagate_moved): also flag[i] = mark[i] | flag[parent], i.e. the node or one of its ancestors was marked (World::transformEntity
// recurses into every child of a moved entity, world.cpp:272-278).  The <false> instantiation is the plain propagate; mark / flag unused.
template <bool FLAGS>
__global__ void __launch_bounds__(HT) propagate_level_kernel(uint32_t begin, uint32_t end, const int* __restrict__ parent, SoaTransforms L, SoaTransforms G,
	const uint8_t* __restrict__ mark, uint8_t* __restrict__ flag)
{
	const uint32_t i = begin + blockIdx.x * HT + threadIdx.x;
	const bool active = i < end;
	int p = 0;
	D3 lpos = d3(0, 0, 0);
	float4 lr = make_float4(0, 0, 0, 1);
	V3 lscale = v3(1, 1, 1);
	uint8_t m = 0;
	if (active) {
		p = parent[i];
		lpos = d3(L.px[i], L.py[i], L.pz[i]);
		lr = L.rot[i];
		lscale = v3(L.sx[i], L.sy[i], L.sz[i]);
		if (FLAGS) m = mark[i];
	}
	cudaGridDependencySynchronize();
	if (!active) return;
	if (FLAGS) flag[i] = m | flag[p];
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

template <bool FLAGS>
__global__ void __launch_bounds__(SMALL_THREADS) propagate_small_levels_kernel(const __grid_constant__ SmallLevels S, const int* __restrict__ parent, SoaTransforms L, SoaTransforms G,
	const uint8_t* __restrict__ mark, uint8_t* __restrict__ flag)
{
	for (uint32_t l = 0; l < S.n; ++l) {
		for (uint32_t i = S.start[l] + threadIdx.x; i < S.start[l + 1]; i += SMALL_THREADS) {
			compose_node(i, parent, L, G);
			if (FLAGS) flag[i] = mark[i] | flag[parent[i]];
		}
		__syncthreads();
	}
}

// render_module.cpp:1544-1554: radius of the world bounding sphere of a moved model instance (level position i); its centre is the global position
__device__ __forceinline__ float sphere_radius(const SoaTransforms& G, uint32_t i, float bounding_radius) {
	const float sx = G.sx[i], sy = G.sy[i], sz = G.sz[i];
	const float bc = sy > sz ? sy : sz; // maximum(a, b, c) = a > max(b, c) ? a : max(b, c), math.h:468-475
	const float m = sx > bc ? sx : bc;
	return LB_FMUL(bounding_radius, m);
}

__global__ void __launch_bounds__(HT) spheres_kernel(SoaTransforms G, const uint32_t* __restrict__ order, const float* __restrict__ bounding_radius, uint32_t n,
	double* __restrict__ out_pos3, float* __restrict__ out_radius)
{
	const uint32_t i = blockIdx.x * HT + threadIdx.x;
	if (i >= n) return;
	const uint32_t node = order[i];
	out_pos3[3 * (size_t)node + 0] = G.px[i];
	out_pos3[3 * (size_t)node + 1] = G.py[i];
	out_pos3[3 * (size_t)node + 2] = G.pz[i];
	out_radius[node] = sphere_radius(G, i, bounding_radius[node]);
}

// ---- The moved list of propagate_moved: nodes i (ascending) with flag[pos_of_node[i]] and entity[i] >= 0 ----
// Two launches: every tile of MT nodes counts its listed nodes; then every tile sums the counts of the tiles before it (as many loads as
// tiles: a few hundred at 1 M nodes) and writes its nodes in order, round by round of CT nodes with a ballot per warp.  No atomics: the
// order is the node order whatever the schedule.
constexpr int CT = 256, CT_WARPS = CT / 32, MT_ROUNDS = 8;
constexpr uint32_t MT = CT * MT_ROUNDS;

struct MovedOut { int32_t* entity; lb200_transform* transform; double* pos3; float* radius; uint32_t* count; };

__device__ __forceinline__ bool listed(uint32_t i, uint32_t n, const uint32_t* __restrict__ pos_of_node, const uint8_t* __restrict__ flag,
	const int32_t* __restrict__ entity)
{
	return i < n && entity[i] >= 0 && flag[pos_of_node[i]];
}

// sum of one value per thread over the block, in every thread.  All CT threads; s_warp is free again on return.
__device__ __forceinline__ uint32_t block_sum(uint32_t v, uint32_t* s_warp) {
	v = __reduce_add_sync(0xffffffffu, v);
	if ((threadIdx.x & 31u) == 0) s_warp[threadIdx.x >> 5] = v;
	__syncthreads();
	uint32_t t = 0;
#pragma unroll
	for (int w = 0; w < CT_WARPS; ++w) t += s_warp[w];
	__syncthreads();
	return t;
}

__global__ void __launch_bounds__(CT) moved_count_kernel(uint32_t n, const uint32_t* __restrict__ pos_of_node, const uint8_t* __restrict__ flag,
	const int32_t* __restrict__ entity, uint32_t* __restrict__ tile_count)
{
	__shared__ uint32_t s_warp[CT_WARPS];
	uint32_t c = 0;
#pragma unroll
	for (int r = 0; r < MT_ROUNDS; ++r) c += listed(blockIdx.x * MT + r * CT + threadIdx.x, n, pos_of_node, flag, entity);
	c = block_sum(c, s_warp);
	if (threadIdx.x == 0) tile_count[blockIdx.x] = c;
}

__global__ void __launch_bounds__(CT) moved_gather_kernel(uint32_t n, const uint32_t* __restrict__ pos_of_node, const uint8_t* __restrict__ flag,
	const int32_t* __restrict__ entity, const uint32_t* __restrict__ tile_count, SoaTransforms G, const float* __restrict__ bounding_radius, MovedOut out)
{
	__shared__ uint32_t s_warp[CT_WARPS];
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	uint32_t before = 0;
	for (uint32_t t = threadIdx.x; t < blockIdx.x; t += CT) before += tile_count[t];
	uint32_t o = block_sum(before, s_warp); // the tile's first output slot
	for (int r = 0; r < MT_ROUNDS; ++r) {
		const uint32_t i = blockIdx.x * MT + r * CT + threadIdx.x;
		const bool f = listed(i, n, pos_of_node, flag, entity);
		const uint32_t ballot = __ballot_sync(0xffffffffu, f);
		if (lane == 0) s_warp[warp] = __popc(ballot);
		__syncthreads();
		uint32_t at = o + __popc(ballot & ((1u << lane) - 1u)), total = 0;
#pragma unroll
		for (int w = 0; w < CT_WARPS; ++w) { const uint32_t c = s_warp[w]; at += (uint32_t)w < warp ? c : 0u; total += c; }
		__syncthreads();
		o += total;
		if (!f) continue;
		const uint32_t k = pos_of_node[i];
		out.entity[at] = entity[i];
		lb200_transform t;
		t.pos[0] = G.px[k]; t.pos[1] = G.py[k]; t.pos[2] = G.pz[k];
		const float4 q = G.rot[k];
		t.rot[0] = q.x; t.rot[1] = q.y; t.rot[2] = q.z; t.rot[3] = q.w;
		t.scale[0] = G.sx[k]; t.scale[1] = G.sy[k]; t.scale[2] = G.sz[k];
		out.transform[at] = t;
		if (bounding_radius) {
			out.pos3[3 * (size_t)at + 0] = t.pos[0];
			out.pos3[3 * (size_t)at + 1] = t.pos[1];
			out.pos3[3 * (size_t)at + 2] = t.pos[2];
			out.radius[at] = sphere_radius(G, k, bounding_radius[i]);
		}
	}
	if (blockIdx.x == gridDim.x - 1 && threadIdx.x == 0) *out.count = o;
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

// ---- Bone attachments (lb200_hierarchy_set_attachments / lb200_hierarchy_propagate_attached) ----
// An attached node's global is set by its attachment, and compose o computeLocal is not exact: recomposing the node from the local computed
// for it would move it by an ulp.  So the propagate of a frame with attachments skips a pinned (attached) node unless it is marked (its local
// was written) or its parent's flag is set in this pass (an ancestor moved, World::transformEntity recomposes the node from its local).
__global__ void __launch_bounds__(HT) propagate_pinned_level_kernel(uint32_t begin, uint32_t end, const int* __restrict__ parent, SoaTransforms L, SoaTransforms G,
	const uint8_t* __restrict__ mark, const uint8_t* __restrict__ pinned, uint8_t* __restrict__ flag)
{
	const uint32_t i = begin + blockIdx.x * HT + threadIdx.x;
	const bool active = i < end;
	int p = 0;
	uint8_t m = 0, pin = 0;
	if (active) { p = parent[i]; m = mark[i]; pin = pinned[i]; }
	cudaGridDependencySynchronize();
	if (!active) return;
	const uint8_t f = m | flag[p];
	flag[i] = f;
	if (!pin || f) compose_node(i, parent, L, G);
}

__global__ void __launch_bounds__(SMALL_THREADS) propagate_pinned_small_levels_kernel(const __grid_constant__ SmallLevels S, const int* __restrict__ parent,
	SoaTransforms L, SoaTransforms G, const uint8_t* __restrict__ mark, const uint8_t* __restrict__ pinned, uint8_t* __restrict__ flag)
{
	for (uint32_t l = 0; l < S.n; ++l) {
		for (uint32_t i = S.start[l] + threadIdx.x; i < S.start[l + 1]; i += SMALL_THREADS) {
			const uint8_t f = mark[i] | flag[parent[i]];
			flag[i] = f;
			if (!pinned[i] || f) compose_node(i, parent, L, G);
		}
		__syncthreads();
	}
}

// One attachment of the table in round order: level positions of the attached and the parent node, the parent's node index (its entity
// id decides whether its move triggers), the system slot, instance, bone and BoneAttachment::relative_transform (pos xyz, rot xyzw).
struct AttachRecord { uint32_t pos_a, pos_p, node_p, slot, instance, bone; float rel[7]; };
// One animation system of a propagate_attached call: its absolute poses and whether it was updated this frame
struct AttachSystem { const float* pos; const float* rot; uint32_t bone_count, posed; };

// The attachments [begin, end) of one round.  Active (the system was posed, or the parent node moved so far in this call and listens):
// RenderModuleImpl::updateBoneAttachment (render_module.cpp:377-405) into the SoA globals, then World::setTransform's update_local
// (world.cpp:267-270) for a node with a world parent.  The node is flagged (moved) and stamped: the round's recompose starts below it.
__global__ void __launch_bounds__(HT) attach_round_kernel(const AttachRecord* __restrict__ rec, uint32_t begin, uint32_t end, const AttachSystem* __restrict__ systems,
	const int32_t* __restrict__ entity, const int* __restrict__ parent, SoaTransforms L, SoaTransforms G, uint8_t* __restrict__ flag, uint32_t* __restrict__ stamps,
	uint32_t stamp)
{
	const uint32_t k = begin + blockIdx.x * HT + threadIdx.x;
	if (k >= end) return;
	const AttachRecord x = rec[k];
	const AttachSystem sys = systems[x.slot];
	if (!sys.posed && !(flag[x.pos_p] && entity[x.node_p] >= 0)) return;
	const size_t bi = (size_t)x.instance * sys.bone_count + x.bone;
	Rigid b;
	b.pos = v3(sys.pos[3 * bi], sys.pos[3 * bi + 1], sys.pos[3 * bi + 2]);
	b.rot = q4(sys.rot[4 * bi], sys.rot[4 * bi + 1], sys.rot[4 * bi + 2], sys.rot[4 * bi + 3]);
	Rigid rel;
	rel.pos = v3(x.rel[0], x.rel[1], x.rel[2]);
	rel.rot = q4(x.rel[3], x.rel[4], x.rel[5], x.rel[6]);
	const uint32_t p = x.pos_p, a = x.pos_a;
	const float4 pr = G.rot[p];
	D3 pos;
	Q4 rot;
	compose_rigid(d3(G.px[p], G.py[p], G.pz[p]), q4(pr.x, pr.y, pr.z, pr.w), v3(G.sx[p], G.sy[p], G.sz[p]), rmul(b, rel), pos, rot); // math.cpp:859-861, 763
	G.px[a] = pos.x; G.py[a] = pos.y; G.pz[a] = pos.z;
	G.rot[a] = make_float4(rot.x, rot.y, rot.z, rot.w); // the scale stays the node's own (result.scale = original_scale)
	const int w = parent[a];
	if (w >= 0) compute_local_node(a, w, G, L);
	flag[a] = 1;
	stamps[a] = stamp;
}

// The recompose behind a round: a node whose parent was written in this round (stamp) is composed from its local, flagged and stamped.
__global__ void __launch_bounds__(HT) recompose_level_kernel(uint32_t begin, uint32_t end, const int* __restrict__ parent, SoaTransforms L, SoaTransforms G,
	uint32_t* __restrict__ stamps, uint32_t stamp, uint8_t* __restrict__ flag)
{
	const uint32_t i = begin + blockIdx.x * HT + threadIdx.x;
	const bool active = i < end;
	const int p = active ? parent[i] : 0;
	cudaGridDependencySynchronize();
	if (!active || stamps[p] != stamp) return;
	compose_node(i, parent, L, G);
	stamps[i] = stamp;
	flag[i] = 1;
}

__global__ void __launch_bounds__(SMALL_THREADS) recompose_small_levels_kernel(const __grid_constant__ SmallLevels S, const int* __restrict__ parent,
	SoaTransforms L, SoaTransforms G, uint32_t* __restrict__ stamps, uint32_t stamp, uint8_t* __restrict__ flag)
{
	for (uint32_t l = 0; l < S.n; ++l) {
		for (uint32_t i = S.start[l] + threadIdx.x; i < S.start[l + 1]; i += SMALL_THREADS) {
			if (stamps[parent[i]] != stamp) continue;
			compose_node(i, parent, L, G);
			stamps[i] = stamp;
			flag[i] = 1;
		}
		__syncthreads();
	}
}

// The round build.  Attachment k -> its attached node's level position: the position's attachment and pin; every round starts at 1.
__global__ void __launch_bounds__(HT) attach_index_kernel(const uint32_t* __restrict__ attached, uint32_t count, const uint32_t* __restrict__ pos_of_node,
	int32_t* __restrict__ att_of_pos, uint8_t* __restrict__ pinned, uint32_t* __restrict__ round)
{
	const uint32_t k = blockIdx.x * HT + threadIdx.x;
	if (k >= count) return;
	const uint32_t a = pos_of_node[attached[k]];
	att_of_pos[a] = (int32_t)k;
	pinned[a] = 1;
	round[k] = 1;
}

struct RoundState { uint32_t changed, max_round, count, pad; }; // count: the pairs the round sort takes

// max(r, 1 + the round of every attachment whose attached node is q or an ancestor of q)
__device__ __forceinline__ uint32_t rounds_above(int q, const int* __restrict__ parent, const int32_t* __restrict__ att_of_pos, const uint32_t* round, uint32_t r) {
	for (; q >= 0; q = parent[q]) {
		const int32_t y = att_of_pos[q];
		if (y >= 0) r = max(r, __ldcg(round + y) + 1);
	}
	return r;
}

// One step towards the least fixed point of round[X] = 1 + max(round[Y]) over the attachments Y whose attached node is an ancestor-or-self of
// X's parent node or a strict ancestor of X's attached node (1 when there is none).  In place: rounds only grow, and every value stays at or
// below the fixed point.  A cycle has none: its rounds grow past the attachment count.
__global__ void __launch_bounds__(HT) attach_rounds_kernel(const uint32_t* __restrict__ attached, const uint32_t* __restrict__ parent_node, uint32_t count,
	const uint32_t* __restrict__ pos_of_node, const int* __restrict__ parent, const int32_t* __restrict__ att_of_pos, uint32_t* round, RoundState* st)
{
	const uint32_t k = blockIdx.x * HT + threadIdx.x;
	if (k >= count) return;
	uint32_t r = rounds_above((int)pos_of_node[parent_node[k]], parent, att_of_pos, round, 1u);
	r = rounds_above(parent[pos_of_node[attached[k]]], parent, att_of_pos, round, r);
	if (r > __ldcg(round + k)) {
		__stcg(round + k, r);
		st->changed = 1;
	}
	atomicMax(&st->max_round, r);
}

__global__ void __launch_bounds__(HT) attach_keys_kernel(const uint32_t* __restrict__ round, uint32_t count, uint64_t* __restrict__ keys, uint64_t* __restrict__ values,
	RoundState* st)
{
	const uint32_t k = blockIdx.x * HT + threadIdx.x;
	if (k == 0) st->count = count;
	if (k >= count) return;
	keys[k] = round[k];
	values[k] = k;
}

// The table sorted by round -> records in round order; starts[r - 1] = the first record of round r (R + 1 entries, rounds are contiguous:
// a round r > 1 exists because of one of round r - 1), starts[R + 1 + r - 1] = the smallest attached level position of round r (pre-set
// to all ones): its level is where the round's recompose starts.
__global__ void __launch_bounds__(HT) attach_records_kernel(const uint64_t* __restrict__ keys, const uint64_t* __restrict__ values, uint32_t count, uint32_t n_rounds,
	const uint32_t* __restrict__ table, const float* __restrict__ relative7, const uint32_t* __restrict__ pos_of_node, AttachRecord* __restrict__ rec,
	uint32_t* __restrict__ starts)
{
	const uint32_t j = blockIdx.x * HT + threadIdx.x;
	if (j >= count) return;
	const uint32_t k = (uint32_t)values[j], r = (uint32_t)keys[j];
	AttachRecord x;
	x.pos_a = pos_of_node[table[k]];
	x.node_p = table[count + k];
	x.pos_p = pos_of_node[x.node_p];
	x.slot = table[2 * (size_t)count + k];
	x.instance = table[3 * (size_t)count + k];
	x.bone = table[4 * (size_t)count + k];
#pragma unroll
	for (int c = 0; c < 7; ++c) x.rel[c] = relative7[7 * (size_t)k + c];
	rec[j] = x;
	if (j == 0 || keys[j - 1] != keys[j]) starts[r - 1] = j;
	if (j + 1 == count) starts[n_rounds] = count;
	atomicMin(&starts[n_rounds + r], x.pos_a);
}

// ---- The level-order builder ----
// Level 0 = the roots in ascending node index; level l + 1 = the children of level l's nodes, walked in level order, each node's children
// in ascending node index.  parent_pos = the parent's level position.
constexpr int BT = 512;                      // threads of expand_levels_kernel; a level is expanded in tiles of BT positions
constexpr int BT_WARPS = BT / 32;
constexpr uint32_t SOLO_LEVEL_NODES = 4096;  // levels up to this many nodes are expanded by block 0 alone, without a grid barrier

struct BuildState { // zeroed before every build
	GridBar bar;
	uint32_t count, pad;              // count: the number of pairs the sort takes (n)
	unsigned long long bad_parent;    // max over the nodes whose parent is >= n of (node + 1) << 32 | parent; 0 = none
	uint32_t depth, placed, distinct; // non-empty levels, nodes placed in them, placed nodes that have a child
	uint32_t next_b, next_e, next_l;  // block 0 -> the grid after a run of narrow levels: the level to go on with and its number
};

// (key = parent, value = node) in node order.  Roots get key n, nodes with an out-of-range parent key n + 1: after the stable sort every
// parent's children are one run in ascending node index, and the roots are the run of key n.
__global__ void __launch_bounds__(HT) child_keys_kernel(const int32_t* __restrict__ parents, uint32_t n, uint64_t* __restrict__ keys, uint64_t* __restrict__ nodes,
	BuildState* st)
{
	const uint32_t i = blockIdx.x * HT + threadIdx.x;
	if (i == 0) st->count = n;
	if (i >= n) return;
	const int32_t p = parents[i];
	uint64_t key = p < 0 ? (uint64_t)n : (uint64_t)p;
	if (p >= 0 && (uint32_t)p >= n) {
		atomicMax(&st->bad_parent, ((unsigned long long)(i + 1) << 32) | (uint32_t)p); // the highest such node, as create's descending loop reports it
		key = (uint64_t)n + 1;
	}
	keys[i] = key;
	nodes[i] = i;
}

struct BuildArgs {
	const uint64_t* keys; const uint64_t* nodes; // the sorted pairs
	uint32_t n;
	uint32_t* child_begin; uint32_t* child_end;  // [n + 2], zeroed: the children of node k are nodes[child_begin[k], child_end[k]); k = n: the roots
	uint32_t* order; int* parent_pos;            // [n] level position -> node, -> parent's level position
	uint32_t* level_start;                       // [n + 2]
	uint32_t* block_sum;                         // [gridDim]
	BuildState* st;
};

// Inclusive scan of one value per thread over the block; `total` = the block's sum.  All BT threads.
__device__ __forceinline__ uint32_t block_scan(uint32_t v, uint32_t* s_warp, uint32_t& total) {
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	uint32_t x = v;
#pragma unroll
	for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, o); if (lane >= (uint32_t)o) x += y; }
	if (lane == 31) s_warp[warp] = x;
	__syncthreads();
	if (warp == 0) {
		uint32_t w = lane < BT_WARPS ? s_warp[lane] : 0u;
#pragma unroll
		for (int o = 1; o < 32; o <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, w, o); if (lane >= (uint32_t)o) w += y; }
		if (lane < BT_WARPS) s_warp[lane] = w;
	}
	__syncthreads();
	const uint32_t incl = x + (warp ? s_warp[warp - 1] : 0u);
	total = s_warp[BT_WARPS - 1];
	__syncthreads(); // s_warp is free again
	return incl;
}

// Level positions [k0, min(k0 + BT, end)): their children, in level order, to positions out, out + 1, ... of the next level.  The block
// writes the children together (thread q finds its parent by binary search over the tile's scan), so a wide star costs what a chain does.
// Returns the tile's number of children; `parents` counts the positions that have children.  All BT threads.
__device__ uint32_t expand_tile(const BuildArgs& a, uint32_t k0, uint32_t end, uint32_t out, uint32_t* s_incl, uint32_t* s_begin, uint32_t* s_warp, uint32_t& parents) {
	const uint32_t k = k0 + threadIdx.x;
	uint32_t begin = 0, c = 0;
	if (k < end) {
		const uint32_t node = __ldcg(a.order + k);
		begin = __ldcg(a.child_begin + node);
		c = __ldcg(a.child_end + node) - begin;
	}
	parents += c != 0;
	uint32_t total;
	s_incl[threadIdx.x] = block_scan(c, s_warp, total);
	s_begin[threadIdx.x] = begin;
	__syncthreads();
	for (uint32_t q = threadIdx.x; q < total; q += BT) {
		uint32_t lo = 0, hi = BT - 1; // the first tile position whose inclusive child count exceeds q
		while (lo < hi) { const uint32_t mid = (lo + hi) >> 1; if (s_incl[mid] > q) hi = mid; else lo = mid + 1; }
		const uint32_t first = lo ? s_incl[lo - 1] : 0u;
		a.order[out + q] = (uint32_t)a.nodes[s_begin[lo] + (q - first)];
		a.parent_pos[out + q] = (int)(k0 + lo);
	}
	__syncthreads();
	return total;
}

// One cooperative launch for every level, however deep: child runs -> level 0 -> level by level until a level is empty.  A level wider than
// SOLO_LEVEL_NODES is expanded by the whole grid (block g takes a contiguous share of its tiles: count, grid barrier, every block sums the
// shares before its own, expand, grid barrier); narrower ones by block 0 alone while the others wait at one barrier.
__global__ void __launch_bounds__(BT) expand_levels_kernel(BuildArgs a) {
	__shared__ uint32_t s_incl[BT], s_begin[BT], s_warp[BT_WARPS];
	BuildState* st = a.st;
	const uint32_t tid = threadIdx.x, grid = gridDim.x;
	uint32_t passed = 0, parents = 0;
	for (uint32_t j = blockIdx.x * BT + tid; j < a.n; j += grid * BT) {
		const uint64_t k = a.keys[j];
		if (j == 0 || a.keys[j - 1] != k) a.child_begin[k] = j;
		if (j + 1 == a.n || a.keys[j + 1] != k) a.child_end[k] = j + 1;
	}
	grid_barrier(&st->bar, passed);
	const uint32_t roots = __ldcg(a.child_begin + a.n);
	uint32_t b = 0, e = __ldcg(a.child_end + a.n) - roots, l = 0; // level l = positions [b, e)
	for (uint32_t k = blockIdx.x * BT + tid; k < e; k += grid * BT) { a.order[k] = (uint32_t)a.nodes[roots + k]; a.parent_pos[k] = -1; }
	if (blockIdx.x == 0 && tid == 0) { a.level_start[0] = 0; a.level_start[1] = e; }
	grid_barrier(&st->bar, passed);
	while (e > b) {
		if (e - b <= SOLO_LEVEL_NODES) {
			if (blockIdx.x == 0) {
				do {
					uint32_t total = 0;
					for (uint32_t k0 = b; k0 < e; k0 += BT) total += expand_tile(a, k0, e, e + total, s_incl, s_begin, s_warp, parents);
					if (tid == 0) a.level_start[l + 2] = e + total;
					b = e; e += total; ++l;
				} while (e > b && e - b <= SOLO_LEVEL_NODES);
				if (tid == 0) { st->next_b = b; st->next_e = e; st->next_l = l; }
			}
			grid_barrier(&st->bar, passed);
			b = __ldcg(&st->next_b); e = __ldcg(&st->next_e); l = __ldcg(&st->next_l);
			continue;
		}
		const uint32_t tiles = (e - b + BT - 1) / BT;
		const uint32_t tb = (uint32_t)((unsigned long long)blockIdx.x * tiles / grid), te = (uint32_t)((unsigned long long)(blockIdx.x + 1) * tiles / grid);
		const uint32_t kb = b + tb * BT, ke = min(e, b + te * BT);
		uint32_t c = 0;
		for (uint32_t k = kb + tid; k < ke; k += BT) { const uint32_t node = __ldcg(a.order + k); c += __ldcg(a.child_end + node) - __ldcg(a.child_begin + node); }
		uint32_t mine;
		block_scan(c, s_warp, mine);
		if (tid == 0) a.block_sum[blockIdx.x] = mine;
		grid_barrier(&st->bar, passed);
		uint32_t before = 0, all = 0;
		for (uint32_t g = tid; g < grid; g += BT) { const uint32_t s = __ldcg(a.block_sum + g); all += s; if (g < blockIdx.x) before += s; }
		block_scan(before, s_warp, before); // the block's sums: children of the shares before this block's, and of the whole level
		block_scan(all, s_warp, all);
		uint32_t out = e + before;
		for (uint32_t k0 = kb; k0 < ke; k0 += BT) out += expand_tile(a, k0, ke, out, s_incl, s_begin, s_warp, parents);
		if (blockIdx.x == 0 && tid == 0) a.level_start[l + 2] = e + all;
		grid_barrier(&st->bar, passed);
		b = e; e += all; ++l;
	}
#pragma unroll
	for (int o = 16; o > 0; o >>= 1) parents += __shfl_xor_sync(0xffffffffu, parents, o);
	if ((tid & 31u) == 0 && parents) atomicAdd(&st->distinct, parents);
	if (blockIdx.x == 0 && tid == 0) { st->depth = l; st->placed = e; }
}

__device__ __forceinline__ void copy_transform(const SoaTransforms& src, uint32_t from, const SoaTransforms& dst, uint32_t to) {
	dst.px[to] = src.px[from]; dst.py[to] = src.py[from]; dst.pz[to] = src.pz[from];
	dst.rot[to] = src.rot[from];
	dst.sx[to] = src.sx[from]; dst.sy[to] = src.sy[from]; dst.sz[to] = src.sz[from];
}

__device__ __forceinline__ void identity_transform(const SoaTransforms& dst, uint32_t to) {
	dst.px[to] = 0.0; dst.py[to] = 0.0; dst.pz[to] = 0.0;
	dst.rot[to] = make_float4(0.f, 0.f, 0.f, 1.f);
	dst.sx[to] = 1.f; dst.sy[to] = 1.f; dst.sz[to] = 1.f;
}

// The new level order -> pos_of_node, and every node's locals, globals and moved mark from its old level position to its new one, and its
// entity id (the identity transforms, no mark and entity i for nodes i >= old_n, which the hierarchy did not hold before).
__global__ void __launch_bounds__(HT) permute_kernel(const uint32_t* __restrict__ order, uint32_t n, const uint32_t* __restrict__ old_pos_of_node, uint32_t old_n,
	SoaTransforms old_L, SoaTransforms old_G, const uint8_t* __restrict__ old_mark, const int32_t* __restrict__ old_entity,
	uint32_t* __restrict__ pos_of_node, SoaTransforms L, SoaTransforms G, uint8_t* __restrict__ mark, int32_t* __restrict__ entity)
{
	const uint32_t k = blockIdx.x * HT + threadIdx.x;
	if (k >= n) return;
	const uint32_t i = order[k];
	pos_of_node[i] = k;
	if (i < old_n) {
		const uint32_t o = old_pos_of_node[i];
		copy_transform(old_L, o, L, k);
		copy_transform(old_G, o, G, k);
		mark[k] = old_mark[o];
		entity[i] = old_entity[i];
	}
	else {
		identity_transform(L, k);
		identity_transform(G, k);
		mark[k] = 0;
		entity[i] = (int32_t)i;
	}
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
	DeviceArray<uint8_t> d_mark;         // level position -> 1: set_subset / mark_moved named the node since the last propagate_moved
	DeviceArray<int32_t> d_entity;       // caller node index -> entity id of the moved list (-1: never listed)
	// propagate_moved: the flags (level position -> the node or an ancestor is marked), the per-tile counts and the moved list (capacity n),
	// allocated together and released when n changes
	DeviceArray<uint8_t> d_flag; DeviceArray<uint32_t> d_tile_count;
	DeviceArray<int32_t> d_moved_entity; DeviceArray<lb200_transform> d_moved_transform; DeviceArray<double> d_moved_pos; DeviceArray<float> d_moved_radius;
	DeviceArray<uint32_t> d_moved_count; PinnedArray<uint32_t> h_moved_count;
	DeviceArray<lb200_transform> d_stage; // n Transforms (API boundary)
	DeviceArray<float4> d_matrices;       // n relative matrices, 4 float4 each (lb200_hierarchy_get_relative_matrices)
	// the inputs and outputs of spheres_kernel, allocated and released together
	DeviceArray<float> d_radius_in;
	DeviceArray<double> d_sphere_pos;
	DeviceArray<float> d_sphere_radius;
	uint64_t gather_bytes = 0;
	// buildTopology builds the next topology into `next` and swaps it with the current one only once it is known to be valid
	struct Topology { DeviceArray<uint32_t> order, pos_of_node; DeviceArray<int> parent; SoaArrays L, G; DeviceArray<uint8_t> mark; DeviceArray<int32_t> entity; } next;
	// buildTopology's scratch, grown to the largest n built (sizes are the capacities)
	DeviceArray<int32_t> d_parents_in;                            // lb200_hierarchy_set_parents: the caller's parents, uploaded
	DeviceArray<uint64_t> d_keys[2], d_nodes[2];                  // the sorted pairs and the sort's alternate buffers
	DeviceArray<uint32_t> d_child_begin, d_child_end, d_level_start; // n + 2 each
	DeviceArray<uint8_t> d_build_state; DeviceArray<uint32_t> d_block_sum; PinnedArray<uint8_t> h_readback;
	RadixSortScratch sort;
	uint32_t expand_grid = 0; // blocks of expand_levels_kernel that can be co-resident
	// bone attachments: the table of set_attachments in caller node indices, on the device as [attached][parent][system][instance][bone] (u32,
	// att_count each) + 7 floats each, and per system slot the table names the largest instance and bone (host checks of every call)
	// (a vector that scales with the slot value would let one large slot ask for gigabytes)
	struct SlotUse { uint32_t slot, max_instance, max_bone; };
	uint32_t att_count = 0, att_max_node = 0;
	std::vector<SlotUse> att_slots; // the distinct slots the table names, ascending
	DeviceArray<uint32_t> d_att_table; DeviceArray<float> d_att_relative;
	// the rounds of the table in the current topology (rebuilt when att_rounds_valid is false): records in round order, round r = records
	// [att_round_start[r - 1], att_round_start[r]), its recompose starting below level att_round_level[r - 1]; per attachment its round; the
	// pins (level position -> attached) and the stamps of the recomposes (level position -> the last (call, round) that wrote the node)
	bool att_rounds_valid = false;
	std::vector<uint32_t> att_round_start, att_round_level;
	DeviceArray<AttachRecord> d_att_records; DeviceArray<uint32_t> d_att_round;
	DeviceArray<uint8_t> d_pinned; DeviceArray<uint32_t> d_stamp; uint32_t stamp = 0;
	DeviceArray<AttachSystem> d_att_systems; std::vector<AttachSystem> att_systems;
};

namespace {

// level starts read back together with the build's counters; a deeper hierarchy takes a second read-back for the rest
constexpr uint32_t READBACK_LEVELS = 64;

int growBuildScratch(lb200_hierarchy* h, uint32_t n) {
	lb200_ctx* ctx = h->ctx;
	if (!h->d_build_state) {
		LB200_CUDA(ctx, h->d_build_state.alloc(sizeof(BuildState)));
		LB200_CUDA(ctx, h->h_readback.alloc(sizeof(BuildState) + sizeof(uint32_t) * READBACK_LEVELS));
		int rc = lb200_radix_sort_alloc_scratch(ctx, (uint32_t)ctx->sm_count * 2, h->sort);
		if (!rc) rc = lb200_coop_grid_limit(ctx, (const void*)expand_levels_kernel, BT, 0, &h->expand_grid);
		if (rc) { h->d_build_state.reset(); return rc; }
		LB200_CUDA(ctx, h->d_block_sum.alloc(h->expand_grid));
	}
	if (h->d_parents_in.size() >= n) return LB200_OK;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // the stream may still use the old scratch
	LB200_CUDA(ctx, h->d_parents_in.alloc(n));
	for (int b = 0; b < 2; ++b) {
		LB200_CUDA(ctx, h->d_keys[b].alloc(n));
		LB200_CUDA(ctx, h->d_nodes[b].alloc(n));
	}
	LB200_CUDA(ctx, h->d_child_begin.alloc((size_t)n + 2));
	LB200_CUDA(ctx, h->d_child_end.alloc((size_t)n + 2));
	LB200_CUDA(ctx, h->d_level_start.alloc(std::max((size_t)n + 2, (size_t)READBACK_LEVELS)));
	return LB200_OK;
}

// The level order of `dev_parents` (n entries, device) -> the hierarchy, keeping every node's transforms.  Refused (LB200_ERR_INVALID, with
// create's error texts) for a parent >= n or a cycle; the hierarchy is then left as it was.  Launches: child keys, sort, expansion, permute,
// whatever the depth; read-backs: the counters with the first READBACK_LEVELS level starts, and the rest of the level starts if deeper.
int buildTopology(lb200_hierarchy* h, const int32_t* dev_parents, uint32_t n, uint32_t max_blocks) {
	lb200_ctx* ctx = h->ctx;
	cudaStream_t s = ctx->stream;
	int rc = growBuildScratch(h, n);
	if (rc) return rc;
	lb200_hierarchy::Topology& next = h->next;
	if (next.order.size() != n) {
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		LB200_CUDA(ctx, next.order.alloc(n));
		LB200_CUDA(ctx, next.pos_of_node.alloc(n));
		LB200_CUDA(ctx, next.parent.alloc(n));
		rc = next.L.alloc(ctx, n);
		if (!rc) rc = next.G.alloc(ctx, n);
		if (!rc && next.mark.alloc(n) != cudaSuccess) rc = LB200_ERR_CUDA;
		if (!rc && next.entity.alloc(n) != cudaSuccess) rc = LB200_ERR_CUDA;
		if (rc) { next.order.reset(); return rc; }
	}
	DeviceArray<lb200_transform> stage;
	if (n != h->n) LB200_CUDA(ctx, stage.alloc(n));

	BuildState* st = reinterpret_cast<BuildState*>(h->d_build_state.get());
	LB200_CUDA(ctx, cudaMemsetAsync(st, 0, sizeof(BuildState), s));
	LB200_CUDA(ctx, cudaMemsetAsync(h->d_child_begin, 0, sizeof(uint32_t) * ((size_t)n + 2), s));
	LB200_CUDA(ctx, cudaMemsetAsync(h->d_child_end, 0, sizeof(uint32_t) * ((size_t)n + 2), s));
	child_keys_kernel<<<(n + HT - 1) / HT, HT, 0, s>>>(dev_parents, n, h->d_keys[0], h->d_nodes[0], st);
	LB200_CHECK_LAUNCH(ctx);
	rc = lb200_radix_sort_pairs(ctx, s, h->d_keys[0], h->d_keys[1], h->d_nodes[0], h->d_nodes[1], &st->count, n, h->sort, max_blocks, false, nullptr);
	if (rc) return rc;
	BuildArgs args{h->d_keys[0], h->d_nodes[0], n, h->d_child_begin, h->d_child_end, next.order, next.parent, h->d_level_start, h->d_block_sum, st};
	const uint32_t grid = std::max(1u, std::min(std::min(h->expand_grid, max_blocks ? max_blocks : UINT32_MAX), (n + BT - 1) / BT));
	void* kargs[] = {&args};
	LB200_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)expand_levels_kernel, dim3(grid), dim3(BT), kargs, 0, s));
	LB200_CHECK_LAUNCH(ctx);
	uint8_t* rb = h->h_readback;
	uint32_t* rb_levels = reinterpret_cast<uint32_t*>(rb + sizeof(BuildState));
	LB200_CUDA(ctx, cudaMemcpyAsync(rb, st, sizeof(BuildState), cudaMemcpyDeviceToHost, s));
	LB200_CUDA(ctx, cudaMemcpyAsync(rb_levels, h->d_level_start, sizeof(uint32_t) * std::min((size_t)n + 2, (size_t)READBACK_LEVELS), cudaMemcpyDeviceToHost, s));
	LB200_CUDA(ctx, cudaStreamSynchronize(s));
	BuildState r;
	memcpy(&r, rb, sizeof(BuildState));
	if (r.bad_parent) { lb200_set_error(ctx, "parent index %d out of range", (int32_t)(uint32_t)r.bad_parent); return LB200_ERR_INVALID; }
	if (r.placed != n) { lb200_set_error(ctx, "hierarchy has a cycle (%zu of %u nodes reachable from roots)", (size_t)r.placed, n); return LB200_ERR_INVALID; }
	std::vector<uint32_t> level_start(r.depth + 1);
	if (r.depth + 1 <= READBACK_LEVELS) memcpy(level_start.data(), rb_levels, sizeof(uint32_t) * (r.depth + 1));
	else {
		LB200_CUDA(ctx, cudaMemcpyAsync(level_start.data(), h->d_level_start, sizeof(uint32_t) * (r.depth + 1), cudaMemcpyDeviceToHost, s));
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
	}

	permute_kernel<<<(n + HT - 1) / HT, HT, 0, s>>>(next.order, n, h->d_pos_of_node, h->n, h->L, h->G, h->d_mark, h->d_entity,
		next.pos_of_node, next.L, next.G, next.mark, next.entity);
	LB200_CHECK_LAUNCH(ctx);
	// valid: the new topology becomes the current one (the old arrays are kept for the next build: nothing is freed at an unchanged n)
	std::swap(h->d_order, next.order);
	std::swap(h->d_pos_of_node, next.pos_of_node);
	std::swap(h->d_parent, next.parent);
	std::swap(h->L, next.L);
	std::swap(h->G, next.G);
	std::swap(h->d_mark, next.mark);
	std::swap(h->d_entity, next.entity);
	if (n != h->n) { // everything sized by n follows; the bounding radii go with the spheres, so the next sphere refresh has to pass them
		h->d_stage = std::move(stage);
		h->d_matrices.reset();
		h->d_radius_in.reset(); h->d_sphere_pos.reset(); h->d_sphere_radius.reset();
		h->d_flag.reset(); h->d_tile_count.reset();
		h->d_moved_entity.reset(); h->d_moved_transform.reset(); h->d_moved_pos.reset(); h->d_moved_radius.reset();
	}
	h->n = n;
	h->level_start = std::move(level_start);
	h->gather_bytes = (uint64_t)r.distinct * 52;
	h->att_rounds_valid = false; // the attachments' level positions, pins and rounds belong to the old level order
	return LB200_OK;
}

int upload(lb200_hierarchy* h, const lb200_transform* src, SoaTransforms dst, uint32_t count_levelorder) {
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_stage, src, sizeof(lb200_transform) * (size_t)h->n, cudaMemcpyHostToDevice, ctx->stream));
	aos_to_soa_kernel<<<(count_levelorder + HT - 1) / HT, HT, 0, ctx->stream>>>(h->d_stage, h->d_order, count_levelorder, dst);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

// One pass over levels [first, depth): the narrow levels at its top run in one block (small(S) launches it), then level(cfg, begin, end)
// launches one kernel per level, chained by programmatic stream serialization.
template <class Small, class Level>
int launchLevels(lb200_hierarchy* h, size_t first, Small small, Level level) {
	lb200_ctx* ctx = h->ctx;
	const size_t n_levels = h->level_start.size() - 1;
	size_t l = first;
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
		small(S);
		LB200_CHECK_LAUNCH(ctx);
	}
	bool chained = S.n != 0; // the first kernel of a pass is a plain launch: whatever precedes it has fully completed
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
		LB200_CUDA(ctx, level(cfg, begin, end));
		LB200_CHECK_LAUNCH(ctx);
	}
	return LB200_OK;
}

// The level launches of lb200_hierarchy_propagate (FLAGS = false) and lb200_hierarchy_propagate_moved (FLAGS = true: the flags of the
// roots have to be in place before).
template <bool FLAGS>
int propagateLevels(lb200_hierarchy* h) {
	const uint8_t* mark = FLAGS ? (const uint8_t*)h->d_mark : nullptr;
	uint8_t* flag = FLAGS ? (uint8_t*)h->d_flag : nullptr;
	return launchLevels(h, 1,
		[&](const SmallLevels& S) { propagate_small_levels_kernel<FLAGS><<<1, SMALL_THREADS, 0, h->ctx->stream>>>(S, h->d_parent, h->L, h->G, mark, flag); },
		[&](const cudaLaunchConfig_t& cfg, uint32_t begin, uint32_t end) {
			return cudaLaunchKernelEx(&cfg, propagate_level_kernel<FLAGS>, begin, end, (const int*)h->d_parent, h->L, h->G, mark, flag);
		});
}

// One of set_subset's / mark_moved's two staging pairs (pinned + device), `bytes` large: the upload before last has left it.  The caller
// records subset_done[*turn] behind its launch.
int stageSubset(lb200_hierarchy* h, size_t bytes, uint8_t** hs, uint8_t** ds, uint32_t* turn) {
	lb200_ctx* ctx = h->ctx;
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
	*turn = h->subset_turn++ & 1u;
	LB200_CUDA(ctx, cudaEventSynchronize(h->subset_done[*turn])); // the upload before last has left this pair of buffers (no wait for the frame in flight)
	*hs = h->h_subset[*turn];
	*ds = h->d_subset[*turn];
	return LB200_OK;
}

int allocMoved(lb200_hierarchy* h) {
	if (h->d_flag) return LB200_OK;
	lb200_ctx* ctx = h->ctx;
	const size_t n = h->n;
	if (!h->h_moved_count) {
		LB200_CUDA(ctx, h->d_moved_count.alloc(1));
		LB200_CUDA(ctx, h->h_moved_count.alloc(1));
	}
	DeviceArray<uint8_t> flag; DeviceArray<uint32_t> tile_count; DeviceArray<int32_t> entity; DeviceArray<lb200_transform> transform;
	DeviceArray<double> pos; DeviceArray<float> radius;
	LB200_CUDA(ctx, flag.alloc(n));
	LB200_CUDA(ctx, tile_count.alloc((n + MT - 1) / MT));
	LB200_CUDA(ctx, entity.alloc(n));
	LB200_CUDA(ctx, transform.alloc(n));
	LB200_CUDA(ctx, pos.alloc(3 * n));
	LB200_CUDA(ctx, radius.alloc(n));
	h->d_flag = std::move(flag); h->d_tile_count = std::move(tile_count);
	h->d_moved_entity = std::move(entity); h->d_moved_transform = std::move(transform); h->d_moved_pos = std::move(pos); h->d_moved_radius = std::move(radius);
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

// propagate_moved's frame around `levels`, the launches that leave the globals and the flags: the radii and the roots' flags before, the
// moved list and the cleared marks after.
template <class Levels>
int movedFrame(lb200_hierarchy* h, const float* bounding_radius, lb200_hierarchy_moved* out, uint32_t* out_count, Levels levels) {
	lb200_ctx* ctx = h->ctx;
	cudaStream_t s = ctx->stream;
	int rc = allocMoved(h);
	if (!rc && bounding_radius) rc = allocSpheres(h);
	if (rc) return rc;
	if (bounding_radius) LB200_CUDA(ctx, cudaMemcpyAsync(h->d_radius_in, bounding_radius, sizeof(float) * h->n, cudaMemcpyHostToDevice, s));
	const float* radius = h->d_radius_in; // NULL: no radii held, no spheres
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_flag, h->d_mark, h->level_start[1], cudaMemcpyDeviceToDevice, s)); // roots: their own mark
	rc = levels();
	if (rc) return rc;
	const uint32_t tiles = (h->n + MT - 1) / MT;
	moved_count_kernel<<<tiles, CT, 0, s>>>(h->n, h->d_pos_of_node, h->d_flag, h->d_entity, h->d_tile_count);
	LB200_CHECK_LAUNCH(ctx);
	const MovedOut mo{h->d_moved_entity, h->d_moved_transform, h->d_moved_pos, h->d_moved_radius, h->d_moved_count};
	moved_gather_kernel<<<tiles, CT, 0, s>>>(h->n, h->d_pos_of_node, h->d_flag, h->d_entity, h->d_tile_count, h->G, radius, mo);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaMemsetAsync(h->d_mark, 0, h->n, s));
	out->entities = h->d_moved_entity;
	out->transforms = h->d_moved_transform;
	out->pos3 = radius ? (const double*)h->d_moved_pos : nullptr;
	out->radius = radius ? (const float*)h->d_moved_radius : nullptr;
	out->count = h->d_moved_count;
	if (out_count) {
		LB200_CUDA(ctx, cudaMemcpyAsync(h->h_moved_count, h->d_moved_count, sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		*out_count = *h->h_moved_count;
	}
	return LB200_OK;
}

// The rounds of the attachment table in the current level order (see attach_rounds_kernel), on the device: the pins, the fixed point (one
// 8-byte read-back per step), the stable radix sort of the table by round, the records in round order with the round starts and every
// round's shallowest attached node (one read-back).  A cycle: LB200_ERR_INVALID, the rounds stay invalid.
int buildRounds(lb200_hierarchy* h) {
	lb200_ctx* ctx = h->ctx;
	cudaStream_t s = ctx->stream;
	const uint32_t count = h->att_count, n = h->n;
	h->att_round_start.clear(); // no rounds to report unless this build succeeds
	if (h->d_pinned.size() != n) {
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		LB200_CUDA(ctx, h->d_pinned.alloc(n));
		LB200_CUDA(ctx, h->d_stamp.alloc(n));
		LB200_CUDA(ctx, cudaMemsetAsync(h->d_stamp, 0, sizeof(uint32_t) * n, s)); // stamps are never 0
	}
	if (h->d_att_round.size() < count) {
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		LB200_CUDA(ctx, h->d_att_round.alloc(count));
		LB200_CUDA(ctx, h->d_att_records.alloc(count));
	}
	DeviceArray<int32_t> att_of_pos; DeviceArray<uint32_t> starts; DeviceArray<RoundState> st;
	LB200_CUDA(ctx, att_of_pos.alloc(n));
	LB200_CUDA(ctx, starts.alloc(2 * (size_t)count + 1));
	LB200_CUDA(ctx, st.alloc(1));
	LB200_CUDA(ctx, cudaMemsetAsync(att_of_pos, 0xff, sizeof(int32_t) * n, s));
	LB200_CUDA(ctx, cudaMemsetAsync(h->d_pinned, 0, n, s));
	const uint32_t* table = h->d_att_table;
	const uint32_t grid = (count + HT - 1) / HT;
	attach_index_kernel<<<grid, HT, 0, s>>>(table, count, h->d_pos_of_node, att_of_pos, h->d_pinned, h->d_att_round);
	LB200_CHECK_LAUNCH(ctx);
	RoundState r{};
	do {
		LB200_CUDA(ctx, cudaMemsetAsync(st, 0, sizeof(RoundState), s));
		attach_rounds_kernel<<<grid, HT, 0, s>>>(table, table + count, count, h->d_pos_of_node, h->d_parent, att_of_pos, h->d_att_round, st);
		LB200_CHECK_LAUNCH(ctx);
		LB200_CUDA(ctx, cudaMemcpyAsync(&r, st, sizeof(RoundState), cudaMemcpyDeviceToHost, s));
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		if (r.max_round > count) { lb200_set_error(ctx, "bone attachments form a cycle (an attached node is an ancestor of its own parent node)"); return LB200_ERR_INVALID; }
	} while (r.changed);
	const uint32_t n_rounds = r.max_round;
	attach_keys_kernel<<<grid, HT, 0, s>>>(h->d_att_round, count, h->d_keys[0], h->d_nodes[0], st);
	LB200_CHECK_LAUNCH(ctx);
	int rc = lb200_radix_sort_pairs(ctx, s, h->d_keys[0], h->d_keys[1], h->d_nodes[0], h->d_nodes[1], &st.get()->count, count, h->sort, 0, false, nullptr);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaMemsetAsync(starts.get() + n_rounds + 1, 0xff, sizeof(uint32_t) * n_rounds, s));
	attach_records_kernel<<<grid, HT, 0, s>>>(h->d_keys[0], h->d_nodes[0], count, n_rounds, table, h->d_att_relative, h->d_pos_of_node, h->d_att_records, starts);
	LB200_CHECK_LAUNCH(ctx);
	std::vector<uint32_t> rb(2 * (size_t)n_rounds + 1);
	LB200_CUDA(ctx, cudaMemcpyAsync(rb.data(), starts, sizeof(uint32_t) * rb.size(), cudaMemcpyDeviceToHost, s));
	LB200_CUDA(ctx, cudaStreamSynchronize(s));
	h->att_round_start.assign(rb.begin(), rb.begin() + n_rounds + 1);
	h->att_round_level.resize(n_rounds);
	for (uint32_t k = 0; k < n_rounds; ++k) // the level of the round's shallowest attached node: the last level starting at or before it
		h->att_round_level[k] = (uint32_t)(std::upper_bound(h->level_start.begin(), h->level_start.end(), rb[n_rounds + 1 + k]) - h->level_start.begin()) - 1;
	h->att_rounds_valid = true;
	return LB200_OK;
}

// next stamp of a recompose; stamps restart (all cleared) when the counter wraps
int nextStamp(lb200_hierarchy* h, uint32_t* stamp) {
	if (++h->stamp == 0) {
		LB200_CUDA(h->ctx, cudaMemsetAsync(h->d_stamp, 0, sizeof(uint32_t) * h->n, h->ctx->stream));
		h->stamp = 1;
	}
	*stamp = h->stamp;
	return LB200_OK;
}

// propagate_attached's launches between the roots' flags and the moved list: the pinned propagate, then per round the attachments and the
// recompose of their subtrees
int attachedLevels(lb200_hierarchy* h) {
	lb200_ctx* ctx = h->ctx;
	cudaStream_t s = ctx->stream;
	int rc = launchLevels(h, 1,
		[&](const SmallLevels& S) { propagate_pinned_small_levels_kernel<<<1, SMALL_THREADS, 0, s>>>(S, h->d_parent, h->L, h->G, h->d_mark, h->d_pinned, h->d_flag); },
		[&](const cudaLaunchConfig_t& cfg, uint32_t begin, uint32_t end) {
			return cudaLaunchKernelEx(&cfg, propagate_pinned_level_kernel, begin, end, (const int*)h->d_parent, h->L, h->G, (const uint8_t*)h->d_mark,
				(const uint8_t*)h->d_pinned, (uint8_t*)h->d_flag);
		});
	if (rc) return rc;
	for (size_t r = 0; r + 1 < h->att_round_start.size(); ++r) {
		const uint32_t begin = h->att_round_start[r], end = h->att_round_start[r + 1];
		uint32_t stamp;
		rc = nextStamp(h, &stamp);
		if (rc) return rc;
		attach_round_kernel<<<(end - begin + HT - 1) / HT, HT, 0, s>>>(h->d_att_records, begin, end, h->d_att_systems, h->d_entity, h->d_parent, h->L, h->G,
			h->d_flag, h->d_stamp, stamp);
		LB200_CHECK_LAUNCH(ctx);
		rc = launchLevels(h, h->att_round_level[r] + 1,
			[&](const SmallLevels& S) { recompose_small_levels_kernel<<<1, SMALL_THREADS, 0, s>>>(S, h->d_parent, h->L, h->G, h->d_stamp, stamp, h->d_flag); },
			[&](const cudaLaunchConfig_t& cfg, uint32_t b, uint32_t e) {
				return cudaLaunchKernelEx(&cfg, recompose_level_kernel, b, e, (const int*)h->d_parent, h->L, h->G, (uint32_t*)h->d_stamp, stamp, (uint8_t*)h->d_flag);
			});
		if (rc) return rc;
	}
	return LB200_OK;
}

} // namespace

extern "C" {

int lb200_hierarchy_create(lb200_ctx* ctx, const int32_t* parents, uint32_t n, lb200_hierarchy** out) {
	if (!out || !parents || !n) return LB200_ERR_INVALID;
	if (!ctx) return LB200_ERR_NO_DEVICE;
	*out = nullptr;
	std::unique_ptr<lb200_hierarchy, decltype(&lb200_hierarchy_destroy)> h(new (std::nothrow) lb200_hierarchy, lb200_hierarchy_destroy);
	if (!h) return LB200_ERR_CUDA;
	h->ctx = ctx;
	const int rc = lb200_hierarchy_set_parents(h.get(), parents, n); // an empty hierarchy re-parented: every node starts as the identity
	if (rc) return rc;
	*out = h.release();
	return LB200_OK;
}

int lb200_hierarchy_set_parents(lb200_hierarchy* h, const int32_t* parents, uint32_t n) {
	if (!h || !parents || !n) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const int rc = growBuildScratch(h, n);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_parents_in, parents, sizeof(int32_t) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
	return buildTopology(h, h->d_parents_in, n, 0);
}

int lb200_hierarchy_set_parents_device(lb200_hierarchy* h, const int32_t* dev_parents, uint32_t n, uint32_t max_blocks) {
	if (!h || !dev_parents || !n) return LB200_ERR_INVALID;
	LB200_CUDA(h->ctx, cudaSetDevice(h->ctx->device));
	return buildTopology(h, dev_parents, n, max_blocks);
}

int lb200_hierarchy_get_level_order(lb200_hierarchy* h, uint32_t* order, int32_t* parent_pos, uint32_t* level_start) {
	if (!h || !order || !parent_pos || !level_start) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(order, h->d_order, sizeof(uint32_t) * (size_t)h->n, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(parent_pos, h->d_parent, sizeof(int32_t) * (size_t)h->n, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	memcpy(level_start, h->level_start.data(), sizeof(uint32_t) * h->level_start.size());
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
	LB200_CUDA(h->ctx, cudaSetDevice(h->ctx->device));
	return propagateLevels<false>(h);
}

int lb200_hierarchy_set_entities(lb200_hierarchy* h, const int32_t* entity_of_node) {
	if (!h || !entity_of_node) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_entity, entity_of_node, sizeof(int32_t) * (size_t)h->n, cudaMemcpyHostToDevice, ctx->stream));
	return LB200_OK;
}

int lb200_hierarchy_mark_moved(lb200_hierarchy* h, const uint32_t* nodes, uint32_t count) {
	if (!h || (count && !nodes)) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	for (uint32_t k = 0; k < count; ++k) {
		if (nodes[k] >= h->n) { lb200_set_error(ctx, "mark_moved: node %u out of range (%u nodes)", nodes[k], h->n); return LB200_ERR_INVALID; }
	}
	if (!count) return LB200_OK;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	uint8_t *hs, *ds; uint32_t turn;
	const int rc = stageSubset(h, sizeof(uint32_t) * (size_t)count, &hs, &ds, &turn);
	if (rc) return rc;
	memcpy(hs, nodes, sizeof(uint32_t) * (size_t)count);
	LB200_CUDA(ctx, cudaMemcpyAsync(ds, hs, sizeof(uint32_t) * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
	mark_nodes_kernel<<<(count + HT - 1) / HT, HT, 0, ctx->stream>>>((const uint32_t*)ds, count, h->d_pos_of_node, h->d_mark);
	LB200_CUDA(ctx, cudaEventRecord(h->subset_done[turn], ctx->stream));
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

int lb200_hierarchy_propagate_moved(lb200_hierarchy* h, const float* bounding_radius, lb200_hierarchy_moved* out, uint32_t* out_count) {
	if (!h || !out) return LB200_ERR_INVALID;
	lb200_range range("transform hierarchy + moved list"); // World::transformEntity, world.cpp:255-282, with its `transformed` fan-out
	LB200_CUDA(h->ctx, cudaSetDevice(h->ctx->device));
	return movedFrame(h, bounding_radius, out, out_count, [&] { return propagateLevels<true>(h); });
}

int lb200_hierarchy_set_attachments(lb200_hierarchy* h, uint32_t n, const uint32_t* attached, const uint32_t* parent, const uint32_t* system,
	const uint32_t* instance, const uint32_t* bone, const float* relative7)
{
	if (!h || (n && (!attached || !parent || !system || !instance || !bone || !relative7))) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	// everything the call may refuse or fail on comes before the table is replaced
	std::vector<uint8_t> seen;
	std::vector<lb200_hierarchy::SlotUse> slots;
	uint32_t max_node = 0;
	try {
		seen.assign(h->n, 0);
		slots.reserve(n);
		for (uint32_t k = 0; k < n; ++k) {
			if (attached[k] >= h->n || parent[k] >= h->n) { lb200_set_error(ctx, "attachment %u: node %u / %u out of range (%u nodes)", k, attached[k], parent[k], h->n); return LB200_ERR_INVALID; }
			if (attached[k] == parent[k]) { lb200_set_error(ctx, "attachment %u: node %u attached to itself", k, attached[k]); return LB200_ERR_INVALID; }
			if (seen[attached[k]]++) { lb200_set_error(ctx, "attachment %u: node %u is attached twice", k, attached[k]); return LB200_ERR_INVALID; }
			max_node = std::max(max_node, std::max(attached[k], parent[k]));
			slots.push_back({system[k], instance[k], bone[k]});
		}
	} catch (const std::bad_alloc&) {
		lb200_set_error(ctx, "set_attachments: out of host memory");
		return LB200_ERR_CUDA;
	}
	// one entry per slot with its largest instance and bone: sort by slot, then fold each run into its first entry
	std::sort(slots.begin(), slots.end(), [](const lb200_hierarchy::SlotUse& a, const lb200_hierarchy::SlotUse& b) { return a.slot < b.slot; });
	size_t distinct = 0;
	for (size_t k = 0; k < slots.size(); ++k) {
		if (distinct && slots[distinct - 1].slot == slots[k].slot) {
			slots[distinct - 1].max_instance = std::max(slots[distinct - 1].max_instance, slots[k].max_instance);
			slots[distinct - 1].max_bone = std::max(slots[distinct - 1].max_bone, slots[k].max_bone);
		}
		else slots[distinct++] = slots[k];
	}
	slots.resize(distinct);
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	DeviceArray<uint32_t> table; DeviceArray<float> relative;
	if (n) {
		LB200_CUDA(ctx, table.alloc(5 * (size_t)n));
		LB200_CUDA(ctx, relative.alloc(7 * (size_t)n));
		const uint32_t* cols[5] = {attached, parent, system, instance, bone};
		for (int c = 0; c < 5; ++c) LB200_CUDA(ctx, cudaMemcpyAsync(table.get() + (size_t)c * n, cols[c], sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
		LB200_CUDA(ctx, cudaMemcpyAsync(relative, relative7, sizeof(float) * 7 * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // the old table may still be read by the stream
	h->d_att_table = std::move(table);
	h->d_att_relative = std::move(relative);
	h->att_count = n;
	h->att_max_node = max_node;
	std::swap(h->att_slots, slots);
	h->att_rounds_valid = false;
	h->att_round_start.clear();
	h->att_round_level.clear();
	return LB200_OK;
}

int lb200_hierarchy_propagate_attached(lb200_hierarchy* h, lb200_animation* const* systems, const uint8_t* posed, uint32_t n_systems,
	const float* bounding_radius, lb200_hierarchy_moved* out, uint32_t* out_count)
{
	if (!h || !out || (n_systems && !systems)) return LB200_ERR_INVALID;
	lb200_range range("transform hierarchy + bone attachments + moved list"); // World::setTransform, world.cpp:337-342 + onModelInstanceMoved, render_module.cpp:1544-1566
	lb200_ctx* ctx = h->ctx;
	const uint32_t count = h->att_count;
	if (!count) { // propagate_moved, whatever systems are passed
		LB200_CUDA(ctx, cudaSetDevice(ctx->device));
		return movedFrame(h, bounding_radius, out, out_count, [&] { return propagateLevels<true>(h); });
	}
	if (h->att_max_node >= h->n) {
		lb200_set_error(ctx, "propagate_attached: the attachment table names node %u, the hierarchy has %u nodes (set the attachments again)", h->att_max_node, h->n);
		return LB200_ERR_STATE;
	}
	if (h->att_slots.back().slot >= n_systems) {
		lb200_set_error(ctx, "propagate_attached: the attachment table names system slot %u, %u systems given", h->att_slots.back().slot, n_systems);
		return LB200_ERR_INVALID;
	}
	h->att_systems.resize(n_systems);
	const lb200_hierarchy::SlotUse* use = h->att_slots.data(); // the next slot the table names (all of them are < n_systems)
	for (uint32_t k = 0; k < n_systems; ++k) {
		AnimationPoses p;
		if (!systems[k]) { lb200_set_error(ctx, "propagate_attached: system %u is NULL", k); return LB200_ERR_STATE; }
		if (lb200_animation_internal_poses(systems[k], &p)) { lb200_set_error(ctx, "propagate_attached: system %u has no absolute poses (update with LB200_PALETTE_POSE)", k); return LB200_ERR_STATE; }
		if (p.ctx != ctx) { lb200_set_error(ctx, "propagate_attached: system %u belongs to another context", k); return LB200_ERR_STATE; }
		if (use != h->att_slots.data() + h->att_slots.size() && use->slot == k) {
			if (use->max_instance >= p.n_instances || use->max_bone >= p.bone_count) {
				lb200_set_error(ctx, "propagate_attached: system %u: instance %u / bone %u out of range (%u instances, %u bones)", k, use->max_instance, use->max_bone,
					p.n_instances, p.bone_count);
				return LB200_ERR_INVALID;
			}
			++use;
		}
		h->att_systems[k] = AttachSystem{p.pos, p.rot, p.bone_count, posed ? (uint32_t)(posed[k] != 0) : 1u};
	}
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!h->att_rounds_valid) {
		const int rc = buildRounds(h);
		if (rc) return rc;
	}
	if (h->d_att_systems.size() < n_systems) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
		LB200_CUDA(ctx, h->d_att_systems.alloc(n_systems));
	}
	LB200_CUDA(ctx, cudaMemcpyAsync(h->d_att_systems, h->att_systems.data(), sizeof(AttachSystem) * n_systems, cudaMemcpyHostToDevice, ctx->stream));
	return movedFrame(h, bounding_radius, out, out_count, [&] { return attachedLevels(h); });
}

int lb200_hierarchy_get_attachment_rounds(lb200_hierarchy* h, uint32_t* rounds, uint32_t* n_rounds) {
	if (!h || !n_rounds) return LB200_ERR_INVALID;
	lb200_ctx* ctx = h->ctx;
	if (h->att_round_start.empty()) { lb200_set_error(ctx, "get_attachment_rounds: no rounds built since the last set_attachments"); return LB200_ERR_STATE; }
	*n_rounds = (uint32_t)h->att_round_start.size() - 1;
	if (rounds) {
		LB200_CUDA(ctx, cudaSetDevice(ctx->device));
		LB200_CUDA(ctx, cudaMemcpyAsync(rounds, h->d_att_round, sizeof(uint32_t) * h->att_count, cudaMemcpyDeviceToHost, ctx->stream));
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
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
	const size_t tr_off = (sizeof(uint32_t) * (size_t)count + 15) & ~(size_t)15;
	uint8_t *hs, *ds; uint32_t turn;
	const int rc = stageSubset(h, tr_off + sizeof(lb200_transform) * (size_t)count, &hs, &ds, &turn);
	if (rc) return rc;
	memcpy(hs, nodes, sizeof(uint32_t) * (size_t)count);
	memcpy(hs + tr_off, values, sizeof(lb200_transform) * (size_t)count);
	LB200_CUDA(ctx, cudaMemcpyAsync(ds, hs, tr_off + sizeof(lb200_transform) * (size_t)count, cudaMemcpyHostToDevice, ctx->stream));
	scatter_transforms_kernel<<<(count + HT - 1) / HT, HT, 0, ctx->stream>>>((const uint32_t*)ds, (const lb200_transform*)(ds + tr_off), count, h->d_pos_of_node,
		globals ? h->G : h->L, h->d_mark);
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
