// Consumer of the visible list on the device (SURVEY.md 8f N1): PipelineImpl::createSortKeys (src/renderer/pipeline.cpp:3789-4018) —
// LOD selection with its smoothing state, sort keys / sort values (:53-143), auto-instancing groups + their instance data (:452-523,
// :3958-4016) — followed by PipelineImpl::radixSort (:4020-4144, radix_sort.cu).  The ids the cull kernel compacted never leave HBM: this stage reads them
// where they lie (lb200_culling's per-type segments + counters) and leaves sorted keys / values and per-group instance data in HBM; the
// host reads back a handful of counters.
//
// Data layout: the walk over the visible list is a random gather by entity id, so everything createSortKeys reads per renderable lives in
// ONE 64-byte record per entity (one DRAM burst): sector 0 = position (fp64) + model index / flags + ModelInstance::lod — all a static
// mesh needs for its LOD and its keys; sector 1 = rotation, scale, Pose::frame — what the instance data adds.  (Round-2 profile of the
// SoA form: 1.33 GB of DRAM reads per 1.5 M visible meshes, six 32-byte sectors per renderable and pass; profiles/r2_B_sortkeys_ncu.txt.)
//
//   create_keys_kernel one cooperative launch (grid = what is co-resident) for one view (create_keys) or every view of a cull_views call
//   (create_keys_views), the views one after the other; per view one thread per visible renderable, grid-stride:
//     pass 1  MESH: sector 0 -> squared distance to the LOD reference point in fp64 -> float, Model::getLODMeshIndices (model.h:173-179),
//             the lod smoothing of :3926-3941 (ModelInstance::lod updated in place), the pose claim (the compare-exchange on Pose::frame,
//             :3890-3897); what the renderable will emit is COUNTED (keys, pose entries per thread; instances per auto-instancer group
//             per block in shared memory) and its decision is stashed as one word.  One block-wide scan + one global atomic per counter
//             and block, one global atomic per (block, group) claim the block's output ranges.
//     -- grid barrier --
//             exclusive scan of the group totals (every block for itself, <= 8192 groups; one block + a second barrier beyond that);
//             block 0 also writes group_offset and one key/value per non-empty group (:3958-3969).
//     pass 2  the stashed decisions are replayed: keys / values (:53-143) at the claimed slots, pose / dirty lists, and for every
//             auto-instanced mesh the 48 bytes of instance data (:3990-4008) straight at group_offset + the block's slice + rank.
// The reference runs createSortKeys on every job worker with one AutoInstancer per worker; this is the one-instancer form (instancer
// index 0 in the group values), every mesh's instances in one group.  Order inside a group and among equal keys is unspecified in the
// reference too (it depends on the workers' race for result pages).
#include "grid_barrier.cuh"
#include "lb200_internal.h"
#include "lb200_math.cuh"

#include <algorithm>
#include <memory>
#include <stdio.h>
#include <stdlib.h>
#include <new>
#include <vector>

namespace {

using namespace lb;

constexpr int SK_THREADS = 256;
constexpr uint64_t SORT_KEY_BUCKET_SHIFT = 56;                 // pipeline.cpp:70-77
constexpr uint64_t SORT_KEY_INSTANCED_FLAG = (uint64_t)1 << 55;
constexpr uint64_t SORT_VALUE_INSTANCER_SHIFT = 16;
constexpr uint64_t SORT_VALUE_MESH_IDX_SHIFT = 40;
constexpr uint64_t SORT_VALUE_TYPE_SHIFT = 32;
enum { DRAW_MESH = 0, DRAW_AUTOINSTANCED = 1, DRAW_SKINNED = 2, DRAW_DECAL = 3, DRAW_CURVE_DECAL = 4 }; // :41-51
enum { RT_MESH = 0, RT_DECAL = 1, RT_LOCAL_LIGHT = 2, RT_CURVE_DECAL = 3 };                                // render_module.h:293-301
enum { CNT_KEYS = 0, CNT_RECS, CNT_INST, CNT_POSE, CNT_DIRTY, CNT_WORDS = 8 };

constexpr uint32_t SK_MAX_VIEWS = LB200_CULL_MAX_VIEWS;
// One view's lb200_sk_view without its tables (those are in EmitArgs::tables, SK_TABLE_WORDS per view)
struct ViewScalars {
	double camera_pos[3], lod_ref_point[3];
	float time_delta, lod_multiplier;
	uint32_t frame_number, is_shadow;
};
static_assert(sizeof(ViewScalars) == 64, "one view's scalars");
constexpr uint32_t SK_TABLE_WORDS = 256 + 64; // bucket_map (256 words) then layer_to_bucket (256 bytes): 1,280 B per view

// Where one view's outputs go (counts: CNT_WORDS counters; group tables: n_groups each)
struct ViewOut {
	uint64_t* keys; uint64_t* values; uint32_t* counts;
	uint32_t* group_count; uint32_t* group_offset; uint32_t* group_cursor;
	uint64_t* group_renderables; float4* instance_data;
	uint32_t* pose_list; uint32_t* dirty_list;
};

struct EmitParams {
	ViewScalars view[SK_MAX_VIEWS]; // views [0, n_views) of the launch
	ViewOut out[SK_MAX_VIEWS];
	uint32_t n_views;
	uint32_t type_base[4]; // offsets of the MESH / DECAL / LOCAL_LIGHT / CURVE_DECAL segments inside every view's ids
	uint32_t id_stride, counter_stride; // view v's ids at visible + v * id_stride, its cull counters at cull_counters + v * counter_stride
	uint32_t cap_keys, cap_recs, cap_pose, cap_dirty;
	uint32_t prefetch_ahead; // records requested into L2 this many grid strides ahead of their use (0 = off; LB200_SK_PREFETCH, default 0)
};

// :57-60
__device__ __forceinline__ uint32_t float_flip(uint32_t bits) { return bits ^ ((uint32_t)(-(int32_t)(bits >> 31)) | 0x80000000u); }
__device__ __forceinline__ uint64_t sext(int32_t e) { return (uint64_t)(int64_t)e; } // EntityPtr::index is an i32: `entity.index | u64` sign-extends

// The same counter for lanes of a warp that add to the same auto-instancer group: one atomic per (warp, group).
__device__ __forceinline__ uint32_t warp_claim_keyed(uint32_t* counters, uint32_t key) {
	const uint32_t active = __activemask();
	const uint32_t lane = threadIdx.x & 31u;
	const uint32_t peers = __match_any_sync(active, key);
	const int leader = __ffs((int)peers) - 1;
	uint32_t base = 0;
	if ((int)lane == leader) base = atomicAdd(&counters[key], (uint32_t)__popc(peers));
	base = __shfl_sync(peers, base, leader);
	return base + (uint32_t)__popc(peers & ((1u << lane) - 1u));
}

struct EmitArgs {
	SkEntity* ent; const uint32_t* __restrict__ decal_sort_key; const uint8_t* __restrict__ decal_layer;
	const lb200_sk_model* __restrict__ models; const lb200_sk_mesh* __restrict__ meshes; const uint32_t* __restrict__ tables;
	const uint8_t* __restrict__ group_layer;
	uint32_t* __restrict__ stash; float4* __restrict__ stash4; uint32_t stash_stride;
	GridBar* bar;
};

// the 64-byte model record / 16-byte mesh record through the read-only path, into registers
__device__ __forceinline__ lb200_sk_model load_model(const lb200_sk_model* p) {
	union { lb200_sk_model m; int4 q[4]; } u;
	const int4* s = reinterpret_cast<const int4*>(p);
	u.q[0] = __ldg(s); u.q[1] = __ldg(s + 1); u.q[2] = __ldg(s + 2); u.q[3] = __ldg(s + 3);
	return u.m;
}
__device__ __forceinline__ lb200_sk_mesh load_mesh(const lb200_sk_mesh* p) {
	union { lb200_sk_mesh m; int4 q; } u;
	u.q = __ldg(reinterpret_cast<const int4*>(p));
	return u.m;
}
__device__ __forceinline__ int lod_from(const lb200_sk_model& m, int l) { return l == 0 ? m.lod_from[0] : l == 1 ? m.lod_from[1] : l == 2 ? m.lod_from[2] : l == 3 ? m.lod_from[3] : m.lod_from[4]; }
__device__ __forceinline__ int lod_to(const lb200_sk_model& m, int l) { return l == 0 ? m.lod_to[0] : l == 1 ? m.lod_to[1] : l == 2 ? m.lod_to[2] : l == 3 ? m.lod_to[3] : m.lod_to[4]; }

// what pass 1 decided for a MESH renderable, one word: model (24) | first lod (3) | second lod too (1) | MOVED (1) | pose claimed here (1) | dirty (1)
constexpr uint32_t CODE_MODEL_MASK = 0xffffffu;
constexpr int CODE_LOD_SHIFT = 24;
constexpr uint32_t CODE_TWO = 1u << 27, CODE_MOVED = 1u << 28, CODE_POSE = 1u << 29, CODE_DIRTY = 1u << 30;

struct Counts { uint32_t k, r, p; };

// What one mesh of a MESH renderable turns into (create_key, :3883-3924), as flags instead of branches: lanes of a warp hold different
// models, so every branch here used to run with a handful of lanes (round-2 profile: 11.8 active threads per instruction on average).
//   skinned                     -> key (mesh sort key) + the instance joins the pose list once per frame
//   MOVED and not a shadow view -> key (mesh sort key)
//   bucket < 0xff               -> an instance of the mesh's auto-instancer group
//   bucket < 0xffff             -> depth-sorted key
struct MeshKind { bool skinned, key, inst, depth; };
__device__ __forceinline__ MeshKind mesh_kind(const lb200_sk_mesh& mm, uint32_t bucket, bool moved_not_shadow) {
	MeshKind k;
	k.skinned = mm.skinned != 0;
	const bool plain = k.skinned || moved_not_shadow;
	k.inst = !plain && bucket < 0xffu;
	k.depth = !plain && bucket >= 0xffu && bucket < 0xffffu;
	k.key = plain || k.depth;
	return k;
}

// MESH renderable, pass 1 (:3868-3956): LOD selection + smoothing state + pose claim; counts what pass 2 will write
__device__ __forceinline__ uint32_t mesh_count(const ViewScalars& W, const ViewOut& O, const EmitArgs& A, const uint32_t* s_bucket_map, uint32_t* s_grp, float lod_multiplier_rcp, int32_t e, uint32_t i, Counts& c) {
	SkEntity* rec = A.ent + e;
	// the whole record, one 64-byte burst (coherent loads: this kernel writes lod / pose_frame)
	const int4* rp = reinterpret_cast<const int4*>(rec);
	const int4 q0 = __ldcg(rp), q1 = __ldcg(rp + 1), q2 = __ldcg(rp + 2), q3 = __ldcg(rp + 3); // L2 only: a record is touched once, L1 stays with the model / mesh tables
	const double px = __hiloint2double(q0.y, q0.x), py = __hiloint2double(q0.w, q0.z), pz = __hiloint2double(q1.y, q1.x);
	const uint32_t model_flags = (uint32_t)q1.z;
	float cur = __int_as_float(q1.w);
	const uint32_t model_idx = model_flags & CODE_MODEL_MASK, fl = model_flags >> 24;
	if (fl & LB200_SK_DIRTY) return CODE_DIRTY | model_idx; // mi.dirty, :3878-3881
	const lb200_sk_model model = load_model(A.models + model_idx);
	const double dx = LB_DSUB(px, W.lod_ref_point[0]), dy = LB_DSUB(py, W.lod_ref_point[1]), dz = LB_DSUB(pz, W.lod_ref_point[2]);
	const float squared_length = (float)LB_DADD(LB_DADD(LB_DMUL(dx, dx), LB_DMUL(dy, dy)), LB_DMUL(dz, dz)); // squaredLength(DVec3), math.cpp:397
	const float sd = LB_FMUL(squared_length, lod_multiplier_rcp);
	const uint32_t lod_idx = sd < model.lod_distances[0] ? 0u : sd < model.lod_distances[1] ? 1u : sd < model.lod_distances[2] ? 2u : sd < model.lod_distances[3] ? 3u : 4u;
	const bool is_shadow = W.is_shadow != 0;
	uint32_t lod0 = lod_idx;
	bool two = false;
	if (cur != (float)lod_idx) { // :3926-3941
		const float d = LB_FSUB((float)lod_idx, cur);
		const float ad = fabsf(d);
		if (ad <= W.time_delta) cur = (float)lod_idx;
		else {
			if (!is_shadow) cur = LB_FADD(cur, LB_FMUL(LB_FDIV(d, ad), W.time_delta));
			lod0 = (uint32_t)cur;
			two = lod0 < 3;
		}
		rec->lod = cur;
	}
	// what pass 2 writes per auto-instanced mesh (:3990-4008) or depth-sorted key (:3915-3922), stashed next to the decision in arrays indexed
	// like the visible list: pass 2 reads them coalesced and never touches the record again
	const double rx = LB_DSUB(px, W.camera_pos[0]), ry = LB_DSUB(py, W.camera_pos[1]), rz = LB_DSUB(pz, W.camera_pos[2]);
	const uint32_t depth_bits = float_flip(__float_as_uint((float)LB_DADD(LB_DADD(LB_DMUL(rx, rx), LB_DMUL(ry, ry)), LB_DMUL(rz, rz))));
	__stcs(A.stash4 + i, make_float4(__int_as_float(q2.x), __int_as_float(q2.y), __int_as_float(q2.z), __int_as_float(q2.w)));                 // rot
	__stcs(A.stash4 + A.stash_stride + i, make_float4((float)rx, (float)ry, (float)rz, __uint_as_float(depth_bits)));                            // Vec3(tr.pos - camera_pos), depth key
	__stcs(A.stash4 + 2 * (size_t)A.stash_stride + i, make_float4(__int_as_float(q3.x), __int_as_float(q3.y), __int_as_float(q3.z), cur));    // scale, lod after the update
	const bool moved_not_shadow = (fl & LB200_SK_MOVED) && !is_shadow;
	uint32_t code = model_idx | (lod0 << CODE_LOD_SHIFT) | (two ? CODE_TWO : 0u) | ((fl & LB200_SK_MOVED) ? CODE_MOVED : 0u);
	// the meshes of lod0 and, while the lod blends over, of lod0 + 1: one loop over both ranges
	const int from0 = lod_from(model, (int)lod0), to0 = lod_to(model, (int)lod0);
	const int from1 = two ? lod_from(model, (int)lod0 + 1) : 0, to1 = two ? lod_to(model, (int)lod0 + 1) : -1;
	const int n0 = max(to0 - from0 + 1, 0), n_all = n0 + max(to1 - from1 + 1, 0);
	bool any_skinned = false;
	for (int j = 0; j < n_all; ++j) {
		const int mesh_idx = j < n0 ? from0 + j : from1 + (j - n0);
		const lb200_sk_mesh mm = load_mesh(A.meshes + model.mesh_base + (uint32_t)mesh_idx);
		const MeshKind kind = mesh_kind(mm, s_bucket_map[mm.layer], moved_not_shadow);
		any_skinned |= kind.skinned;
		c.k += kind.key ? 1u : 0u;
		if (kind.inst) { // AutoInstancer::add, :3913-3914
			if (s_grp) atomicAdd(&s_grp[mm.sort_key], 1u);
			else warp_claim_keyed(O.group_count, mm.sort_key);
		}
	}
	// once per instance and frame the palette has to be built (PoseProcessor::push; the compare-exchange on Pose::frame of :3890-3897 —
	// one thread owns the instance within a view)
	if (any_skinned && (uint32_t)q3.w != W.frame_number) { rec->pose_frame = W.frame_number; code |= CODE_POSE; ++c.p; }
	return code;
}

__device__ __forceinline__ void push_key(const EmitParams& P, const ViewOut& O, uint32_t& slot, uint64_t key, uint64_t value) {
	if (slot < P.cap_keys) { O.keys[slot] = key; O.values[slot] = value; }
	++slot;
}

// MESH renderable, pass 2: replay of the stashed decision, writes
__device__ __forceinline__ void mesh_write(const EmitParams& P, const ViewScalars& W, const ViewOut& O, const EmitArgs& A, const uint32_t* s_bucket_map, uint32_t* s_grp, int32_t e, uint32_t i, uint32_t code, uint32_t& k, uint32_t& p) {
	if (code & CODE_DIRTY) { // queueMaterialOverrideRefresh (rare: its own atomic)
		const uint32_t slot = atomicAdd(&O.counts[CNT_DIRTY], 1u);
		if (slot < P.cap_dirty) O.dirty_list[slot] = (uint32_t)e;
		return;
	}
	const lb200_sk_model model = load_model(A.models + (code & CODE_MODEL_MASK));
	const bool moved_not_shadow = (code & CODE_MOVED) && W.is_shadow == 0;
	const uint32_t lod0 = (code >> CODE_LOD_SHIFT) & 7u;
	const bool two = (code & CODE_TWO) != 0;
	if (code & CODE_POSE) {
		if (p < P.cap_pose) O.pose_list[p] = (uint32_t)e;
		++p;
	}
	const float4 s_rot = __ldcs(A.stash4 + i), s_pos = __ldcs(A.stash4 + A.stash_stride + i), s_scl = __ldcs(A.stash4 + 2 * (size_t)A.stash_stride + i); // coalesced, read once
	const int from0 = lod_from(model, (int)lod0), to0 = lod_to(model, (int)lod0);
	const int from1 = two ? lod_from(model, (int)lod0 + 1) : 0, to1 = two ? lod_to(model, (int)lod0 + 1) : -1;
	const int n0 = max(to0 - from0 + 1, 0), n_all = n0 + max(to1 - from1 + 1, 0);
	for (int j = 0; j < n_all; ++j) {
		const int mesh_idx = j < n0 ? from0 + j : from1 + (j - n0);
		const lb200_sk_mesh mm = load_mesh(A.meshes + model.mesh_base + (uint32_t)mesh_idx);
		const uint32_t bucket = s_bucket_map[mm.layer];
		const MeshKind kind = mesh_kind(mm, bucket, moved_not_shadow);
		const uint64_t mesh_value = sext(e) | ((uint64_t)mesh_idx << SORT_VALUE_MESH_IDX_SHIFT);
		if (kind.key) {
			const uint64_t low = kind.depth ? (uint64_t)__float_as_uint(s_pos.w) : (uint64_t)mm.sort_key;
			push_key(P, O, k, low | ((uint64_t)(uint8_t)bucket << SORT_KEY_BUCKET_SHIFT), mesh_value | ((uint64_t)(kind.skinned ? DRAW_SKINNED : DRAW_MESH) << SORT_VALUE_TYPE_SHIFT));
		}
		if (kind.inst) { // instance data of the auto-instanced mesh, :3990-4008, at the group's offset + this block's slice + rank
			const uint32_t at = s_grp ? atomicAdd(&s_grp[mm.sort_key], 1u) : warp_claim_keyed(O.group_cursor, mm.sort_key);
			if (at < P.cap_recs) {
				__stcs(reinterpret_cast<unsigned long long*>(O.group_renderables) + at, (unsigned long long)mesh_value);
				float4* dst = O.instance_data + (size_t)at * 3;
				__stcs(dst, s_rot);
				__stcs(dst + 1, make_float4(s_pos.x, s_pos.y, s_pos.z, LB_FSUB(s_scl.w, mm.lod))); // camera-relative position, lod - mesh.lod
				__stcs(dst + 2, make_float4(s_scl.x, s_scl.y, s_scl.z, __uint_as_float(mm.material_index)));
			}
		}
	}
}

// block-wide exclusive scan of one value per thread (SK_THREADS threads); returns the thread's prefix, *total = the block's sum
__device__ __forceinline__ uint32_t block_exclusive_scan(uint32_t v, uint32_t* s_warp /* SK_THREADS / 32 */, uint32_t* total) {
	const uint32_t lane = threadIdx.x & 31u, warp = threadIdx.x >> 5;
	uint32_t x = v;
#pragma unroll
	for (int d = 1; d < 32; d <<= 1) {
		const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
		if (lane >= (uint32_t)d) x += y;
	}
	if (lane == 31) s_warp[warp] = x;
	__syncthreads();
	uint32_t before = 0, sum = 0;
#pragma unroll
	for (int w = 0; w < SK_THREADS / 32; ++w) { if ((uint32_t)w < warp) before += s_warp[w]; sum += s_warp[w]; }
	__syncthreads();
	*total = sum;
	return before + x - v;
}

constexpr uint32_t SK_SMEM_GROUPS = 8192; // group counters a block keeps in shared memory (32 KB)

__device__ __forceinline__ void prefetch_l2(const void* p) { asm volatile("prefetch.global.L2 [%0];" ::"l"(p)); }
// entity id at index i of the three segments seen as one index space [MESH | DECAL | CURVE_DECAL]
__device__ __forceinline__ uint32_t visible_at(const EmitParams& P, const uint32_t* __restrict__ visible, uint32_t i, uint32_t n_mesh, uint32_t n_decal) {
	return i < n_mesh ? visible[P.type_base[RT_MESH] + i] : i < n_mesh + n_decal ? visible[P.type_base[RT_DECAL] + (i - n_mesh)] : visible[P.type_base[RT_CURVE_DECAL] + (i - n_mesh - n_decal)];
}

// Views [0, P.n_views) one after the other, each exactly as a launch of its own would run it: pass 1, grid barrier, group scan (+ barrier
// with the group cursors in HBM), pass 2.  A later view sees the lod / pose_frame stores of the earlier ones through the barrier behind
// their pass 1 (records are read with ld.cg, never from L1).  No grid barrier separates a view's pass 2 from the next view's pass 1: pass 2
// reads no record, every view has its own counters, group tables and outputs, and stash slot i is written (pass 1) and read (pass 2) by
// the thread that owns index i in every view, the grid stride being the same.
__global__ void __launch_bounds__(SK_THREADS, 4) create_keys_kernel(const __grid_constant__ EmitParams P, const uint32_t* __restrict__ visible_all,
	const uint32_t* __restrict__ cull_counters_all, EmitArgs A, uint32_t n_groups)
{
	extern __shared__ uint32_t s_grp_mem[];
	__shared__ uint32_t s_warp[SK_THREADS / 32];
	__shared__ uint32_t s_base[2];
	__shared__ uint32_t s_carry;
	__shared__ uint32_t s_bucket_map[256];
	for (uint32_t v = 0; v < P.n_views; ++v) { // v is all the loop carries: what follows is derived from it and the parameters
		uint32_t* s_grp = n_groups <= SK_SMEM_GROUPS ? s_grp_mem : nullptr;
		const uint32_t stride = gridDim.x * SK_THREADS;
		uint32_t barriers_passed = v * (s_grp ? 1u : 2u); // the earlier views' grid barriers
		const ViewScalars& W = P.view[v];
		const ViewOut& O = P.out[v];
		const uint32_t* __restrict__ visible = visible_all + (size_t)v * P.id_stride;
		const uint32_t* __restrict__ cull_counters = cull_counters_all + (size_t)v * P.counter_stride;
		__syncthreads(); // the previous view's pass 2 is done with s_bucket_map / s_grp in this block
		s_bucket_map[threadIdx.x] = __ldg(A.tables + (size_t)v * SK_TABLE_WORDS + threadIdx.x); // SK_THREADS == 256
		if (s_grp) for (uint32_t g = threadIdx.x; g < n_groups; g += SK_THREADS) s_grp[g] = 0;
		__syncthreads();
		// the three segments as one index space: [MESH | DECAL | CURVE_DECAL]
		const uint32_t n_mesh = __ldg(cull_counters + RT_MESH), n_decal = __ldg(cull_counters + RT_DECAL), n_curve = __ldg(cull_counters + RT_CURVE_DECAL);
		const uint32_t n_all = n_mesh + n_decal + n_curve;
		const float lod_multiplier_rcp = LB_FDIV(1.0f, W.lod_multiplier); // :3798-3799

		// ---- pass 1: decide + count ----
		// The walk is a random gather by entity id: the id of the thread's NEXT renderable is read one iteration ahead and its record is
		// requested into L2 while the current one is processed (a dependent chain id -> record -> model -> mesh per renderable otherwise).
		Counts c = {0u, 0u, 0u};
		{
			uint32_t i = blockIdx.x * SK_THREADS + threadIdx.x;
			uint32_t e = i < n_all ? visible_at(P, visible, i, n_mesh, n_decal) : 0u;
			const uint32_t ahead = P.prefetch_ahead * stride;
			for (; i < n_all; i += stride) {
				const uint32_t i_next = i + stride;
				uint32_t e_next = 0;
				if (i_next < n_all) e_next = visible_at(P, visible, i_next, n_mesh, n_decal);
				if (ahead) {
					const uint32_t i_pf = i + ahead;
					if (i_pf < n_all) {
						const uint32_t e_pf = ahead == stride ? e_next : visible_at(P, visible, i_pf, n_mesh, n_decal);
						if (i_pf < n_mesh) { prefetch_l2(A.ent + e_pf); prefetch_l2(reinterpret_cast<const char*>(A.ent + e_pf) + 32); }
						else { prefetch_l2(A.decal_layer + e_pf); prefetch_l2(A.decal_sort_key + e_pf); }
					}
				}
				if (i < n_mesh) A.stash[i] = mesh_count(W, O, A, s_bucket_map, s_grp, lod_multiplier_rcp, (int32_t)e, i, c);
				else { // DECAL / CURVE_DECAL renderable (:3840-3867): one key if its layer is in the view; bucket and material sort key stashed for pass 2
					const uint32_t bucket = (uint8_t)s_bucket_map[A.decal_layer[e]];
					uint32_t key = 0;
					if (bucket < 0xff) { key = A.decal_sort_key[e]; ++c.k; }
					A.stash[i] = bucket;
					A.stash4[i].x = __uint_as_float(key);
				}
				e = e_next;
			}
		}
		uint32_t tk, tp;
		const uint32_t pk = block_exclusive_scan(c.k, s_warp, &tk);
		const uint32_t pp = block_exclusive_scan(c.p, s_warp, &tp);
		if (threadIdx.x == 0) {
			s_base[0] = tk ? atomicAdd(&O.counts[CNT_KEYS], tk) : 0u;
			s_base[1] = tp ? atomicAdd(&O.counts[CNT_POSE], tp) : 0u;
		}
		// the block's slice of every group it has instances of: count -> start inside the group
		if (s_grp) for (uint32_t g = threadIdx.x; g < n_groups; g += SK_THREADS) if (s_grp[g]) s_grp[g] = atomicAdd(&O.group_count[g], s_grp[g]);
		grid_barrier(A.bar, barriers_passed); // every block's counts are in: group totals are final; the view's lod / pose_frame stores are visible

		// ---- group offsets = exclusive scan of the group totals; block 0 publishes them and one key/value per non-empty group (:3958-3969) ----
		if (s_grp || blockIdx.x == 0) {
			const uint8_t* __restrict__ layer_to_bucket = reinterpret_cast<const uint8_t*>(A.tables + (size_t)v * SK_TABLE_WORDS + 256);
			if (threadIdx.x == 0) s_carry = 0;
			__syncthreads();
			for (uint32_t base = 0; base < n_groups; base += SK_THREADS) {
				const uint32_t g = base + threadIdx.x;
				const uint32_t cnt = g < n_groups ? __ldcg(O.group_count + g) : 0u;
				uint32_t total;
				const uint32_t carry = s_carry; // read before the scan's barriers: thread 0 moves it on behind them
				const uint32_t off = carry + block_exclusive_scan(cnt, s_warp, &total);
				if (g < n_groups) {
					if (s_grp) s_grp[g] += off; // cursor of this block inside the group, absolute
					if (blockIdx.x == 0) {
						O.group_offset[g] = off;
						if (!s_grp) O.group_cursor[g] = off;
						if (cnt) {
							const uint32_t slot = atomicAdd(&O.counts[CNT_KEYS], 1u);
							if (slot < P.cap_keys) {
								O.keys[slot] = (uint64_t)g | SORT_KEY_INSTANCED_FLAG | ((uint64_t)__ldg(layer_to_bucket + A.group_layer[g]) << SORT_KEY_BUCKET_SHIFT); // :100-102
								O.values[slot] = (uint64_t)g | ((uint64_t)0 << SORT_VALUE_INSTANCER_SHIFT) | ((uint64_t)DRAW_AUTOINSTANCED << SORT_VALUE_TYPE_SHIFT); // :141-143
							}
						}
					}
				}
				if (threadIdx.x == 0) s_carry += total;
				__syncthreads();
			}
			if (blockIdx.x == 0 && threadIdx.x == 0) { O.counts[CNT_INST] = s_carry; O.counts[CNT_RECS] = s_carry; }
		}
		if (!s_grp) grid_barrier(A.bar, barriers_passed); // more groups than fit in shared memory: everybody waits for block 0's cursors in HBM

		// ---- pass 2: write ----
		uint32_t k = s_base[0] + pk, p = s_base[1] + pp;
		{
			uint32_t i = blockIdx.x * SK_THREADS + threadIdx.x;
			uint32_t e = i < n_all ? visible_at(P, visible, i, n_mesh, n_decal) : 0u;
			for (; i < n_all; i += stride) {
				const uint32_t i_next = i + stride;
				uint32_t e_next = 0;
				if (i_next < n_all) e_next = visible_at(P, visible, i_next, n_mesh, n_decal);
				if (i < n_mesh) mesh_write(P, W, O, A, s_bucket_map, s_grp, (int32_t)e, i, A.stash[i], k, p);
				else {
					const bool curve = i >= n_mesh + n_decal;
					const uint32_t bucket = A.stash[i];
					if (bucket < 0xff) push_key(P, O, k, (uint64_t)__float_as_uint(A.stash4[i].x) | ((uint64_t)bucket << SORT_KEY_BUCKET_SHIFT),
						sext((int32_t)e) | ((uint64_t)(curve ? DRAW_CURVE_DECAL : DRAW_DECAL) << SORT_VALUE_TYPE_SHIFT));
				}
				e = e_next;
			}
		}
	}
}

// ---- per-entity records: packing what the caller hands over as arrays, unpacking the state the pass keeps ----
// Bit 7 of the record's flag byte, internal: the entity is in this frame's moved list.  ent_move_kernel sets it with MOVED, end_frame
// clears both, a spawn clears MOVED (createModelInstance) and leaves it: move -> spawn -> move lists the entity once.  createSortKeys
// reads MOVED and DIRTY only.
constexpr uint32_t FLAG_MOVED = (uint32_t)LB200_SK_MOVED << 24, FLAG_DIRTY = (uint32_t)LB200_SK_DIRTY << 24, FLAG_LISTED = 0x80u << 24;

__global__ void __launch_bounds__(256) ent_init_kernel(SkEntity* ent, uint32_t n) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	int4* r = reinterpret_cast<int4*>(ent + i);
	r[0] = r[1] = r[2] = make_int4(0, 0, 0, 0);
	r[3] = make_int4(0, 0, 0, (int)0xffffffffu); // Pose::frame = 0xffffffff: "never" (pipeline.cpp:3814)
}
__global__ void __launch_bounds__(256) ent_pack_transforms_kernel(SkEntity* ent, const lb200_transform* __restrict__ tr, uint32_t n) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const lb200_transform t = tr[i];
	SkEntity& r = ent[i];
	r.pos[0] = t.pos[0]; r.pos[1] = t.pos[1]; r.pos[2] = t.pos[2];
	r.rot[0] = t.rot[0]; r.rot[1] = t.rot[1]; r.rot[2] = t.rot[2]; r.rot[3] = t.rot[3];
	r.scale[0] = t.scale[0]; r.scale[1] = t.scale[1]; r.scale[2] = t.scale[2];
}
__global__ void __launch_bounds__(256) ent_pack_fields_kernel(SkEntity* ent, uint32_t n, const uint32_t* __restrict__ model_of, const float* __restrict__ lod,
	const uint8_t* __restrict__ flags, const uint32_t* __restrict__ pose_frame)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	SkEntity& r = ent[i];
	if (model_of || flags) {
		uint32_t mf = r.model_flags;
		if (model_of) mf = (mf & ~CODE_MODEL_MASK) | (model_of[i] & CODE_MODEL_MASK);
		if (flags) mf = (mf & CODE_MODEL_MASK) | (((uint32_t)flags[i] << 24) & ~FLAG_LISTED); // the whole flag byte, "listed" included: off
		r.model_flags = mf;
	}
	if (lod) r.lod = lod[i];
	if (pose_frame) r.pose_frame = pose_frame[i];
}
__global__ void __launch_bounds__(256) ent_unpack_state_kernel(const SkEntity* __restrict__ ent, uint32_t n, float* __restrict__ lod, uint32_t* __restrict__ pose_frame) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	lod[i] = ent[i].lod;
	pose_frame[i] = ent[i].pose_frame;
}

// RenderModuleImpl::onModelInstanceMoved (render_module.cpp:1544-1554) for a batch whose new transforms are already in HBM (e.g. bone attachments
// of this frame's poses): the record takes the transform, the instance gets ModelInstance::MOVED and joins the moved list once, and — if
// asked — the sphere CullingSystem::set needs (pos, bounding radius * max scale) is written for lb200_culling_set_many_device.
__global__ void __launch_bounds__(256) ent_move_kernel(SkEntity* ent, uint32_t max_entities, const int32_t* __restrict__ entities, const lb200_transform* __restrict__ tr, uint32_t n,
	const float* __restrict__ bounding_radius, double* __restrict__ out_pos3, float* __restrict__ out_radius, uint32_t* moved_list, uint32_t* moved_count)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const lb200_transform t = tr[i];
	if (out_pos3) { out_pos3[3 * (size_t)i] = t.pos[0]; out_pos3[3 * (size_t)i + 1] = t.pos[1]; out_pos3[3 * (size_t)i + 2] = t.pos[2]; }
	if (out_radius) out_radius[i] = LB_FMUL(bounding_radius[i], fmaxf(fmaxf(t.scale[0], t.scale[1]), t.scale[2])); // maximum(x, y, z), math.h
	const uint32_t e = (uint32_t)entities[i];
	if (e >= max_entities) return;
	SkEntity& r = ent[e];
	r.pos[0] = t.pos[0]; r.pos[1] = t.pos[1]; r.pos[2] = t.pos[2];
	r.rot[0] = t.rot[0]; r.rot[1] = t.rot[1]; r.rot[2] = t.rot[2]; r.rot[3] = t.rot[3];
	r.scale[0] = t.scale[0]; r.scale[1] = t.scale[1]; r.scale[2] = t.scale[2];
	const uint32_t before = atomicOr(&r.model_flags, FLAG_MOVED | FLAG_LISTED);
	if (!(before & (FLAG_MOVED | FLAG_LISTED))) moved_list[atomicAdd(moved_count, 1u)] = e; // m_moved_instances.push(entity), once
}

// RenderModuleImpl::endFrame (render_module.cpp:526-534): MOVED off, prev_frame_transform = the transform of this frame
__global__ void __launch_bounds__(256) ent_end_frame_kernel(SkEntity* ent, const uint32_t* __restrict__ moved_list, uint32_t* moved_count, lb200_transform* __restrict__ prev) {
	const uint32_t n = *moved_count;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint32_t e = moved_list[i];
		SkEntity& r = ent[e];
		r.model_flags &= ~(FLAG_MOVED | FLAG_LISTED);
		lb200_transform t;
		t.pos[0] = r.pos[0]; t.pos[1] = r.pos[1]; t.pos[2] = r.pos[2];
		t.rot[0] = r.rot[0]; t.rot[1] = r.rot[1]; t.rot[2] = r.rot[2]; t.rot[3] = r.rot[3];
		t.scale[0] = r.scale[0]; t.scale[1] = r.scale[1]; t.scale[2] = r.scale[2];
		prev[e] = t;
	}
}
__global__ void reset_word_kernel(uint32_t* w) { *w = 0; }

// ---- spawns: one thread per batch entry ----
// The refusal count of a spawn batch: an id outside [0, max_entity], a model index >= n_models (model_of may be null: no model check) or
// an id listed twice (the second of two entries that stamp the same entity with this batch's sequence number sees it there).
__global__ void __launch_bounds__(256) spawn_check_kernel(const int32_t* __restrict__ entities, uint32_t n, uint32_t max_entity, const uint32_t* __restrict__ model_of,
	uint32_t n_models, uint32_t* stamp, uint32_t seq, uint32_t* refused)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const int32_t e = entities[i];
	bool bad = e < 0 || (uint32_t)e > max_entity || (model_of && model_of[i] >= n_models);
	if (!bad) bad = atomicExch(&stamp[e], seq) == seq;
	if (bad) atomicAdd(refused, 1u);
}

// createModelInstance + setModel + modelLoaded (render_module.cpp:3284-3292, :3107-3148, :2911-2951) of a checked batch: the whole record
// in two 32-byte sectors of 16-byte stores, and prev_frame_transform.  Nothing when the batch was refused.
__global__ void __launch_bounds__(256) spawn_instances_kernel(SkEntity* ent, const int32_t* __restrict__ entities, const uint32_t* __restrict__ model_of,
	const lb200_transform* __restrict__ tr, const uint8_t* __restrict__ dirty, uint32_t n, const lb200_sk_model* __restrict__ models, lb200_transform* __restrict__ prev,
	const uint32_t* __restrict__ refused)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n || *refused) return;
	const uint32_t e = (uint32_t)entities[i], m = model_of[i];
	const lb200_transform t = tr[i];
	float lod = 4.0f; // ModelInstance::lod (render_module.h:221) unless a LOD 3 .. 0 has meshes (modelLoaded, :2942-2948)
	for (int l = 3; l >= 0; --l) {
		if (__ldg(&models[m].lod_to[l]) != -1) { lod = (float)l; break; }
	}
	int4* r = reinterpret_cast<int4*>(ent + e);
	// VALID | ENABLED (:3290): MOVED off; dirty = the instance has a material override (:2950); "listed" stays as it was
	const uint32_t mf = (m & CODE_MODEL_MASK) | (r[1].z & FLAG_LISTED) | (dirty && dirty[i] ? FLAG_DIRTY : 0u);
	r[0] = make_int4(__double2loint(t.pos[0]), __double2hiint(t.pos[0]), __double2loint(t.pos[1]), __double2hiint(t.pos[1]));
	r[1] = make_int4(__double2loint(t.pos[2]), __double2hiint(t.pos[2]), (int)mf, __float_as_int(lod));
	r[2] = make_int4(__float_as_int(t.rot[0]), __float_as_int(t.rot[1]), __float_as_int(t.rot[2]), __float_as_int(t.rot[3]));
	r[3] = make_int4(__float_as_int(t.scale[0]), __float_as_int(t.scale[1]), __float_as_int(t.scale[2]), (int)0xffffffffu); // a new Pose: frame "never" (pose.h:29)
	prev[e] = t; // setModel, :3109
}

// createDecal / createCurveDecal + updateDecalInfo of a checked batch: what createSortKeys reads of a decal (pipeline.cpp:3841-3867)
__global__ void __launch_bounds__(256) spawn_decals_kernel(uint32_t* decal_sort_key, uint8_t* decal_layer, const int32_t* __restrict__ entities, const uint32_t* __restrict__ sort_key,
	const uint8_t* __restrict__ layer, uint32_t n, const uint32_t* __restrict__ refused)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n || *refused) return;
	const uint32_t e = (uint32_t)entities[i];
	decal_sort_key[e] = sort_key[i];
	decal_layer[e] = layer[i];
}

// mi.dirty = false of refreshMaterialOverrides (pipeline.cpp:3685-3721); ids outside the records are skipped
__global__ void __launch_bounds__(256) clear_dirty_kernel(SkEntity* ent, uint32_t max_entities, const int32_t* __restrict__ entities, uint32_t n) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const uint32_t e = (uint32_t)entities[i];
	if (e < max_entities) atomicAnd(&ent[e].model_flags, ~FLAG_DIRTY);
}

} // namespace

constexpr uint32_t NO_MODEL = 0xffffffffu;
constexpr uint32_t SK_TABLE_SLOTS = 4; // pinned staging slots of the view tables: a copy waits for the one SK_TABLE_SLOTS copies before it

namespace {
// What create_keys leaves in HBM for n views: view v's part of each array at + v x its per-view size (EmitArgs).  The plain create_keys
// writes a set of one view, create_keys_views a set of its own.
struct OutputSet {
	uint32_t n_views = 0;
	DeviceArray<uint64_t> keys, values;                            // [n_views][cap_keys]
	DeviceArray<uint32_t> counts; PinnedArray<uint32_t> h_counts;  // [n_views][CNT_WORDS]
	DeviceArray<uint32_t> group_count, group_offset, group_cursor; // [n_views][max_groups]; a launch's views lie n_groups apart
	DeviceArray<uint64_t> group_renderables; DeviceArray<float4> instance_data; // [n_views][cap_recs], [n_views][3 cap_recs]
	DeviceArray<uint32_t> pose_list, dirty_list;                   // [n_views][max_entities]
	uint32_t pose_cap = 0; // capacity of each pose list when create_keys last filled the set (0 = never): entries past it were not written
};
} // namespace

struct lb200_sortkeys {
	lb200_ctx* ctx = nullptr;
	uint32_t max_entities = 0, max_groups = 0;
	uint32_t cap_keys = 0, cap_recs = 0;
	// inputs
	DeviceArray<SkEntity> d_ent;       // one 64-byte record per entity (transform, model / flags, lod and pose-frame state)
	bool have_transforms = false;
	DeviceArray<uint32_t> d_decal_sort_key; DeviceArray<uint8_t> d_decal_layer;
	DeviceArray<lb200_sk_model> d_models; DeviceArray<lb200_sk_mesh> d_meshes; // both set or both empty (lb200_sortkeys_set_models)
	DeviceArray<uint8_t> d_group_layer; // layer of the mesh material a sort key (= auto-instancer group) belongs to
	// the views' bucket_map + layer_to_bucket (SK_TABLE_WORDS each): copied from a pinned slot when they differ from what the device holds
	DeviceArray<uint32_t> d_tables; PinnedArray<uint32_t> h_tables; Event tables_copied[SK_TABLE_SLOTS];
	uint32_t table_slot = 0, tables_views = 0; // next pinned slot; views whose tables d_tables holds (0 = none yet)
	uint32_t tables_now[SK_MAX_VIEWS * SK_TABLE_WORDS] = {};   // ... and what they are
	// outputs
	OutputSet plain;                   // lb200_sortkeys_create_keys
	OutputSet views;                   // lb200_sortkeys_create_keys_views, grown to the most views a call had
	uint32_t views_n = 0, views_groups = 0; // views and group-table stride of the latest create_keys_views (0 = none yet)
	DeviceArray<uint64_t> d_keys_alt, d_values_alt; // the sort's alternate buffers, shared by every view of both sets
	DeviceArray<uint32_t> d_stash; DeviceArray<float4> d_stash4; // the two passes' hand-over: one word + 3 x float4 per visible renderable
	DeviceArray<float> d_lod; DeviceArray<uint32_t> d_pose_frame; // unpacked on request (lb200_sortkeys_device_outputs)
	DeviceArray<uint32_t> d_moved_list, d_moved_count; DeviceArray<lb200_transform> d_prev; // RenderModule::m_moved_instances, ModelInstance::prev_frame_transform (first move or spawn onwards)
	// spawns: per entity the sequence number of the last batch that listed it (duplicate check), the refusal count of a batch and its read-back
	DeviceArray<uint32_t> d_stamp, d_refused; PinnedArray<uint32_t> h_refused;
	uint32_t spawn_seq = 0;
	DeviceArray<GridBar> d_bar;
	RadixSortScratch radix_scratch; // the sort of every view's keys / values, with d_keys_alt / d_values_alt as its alternate buffers
	uint32_t max_mesh_sort_key = 0; // largest sort key of the mesh table: every view's max_sort_key must reach it
	uint32_t model_past_table = NO_MODEL; // first model whose meshes leave the mesh table (create_keys refuses to launch), NO_MODEL if none
	char past_table_text[128] = {};
	uint32_t keys_grid_limit[2] = {0, 0}; // co-resident blocks of create_keys_kernel: group counters in shared memory / in HBM
	// lb200_sortkeys_set_launch (blocks 0 = environment switch, else 2 per SM; -1 = all co-resident; prefetch -1 = environment switch) and
	// what the last create_keys / create_keys_views launched
	int launch_blocks = 0, launch_prefetch = -1;
	uint32_t last_grid = 0, last_prefetch = 0;
	int last_in_smem = 0;
	// lb200_sortkeys_build_palettes, allocated by the first build: the palette buffer (2 float4 = one dual quaternion per bone, grown to the
	// largest capacity a build needed), per entity the first bone of its slice, the bones written; per entity the instance that lists it,
	// as (number << 32 | stamp of the build that wrote it); the build sequence the stamps come from
	DeviceArray<float4> d_pal_dq; DeviceArray<uint32_t> d_pal_offset, d_pal_n_bones; DeviceArray<unsigned long long> d_pal_map;
	uint32_t pal_seq = 0;
};

namespace {
// host array (may be null: nothing to upload) -> temporary device buffer on the context stream (setters are not on the per-frame path)
template <typename T> int upload_temp(lb200_ctx* ctx, const T* host, size_t n, DeviceArray<T>& dev) {
	if (!host) return LB200_OK;
	LB200_CUDA(ctx, dev.alloc(n));
	LB200_CUDA(ctx, cudaMemcpyAsync(dev, host, sizeof(T) * n, cudaMemcpyHostToDevice, ctx->stream));
	return LB200_OK;
}

// An output set of n views, allocated whole before it replaces `out` (on failure `out` is left as it was)
int alloc_outputs(const lb200_sortkeys* sk, uint32_t n, OutputSet& out) {
	lb200_ctx* ctx = sk->ctx;
	const size_t keys = (size_t)n * sk->cap_keys, recs = (size_t)n * sk->cap_recs, groups = (size_t)n * sk->max_groups, lists = (size_t)n * sk->max_entities;
	OutputSet o;
	o.n_views = n;
	LB200_CUDA(ctx, o.keys.alloc(keys));
	LB200_CUDA(ctx, o.values.alloc(keys));
	LB200_CUDA(ctx, o.counts.alloc((size_t)n * CNT_WORDS));
	LB200_CUDA(ctx, o.h_counts.alloc((size_t)n * CNT_WORDS));
	LB200_CUDA(ctx, o.group_count.alloc(groups));
	LB200_CUDA(ctx, o.group_offset.alloc(groups));
	LB200_CUDA(ctx, o.group_cursor.alloc(groups));
	LB200_CUDA(ctx, o.group_renderables.alloc(recs));
	LB200_CUDA(ctx, o.instance_data.alloc(3 * recs)); // 48 bytes per instance
	LB200_CUDA(ctx, o.pose_list.alloc(lists));
	LB200_CUDA(ctx, o.dirty_list.alloc(lists));
	out = std::move(o);
	return LB200_OK;
}

// What create_keys checks of one view against the tables and the culling system (LB200_ERR_INVALID)
int check_view(lb200_sortkeys* sk, const lb200_sk_view& view) {
	lb200_ctx* ctx = sk->ctx;
	if (view.max_sort_key >= sk->max_groups) { lb200_set_error(ctx, "view.max_sort_key %u >= max_groups %u", view.max_sort_key, sk->max_groups); return LB200_ERR_INVALID; }
	if (sk->model_past_table != NO_MODEL) { lb200_set_error(ctx, "create_keys: %s", sk->past_table_text); return LB200_ERR_INVALID; }
	if (view.max_sort_key < sk->max_mesh_sort_key) { lb200_set_error(ctx, "view.max_sort_key %u < sort key %u of the mesh table", view.max_sort_key, sk->max_mesh_sort_key); return LB200_ERR_INVALID; }
	return LB200_OK;
}
int check_entity_range(lb200_sortkeys* sk, lb200_culling* cs) {
	// the kernel indexes the entity records, the decal arrays and the stash by the culled ids without a bounds check
	const uint32_t entity_range = lb200_culling_internal_entity_range(cs);
	if (entity_range > sk->max_entities) { lb200_set_error(sk->ctx, "the culling system holds entity ids up to %u, max_entities is %u", entity_range - 1, sk->max_entities); return LB200_ERR_INVALID; }
	return LB200_OK;
}

// The views' bucket_map + layer_to_bucket into d_tables, unless d_tables holds them already
int upload_tables(lb200_sortkeys* sk, const lb200_sk_view* views, uint32_t n) {
	lb200_ctx* ctx = sk->ctx;
	uint32_t t[SK_MAX_VIEWS * SK_TABLE_WORDS];
	for (uint32_t v = 0; v < n; ++v) {
		memcpy(t + v * SK_TABLE_WORDS, views[v].bucket_map, sizeof(views[v].bucket_map));
		memcpy(t + v * SK_TABLE_WORDS + 256, views[v].layer_to_bucket, sizeof(views[v].layer_to_bucket));
	}
	const size_t bytes = sizeof(uint32_t) * SK_TABLE_WORDS * n;
	if (n <= sk->tables_views && !memcmp(t, sk->tables_now, bytes)) return LB200_OK;
	const uint32_t slot = sk->table_slot;
	uint32_t* h = sk->h_tables + (size_t)slot * SK_MAX_VIEWS * SK_TABLE_WORDS;
	LB200_CUDA(ctx, cudaEventSynchronize(sk->tables_copied[slot])); // the copy that last used this slot has been made
	memcpy(h, t, bytes);
	sk->tables_views = 0; // unknown until the copy is enqueued
	LB200_CUDA(ctx, cudaMemcpyAsync(sk->d_tables, h, bytes, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaEventRecord(sk->tables_copied[slot], ctx->stream));
	sk->table_slot = (slot + 1) % SK_TABLE_SLOTS;
	memcpy(sk->tables_now, t, bytes);
	sk->tables_views = n;
	return LB200_OK;
}

// view v of `set`, whose group tables lie `groups` apart
ViewOut view_out(const lb200_sortkeys* sk, const OutputSet& set, uint32_t v, uint32_t groups) {
	const size_t k = (size_t)v * sk->cap_keys, r = (size_t)v * sk->cap_recs, g = (size_t)v * groups, l = (size_t)v * sk->max_entities;
	return {set.keys + k, set.values + k, set.counts + (size_t)v * CNT_WORDS, set.group_count + g, set.group_offset + g, set.group_cursor + g,
		set.group_renderables + r, set.instance_data + 3 * r, set.pose_list + l, set.dirty_list + l};
}
void view_pointers(const lb200_sortkeys* sk, const OutputSet& set, uint32_t v, uint32_t groups, lb200_sk_outputs* out) {
	const ViewOut o = view_out(sk, set, v, groups);
	out->keys = o.keys; out->values = o.values; out->group_count = o.group_count; out->group_offset = o.group_offset;
	out->group_renderables = o.group_renderables; out->instance_data = o.instance_data; out->pose_list = o.pose_list; out->dirty_list = o.dirty_list;
}

// createSortKeys of cv's views [0, n) into `out` (one cooperative launch), + radixSort of each view if `sort`, + one read-back of every view's
// counters into results[0, n) if `want_counts`
int launch_keys(lb200_sortkeys* sk, const CullViewsResult& cv, const lb200_sk_view* views, uint32_t n, OutputSet& out, int sort, int want_counts, lb200_sk_result* results) {
	lb200_ctx* ctx = sk->ctx;
	cudaStream_t s = ctx->stream;
	int rc = upload_tables(sk, views, n);
	if (rc) return rc;
	uint32_t n_groups = views[0].max_sort_key + 1;
	LB200_CUDA(ctx, cudaMemsetAsync(out.counts, 0, sizeof(uint32_t) * CNT_WORDS * n, s));
	LB200_CUDA(ctx, cudaMemsetAsync(out.group_count, 0, sizeof(uint32_t) * n_groups * n, s));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_bar, 0, sizeof(GridBar), s));
	EmitParams EP = {};
	for (uint32_t v = 0; v < n; ++v) {
		ViewScalars& w = EP.view[v];
		for (int c = 0; c < 3; ++c) { w.camera_pos[c] = views[v].camera_pos[c]; w.lod_ref_point[c] = views[v].lod_ref_point[c]; }
		w.time_delta = views[v].time_delta; w.lod_multiplier = views[v].lod_multiplier; w.frame_number = views[v].frame_number; w.is_shadow = views[v].is_shadow;
	}
	EP.n_views = n;
	for (int t = 0; t < 4; ++t) EP.type_base[t] = cv.type_base[t];
	EP.id_stride = cv.id_stride; EP.counter_stride = cv.counter_stride;
	EP.cap_keys = sk->cap_keys; EP.cap_recs = sk->cap_recs; EP.cap_pose = sk->max_entities; EP.cap_dirty = sk->max_entities;
	static const uint32_t prefetch_ahead = [] { const char* e = getenv("LB200_SK_PREFETCH"); const int v = e ? atoi(e) : 0; return (uint32_t)std::max(0, std::min(v, 4)); }(); // off: on H100 the prefetch slows the pass (DESIGN.md 4.5)
	EP.prefetch_ahead = sk->launch_prefetch >= 0 ? (uint32_t)sk->launch_prefetch : prefetch_ahead;
	const bool in_smem = n_groups <= SK_SMEM_GROUPS;
	size_t smem = in_smem ? sizeof(uint32_t) * n_groups : 0;
	uint32_t& limit = sk->keys_grid_limit[in_smem ? 0 : 1];
	if (!limit) { // co-resident blocks with the largest group table this path can ask for, so that the number holds for every view
		rc = lb200_coop_grid_limit(ctx,(const void*)create_keys_kernel, SK_THREADS, in_smem ? sizeof(uint32_t) * SK_SMEM_GROUPS : 0, &limit);
		if (rc) return rc;
	}
	const uint32_t work = cv.type_counts[RT_MESH] + cv.type_counts[RT_DECAL] + cv.type_counts[RT_CURVE_DECAL]; // upper bound of any view's visible renderables
	static const uint32_t blocks_per_sm = [] { const char* e = getenv("LB200_SK_BLOCKS_PER_SM"); const int v = e ? atoi(e) : 2; return (uint32_t)std::max(0, v); }(); // fewer resident blocks than fit (0 = all): 2 is fastest on H100
	uint32_t grid = std::max(1u, std::min(blocks_per_sm ? std::min(limit, blocks_per_sm * (uint32_t)ctx->sm_count) : limit, (work + SK_THREADS - 1) / SK_THREADS));
	if (sk->launch_blocks < 0) grid = limit; // lb200_sortkeys_set_launch: not capped by the work, so that threads with nothing to do still take part
	else if (sk->launch_blocks > 0) grid = std::min((uint32_t)sk->launch_blocks, limit);
	for (uint32_t v = 0; v < n; ++v) EP.out[v] = view_out(sk, out, v, n_groups);
	EmitArgs EA = {sk->d_ent, sk->d_decal_sort_key, sk->d_decal_layer, sk->d_models, sk->d_meshes, sk->d_tables, sk->d_group_layer, sk->d_stash, sk->d_stash4, sk->max_entities, sk->d_bar};
	const uint32_t* visible = cv.ids;
	const uint32_t* cull_counters = cv.counters;
	void* args[] = {&EP, &visible, &cull_counters, &EA, &n_groups};
	LB200_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)create_keys_kernel, dim3(grid), dim3(SK_THREADS), args, smem, s));
	LB200_CHECK_LAUNCH(ctx);
	sk->last_grid = grid; sk->last_in_smem = in_smem ? 1 : 0; sk->last_prefetch = EP.prefetch_ahead;
	out.pose_cap = EP.cap_pose;
	if (sort) {
		lb200_range r2("radixSort"); // pipeline.cpp:4101
		for (uint32_t v = 0; v < n; ++v) { // every view: whether a view has keys is known on the device only
			const size_t at = (size_t)v * sk->cap_keys;
			rc = lb200_radix_sort_pairs(ctx, s, out.keys + at, sk->d_keys_alt, out.values + at, sk->d_values_alt, out.counts + v * CNT_WORDS + CNT_KEYS, sk->cap_keys,
				sk->radix_scratch, 0, false, nullptr);
			if (rc) return rc;
		}
	}
	if (want_counts) {
		if (!results) return LB200_ERR_INVALID;
		LB200_CUDA(ctx, cudaMemcpyAsync(out.h_counts, out.counts, sizeof(uint32_t) * CNT_WORDS * n, cudaMemcpyDeviceToHost, s));
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		rc = LB200_OK;
		for (uint32_t v = 0; v < n; ++v) {
			const uint32_t* hc = out.h_counts + v * CNT_WORDS;
			lb200_sk_result& r = results[v];
			r.n_keys = hc[CNT_KEYS]; r.n_instances = hc[CNT_INST]; r.n_pose = hc[CNT_POSE]; r.n_dirty = hc[CNT_DIRTY]; r.n_groups = n_groups;
			if (!rc && (r.n_keys > sk->cap_keys || hc[CNT_RECS] > sk->cap_recs)) {
				lb200_set_error(ctx, "create_keys: view %u: %u keys / %u instances exceed the capacities %u / %u", v, r.n_keys, hc[CNT_RECS], sk->cap_keys, sk->cap_recs);
				rc = LB200_ERR_CAPACITY;
			}
		}
		return rc;
	}
	return LB200_OK;
}

// ModelInstance::lod / Pose::frame unpacked from the entity records into plain arrays (on the context stream)
int unpack_state(lb200_sortkeys* sk, lb200_sk_outputs* out) {
	lb200_ctx* ctx = sk->ctx;
	if (!sk->d_lod || !sk->d_pose_frame) {
		DeviceArray<float> lod; DeviceArray<uint32_t> pose_frame;
		LB200_CUDA(ctx, lod.alloc(sk->max_entities));
		LB200_CUDA(ctx, pose_frame.alloc(sk->max_entities));
		sk->d_lod = std::move(lod); sk->d_pose_frame = std::move(pose_frame);
	}
	ent_unpack_state_kernel<<<(sk->max_entities + 255) / 256, 256, 0, ctx->stream>>>(sk->d_ent, sk->max_entities, sk->d_lod, sk->d_pose_frame);
	LB200_CHECK_LAUNCH(ctx);
	out->lod = sk->d_lod; out->pose_frame = sk->d_pose_frame;
	return LB200_OK;
}

// the moved list and prev_frame_transform, allocated by the first move or spawn (end_frame tests d_moved_list alone: all three or none)
int ensure_moved(lb200_sortkeys* sk) {
	lb200_ctx* ctx = sk->ctx;
	if (sk->d_moved_list && sk->d_moved_count && sk->d_prev) return LB200_OK;
	DeviceArray<uint32_t> moved_list, moved_count; DeviceArray<lb200_transform> prev;
	LB200_CUDA(ctx, moved_list.alloc(sk->max_entities));
	LB200_CUDA(ctx, moved_count.alloc(1));
	LB200_CUDA(ctx, cudaMemsetAsync(moved_count, 0, sizeof(uint32_t), ctx->stream));
	LB200_CUDA(ctx, prev.alloc(sk->max_entities));
	LB200_CUDA(ctx, cudaMemsetAsync(prev, 0, sizeof(lb200_transform) * (size_t)sk->max_entities, ctx->stream));
	sk->d_moved_list = std::move(moved_list); sk->d_moved_count = std::move(moved_count); sk->d_prev = std::move(prev);
	return LB200_OK;
}

// `to` holds the first n_old elements of `from` (on the context stream), the rest filled with byte `fill` (fill < 0: left as allocated)
template <typename T> int grow_copy(lb200_ctx* ctx, const DeviceArray<T>& from, size_t n_old, size_t n_new, int fill, DeviceArray<T>& to) {
	LB200_CUDA(ctx, to.alloc(n_new));
	if (n_old) LB200_CUDA(ctx, cudaMemcpyAsync(to, from, sizeof(T) * n_old, cudaMemcpyDeviceToDevice, ctx->stream));
	if (fill >= 0) LB200_CUDA(ctx, cudaMemsetAsync(to + n_old, fill, sizeof(T) * (n_new - n_old), ctx->stream));
	return LB200_OK;
}
// a set's pose / dirty lists ([n_views][max_entities]) at the row stride `cap`, each view's row copied over
int grow_lists(lb200_ctx* ctx, const DeviceArray<uint32_t>& from, uint32_t n_views, uint32_t old_cap, uint32_t cap, DeviceArray<uint32_t>& to) {
	LB200_CUDA(ctx, to.alloc((size_t)n_views * cap));
	LB200_CUDA(ctx, cudaMemcpy2DAsync(to, sizeof(uint32_t) * cap, from, sizeof(uint32_t) * old_cap, sizeof(uint32_t) * old_cap, n_views, cudaMemcpyDeviceToDevice, ctx->stream));
	return LB200_OK;
}

// Every per-entity array grown to `cap` entity ids: allocated and filled first, swapped in once the stream has finished the copies, so
// that a failure leaves the object as it was.  Records, decal arrays, moved list, prev_frame_transform and the pose / dirty lists of both
// output sets keep their contents (the new records in ent_init_kernel's state); the stash and the unpacked lod / pose-frame arrays hold
// nothing across calls and are allocated anew; `stamp` (cap entries, the batch that asked for the growth already checked with it)
// becomes the stamp array.
int grow_entities(lb200_sortkeys* sk, size_t cap, DeviceArray<uint32_t>& stamp) {
	lb200_ctx* ctx = sk->ctx;
	const size_t old = sk->max_entities;
	cudaStream_t s = ctx->stream;
	DeviceArray<SkEntity> ent;
	LB200_CUDA(ctx, ent.alloc(cap));
	LB200_CUDA(ctx, cudaMemcpyAsync(ent, sk->d_ent, sizeof(SkEntity) * old, cudaMemcpyDeviceToDevice, s));
	ent_init_kernel<<<(uint32_t)((cap - old + 255) / 256), 256, 0, s>>>(ent + old, (uint32_t)(cap - old));
	LB200_CHECK_LAUNCH(ctx);
	DeviceArray<uint32_t> decal_sort_key, stash, moved_list, pose_frame, plain_pose, plain_dirty, views_pose, views_dirty;
	DeviceArray<uint8_t> decal_layer; DeviceArray<float4> stash4; DeviceArray<lb200_transform> prev; DeviceArray<float> lod;
	DeviceArray<uint32_t> pal_offset; DeviceArray<unsigned long long> pal_map;
	int rc = grow_copy(ctx, sk->d_decal_sort_key, old, cap, 0, decal_sort_key);
	if (!rc) rc = grow_copy(ctx, sk->d_decal_layer, old, cap, 0, decal_layer);
	if (rc) return rc;
	LB200_CUDA(ctx, stash.alloc(cap));
	LB200_CUDA(ctx, stash4.alloc(3 * cap));
	if (sk->d_moved_list) {
		rc = grow_copy(ctx, sk->d_moved_list, old, cap, -1, moved_list);
		if (!rc) rc = grow_copy(ctx, sk->d_prev, old, cap, 0, prev);
		if (rc) return rc;
	}
	if (sk->d_lod) {
		LB200_CUDA(ctx, lod.alloc(cap));
		LB200_CUDA(ctx, pose_frame.alloc(cap));
	}
	if (sk->d_pal_offset) { // the palette offsets keep theirs; the entity -> instance map is rebuilt by every build and starts stamp-free
		rc = grow_copy(ctx, sk->d_pal_offset, old, cap, 0xff, pal_offset);
		if (rc) return rc;
		LB200_CUDA(ctx, pal_map.alloc(cap));
		LB200_CUDA(ctx, cudaMemsetAsync(pal_map, 0, sizeof(unsigned long long) * cap, s));
	}
	rc = grow_lists(ctx, sk->plain.pose_list, sk->plain.n_views, (uint32_t)old, (uint32_t)cap, plain_pose);
	if (!rc) rc = grow_lists(ctx, sk->plain.dirty_list, sk->plain.n_views, (uint32_t)old, (uint32_t)cap, plain_dirty);
	if (!rc && sk->views.n_views) {
		rc = grow_lists(ctx, sk->views.pose_list, sk->views.n_views, (uint32_t)old, (uint32_t)cap, views_pose);
		if (!rc) rc = grow_lists(ctx, sk->views.dirty_list, sk->views.n_views, (uint32_t)old, (uint32_t)cap, views_dirty);
	}
	if (rc) return rc;
	LB200_CUDA(ctx, cudaStreamSynchronize(s)); // the copies are done and nothing enqueued still uses the old arrays
	sk->d_ent = std::move(ent);
	sk->d_decal_sort_key = std::move(decal_sort_key); sk->d_decal_layer = std::move(decal_layer);
	sk->d_stash = std::move(stash); sk->d_stash4 = std::move(stash4); sk->d_stamp = std::move(stamp);
	if (sk->d_moved_list) { sk->d_moved_list = std::move(moved_list); sk->d_prev = std::move(prev); }
	if (sk->d_lod) { sk->d_lod = std::move(lod); sk->d_pose_frame = std::move(pose_frame); }
	if (sk->d_pal_offset) { sk->d_pal_offset = std::move(pal_offset); sk->d_pal_map = std::move(pal_map); }
	sk->plain.pose_list = std::move(plain_pose); sk->plain.dirty_list = std::move(plain_dirty);
	if (sk->views.n_views) { sk->views.pose_list = std::move(views_pose); sk->views.dirty_list = std::move(views_dirty); }
	sk->max_entities = (uint32_t)cap;
	return LB200_OK;
}

// The read-back of a spawn batch's refusal count (synchronises the stream)
int spawn_result(lb200_sortkeys* sk, const char* what, const char* reasons, uint32_t max_entity) {
	lb200_ctx* ctx = sk->ctx;
	LB200_CUDA(ctx, cudaMemcpyAsync(sk->h_refused, sk->d_refused, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	if (const uint32_t bad = *sk->h_refused) {
		lb200_set_error(ctx, "%s: %u entries refused (%s; ids in [0, %u]): nothing spawned", what, bad, reasons, max_entity);
		return LB200_ERR_INVALID;
	}
	return LB200_OK;
}

// What both spawn calls do ahead of their writes: the refusal count of the batch (model check if model_of).  A batch whose max_entity
// needs more entity ids is checked against a stamp array of the grown size first, and only a batch without refusals grows the object
// (one more synchronisation, on a call that waits for the stream anyway): a refused call changes nothing.
int spawn_check(lb200_sortkeys* sk, const int32_t* entities, uint32_t n, uint32_t max_entity, const uint32_t* model_of, const char* what, const char* reasons) {
	lb200_ctx* ctx = sk->ctx;
	cudaStream_t s = ctx->stream;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!sk->d_refused) {
		DeviceArray<uint32_t> refused; PinnedArray<uint32_t> h_refused;
		LB200_CUDA(ctx, refused.alloc(1));
		LB200_CUDA(ctx, h_refused.alloc(1));
		sk->d_refused = std::move(refused); sk->h_refused = std::move(h_refused);
	}
	const bool grow = (size_t)max_entity >= sk->max_entities;
	const size_t stamps = grow ? grownCapacity(sk->max_entities, 4096, (size_t)max_entity + 1) : sk->max_entities;
	DeviceArray<uint32_t> grown_stamp;
	if (grow || !sk->d_stamp) { // zero: no stamp holds a batch number yet
		DeviceArray<uint32_t>& st = grow ? grown_stamp : sk->d_stamp;
		LB200_CUDA(ctx, st.alloc(stamps));
		LB200_CUDA(ctx, cudaMemsetAsync(st, 0, sizeof(uint32_t) * stamps, s));
	}
	uint32_t* stamp = grow ? grown_stamp.get() : sk->d_stamp.get();
	if (++sk->spawn_seq == 0) { // wrapped: no stamp may hold the new number already
		LB200_CUDA(ctx, cudaMemsetAsync(stamp, 0, sizeof(uint32_t) * stamps, s));
		sk->spawn_seq = 1;
	}
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_refused, 0, sizeof(uint32_t), s));
	spawn_check_kernel<<<(n + 255) / 256, 256, 0, s>>>(entities, n, max_entity, model_of, (uint32_t)sk->d_models.size(), stamp, sk->spawn_seq, sk->d_refused);
	LB200_CHECK_LAUNCH(ctx);
	if (!grow) return LB200_OK;
	const int rc = spawn_result(sk, what, reasons, max_entity);
	if (rc) return rc;
	return grow_entities(sk, stamps, grown_stamp);
}

// ---- PoseProcessor::push + computeSkeletonDualQuats (pipeline.cpp:3730-3787, 2680-2745) for the pose lists create_keys left ----
// Every build numbers the instances of its systems that have entity ids 0, 1, ... in system order and maps each entity to the number of
// the instance that lists it (pal_map_kernel: one 64-bit exchange per instance, stamped with the build).  pal_build_kernel then walks the
// pose lists: the first listing of a mapped entity claims the map entry (stamp -> stamp + 1) and writes the instance's palette into a
// slice of the build's buffer; a listing of an unmapped entity writes PAL_NONE.  Stale entries carry an older stamp: nothing is cleared.
constexpr uint32_t PAL_MAX_SYSTEMS = 64; // systems per launch (parameter block of ~3.6 KB); longer lists run as consecutive launches
constexpr int PAL_THREADS = 256;
constexpr uint32_t PAL_LANES = 8;        // lanes per listed entity, the bones strided over them
constexpr uint32_t PAL_NONE = 0xffffffffu;

struct PalSystem {
	const float* pos; const float4* rot;                // absolute poses, instance-major (what LB200_PALETTE_POSE fills)
	const float4* inv_bind_pos; const float4* inv_bind_rot;
	const int32_t* entity;                              // entity id of instances [0, n)
	uint32_t bone_count, n, base, pad;                  // instance i has number base + i
};
struct PalParams {
	PalSystem sys[PAL_MAX_SYSTEMS];
	uint32_t n_systems, first, end; // the launch's systems own numbers [first, end)
	uint32_t stamp;                 // even; an entry this build claimed holds stamp + 1
	const uint32_t* list[SK_MAX_VIEWS]; const uint32_t* count[SK_MAX_VIEWS]; // the pose lists and their counts (device)
	uint32_t n_lists, cap_pose, max_entities;
	uint32_t write_none;            // the first launch of a build: listed entities without an instance get PAL_NONE
	unsigned long long* map; uint32_t* offset; float4* dq; uint32_t* n_bones;
};

// blockIdx.y = system of the launch, its instances grid-strided over blockIdx.x
__global__ void __launch_bounds__(PAL_THREADS) pal_map_kernel(const __grid_constant__ PalParams P) {
	const PalSystem& S = P.sys[blockIdx.y];
	for (uint32_t i = blockIdx.x * PAL_THREADS + threadIdx.x; i < S.n; i += gridDim.x * PAL_THREADS) {
		const int32_t e = S.entity[i];
		if (e >= 0 && (uint32_t)e < P.max_entities) atomicExch(P.map + e, ((unsigned long long)(S.base + i) << 32) | P.stamp);
	}
}

// PAL_LANES lanes per listed entity, the lists of every view as one index space, grid-strided a warp (32 / PAL_LANES entities) at a time.
// The arithmetic is the pose kernel's palette epilogue: the same rmul + to_dual_quat of the same inputs, so the bits are the same.
__global__ void __launch_bounds__(PAL_THREADS) pal_build_kernel(const __grid_constant__ PalParams P) {
	constexpr uint32_t PER_WARP = 32 / PAL_LANES;
	__shared__ uint32_t s_end[SK_MAX_VIEWS]; // inclusive prefix of the clamped list lengths
	if (threadIdx.x == 0) {
		uint32_t total = 0;
		for (uint32_t v = 0; v < P.n_lists; ++v) { total += min(__ldcg(P.count[v]), P.cap_pose); s_end[v] = total; }
	}
	__syncthreads();
	const uint32_t total = s_end[P.n_lists - 1];
	const uint32_t lane = threadIdx.x & 31u, sub = lane % PAL_LANES, leader = lane - sub;
	const uint32_t warps = gridDim.x * (PAL_THREADS / 32);
	for (uint32_t at = (blockIdx.x * (PAL_THREADS / 32) + threadIdx.x / 32) * PER_WARP; at < total; at += warps * PER_WARP) { // warp-uniform
		const uint32_t k = at + lane / PAL_LANES;
		uint32_t e = 0, g = 0, s = 0, bones = 0;
		if (sub == 0 && k < total) {
			uint32_t v = 0;
			while (k >= s_end[v]) ++v;
			e = __ldcg(P.list[v] + (k - (v ? s_end[v - 1] : 0u)));
			const unsigned long long w = __ldcg(P.map + e);
			const uint32_t stamp = (uint32_t)w;
			g = (uint32_t)(w >> 32);
			if (stamp == P.stamp) {
				if (g >= P.first && g < P.end && atomicCAS(P.map + e, w, w + 1) == w) { // the entity's first listing builds it
					uint32_t lo = 0, hi = P.n_systems - 1; // the last system whose numbers start at or below g
					while (lo < hi) {
						const uint32_t mid = (lo + hi + 1) >> 1;
						if (P.sys[mid].base <= g) lo = mid;
						else hi = mid - 1;
					}
					s = lo;
					bones = P.sys[s].bone_count;
				}
			}
			else if (stamp != P.stamp + 1 && P.write_none) P.offset[e] = PAL_NONE; // no instance of the build lists e
		}
		// the warp's slices with one atomic: inclusive scan of the bones its leaders build
		uint32_t incl = bones;
#pragma unroll
		for (int d = 1; d < 32; d <<= 1) {
			const uint32_t y = __shfl_up_sync(0xffffffffu, incl, d);
			if (lane >= (uint32_t)d) incl += y;
		}
		uint32_t base = 0;
		if (lane == 31 && incl) base = atomicAdd(P.n_bones, incl);
		base = __shfl_sync(0xffffffffu, base, 31);
		const uint32_t first = __shfl_sync(0xffffffffu, base + incl - bones, leader);
		e = __shfl_sync(0xffffffffu, e, leader);
		g = __shfl_sync(0xffffffffu, g, leader);
		s = __shfl_sync(0xffffffffu, s, leader);
		bones = __shfl_sync(0xffffffffu, bones, leader);
		if (!bones) continue;
		const PalSystem& S = P.sys[s];
		if (sub == 0) P.offset[e] = first;
		const size_t src = (size_t)(g - S.base) * bones;
		float4* out = P.dq + 2 * (size_t)first;
		for (uint32_t b = sub; b < bones; b += PAL_LANES) {
			const float* p = S.pos + 3 * (src + b);
			const float4 r = __ldg(S.rot + src + b);
			const float4 ip = __ldg(S.inv_bind_pos + b), ir = __ldg(S.inv_bind_rot + b);
			Rigid pose, inv;
			pose.pos = v3(__ldg(p), __ldg(p + 1), __ldg(p + 2));
			pose.rot = q4(r.x, r.y, r.z, r.w);
			inv.pos = v3(ip.x, ip.y, ip.z);
			inv.rot = q4(ir.x, ir.y, ir.z, ir.w);
			const DualQ dq = to_dual_quat(rmul(pose, inv));
			out[2 * b] = make_float4(dq.r.x, dq.r.y, dq.r.z, dq.r.w);
			out[2 * b + 1] = make_float4(dq.d.x, dq.d.y, dq.d.z, dq.d.w);
		}
	}
}

} // namespace

void lb200_sortkeys_internal_records(const lb200_sortkeys* sk, SortKeysRecords* out) {
	*out = {sk->ctx, sk->d_ent, sk->max_entities, sk->have_transforms};
}

extern "C" {

int lb200_sortkeys_create(lb200_ctx* ctx, uint32_t max_entities, uint32_t max_groups, uint32_t max_keys, uint32_t max_instances, lb200_sortkeys** out) {
	if (!ctx || !out || !max_entities || !max_groups) return LB200_ERR_INVALID;
	*out = nullptr;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	std::unique_ptr<lb200_sortkeys, decltype(&lb200_sortkeys_destroy)> sk(new (std::nothrow) lb200_sortkeys, lb200_sortkeys_destroy);
	if (!sk) return LB200_ERR_CUDA;
	sk->ctx = ctx;
	sk->max_entities = max_entities; sk->max_groups = max_groups;
	sk->cap_keys = max_keys ? max_keys : max_entities; sk->cap_recs = max_instances ? max_instances : max_entities;
	const size_t E = max_entities;
	LB200_CUDA(ctx, sk->d_ent.alloc(E));
	ent_init_kernel<<<(uint32_t)((E + 255) / 256), 256, 0, ctx->stream>>>(sk->d_ent, max_entities);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, sk->d_decal_sort_key.alloc(E));
	LB200_CUDA(ctx, sk->d_decal_layer.alloc(E));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_decal_sort_key, 0, sizeof(uint32_t) * E, ctx->stream));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_decal_layer, 0, E, ctx->stream));
	int rc = alloc_outputs(sk.get(), 1, sk->plain);
	if (rc) return rc;
	LB200_CUDA(ctx, sk->d_keys_alt.alloc(sk->cap_keys));
	LB200_CUDA(ctx, sk->d_values_alt.alloc(sk->cap_keys));
	LB200_CUDA(ctx, sk->d_group_layer.alloc(max_groups));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_group_layer, 0, max_groups, ctx->stream));
	LB200_CUDA(ctx, sk->d_tables.alloc((size_t)SK_MAX_VIEWS * SK_TABLE_WORDS));
	LB200_CUDA(ctx, sk->h_tables.alloc((size_t)SK_TABLE_SLOTS * SK_MAX_VIEWS * SK_TABLE_WORDS));
	for (Event& ev : sk->tables_copied) LB200_CUDA(ctx, cudaEventCreateWithFlags(ev.create(), cudaEventDisableTiming));
	LB200_CUDA(ctx, sk->d_stash.alloc(E));
	LB200_CUDA(ctx, sk->d_stash4.alloc(3 * E));
	LB200_CUDA(ctx, sk->d_bar.alloc(1));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_bar, 0, sizeof(GridBar), ctx->stream));
	rc = lb200_radix_sort_alloc_scratch(ctx, (uint32_t)ctx->sm_count * 2, sk->radix_scratch);
	if (rc) return rc;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	*out = sk.release();
	return LB200_OK;
}

void lb200_sortkeys_destroy(lb200_sortkeys* sk) {
	if (!sk) return;
	cudaSetDevice(sk->ctx->device);
	cudaStreamSynchronize(sk->ctx->stream);
	delete sk;
}

int lb200_sortkeys_set_models(lb200_sortkeys* sk, const lb200_sk_model* models, uint32_t n_models, const lb200_sk_mesh* meshes, uint32_t n_meshes) {
	if (!sk || !models || !meshes || !n_models || !n_meshes) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	if (n_models > CODE_MODEL_MASK + 1u) { lb200_set_error(ctx, "%u models: the entity record keeps 24 bits of model index", n_models); return LB200_ERR_INVALID; }
	uint32_t max_key = 0;
	for (uint32_t i = 0; i < n_meshes; ++i) {
		if (meshes[i].sort_key >= sk->max_groups) { lb200_set_error(ctx, "mesh %u: sort key %u >= max_groups %u", i, meshes[i].sort_key, sk->max_groups); return LB200_ERR_INVALID; }
		max_key = std::max(max_key, meshes[i].sort_key);
	}
	// the kernel reads meshes[mesh_base + j] for every j of the drawn LOD ranges without a bounds check: a LOD range has to stay inside its
	// model's meshes (refused here), and the model's meshes inside the mesh table (create_keys refuses to launch until they do, so that a
	// table can be set ahead of the meshes it will be paired with)
	uint32_t model_past_table = NO_MODEL;
	for (uint32_t m = 0; m < n_models; ++m) {
		const lb200_sk_model& md = models[m];
		if (model_past_table == NO_MODEL && (md.mesh_base > n_meshes || md.mesh_count > n_meshes - md.mesh_base)) model_past_table = m;
		for (int l = 0; l < 5; ++l) {
			if (md.lod_from[l] > md.lod_to[l]) continue; // empty LOD: nothing drawn
			if (md.lod_from[l] < 0 || (uint32_t)md.lod_to[l] >= md.mesh_count) {
				lb200_set_error(ctx, "model %u: LOD %d meshes [%d, %d] leave the model's %u meshes", m, l, md.lod_from[l], md.lod_to[l], md.mesh_count);
				return LB200_ERR_INVALID;
			}
		}
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	sk->d_models.reset(); sk->d_meshes.reset(); // both go before either is allocated again
	DeviceArray<lb200_sk_model> d_models; DeviceArray<lb200_sk_mesh> d_meshes;
	LB200_CUDA(ctx, d_models.alloc(n_models));
	LB200_CUDA(ctx, d_meshes.alloc(n_meshes));
	sk->d_models = std::move(d_models); sk->d_meshes = std::move(d_meshes);
	LB200_CUDA(ctx, cudaMemcpyAsync(sk->d_models, models, sizeof(lb200_sk_model) * n_models, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(sk->d_meshes, meshes, sizeof(lb200_sk_mesh) * n_meshes, cudaMemcpyHostToDevice, ctx->stream));
	// a sort key stands for one (mesh, material) pair (RenderModule::computeSortKey): the layer a group's key is bucketed by (:3958-3969)
	// is that material's, the same for every instance of the group
	uint8_t* layer = new (std::nothrow) uint8_t[sk->max_groups];
	if (!layer) return LB200_ERR_CUDA;
	memset(layer, 0, sk->max_groups);
	for (uint32_t i = 0; i < n_meshes; ++i) layer[meshes[i].sort_key] = meshes[i].layer;
	const cudaError_t e = cudaMemcpyAsync(sk->d_group_layer, layer, sk->max_groups, cudaMemcpyHostToDevice, ctx->stream);
	cudaStreamSynchronize(ctx->stream);
	delete[] layer;
	LB200_CUDA(ctx, e);
	sk->max_mesh_sort_key = max_key;
	sk->model_past_table = model_past_table;
	if (model_past_table != NO_MODEL) {
		const lb200_sk_model& md = models[model_past_table];
		snprintf(sk->past_table_text, sizeof(sk->past_table_text), "model %u: meshes [%u, %u + %u) leave the %u-mesh table", model_past_table, md.mesh_base, md.mesh_base,
			md.mesh_count, n_meshes);
	}
	return LB200_OK;
}

// per-entity state, arrays indexed by entity id (n <= max_entities); null pointers leave that field as it is
int lb200_sortkeys_set_instances(lb200_sortkeys* sk, uint32_t n, const uint32_t* model_of, const float* lod, const uint8_t* flags, const uint32_t* pose_frame,
	const uint32_t* decal_sort_key, const uint8_t* decal_layer)
{
	if (!sk || n > sk->max_entities) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	if (!n) return LB200_OK;
	DeviceArray<uint32_t> t_model, t_pose; DeviceArray<float> t_lod; DeviceArray<uint8_t> t_flags;
	int rc = upload_temp(ctx, model_of, n, t_model);
	if (!rc) rc = upload_temp(ctx, lod, n, t_lod);
	if (!rc) rc = upload_temp(ctx, flags, n, t_flags);
	if (!rc) rc = upload_temp(ctx, pose_frame, n, t_pose);
	if (rc) return rc;
	if (t_model || t_lod || t_flags || t_pose) {
		ent_pack_fields_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(sk->d_ent, n, t_model, t_lod, t_flags, t_pose);
		LB200_CHECK_LAUNCH(ctx);
	}
	if (decal_sort_key) LB200_CUDA(ctx, cudaMemcpyAsync(sk->d_decal_sort_key, decal_sort_key, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	if (decal_layer) LB200_CUDA(ctx, cudaMemcpyAsync(sk->d_decal_layer, decal_layer, n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

int lb200_sortkeys_set_transforms(lb200_sortkeys* sk, const lb200_transform* transforms, uint32_t n) {
	if (!sk || !transforms || n > sk->max_entities) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	DeviceArray<lb200_transform> tmp;
	const int rc = upload_temp(ctx, transforms, n, tmp);
	if (rc) return rc;
	if (n) {
		ent_pack_transforms_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(sk->d_ent, tmp, n);
		LB200_CHECK_LAUNCH(ctx);
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // before tmp is freed
	sk->have_transforms = true;
	return LB200_OK;
}

// World::getTransforms() already in HBM (e.g. lb200_hierarchy's globals): packed into the entity records on the context stream, now —
// call again after the array changed.
int lb200_sortkeys_set_transforms_device(lb200_sortkeys* sk, const lb200_transform* dev_transforms, uint32_t n) {
	if (!sk || !dev_transforms || n > sk->max_entities) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	if (n) {
		ent_pack_transforms_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(sk->d_ent, dev_transforms, n);
		LB200_CHECK_LAUNCH(ctx);
	}
	sk->have_transforms = true;
	return LB200_OK;
}

int lb200_sortkeys_create_keys(lb200_sortkeys* sk, lb200_culling* cs, const lb200_sk_view* view, int sort, int want_counts, lb200_sk_result* result) {
	if (!sk || !cs || !view) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	lb200_range range("create keys"); // pipeline.cpp:3818
	if (!sk->have_transforms || !sk->d_models) { lb200_set_error(ctx, "create_keys needs set_models and set_transforms first"); return LB200_ERR_STATE; }
	int rc = check_view(sk, *view);
	if (rc) return rc;
	CullViewsResult cv = {1, 0, 0, nullptr, nullptr, nullptr, nullptr};
	rc = lb200_culling_internal_last(cs, &cv.ids, &cv.counters, &cv.type_base, &cv.type_counts);
	if (rc) return rc;
	rc = check_entity_range(sk, cs);
	if (rc) return rc;
	return launch_keys(sk, cv, view, 1, sk->plain, sort, want_counts, result);
}

int lb200_sortkeys_create_keys_views(lb200_sortkeys* sk, lb200_culling* cs, const lb200_sk_view* views, uint32_t n_views, int sort, int want_counts, lb200_sk_result* results) {
	if (!sk || !cs || !views || (want_counts && !results)) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	lb200_range range("create keys"); // pipeline.cpp:3818
	if (n_views < 1 || n_views > SK_MAX_VIEWS) { lb200_set_error(ctx, "create_keys_views: n_views %u is not 1..%u", n_views, SK_MAX_VIEWS); return LB200_ERR_INVALID; }
	if (!sk->have_transforms || !sk->d_models) { lb200_set_error(ctx, "create_keys_views needs set_models and set_transforms first"); return LB200_ERR_STATE; }
	CullViewsResult cv;
	int rc = lb200_culling_internal_views(cs, &cv);
	if (rc) return rc;
	if (n_views != cv.n_views) { lb200_set_error(ctx, "create_keys_views: %u views, the latest cull_views culled %u", n_views, cv.n_views); return LB200_ERR_INVALID; }
	for (uint32_t v = 0; v < n_views; ++v) {
		// Renderer::getMaxSortKey() is renderer-wide: it sizes the launch's group tables
		if (views[v].max_sort_key != views[0].max_sort_key) {
			lb200_set_error(ctx, "create_keys_views: view %u has max_sort_key %u, view 0 %u", v, views[v].max_sort_key, views[0].max_sort_key);
			return LB200_ERR_INVALID;
		}
		rc = check_view(sk, views[v]);
		if (rc) return rc;
	}
	rc = check_entity_range(sk, cs);
	if (rc) return rc;
	if (sk->views.n_views < n_views) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // nothing enqueued still uses the old set
		sk->views_n = 0;
		sk->views = OutputSet();
		rc = alloc_outputs(sk, n_views, sk->views);
		if (rc) return rc;
	}
	sk->views_n = n_views;
	sk->views_groups = views[0].max_sort_key + 1;
	return launch_keys(sk, cv, views, n_views, sk->views, sort, want_counts, results);
}

int lb200_sortkeys_set_launch(lb200_sortkeys* sk, int blocks, int prefetch_ahead) {
	if (!sk) return LB200_ERR_INVALID;
	if (blocks < -1) { lb200_set_error(sk->ctx, "set_launch: blocks %d is not -1, 0 or a block count", blocks); return LB200_ERR_INVALID; }
	if (prefetch_ahead < -1 || prefetch_ahead > 4) { lb200_set_error(sk->ctx, "set_launch: prefetch_ahead %d is not -1 or 0..4", prefetch_ahead); return LB200_ERR_INVALID; }
	sk->launch_blocks = blocks;
	sk->launch_prefetch = prefetch_ahead;
	return LB200_OK;
}

int lb200_sortkeys_get_launch(lb200_sortkeys* sk, uint32_t* grid, int* groups_in_smem, uint32_t* prefetch_ahead) {
	if (!sk) return LB200_ERR_INVALID;
	if (grid) *grid = sk->last_grid;
	if (groups_in_smem) *groups_in_smem = sk->last_in_smem;
	if (prefetch_ahead) *prefetch_ahead = sk->last_prefetch;
	return LB200_OK;
}

// device pointers of the last create_keys (valid until the next one): sorted keys / values, group tables, instance data, lists; the
// lod / pose-frame state is unpacked from the entity records into plain arrays for the caller (on the context stream)
int lb200_sortkeys_device_outputs(lb200_sortkeys* sk, lb200_sk_outputs* out) {
	if (!sk || !out) return LB200_ERR_INVALID;
	const int rc = unpack_state(sk, out);
	if (rc) return rc;
	view_pointers(sk, sk->plain, 0, sk->max_groups, out);
	return LB200_OK;
}

// the same for view k of the latest create_keys_views (valid until the next one)
int lb200_sortkeys_view_outputs(lb200_sortkeys* sk, uint32_t k, lb200_sk_outputs* out) {
	if (!sk || !out) return LB200_ERR_INVALID;
	if (!sk->views_n) { lb200_set_error(sk->ctx, "view_outputs needs a preceding create_keys_views"); return LB200_ERR_STATE; }
	if (k >= sk->views_n) { lb200_set_error(sk->ctx, "view_outputs: view %u of a create_keys_views call of %u views", k, sk->views_n); return LB200_ERR_INVALID; }
	const int rc = unpack_state(sk, out);
	if (rc) return rc;
	view_pointers(sk, sk->views, k, sk->views_groups, out);
	return LB200_OK;
}

// RenderModule::onModelInstanceMoved for n instances whose new transforms lie in HBM (SURVEY 8f N4): transforms into the entity records,
// ModelInstance::MOVED on, the instances join the moved list (createSortKeys draws them as DRAW_MESH until lb200_sortkeys_end_frame).
// With dev_bounding_radius: (pos, radius * max scale) per instance into dev_out_pos3 / dev_out_radius, the arguments of
// lb200_culling_set_many_device (render_module.cpp:1552-1554).
int lb200_sortkeys_move_device(lb200_sortkeys* sk, const int32_t* dev_entities, const lb200_transform* dev_transforms, uint32_t n, const float* dev_bounding_radius,
	double* dev_out_pos3, float* dev_out_radius)
{
	if (!sk || !dev_entities || !dev_transforms || (dev_out_radius && !dev_bounding_radius)) return LB200_ERR_INVALID;
	if (!n) return LB200_OK;
	lb200_ctx* ctx = sk->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const int rc = ensure_moved(sk);
	if (rc) return rc;
	ent_move_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(sk->d_ent, sk->max_entities, dev_entities, dev_transforms, n, dev_bounding_radius, dev_out_pos3, dev_out_radius, sk->d_moved_list, sk->d_moved_count);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

// RenderModule::endFrame (render_module.cpp:526-534) for the instances moved since the last call
int lb200_sortkeys_end_frame(lb200_sortkeys* sk) {
	if (!sk) return LB200_ERR_INVALID;
	if (!sk->d_moved_list) return LB200_OK; // nothing ever moved through this object
	lb200_ctx* ctx = sk->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	ent_end_frame_kernel<<<(uint32_t)ctx->sm_count * 2, 256, 0, ctx->stream>>>(sk->d_ent, sk->d_moved_list, sk->d_moved_count, sk->d_prev);
	LB200_CHECK_LAUNCH(ctx);
	reset_word_kernel<<<1, 1, 0, ctx->stream>>>(sk->d_moved_count);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

// ModelInstance::prev_frame_transform per entity (device array, zero until an instance has been through move + end_frame or a spawn), valid
// while sk lives and until a spawn grows it
int lb200_sortkeys_prev_transforms(lb200_sortkeys* sk, const lb200_transform** dev_prev) {
	if (!sk || !dev_prev) return LB200_ERR_INVALID;
	*dev_prev = sk->d_prev;
	return LB200_OK;
}

int lb200_sortkeys_moved_list(lb200_sortkeys* sk, const uint32_t** dev_list, uint32_t* n) {
	if (!sk || !dev_list || !n) return LB200_ERR_INVALID;
	*dev_list = sk->d_moved_list;
	*n = 0;
	if (!sk->d_moved_count) return LB200_OK;
	lb200_ctx* ctx = sk->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(n, sk->d_moved_count, sizeof(uint32_t), cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

uint32_t lb200_sortkeys_max_entities(const lb200_sortkeys* sk) { return sk ? sk->max_entities : 0u; }

// createModelInstance + setModel + modelLoaded for a batch of new model instances whose data lies in device memory (SURVEY 8f N1)
int lb200_sortkeys_spawn_instances_device(lb200_sortkeys* sk, const int32_t* dev_entities, const uint32_t* dev_model_of, const lb200_transform* dev_transforms,
	const uint8_t* dev_dirty, uint32_t n, uint32_t max_entity)
{
	if (!sk) return LB200_ERR_INVALID;
	if (!n) return LB200_OK;
	if (!dev_entities || !dev_model_of || !dev_transforms) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	if (!sk->d_models) { lb200_set_error(ctx, "spawn_instances_device needs set_models first"); return LB200_ERR_STATE; }
	if (max_entity > (uint32_t)INT32_MAX) { lb200_set_error(ctx, "spawn_instances_device: max_entity %u is not an entity id", max_entity); return LB200_ERR_INVALID; }
	const char* what = "spawn_instances_device";
	const char* reasons = "an id out of range, an id listed twice or a model index past the model table";
	int rc = spawn_check(sk, dev_entities, n, max_entity, dev_model_of, what, reasons);
	if (!rc) rc = ensure_moved(sk);
	if (rc) return rc;
	spawn_instances_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(sk->d_ent, dev_entities, dev_model_of, dev_transforms, dev_dirty, n, sk->d_models, sk->d_prev, sk->d_refused);
	LB200_CHECK_LAUNCH(ctx);
	rc = spawn_result(sk, what, reasons, max_entity);
	if (!rc) sk->have_transforms = true; // create_keys reads only the records of culled ids: a spawned one holds its transform
	return rc;
}

// createDecal / createCurveDecal + updateDecalInfo for a batch of new decals whose data lies in device memory
int lb200_sortkeys_spawn_decals_device(lb200_sortkeys* sk, const int32_t* dev_entities, const uint32_t* dev_sort_key, const uint8_t* dev_layer, uint32_t n, uint32_t max_entity) {
	if (!sk) return LB200_ERR_INVALID;
	if (!n) return LB200_OK;
	if (!dev_entities || !dev_sort_key || !dev_layer) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	if (max_entity > (uint32_t)INT32_MAX) { lb200_set_error(ctx, "spawn_decals_device: max_entity %u is not an entity id", max_entity); return LB200_ERR_INVALID; }
	const char* what = "spawn_decals_device";
	const char* reasons = "an id out of range or an id listed twice";
	const int rc = spawn_check(sk, dev_entities, n, max_entity, nullptr, what, reasons);
	if (rc) return rc;
	spawn_decals_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(sk->d_decal_sort_key, sk->d_decal_layer, dev_entities, dev_sort_key, dev_layer, n, sk->d_refused);
	LB200_CHECK_LAUNCH(ctx);
	return spawn_result(sk, what, reasons, max_entity);
}

int lb200_sortkeys_clear_dirty_device(lb200_sortkeys* sk, const int32_t* dev_entities, uint32_t n) {
	if (!sk) return LB200_ERR_INVALID;
	if (!n) return LB200_OK;
	if (!dev_entities) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	clear_dirty_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(sk->d_ent, sk->max_entities, dev_entities, n);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}


int lb200_sortkeys_build_palettes(lb200_sortkeys* sk, lb200_animation* const* systems, uint32_t n_systems, int views, lb200_sk_palettes* out) {
	if (!sk) return LB200_ERR_INVALID;
	lb200_ctx* ctx = sk->ctx;
	lb200_range range("PoseProcessor"); // pipeline.cpp:3730
	if (!out || (n_systems && !systems) || (views != 0 && views != 1)) { lb200_set_error(ctx, "build_palettes: no outputs, no system array or views %d not 0 / 1", views); return LB200_ERR_INVALID; }
	std::vector<AnimationPaletteSource> src(n_systems);
	for (uint32_t k = 0; k < n_systems; ++k) {
		if (!systems[k]) { lb200_set_error(ctx, "build_palettes: system %u is NULL", k); return LB200_ERR_INVALID; }
		lb200_animation_internal_palette_source(systems[k], &src[k]);
		if (src[k].ctx != ctx) { lb200_set_error(ctx, "build_palettes: system %u belongs to another context", k); return LB200_ERR_INVALID; }
	}
	{
		std::vector<const lb200_animation*> sorted(systems, systems + n_systems);
		std::sort(sorted.begin(), sorted.end());
		if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) { lb200_set_error(ctx, "build_palettes: a system is listed twice"); return LB200_ERR_INVALID; }
	}
	uint64_t cap = 0; // bones of every instance with an entity id: each feeds one slice at most
	for (uint32_t k = 0; k < n_systems; ++k) {
		if (src[k].n_listed && !src[k].pos) { lb200_set_error(ctx, "build_palettes: system %u has no absolute poses (update with LB200_PALETTE_POSE)", k); return LB200_ERR_STATE; }
		cap += (uint64_t)src[k].n_listed * src[k].bone_count;
	}
	const OutputSet& set = views ? sk->views : sk->plain;
	const uint32_t n_lists = views ? sk->views_n : 1u;
	if (!n_lists || !set.pose_cap) { lb200_set_error(ctx, "build_palettes needs a preceding %s", views ? "create_keys_views" : "create_keys"); return LB200_ERR_STATE; }
	if (cap >= PAL_NONE) { lb200_set_error(ctx, "build_palettes: %llu bones do not fit 32-bit offsets", (unsigned long long)cap); return LB200_ERR_INVALID; }
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	cudaStream_t st = ctx->stream;
	// every buffer before anything is launched or replaced
	const size_t E = sk->max_entities;
	DeviceArray<uint32_t> offset, n_bones; DeviceArray<unsigned long long> map; DeviceArray<float4> dq;
	if (!sk->d_pal_offset) {
		LB200_CUDA(ctx, offset.alloc(E));
		LB200_CUDA(ctx, n_bones.alloc(1));
		LB200_CUDA(ctx, map.alloc(E));
	}
	const size_t have = sk->d_pal_dq.size() / 2;
	if (!sk->d_pal_dq || have < cap) LB200_CUDA(ctx, dq.alloc(2 * grownCapacity(have, 4096, (size_t)cap)));
	if (offset) {
		LB200_CUDA(ctx, cudaMemsetAsync(offset, 0xff, sizeof(uint32_t) * E, st));
		LB200_CUDA(ctx, cudaMemsetAsync(map, 0, sizeof(unsigned long long) * E, st));
		sk->d_pal_offset = std::move(offset); sk->d_pal_n_bones = std::move(n_bones); sk->d_pal_map = std::move(map);
	}
	if (dq) {
		if (sk->d_pal_dq) LB200_CUDA(ctx, cudaStreamSynchronize(st)); // nothing enqueued still writes or reads the old buffer
		sk->d_pal_dq = std::move(dq);
	}
	if (++sk->pal_seq == 0x80000000u) { // the stamps would wrap: no entry may hold the new one already
		LB200_CUDA(ctx, cudaMemsetAsync(sk->d_pal_map, 0, sizeof(unsigned long long) * E, st));
		sk->pal_seq = 1;
	}
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_pal_n_bones, 0, sizeof(uint32_t), st));
	PalParams P = {};
	P.stamp = 2 * sk->pal_seq;
	P.n_lists = n_lists; P.cap_pose = set.pose_cap; P.max_entities = sk->max_entities;
	for (uint32_t v = 0; v < n_lists; ++v) {
		P.list[v] = set.pose_list + (size_t)v * sk->max_entities;
		P.count[v] = set.counts + (size_t)v * CNT_WORDS + CNT_POSE;
	}
	P.map = sk->d_pal_map; P.offset = sk->d_pal_offset; P.dq = sk->d_pal_dq; P.n_bones = sk->d_pal_n_bones;
	// the launches' systems, numbered in list order; the map of every launch goes in before the first build reads it
	const uint32_t n_launches = std::max(1u, (n_systems + PAL_MAX_SYSTEMS - 1) / PAL_MAX_SYSTEMS);
	uint32_t number = 0;
	std::vector<uint32_t> first_number(n_launches + 1, 0);
	for (uint32_t l = 0; l < n_launches; ++l) {
		first_number[l] = number;
		for (uint32_t k = l * PAL_MAX_SYSTEMS; k < std::min(n_systems, (l + 1) * PAL_MAX_SYSTEMS); ++k) number += src[k].n_listed;
	}
	first_number[n_launches] = number;
	auto fill = [&](uint32_t l) {
		P.n_systems = 0;
		uint32_t base = first_number[l], most = 0;
		for (uint32_t k = l * PAL_MAX_SYSTEMS; k < std::min(n_systems, (l + 1) * PAL_MAX_SYSTEMS); ++k) {
			const AnimationPaletteSource& a = src[k];
			PalSystem& S = P.sys[P.n_systems++];
			S.pos = a.pos; S.rot = reinterpret_cast<const float4*>(a.rot); S.inv_bind_pos = a.inv_bind_pos; S.inv_bind_rot = a.inv_bind_rot; S.entity = a.entity;
			S.bone_count = a.bone_count; S.n = a.n_listed; S.base = base;
			base += a.n_listed;
			most = std::max(most, a.n_listed);
		}
		P.first = first_number[l]; P.end = first_number[l + 1];
		return most;
	};
	for (uint32_t l = 0; l < n_launches; ++l) {
		const uint32_t most = fill(l);
		if (!most) continue;
		pal_map_kernel<<<dim3(std::min(256u, (most + PAL_THREADS - 1) / PAL_THREADS), P.n_systems), PAL_THREADS, 0, st>>>(P);
		LB200_CHECK_LAUNCH(ctx);
	}
	const uint64_t listed = (uint64_t)n_lists * set.pose_cap; // the lists' capacity: the counts stay on the device
	const uint32_t per_block = PAL_THREADS / PAL_LANES;
	const uint32_t grid = (uint32_t)std::max<uint64_t>(1, std::min<uint64_t>((uint64_t)ctx->sm_count * 8, (listed + per_block - 1) / per_block));
	for (uint32_t l = 0; l < n_launches; ++l) {
		fill(l);
		P.write_none = l == 0;
		pal_build_kernel<<<grid, PAL_THREADS, 0, st>>>(P);
		LB200_CHECK_LAUNCH(ctx);
	}
	out->dual_quats = reinterpret_cast<const float*>(sk->d_pal_dq.get());
	out->offset = sk->d_pal_offset;
	out->n_bones = sk->d_pal_n_bones;
	return LB200_OK;
}

} // extern "C"
