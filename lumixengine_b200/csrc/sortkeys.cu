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
//   create_keys_kernel one cooperative launch (grid = what is co-resident), one thread per visible renderable, grid-stride:
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

// One entity = one 64-byte DRAM burst.  Sector 0 is all a static mesh needs for LOD selection and keys, sector 1 is what instance data adds.
struct alignas(64) SkEntity {
	double pos[3];        // Transform::pos
	uint32_t model_flags; // model index (24 bits) | LB200_SK_* flags << 24
	float lod;            // ModelInstance::lod (smoothing state, updated by the pass)
	float rot[4];         // Transform::rot
	float scale[3];       // Transform::scale
	uint32_t pose_frame;  // Pose::frame (0xffffffff = never)
};
static_assert(sizeof(SkEntity) == 64, "one burst per entity");

struct EmitParams {
	lb200_sk_view view;
	uint32_t type_base[4]; // offsets of the MESH / DECAL / LOCAL_LIGHT / CURVE_DECAL segments inside out_ids
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
	const lb200_sk_model* __restrict__ models; const lb200_sk_mesh* __restrict__ meshes;
	uint64_t* __restrict__ keys; uint64_t* __restrict__ values; uint32_t* counts;
	uint32_t* group_count; uint32_t* group_offset; uint32_t* group_cursor; const uint8_t* __restrict__ group_layer;
	uint64_t* __restrict__ group_renderables; float4* __restrict__ instance_data;
	uint32_t* __restrict__ pose_list; uint32_t* __restrict__ dirty_list; uint32_t* __restrict__ stash; float4* __restrict__ stash4; uint32_t stash_stride;
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
__device__ __forceinline__ uint32_t mesh_count(const EmitParams& P, const EmitArgs& A, const uint32_t* s_bucket_map, uint32_t* s_grp, float lod_multiplier_rcp, int32_t e, uint32_t i, Counts& c) {
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
	const double dx = LB_DSUB(px, P.view.lod_ref_point[0]), dy = LB_DSUB(py, P.view.lod_ref_point[1]), dz = LB_DSUB(pz, P.view.lod_ref_point[2]);
	const float squared_length = (float)LB_DADD(LB_DADD(LB_DMUL(dx, dx), LB_DMUL(dy, dy)), LB_DMUL(dz, dz)); // squaredLength(DVec3), math.cpp:397
	const float sd = LB_FMUL(squared_length, lod_multiplier_rcp);
	const uint32_t lod_idx = sd < model.lod_distances[0] ? 0u : sd < model.lod_distances[1] ? 1u : sd < model.lod_distances[2] ? 2u : sd < model.lod_distances[3] ? 3u : 4u;
	const bool is_shadow = P.view.is_shadow != 0;
	uint32_t lod0 = lod_idx;
	bool two = false;
	if (cur != (float)lod_idx) { // :3926-3941
		const float d = LB_FSUB((float)lod_idx, cur);
		const float ad = fabsf(d);
		if (ad <= P.view.time_delta) cur = (float)lod_idx;
		else {
			if (!is_shadow) cur = LB_FADD(cur, LB_FMUL(LB_FDIV(d, ad), P.view.time_delta));
			lod0 = (uint32_t)cur;
			two = lod0 < 3;
		}
		rec->lod = cur;
	}
	// what pass 2 writes per auto-instanced mesh (:3990-4008) or depth-sorted key (:3915-3922), stashed next to the decision in arrays indexed
	// like the visible list: pass 2 reads them coalesced and never touches the record again
	const double rx = LB_DSUB(px, P.view.camera_pos[0]), ry = LB_DSUB(py, P.view.camera_pos[1]), rz = LB_DSUB(pz, P.view.camera_pos[2]);
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
			else warp_claim_keyed(A.group_count, mm.sort_key);
		}
	}
	// once per instance and frame the palette has to be built (PoseProcessor::push; the compare-exchange on Pose::frame of :3890-3897 —
	// one thread owns the instance within a view)
	if (any_skinned && (uint32_t)q3.w != P.view.frame_number) { rec->pose_frame = P.view.frame_number; code |= CODE_POSE; ++c.p; }
	return code;
}

__device__ __forceinline__ void push_key(const EmitParams& P, const EmitArgs& A, uint32_t& slot, uint64_t key, uint64_t value) {
	if (slot < P.cap_keys) { A.keys[slot] = key; A.values[slot] = value; }
	++slot;
}

// MESH renderable, pass 2: replay of the stashed decision, writes
__device__ __forceinline__ void mesh_write(const EmitParams& P, const EmitArgs& A, const uint32_t* s_bucket_map, uint32_t* s_grp, int32_t e, uint32_t i, uint32_t code, uint32_t& k, uint32_t& p) {
	if (code & CODE_DIRTY) { // queueMaterialOverrideRefresh (rare: its own atomic)
		const uint32_t slot = atomicAdd(&A.counts[CNT_DIRTY], 1u);
		if (slot < P.cap_dirty) A.dirty_list[slot] = (uint32_t)e;
		return;
	}
	const lb200_sk_model model = load_model(A.models + (code & CODE_MODEL_MASK));
	const bool moved_not_shadow = (code & CODE_MOVED) && P.view.is_shadow == 0;
	const uint32_t lod0 = (code >> CODE_LOD_SHIFT) & 7u;
	const bool two = (code & CODE_TWO) != 0;
	if (code & CODE_POSE) {
		if (p < P.cap_pose) A.pose_list[p] = (uint32_t)e;
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
			push_key(P, A, k, low | ((uint64_t)(uint8_t)bucket << SORT_KEY_BUCKET_SHIFT), mesh_value | ((uint64_t)(kind.skinned ? DRAW_SKINNED : DRAW_MESH) << SORT_VALUE_TYPE_SHIFT));
		}
		if (kind.inst) { // instance data of the auto-instanced mesh, :3990-4008, at the group's offset + this block's slice + rank
			const uint32_t at = s_grp ? atomicAdd(&s_grp[mm.sort_key], 1u) : warp_claim_keyed(A.group_cursor, mm.sort_key);
			if (at < P.cap_recs) {
				__stcs(reinterpret_cast<unsigned long long*>(A.group_renderables) + at, (unsigned long long)mesh_value);
				float4* dst = A.instance_data + (size_t)at * 3;
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

__global__ void __launch_bounds__(SK_THREADS, 4) create_keys_kernel(const __grid_constant__ EmitParams P, const uint32_t* __restrict__ visible,
	const uint32_t* __restrict__ cull_counters, EmitArgs A, uint32_t n_groups)
{
	extern __shared__ uint32_t s_grp_mem[];
	__shared__ uint32_t s_warp[SK_THREADS / 32];
	__shared__ uint32_t s_base[2];
	__shared__ uint32_t s_carry;
	__shared__ uint32_t s_bucket_map[256];
	s_bucket_map[threadIdx.x] = P.view.bucket_map[threadIdx.x]; // SK_THREADS == 256
	uint32_t* s_grp = n_groups <= SK_SMEM_GROUPS ? s_grp_mem : nullptr;
	if (s_grp) for (uint32_t g = threadIdx.x; g < n_groups; g += SK_THREADS) s_grp[g] = 0;
	__syncthreads();
	// the three segments as one index space: [MESH | DECAL | CURVE_DECAL]
	const uint32_t n_mesh = __ldg(cull_counters + RT_MESH), n_decal = __ldg(cull_counters + RT_DECAL), n_curve = __ldg(cull_counters + RT_CURVE_DECAL);
	const uint32_t n_all = n_mesh + n_decal + n_curve;
	const float lod_multiplier_rcp = LB_FDIV(1.0f, P.view.lod_multiplier); // :3798-3799
	const uint32_t stride = gridDim.x * SK_THREADS;

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
			if (i < n_mesh) A.stash[i] = mesh_count(P, A, s_bucket_map, s_grp, lod_multiplier_rcp, (int32_t)e, i, c);
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
		s_base[0] = tk ? atomicAdd(&A.counts[CNT_KEYS], tk) : 0u;
		s_base[1] = tp ? atomicAdd(&A.counts[CNT_POSE], tp) : 0u;
	}
	// the block's slice of every group it has instances of: count -> start inside the group
	if (s_grp) for (uint32_t g = threadIdx.x; g < n_groups; g += SK_THREADS) if (s_grp[g]) s_grp[g] = atomicAdd(&A.group_count[g], s_grp[g]);
	uint32_t barriers_passed = 0;
	grid_barrier(A.bar, barriers_passed); // every block's counts are in: group totals are final

	// ---- group offsets = exclusive scan of the group totals; block 0 publishes them and one key/value per non-empty group (:3958-3969) ----
	if (s_grp || blockIdx.x == 0) {
		if (threadIdx.x == 0) s_carry = 0;
		__syncthreads();
		for (uint32_t base = 0; base < n_groups; base += SK_THREADS) {
			const uint32_t g = base + threadIdx.x;
			const uint32_t cnt = g < n_groups ? __ldcg(A.group_count + g) : 0u;
			uint32_t total;
			const uint32_t carry = s_carry; // read before the scan's barriers: thread 0 moves it on behind them
			const uint32_t off = carry + block_exclusive_scan(cnt, s_warp, &total);
			if (g < n_groups) {
				if (s_grp) s_grp[g] += off; // cursor of this block inside the group, absolute
				if (blockIdx.x == 0) {
					A.group_offset[g] = off;
					if (!s_grp) A.group_cursor[g] = off;
					if (cnt) {
						const uint32_t slot = atomicAdd(&A.counts[CNT_KEYS], 1u);
						if (slot < P.cap_keys) {
							A.keys[slot] = (uint64_t)g | SORT_KEY_INSTANCED_FLAG | ((uint64_t)P.view.layer_to_bucket[A.group_layer[g]] << SORT_KEY_BUCKET_SHIFT); // :100-102
							A.values[slot] = (uint64_t)g | ((uint64_t)0 << SORT_VALUE_INSTANCER_SHIFT) | ((uint64_t)DRAW_AUTOINSTANCED << SORT_VALUE_TYPE_SHIFT); // :141-143
						}
					}
				}
			}
			if (threadIdx.x == 0) s_carry += total;
			__syncthreads();
		}
		if (blockIdx.x == 0 && threadIdx.x == 0) { A.counts[CNT_INST] = s_carry; A.counts[CNT_RECS] = s_carry; }
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
			if (i < n_mesh) mesh_write(P, A, s_bucket_map, s_grp, (int32_t)e, i, A.stash[i], k, p);
			else {
				const bool curve = i >= n_mesh + n_decal;
				const uint32_t bucket = A.stash[i];
				if (bucket < 0xff) push_key(P, A, k, (uint64_t)__float_as_uint(A.stash4[i].x) | ((uint64_t)bucket << SORT_KEY_BUCKET_SHIFT),
					sext((int32_t)e) | ((uint64_t)(curve ? DRAW_CURVE_DECAL : DRAW_DECAL) << SORT_VALUE_TYPE_SHIFT));
			}
			e = e_next;
		}
	}
}

// ---- per-entity records: packing what the caller hands over as arrays, unpacking the state the pass keeps ----
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
		if (flags) mf = (mf & CODE_MODEL_MASK) | ((uint32_t)flags[i] << 24);
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
	const uint32_t before = atomicOr(&r.model_flags, (uint32_t)LB200_SK_MOVED << 24);
	if (!(before & ((uint32_t)LB200_SK_MOVED << 24))) moved_list[atomicAdd(moved_count, 1u)] = e; // m_moved_instances.push(entity), once
}

// RenderModuleImpl::endFrame (render_module.cpp:526-534): MOVED off, prev_frame_transform = the transform of this frame
__global__ void __launch_bounds__(256) ent_end_frame_kernel(SkEntity* ent, const uint32_t* __restrict__ moved_list, uint32_t* moved_count, lb200_transform* __restrict__ prev) {
	const uint32_t n = *moved_count;
	for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
		const uint32_t e = moved_list[i];
		SkEntity& r = ent[e];
		r.model_flags &= ~((uint32_t)LB200_SK_MOVED << 24);
		lb200_transform t;
		t.pos[0] = r.pos[0]; t.pos[1] = r.pos[1]; t.pos[2] = r.pos[2];
		t.rot[0] = r.rot[0]; t.rot[1] = r.rot[1]; t.rot[2] = r.rot[2]; t.rot[3] = r.rot[3];
		t.scale[0] = r.scale[0]; t.scale[1] = r.scale[1]; t.scale[2] = r.scale[2];
		prev[e] = t;
	}
}
__global__ void reset_word_kernel(uint32_t* w) { *w = 0; }

} // namespace

constexpr uint32_t NO_MODEL = 0xffffffffu;

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
	// outputs
	DeviceArray<uint64_t> d_keys[2], d_values[2];
	DeviceArray<uint32_t> d_counts; PinnedArray<uint32_t> h_counts;
	DeviceArray<uint32_t> d_group_count, d_group_offset, d_group_cursor;
	DeviceArray<uint64_t> d_group_renderables; DeviceArray<float4> d_instance_data;
	DeviceArray<uint32_t> d_pose_list, d_dirty_list, d_stash; DeviceArray<float4> d_stash4; // the two passes' hand-over: one word + 3 x float4 per visible renderable
	DeviceArray<float> d_lod; DeviceArray<uint32_t> d_pose_frame; // unpacked on request (lb200_sortkeys_device_outputs)
	DeviceArray<uint32_t> d_moved_list, d_moved_count; DeviceArray<lb200_transform> d_prev; // RenderModule::m_moved_instances, ModelInstance::prev_frame_transform (first move onwards)
	DeviceArray<GridBar> d_bar;
	RadixSortScratch radix_scratch; // the sort of d_keys / d_values, with d_keys[1] / d_values[1] as its alternate buffers
	uint32_t last_groups = 0;
	uint32_t max_mesh_sort_key = 0; // largest sort key of the mesh table: every view's max_sort_key must reach it
	uint32_t model_past_table = NO_MODEL; // first model whose meshes leave the mesh table (create_keys refuses to launch), NO_MODEL if none
	char past_table_text[128] = {};
	uint32_t keys_grid_limit[2] = {0, 0}; // co-resident blocks of create_keys_kernel: group counters in shared memory / in HBM
	// lb200_sortkeys_set_launch (blocks 0 = environment switch, else 2 per SM; -1 = all co-resident; prefetch -1 = environment switch) and
	// what the last create_keys launched
	int launch_blocks = 0, launch_prefetch = -1;
	uint32_t last_grid = 0, last_prefetch = 0;
	int last_in_smem = 0;
};

namespace {
// host array (may be null: nothing to upload) -> temporary device buffer on the context stream (setters are not on the per-frame path)
template <typename T> int upload_temp(lb200_ctx* ctx, const T* host, size_t n, DeviceArray<T>& dev) {
	if (!host) return LB200_OK;
	LB200_CUDA(ctx, dev.alloc(n));
	LB200_CUDA(ctx, cudaMemcpyAsync(dev, host, sizeof(T) * n, cudaMemcpyHostToDevice, ctx->stream));
	return LB200_OK;
}
} // namespace

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
	for (int b = 0; b < 2; ++b) {
		LB200_CUDA(ctx, sk->d_keys[b].alloc(sk->cap_keys));
		LB200_CUDA(ctx, sk->d_values[b].alloc(sk->cap_keys));
	}
	LB200_CUDA(ctx, sk->d_counts.alloc(CNT_WORDS));
	LB200_CUDA(ctx, sk->h_counts.alloc(CNT_WORDS));
	LB200_CUDA(ctx, sk->d_group_count.alloc(max_groups));
	LB200_CUDA(ctx, sk->d_group_offset.alloc(max_groups));
	LB200_CUDA(ctx, sk->d_group_cursor.alloc(max_groups));
	LB200_CUDA(ctx, sk->d_group_layer.alloc(max_groups));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_group_layer, 0, max_groups, ctx->stream));
	LB200_CUDA(ctx, sk->d_group_renderables.alloc(sk->cap_recs));
	LB200_CUDA(ctx, sk->d_instance_data.alloc(3 * (size_t)sk->cap_recs)); // 48 bytes per instance
	LB200_CUDA(ctx, sk->d_pose_list.alloc(E));
	LB200_CUDA(ctx, sk->d_dirty_list.alloc(E));
	LB200_CUDA(ctx, sk->d_stash.alloc(E));
	LB200_CUDA(ctx, sk->d_stash4.alloc(3 * E));
	LB200_CUDA(ctx, sk->d_bar.alloc(1));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_bar, 0, sizeof(GridBar), ctx->stream));
	const int rc = lb200_radix_sort_alloc_scratch(ctx, (uint32_t)ctx->sm_count * 2, sk->radix_scratch);
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
	if (view->max_sort_key >= sk->max_groups) { lb200_set_error(ctx, "view.max_sort_key %u >= max_groups %u", view->max_sort_key, sk->max_groups); return LB200_ERR_INVALID; }
	if (sk->model_past_table != NO_MODEL) { lb200_set_error(ctx, "create_keys: %s", sk->past_table_text); return LB200_ERR_INVALID; }
	if (view->max_sort_key < sk->max_mesh_sort_key) { lb200_set_error(ctx, "view.max_sort_key %u < sort key %u of the mesh table", view->max_sort_key, sk->max_mesh_sort_key); return LB200_ERR_INVALID; }
	const uint32_t *visible = nullptr, *cull_counters = nullptr, *type_base = nullptr, *type_counts = nullptr;
	int rc = lb200_culling_internal_last(cs, &visible, &cull_counters, &type_base, &type_counts);
	if (rc) return rc;
	// the kernel indexes the entity records, the decal arrays and the stash by the culled ids without a bounds check
	const uint32_t entity_range = lb200_culling_internal_entity_range(cs);
	if (entity_range > sk->max_entities) { lb200_set_error(ctx, "the culling system holds entity ids up to %u, max_entities is %u", entity_range - 1, sk->max_entities); return LB200_ERR_INVALID; }
	cudaStream_t s = ctx->stream;
	uint32_t n_groups = view->max_sort_key + 1;
	sk->last_groups = n_groups;
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_counts, 0, sizeof(uint32_t) * CNT_WORDS, s));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_group_count, 0, sizeof(uint32_t) * n_groups, s));
	LB200_CUDA(ctx, cudaMemsetAsync(sk->d_bar, 0, sizeof(GridBar), s));
	EmitParams EP;
	EP.view = *view;
	for (int t = 0; t < 4; ++t) EP.type_base[t] = type_base[t];
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
	const uint32_t work = type_counts[RT_MESH] + type_counts[RT_DECAL] + type_counts[RT_CURVE_DECAL]; // upper bound of visible renderables
	static const uint32_t blocks_per_sm = [] { const char* e = getenv("LB200_SK_BLOCKS_PER_SM"); const int v = e ? atoi(e) : 2; return (uint32_t)std::max(0, v); }(); // fewer resident blocks than fit (0 = all): 2 is fastest on H100
	uint32_t grid = std::max(1u, std::min(blocks_per_sm ? std::min(limit, blocks_per_sm * (uint32_t)ctx->sm_count) : limit, (work + SK_THREADS - 1) / SK_THREADS));
	if (sk->launch_blocks < 0) grid = limit; // lb200_sortkeys_set_launch: not capped by the work, so that threads with nothing to do still take part
	else if (sk->launch_blocks > 0) grid = std::min((uint32_t)sk->launch_blocks, limit);
	EmitArgs EA = {sk->d_ent, sk->d_decal_sort_key, sk->d_decal_layer, sk->d_models, sk->d_meshes, sk->d_keys[0], sk->d_values[0], sk->d_counts,
		sk->d_group_count, sk->d_group_offset, sk->d_group_cursor, sk->d_group_layer, sk->d_group_renderables, sk->d_instance_data, sk->d_pose_list, sk->d_dirty_list, sk->d_stash, sk->d_stash4, sk->max_entities, sk->d_bar};
	void* args[] = {&EP, &visible, &cull_counters, &EA, &n_groups};
	LB200_CUDA(ctx, cudaLaunchCooperativeKernel((const void*)create_keys_kernel, dim3(grid), dim3(SK_THREADS), args, smem, s));
	LB200_CHECK_LAUNCH(ctx);
	sk->last_grid = grid; sk->last_in_smem = in_smem ? 1 : 0; sk->last_prefetch = EP.prefetch_ahead;
	if (sort) {
		lb200_range r2("radixSort"); // pipeline.cpp:4101
		rc = lb200_radix_sort_pairs(ctx, s, sk->d_keys[0], sk->d_keys[1], sk->d_values[0], sk->d_values[1], sk->d_counts + CNT_KEYS, sk->cap_keys, sk->radix_scratch, 0, false, nullptr);
		if (rc) return rc;
	}
	if (want_counts) {
		if (!result) return LB200_ERR_INVALID;
		LB200_CUDA(ctx, cudaMemcpyAsync(sk->h_counts, sk->d_counts, sizeof(uint32_t) * CNT_WORDS, cudaMemcpyDeviceToHost, s));
		LB200_CUDA(ctx, cudaStreamSynchronize(s));
		result->n_keys = sk->h_counts[CNT_KEYS]; result->n_instances = sk->h_counts[CNT_INST]; result->n_pose = sk->h_counts[CNT_POSE];
		result->n_dirty = sk->h_counts[CNT_DIRTY]; result->n_groups = n_groups;
		if (result->n_keys > sk->cap_keys || sk->h_counts[CNT_RECS] > sk->cap_recs) { lb200_set_error(ctx, "create_keys: %u keys / %u instances exceed the capacities %u / %u", result->n_keys, sk->h_counts[CNT_RECS], sk->cap_keys, sk->cap_recs); return LB200_ERR_CAPACITY; }
	}
	return LB200_OK;
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
	lb200_ctx* ctx = sk->ctx;
	if (!sk->d_lod || !sk->d_pose_frame) {
		DeviceArray<float> lod; DeviceArray<uint32_t> pose_frame;
		LB200_CUDA(ctx, lod.alloc(sk->max_entities));
		LB200_CUDA(ctx, pose_frame.alloc(sk->max_entities));
		sk->d_lod = std::move(lod); sk->d_pose_frame = std::move(pose_frame);
	}
	ent_unpack_state_kernel<<<(sk->max_entities + 255) / 256, 256, 0, ctx->stream>>>(sk->d_ent, sk->max_entities, sk->d_lod, sk->d_pose_frame);
	LB200_CHECK_LAUNCH(ctx);
	out->keys = sk->d_keys[0]; out->values = sk->d_values[0]; out->group_count = sk->d_group_count; out->group_offset = sk->d_group_offset;
	out->group_renderables = sk->d_group_renderables; out->instance_data = sk->d_instance_data; out->pose_list = sk->d_pose_list; out->dirty_list = sk->d_dirty_list;
	out->lod = sk->d_lod; out->pose_frame = sk->d_pose_frame;
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
	if (!sk->d_moved_list || !sk->d_moved_count || !sk->d_prev) { // end_frame tests d_moved_list alone: all three or none
		DeviceArray<uint32_t> moved_list, moved_count; DeviceArray<lb200_transform> prev;
		LB200_CUDA(ctx, moved_list.alloc(sk->max_entities));
		LB200_CUDA(ctx, moved_count.alloc(1));
		LB200_CUDA(ctx, cudaMemsetAsync(moved_count, 0, sizeof(uint32_t), ctx->stream));
		LB200_CUDA(ctx, prev.alloc(sk->max_entities));
		LB200_CUDA(ctx, cudaMemsetAsync(prev, 0, sizeof(lb200_transform) * (size_t)sk->max_entities, ctx->stream));
		sk->d_moved_list = std::move(moved_list); sk->d_moved_count = std::move(moved_count); sk->d_prev = std::move(prev);
	}
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

// ModelInstance::prev_frame_transform per entity (device array, zero until an instance has been through move + end_frame), valid while sk lives
int lb200_sortkeys_prev_transforms(lb200_sortkeys* sk, const lb200_transform** dev_prev) {
	if (!sk || !dev_prev) return LB200_ERR_INVALID;
	*dev_prev = sk->d_prev;
	return LB200_OK;
}

} // extern "C"
