/* TEST INFRASTRUCTURE — CPU restatement of the consumer of the visible list: PipelineImpl::createSortKeys (sort keys, LOD selection with
 * its smoothing state, auto-instancing groups + instance data) and PipelineImpl::radixSort, on flat arrays.  Never linked into or executed
 * by the product (see oracle_math.h).
 *
 * Reference: src/renderer/pipeline.cpp
 *   :53-60    floatFlip
 *   :62-143   sort key / sort value layout and packers (makeMeshSortKey, makeDepthSortKey, makeAutoInstancedSortKey, makeDecalSortKey,
 *             makeMeshSortValue, makeSkinnedSortValue, makeAutoInstancedSortValue, makeDecalSortValue, makeCurveDecalSortValue)
 *   :452-523  AutoInstancer (groups of renderables per mesh sort key)
 *   :3789-4018 createSortKeys
 *   :4020-4144 Histogram + radixSort (6 stable passes of 11 bits; a pass whose keys all fall into bin 0 is skipped)
 * src/renderer/model.h:173-179 Model::getLODMeshIndices
 *
 * The reference runs createSortKeys on every job worker with one AutoInstancer per worker; the instancer index goes into the sort value
 * of a group (makeAutoInstancedSortValue) and the groups of one mesh are split over the workers.  This restatement is the one-worker
 * run: a single instancer (index 0), every mesh's instances in one group.  Pinned pieces (tests/golden/sortkeys_kat.npz, reference-run):
 * the packers, getLODMeshIndices and radixSort, which oracle/build_ref.py compiles from the reference file itself. */
#include "oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

enum { DRAW_MESH = 0, DRAW_AUTOINSTANCED = 1, DRAW_SKINNED = 2, DRAW_DECAL = 3, DRAW_CURVE_DECAL = 4 }; /* pipeline.cpp:41-51 */
enum { RT_MESH = 0, RT_DECAL = 1, RT_LOCAL_LIGHT = 2, RT_CURVE_DECAL = 3 };                                /* render_module.h:293-301 */

#define SORT_KEY_BUCKET_SHIFT 56
#define SORT_KEY_INSTANCED_FLAG ((uint64_t)1 << 55)
#define SORT_VALUE_INSTANCER_SHIFT 16
#define SORT_VALUE_MESH_IDX_SHIFT 40
#define SORT_VALUE_TYPE_SHIFT 32

/* pipeline.cpp:57-60 */
uint32_t oracle_float_flip(uint32_t float_bits_value) {
	uint32_t mask = (uint32_t)(-(int32_t)(float_bits_value >> 31)) | 0x80000000u;
	return float_bits_value ^ mask;
}
/* :91-93 (the bucket parameter is a u8: a u32 bucket-map entry is truncated on the way in) */
uint64_t oracle_make_mesh_sort_key(uint32_t mesh_sort_key, uint8_t bucket) { return mesh_sort_key | ((uint64_t)bucket << SORT_KEY_BUCKET_SHIFT); }
/* :95-98 */
uint64_t oracle_make_depth_sort_key(float depth_squared, uint8_t bucket) {
	uint32_t bits;
	memcpy(&bits, &depth_squared, 4);
	return oracle_float_flip(bits) | ((uint64_t)bucket << SORT_KEY_BUCKET_SHIFT);
}
/* :100-102 */
uint64_t oracle_make_autoinstanced_sort_key(int32_t instancer_index, uint8_t bucket) {
	return (uint64_t)(int64_t)instancer_index | SORT_KEY_INSTANCED_FLAG | ((uint64_t)bucket << SORT_KEY_BUCKET_SHIFT);
}
/* :83-85 */
uint64_t oracle_make_decal_sort_key(uint32_t material_sort_key, uint8_t bucket) { return material_sort_key | ((uint64_t)bucket << SORT_KEY_BUCKET_SHIFT); }
/* :125-143; EntityPtr::index is an i32: `entity.index | u64` sign-extends it */
uint64_t oracle_make_decal_sort_value(int32_t entity) { return (uint64_t)(int64_t)entity | ((uint64_t)DRAW_DECAL << SORT_VALUE_TYPE_SHIFT); }
uint64_t oracle_make_curve_decal_sort_value(int32_t entity) { return (uint64_t)(int64_t)entity | ((uint64_t)DRAW_CURVE_DECAL << SORT_VALUE_TYPE_SHIFT); }
uint64_t oracle_make_skinned_sort_value(int32_t entity, uint32_t mesh_idx) {
	return (uint64_t)(int64_t)entity | ((uint64_t)DRAW_SKINNED << SORT_VALUE_TYPE_SHIFT) | ((uint64_t)mesh_idx << SORT_VALUE_MESH_IDX_SHIFT);
}
uint64_t oracle_make_mesh_sort_value(int32_t entity, uint32_t mesh_idx) {
	return (uint64_t)(int64_t)entity | ((uint64_t)DRAW_MESH << SORT_VALUE_TYPE_SHIFT) | ((uint64_t)mesh_idx << SORT_VALUE_MESH_IDX_SHIFT);
}
uint64_t oracle_make_autoinstanced_sort_value(uint32_t batch_idx, uint32_t instancer_idx) {
	return batch_idx | (instancer_idx << SORT_VALUE_INSTANCER_SHIFT) | ((uint64_t)DRAW_AUTOINSTANCED << SORT_VALUE_TYPE_SHIFT);
}

/* model.h:173-179 */
uint32_t oracle_lod_mesh_indices(const float* lod_distances4, float squared_distance) {
	if (squared_distance < lod_distances4[0]) return 0;
	if (squared_distance < lod_distances4[1]) return 1;
	if (squared_distance < lod_distances4[2]) return 2;
	if (squared_distance < lod_distances4[3]) return 3;
	return 4;
}

/* pipeline.cpp:4100-4144 (+ the histogram of :4020-4097, which is a plain count): LSD radix sort, 6 passes of 11 bits, stable.
 * reference_copy_back != 0 reproduces the reference's last lines literally (:4140-4143): `if (keys == _keys) memcpy(_keys, keys, ...)` —
 * the copy back to the caller's arrays happens when it is NOT needed and is skipped when the sorted data sits in the temporary buffer,
 * i.e. after an odd number of executed passes the caller sees the state before the last executed pass.  That form exists only to pin this
 * restatement against the reference build (tests/golden/sortkeys_kat.npz); with 0 the caller gets the sorted sequence, which is what
 * the product delivers and what the reference delivers whenever its number of executed passes is even. */
void oracle_radix_sort_ex(uint64_t* keys_io, uint64_t* values_io, uint32_t size, int reference_copy_back) {
	enum { BITS = 11, SIZE = 1 << BITS, MASK = SIZE - 1, PASSES = 6 };
	if (size == 0) return;
	uint64_t* tmp = (uint64_t*)malloc(sizeof(uint64_t) * 2 * (size_t)size);
	uint32_t* hist = (uint32_t*)calloc((size_t)PASSES * SIZE, sizeof(uint32_t));
	uint64_t *keys = keys_io, *values = values_io, *tmp_keys = tmp, *tmp_values = tmp + size;
	for (uint32_t i = 0; i < size; ++i) {
		const uint64_t key = keys[i];
		for (int p = 0; p < PASSES; ++p) ++hist[p * SIZE + (uint16_t)((p == 5 ? (key >> 55) : (key >> (BITS * p))) & (p == 5 ? 0xffffu : MASK))];
	}
	uint16_t shift = 0;
	for (int pass = 0; pass < PASSES; ++pass) {
		uint32_t* h = hist + pass * SIZE;
		uint32_t offset = 0;
		for (int i = 0; i < SIZE; ++i) {
			const uint32_t count = h[i];
			h[i] = offset;
			offset += count;
		}
		if (h[1] != size) { /* :4120: every key in bin 0 -> nothing to move */
			for (uint32_t i = 0; i < size; ++i) {
				const uint64_t key = keys[i];
				const uint16_t index = (uint16_t)((key >> shift) & MASK);
				const uint32_t dest = h[index]++;
				tmp_keys[dest] = key;
				tmp_values[dest] = values[i];
			}
			uint64_t* t;
			t = tmp_keys; tmp_keys = keys; keys = t;
			t = tmp_values; tmp_values = values; values = t;
		}
		shift += BITS;
	}
	if (keys != keys_io && !reference_copy_back) {
		memcpy(keys_io, keys, sizeof(uint64_t) * size);
		memcpy(values_io, values, sizeof(uint64_t) * size);
	}
	free(tmp);
	free(hist);
}
void oracle_radix_sort(uint64_t* keys_io, uint64_t* values_io, uint32_t size) { oracle_radix_sort_ex(keys_io, values_io, size, 0); }

/* ---- createSortKeys on flat inputs ---- */
typedef struct {
	uint64_t* keys; uint64_t* values; uint32_t cap, n;
} Inserter;
static void push(Inserter* s, uint64_t key, uint64_t value) {
	if (s->n < s->cap) { s->keys[s->n] = key; s->values[s->n] = value; }
	++s->n;
}

typedef struct { uint32_t group; uint64_t renderable; } InstRec;

/* Returns 0, or -1 if an output capacity was too small (the counts are still complete).
 * Per entity arrays are indexed by entity id.  group_offset / group_count have max_sort_key + 1 entries; instances of group g are
 * group_renderables / instance_data48 [group_offset[g], group_offset[g] + group_count[g]) in visit order. */
int oracle_create_sort_keys(const uint32_t* visible_ids, const uint8_t* visible_types, uint32_t n_visible, const OTransform* transforms,
	const uint32_t* model_of, float* lod, const uint8_t* flags, uint32_t* pose_frame, const uint32_t* decal_sort_key, const uint8_t* decal_layer,
	const OracleSkModel* models, const OracleSkMesh* meshes, const OracleSkView* view,
	uint64_t* keys, uint64_t* values, uint32_t cap_keys, uint32_t* n_keys,
	uint32_t* group_count, uint32_t* group_offset, uint64_t* group_renderables, uint8_t* instance_data48, uint32_t cap_instances, uint32_t* n_instances,
	uint32_t* pose_list, uint32_t cap_pose, uint32_t* n_pose, uint32_t* dirty_list, uint32_t cap_dirty, uint32_t* n_dirty)
{
	Inserter ins = {keys, values, cap_keys, 0};
	const uint32_t n_groups = view->max_sort_key + 1; /* :3830 instancer.init(getMaxSortKey() + 1) */
	memset(group_count, 0, sizeof(uint32_t) * n_groups);
	size_t cap_recs = (size_t)n_visible * 2 + 64;
	InstRec* recs = (InstRec*)malloc(sizeof(InstRec) * cap_recs);
	uint32_t n_recs = 0, np = 0, nd = 0;
	const float global_lod_multiplier_rcp = 1 / view->lod_multiplier; /* :3798-3799 */
	const float time_delta = view->time_delta;
	const int is_shadow = view->is_shadow != 0;
	const uint32_t frame_number = view->frame_number;

	for (uint32_t vi = 0; vi < n_visible; ++vi) {
		const int32_t e = (int32_t)visible_ids[vi];
		switch (visible_types[vi]) {
			case RT_LOCAL_LIGHT: break; /* :3839 */
			case RT_DECAL:          /* :3840-3853 */
			case RT_CURVE_DECAL: {  /* :3854-3867 */
				const int layer = decal_layer[e];
				const uint8_t bucket = (uint8_t)view->bucket_map[layer];
				if (bucket < 0xff) {
					push(&ins, oracle_make_decal_sort_key(decal_sort_key[e], bucket),
						visible_types[vi] == RT_DECAL ? oracle_make_decal_sort_value(e) : oracle_make_curve_decal_sort_value(e));
				}
				break;
			}
			case RT_MESH: { /* :3868-3956 */
				const OracleSkModel* model = &models[model_of[e]];
				const ODVec3 pos = transforms[e].pos;
				const ODVec3 lrp = {view->lod_ref_point[0], view->lod_ref_point[1], view->lod_ref_point[2]};
				const ODVec3 dd = odv3_sub(pos, lrp);
				const float squared_length = (float)(dd.x * dd.x + dd.y * dd.y + dd.z * dd.z); /* squaredLength(DVec3), math.cpp */
				const uint32_t lod_idx = oracle_lod_mesh_indices(model->lod_distances, squared_length * global_lod_multiplier_rcp);
				if (flags[e] & 2) { /* mi.dirty, :3878-3881 */
					if (nd < cap_dirty) dirty_list[nd] = (uint32_t)e;
					++nd;
					break;
				}
				int lods[2], n_lods = 0;
				if (lod[e] != (float)lod_idx) { /* :3926-3941 */
					const float d = (float)lod_idx - lod[e];
					const float ad = fabsf(d);
					if (ad <= time_delta) {
						lod[e] = (float)lod_idx;
						lods[n_lods++] = (int)lod_idx;
					}
					else {
						if (!is_shadow) lod[e] += d / ad * time_delta;
						const uint32_t cur_lod_idx = (uint32_t)lod[e];
						lods[n_lods++] = (int)cur_lod_idx;
						if (cur_lod_idx < 3) lods[n_lods++] = (int)cur_lod_idx + 1;
					}
				}
				else lods[n_lods++] = (int)lod_idx;
				for (int li = 0; li < n_lods; ++li) { /* create_key, :3883-3924 */
					for (int mesh_idx = model->lod_from[lods[li]]; mesh_idx <= model->lod_to[lods[li]]; ++mesh_idx) {
						const OracleSkMesh* mm = &meshes[model->mesh_base + (uint32_t)mesh_idx];
						const uint32_t bucket = view->bucket_map[mm->layer];
						if (mm->skinned) {
							if (pose_frame[e] != frame_number) { /* the compare-exchange loop of :3890-3897, one thread */
								pose_frame[e] = frame_number;
								if (np < cap_pose) pose_list[np] = (uint32_t)e;
								++np;
							}
							push(&ins, oracle_make_mesh_sort_key(mm->sort_key, (uint8_t)bucket), oracle_make_skinned_sort_value(e, (uint32_t)mesh_idx));
						}
						else if ((flags[e] & 1) && !is_shadow) { /* ModelInstance::MOVED */
							push(&ins, oracle_make_mesh_sort_key(mm->sort_key, (uint8_t)bucket), oracle_make_mesh_sort_value(e, (uint32_t)mesh_idx));
						}
						else if (bucket < 0xff) {
							if (n_recs == cap_recs) { cap_recs *= 2; recs = (InstRec*)realloc(recs, sizeof(InstRec) * cap_recs); }
							recs[n_recs].group = mm->sort_key;
							recs[n_recs].renderable = (uint64_t)(int64_t)e | ((uint64_t)mesh_idx << SORT_VALUE_MESH_IDX_SHIFT); /* :3913 */
							++n_recs;
							++group_count[mm->sort_key];
						}
						else if (bucket < 0xffff) { /* depth sorted, :3915-3922 */
							const ODVec3 cp = {view->camera_pos[0], view->camera_pos[1], view->camera_pos[2]};
							const ODVec3 rel = odv3_sub(pos, cp);
							const float sq = (float)(rel.x * rel.x + rel.y * rel.y + rel.z * rel.z);
							push(&ins, oracle_make_depth_sort_key(sq, (uint8_t)bucket), oracle_make_mesh_sort_value(e, (uint32_t)mesh_idx));
						}
					}
				}
				break;
			}
			default: break;
		}
	}
	/* groups in key order, their instances in visit order (AutoInstancer::add appends, :505-523) */
	uint32_t off = 0;
	for (uint32_t g = 0; g < n_groups; ++g) { group_offset[g] = off; off += group_count[g]; }
	uint32_t* cursor = (uint32_t*)malloc(sizeof(uint32_t) * n_groups);
	memcpy(cursor, group_offset, sizeof(uint32_t) * n_groups);
	const uint32_t first_none = 0xffffffffu;
	uint32_t* first = (uint32_t*)malloc(sizeof(uint32_t) * n_groups);
	for (uint32_t g = 0; g < n_groups; ++g) first[g] = first_none;
	for (uint32_t r = 0; r < n_recs; ++r) {
		const uint32_t g = recs[r].group;
		const uint32_t at = cursor[g]++;
		if (first[g] == first_none) first[g] = r;
		if (at >= cap_instances) continue;
		group_renderables[at] = recs[r].renderable;
		/* fill instance data, :3990-4008: rot (16 B), Vec3(pos - camera_pos) (12 B), lod - mesh.lod (4 B), scale (12 B), material index (4 B) */
		const int32_t e = (int32_t)(recs[r].renderable & 0xffffffffu);
		const uint32_t mesh_idx = (uint32_t)(recs[r].renderable >> SORT_VALUE_MESH_IDX_SHIFT);
		const OracleSkMesh* mm = &meshes[models[model_of[e]].mesh_base + mesh_idx];
		const OTransform* tr = &transforms[e];
		const ODVec3 cp = {view->camera_pos[0], view->camera_pos[1], view->camera_pos[2]};
		const OVec3 lpos = ov3_from_d(odv3_sub(tr->pos, cp));
		const float lod_d = lod[e] - mm->lod; /* the instance's lod after every update of this pass; :3968 mesh_lod is the group's first mesh's */
		uint8_t* dst = instance_data48 + (size_t)at * 48;
		memcpy(dst, &tr->rot, 16);
		memcpy(dst + 16, &lpos, 12);
		memcpy(dst + 28, &lod_d, 4);
		memcpy(dst + 32, &tr->scale, 12);
		memcpy(dst + 44, &mm->material_index, 4);
	}
	/* one sort key per non-empty group, :3958-3969: bucket = layer_to_bucket[layer of the group's first renderable's material] */
	for (uint32_t g = 0; g < n_groups; ++g) {
		if (first[g] == first_none) continue;
		const int32_t e = (int32_t)(recs[first[g]].renderable & 0xffffffffu);
		const uint32_t mesh_idx = (uint32_t)(recs[first[g]].renderable >> SORT_VALUE_MESH_IDX_SHIFT);
		const uint8_t layer = meshes[models[model_of[e]].mesh_base + mesh_idx].layer;
		push(&ins, oracle_make_autoinstanced_sort_key((int32_t)g, view->layer_to_bucket[layer]), oracle_make_autoinstanced_sort_value(g, 0));
	}
	free(first); free(cursor); free(recs);
	*n_keys = ins.n; *n_instances = off; *n_pose = np; *n_dirty = nd;
	return (ins.n > cap_keys || off > cap_instances || np > cap_pose || nd > cap_dirty) ? -1 : 0;
}
