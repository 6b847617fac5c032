/* TEST INFRASTRUCTURE — CPU restatement of root motion in the pose path (see oracle_math.h for the rules of use), built into
 * oracle/liboracle_root_motion.so by oracle/Makefile on top of the pose restatement of oracle_anim.c
 * (liboracle_lumix.so) and the IK restatement of oracle_ik.c (liboracle_ik.so):
 *
 *   src/animation/animation.cpp:214-270   Animation::setRootMotionBone on a freshly loaded Animation (oracle_root_motion_tables)
 *   src/animation/animation.cpp:97-115    AnimationSampler::maskRootMotion
 *   src/animation/animation.cpp:336-364   Animation::getRotation (unpackChannel through double)
 *   src/animation/animation.cpp:30-95     AnimationSampler::getRotation, pose_rotations for the root-motion track (:33-37)
 *   src/animation/animation.cpp:117-204   AnimationSampler::getRelativePose<mask=false, weight>, pose_translations for the root-motion
 *                                         track through Animation::getTranslation (:318-321)
 *   src/animation/controller.cpp:142-157, 267-293  getPose / evalBlendStack, as oracle_pose_stack_ik (oracle_stack_rm)
 */
#include <stdlib.h>

#include "oracle.h"

enum { RM_Y = 1, RM_XZ = 2, RM_ROT = 4 }; /* Animation::Flags, animation.h:73-78 */

/* one clip's root motion as lb200_root_motion: flags, translation track, rotation track */
typedef struct { uint32_t flags; int32_t translation_track; int32_t rotation_track; } OracleRootMotion;

void oracle_eval_ik(const OracleSkeleton* sk, float alpha, OVec3 target, uint32_t leaf, uint32_t bones_count, OVec3* pos, OQuat* rot);

static inline float o_max(float a, float b) { return a > b ? a : b; } /* math.h */
static inline float o_min(float a, float b) { return a < b ? a : b; }

/* math.cpp:378-389 normalize(Quat) */
static inline OQuat oquat_normalize(OQuat q) {
	const float inv_len = 1 / sqrtf(q.x * q.x + q.y * q.y + q.z * q.z + q.w * q.w);
	return oquat(q.x * inv_len, q.y * inv_len, q.z * inv_len, q.w * inv_len);
}

/* animation.cpp:313-316 unpackChannel */
static inline float o_unpack_channel(uint64_t val, float min, float to_float_range, uint32_t bitsize) {
	const uint64_t mask = ((uint64_t)1 << bitsize) - 1;
	return (float)(min + to_float_range * (double)(val & mask));
}

/* animation.cpp:336-364 Animation::getRotation of one packed sample, already shifted to its first bit: unpackChannel (through double) per
 * channel, then the smallest-three reconstruction */
static inline OQuat o_unpack_rotation_d(uint64_t packed, const float* min, const float* to_range, const uint8_t* bitsizes, uint8_t skipped_channel) {
	const int is_negative = (int)(packed & 1);
	packed >>= 1;
	OVec3 v;
	v.x = o_unpack_channel(packed, min[0], to_range[0], bitsizes[0]);
	packed >>= bitsizes[0];
	v.y = o_unpack_channel(packed, min[1], to_range[1], bitsizes[1]);
	packed >>= bitsizes[1];
	v.z = o_unpack_channel(packed, min[2], to_range[2], bitsizes[2]);
	const float rem = 1 - ov3_dot(v, v);
	const float skipped = sqrtf(0.f > rem ? 0.f : rem) * (is_negative ? -1 : 1); /* maximum(0.f, x), math.h */
	switch (skipped_channel) {
		case 0: return oquat(skipped, v.x, v.y, v.z);
		case 1: return oquat(v.x, skipped, v.y, v.z);
		case 2: return oquat(v.x, v.y, skipped, v.z);
		default: return oquat(v.x, v.y, v.z, skipped);
	}
}

static inline uint64_t load_u64(const uint8_t* p) {
	uint64_t v;
	memcpy(&v, p, sizeof(v));
	return v;
}

/* animation.cpp:322-334 Animation::getTranslation of the packed track */
static OVec3 packed_translation(const OracleClip* c, uint32_t frame, const OracleTrack* track) {
	const uint32_t offset = c->translations_frame_size_bits * frame + track->offset_bits;
	uint64_t tmp = load_u64(&c->translation_stream[offset / 8]);
	tmp >>= offset & 7;
	OVec3 res;
	res.x = o_unpack_channel(tmp, track->min[0], track->to_range[0], track->bitsizes[0]);
	tmp >>= track->bitsizes[0];
	res.y = o_unpack_channel(tmp, track->min[1], track->to_range[1], track->bitsizes[1]);
	tmp >>= track->bitsizes[1];
	res.z = o_unpack_channel(tmp, track->min[2], track->to_range[2], track->bitsizes[2]);
	return res;
}

/* animation.cpp:338-364 Animation::getRotation of the packed track */
static OQuat packed_rotation_d(const OracleClip* c, uint32_t frame, const OracleTrack* track) {
	const uint32_t offset = c->rotations_frame_size_bits * frame + track->offset_bits;
	uint64_t packed = load_u64(&c->rotation_stream[offset / 8]);
	packed >>= offset & 7;
	return o_unpack_rotation_d(packed, track->min, track->to_range, track->bitsizes, track->skipped_channel);
}

/* animation.cpp:97-115 */
static OLocalRigidTransform mask_root_motion(uint32_t flags, OLocalRigidTransform t) {
	OLocalRigidTransform rm;
	rm.pos = ov3(0, 0, 0);
	rm.rot = oquat(0, 0, 0, 1);
	if (flags & RM_Y) rm.pos.y = t.pos.y;
	if (flags & RM_XZ) {
		rm.pos.x = t.pos.x;
		rm.pos.z = t.pos.z;
	}
	if (flags & RM_ROT) {
		rm.rot.y = t.rot.y;
		rm.rot.w = t.rot.w;
		rm.rot = oquat_normalize(rm.rot);
	}
	return rm;
}

/* animation.cpp:214-270 setRootMotionBone on a freshly loaded Animation whose m_flags are `flags` and whose root-motion bone's first
 * animated tracks are t / r (-1: none): pose_t / pose_r[frame_count + 1] receive pose_translations / pose_rotations.  Returns 0 when the
 * call returns early (:216, no root-motion flag) and the clip keeps its packed tracks, 1 otherwise. */
int oracle_root_motion_tables(const OracleClip* c, uint32_t flags, int32_t t, int32_t r, OVec3* pose_t, OQuat* pose_r) {
	if ((flags & (RM_Y | RM_XZ | RM_ROT)) == 0) return 0;
	const int have_translations = t >= 0 && (flags & (RM_Y | RM_XZ)); /* :240-246: the arrays are sized, or left empty */
	const int have_rotations = r >= 0 && (flags & RM_ROT);
	OVec3 translation0 = ov3(0, 0, 0);
	OQuat rotation0 = oquat(0, 0, 0, 1);
	for (uint32_t f = 0; f < c->frame_count + 1; ++f) {
		OLocalRigidTransform tmp;
		tmp.pos = ov3(0, 0, 0);
		tmp.rot = oquat(0, 0, 0, 1);
		if (t >= 0) tmp.pos = packed_translation(c, f, &c->translations[t]);
		if (r >= 0) tmp.rot = packed_rotation_d(c, f, &c->rotations[r]);
		const OLocalRigidTransform rm = mask_root_motion(flags, tmp);
		if (f == 0) {
			translation0 = rm.pos;
			rotation0 = rm.rot;
		}
		OLocalRigidTransform rm0;
		rm0.pos = have_translations ? translation0 : ov3(0, 0, 0);
		rm0.rot = have_rotations ? rotation0 : oquat(0, 0, 0, 1);
		tmp = olrt_mul(olrt_mul(rm0, olrt_inverted(rm)), tmp); /* :257 */
		pose_t[f] = tmp.pos;
		pose_r[f] = tmp.rot;
	}
	return 1;
}

/* a clip and its root-motion tables: the track indices the sampler substitutes (-1: none) */
typedef struct {
	const OracleClip* clip;
	int32_t t, r;
	OVec3* pose_t;
	OQuat* pose_r;
} RmClip;

static OVec3 get_translation(const RmClip* c, uint32_t frame, uint32_t track) {
	if ((int32_t)track == c->t) return c->pose_t[frame]; /* :321 */
	return packed_translation(c->clip, frame, &c->clip->translations[track]);
}

/* animation.cpp:30-95 (float unpack, simd_nlerp of the two frames) */
static OQuat get_rotation(const RmClip* rc, uint32_t frame, uint32_t track_idx, float t) {
	if ((int32_t)track_idx == rc->r) return oquat_simd_nlerp(rc->pose_r[frame], rc->pose_r[frame + 1], t); /* :33-37 */
	const OracleClip* c = rc->clip;
	const OracleTrack* track = &c->rotations[track_idx];
	OQuat q[2];
	for (int k = 0; k < 2; ++k) {
		const uint32_t offset = c->rotations_frame_size_bits * (frame + k) + track->offset_bits;
		uint64_t packed = load_u64(&c->rotation_stream[offset / 8]);
		packed >>= offset & 7;
		const int is_negative = (int)(packed & 1);
		packed >>= 1;
		const uint64_t mask_x = ((uint64_t)1 << track->bitsizes[0]) - 1;
		const uint64_t mask_y = ((uint64_t)1 << track->bitsizes[1]) - 1;
		const uint64_t mask_z = ((uint64_t)1 << track->bitsizes[2]) - 1;
		const uint64_t packed_y = packed >> track->bitsizes[0];
		const uint64_t packed_z = packed_y >> track->bitsizes[1];
		OVec3 v;
		v.x = track->min[0] + track->to_range[0] * (float)(packed & mask_x);
		v.y = track->min[1] + track->to_range[1] * (float)(packed_y & mask_y);
		v.z = track->min[2] + track->to_range[2] * (float)(packed_z & mask_z);
		const float skipped = sqrtf(o_max(0.f, 1 - ov3_dot(v, v))) * (is_negative ? -1 : 1);
		switch (track->skipped_channel) {
			case 0: q[k] = oquat(skipped, v.x, v.y, v.z); break;
			case 1: q[k] = oquat(v.x, skipped, v.y, v.z); break;
			case 2: q[k] = oquat(v.x, v.y, skipped, v.z); break;
			default: q[k] = oquat(v.x, v.y, v.z, skipped); break;
		}
	}
	return oquat_simd_nlerp(q[0], q[1], t);
}

/* animation.cpp:117-204 with use_mask = false; the weighted form when weight < 0.9999 (:294-311) */
static void sample(const RmClip* rc, uint32_t time_ticks, float weight, OVec3* pos, OQuat* rot) {
	const OracleClip* anim = rc->clip;
	const int use_weight = weight < 0.9999f;
	const float frame = (float)(time_ticks / (double)(1 << 15) * anim->fps);
	const float s = o_min(o_max(frame, 0.f), (float)anim->frame_count - 0.00001f);
	const uint32_t idx = (uint32_t)s;
	const float t = s - (float)idx;
	for (uint32_t i = 0; i < anim->n_const_translations; ++i) {
		const OracleConstTranslation* track = &anim->const_translations[i];
		const OVec3 v = ov3(track->value[0], track->value[1], track->value[2]);
		pos[track->bone_index] = use_weight ? ov3_lerp(pos[track->bone_index], v, weight) : v;
	}
	for (uint32_t i = 0; i < anim->n_translations; ++i) {
		const uint32_t b = anim->translations[i].bone_index;
		const OVec3 p = ov3_lerp(get_translation(rc, idx, i), get_translation(rc, idx + 1, i), t);
		pos[b] = use_weight ? ov3_lerp(pos[b], p, weight) : p;
	}
	for (uint32_t i = 0; i < anim->n_const_rotations; ++i) {
		const OracleConstRotation* track = &anim->const_rotations[i];
		const OQuat v = oquat(track->value[0], track->value[1], track->value[2], track->value[3]);
		rot[track->bone_index] = use_weight ? oquat_simd_nlerp(rot[track->bone_index], v, weight) : v;
	}
	for (uint32_t i = 0; i < anim->n_rotations; ++i) {
		const uint32_t b = anim->rotations[i].bone_index;
		const OQuat q = get_rotation(rc, idx, i, t);
		rot[b] = use_weight ? oquat_simd_nlerp(rot[b], q, weight) : q;
	}
}

/* The relative pose of Model::getRelativePose + the samples in order, with IK ops between them (as oracle_pose_stack_ik), over clips
 * with root motion (rm[c] per clip, as lb200_root_motion), then Pose::computeAbsolute.  Each sample's time is taken as getPose takes it
 * (time % length when looped, else min(time, length)).  Returns -1 when the tables cannot be allocated. */
int oracle_stack_rm(const OracleSkeleton* sk, const OracleClip* clips, uint32_t n_clips, const OracleRootMotion* rm, const uint32_t* clip,
	const uint32_t* time_ticks, const float* weight, const uint32_t* looped, uint32_t n_samples, const uint32_t* ik_after, const uint32_t* ik_leaf,
	const uint32_t* ik_bones, const float* ik_alpha, const float* ik_target3, uint32_t n_ik, OVec3* pos, OQuat* rot)
{
	RmClip* rc = (RmClip*)calloc(n_clips ? n_clips : 1, sizeof(RmClip));
	if (!rc) return -1;
	int status = 0;
	for (uint32_t c = 0; c < n_clips; ++c) {
		rc[c].clip = &clips[c];
		rc[c].t = rc[c].r = -1;
		/* one entry past the reference's frame_count + 1: a sample at or past the end of a clip of 257 frames or more reads entry
		 * frame_count + 1 at t == 0 (see sample()); it repeats the last entry, whose value that lerp / nlerp then gives */
		const size_t n = (size_t)clips[c].frame_count + 2;
		rc[c].pose_t = (OVec3*)malloc(sizeof(OVec3) * n);
		rc[c].pose_r = (OQuat*)malloc(sizeof(OQuat) * n);
		if (!rc[c].pose_t || !rc[c].pose_r) { status = -1; continue; }
		if (rm && oracle_root_motion_tables(&clips[c], rm[c].flags, rm[c].translation_track, rm[c].rotation_track, rc[c].pose_t, rc[c].pose_r)) {
			rc[c].t = rm[c].translation_track; /* :268-269 */
			rc[c].r = rm[c].rotation_track;
			rc[c].pose_t[n - 1] = rc[c].pose_t[n - 2];
			rc[c].pose_r[n - 1] = rc[c].pose_r[n - 2];
		}
	}
	if (status == 0) {
		for (uint32_t i = 0; i < sk->bone_count; ++i) { /* model.cpp:226-237 */
			pos[i] = sk->bind_relative[i].pos;
			rot[i] = sk->bind_relative[i].rot;
		}
		uint32_t ik = 0;
		for (uint32_t k = 0; k <= n_samples; ++k) {
			for (; ik < n_ik && ik_after[ik] == k; ++ik) {
				oracle_eval_ik(sk, ik_alpha[ik], ov3(ik_target3[3 * ik], ik_target3[3 * ik + 1], ik_target3[3 * ik + 2]), ik_leaf[ik], ik_bones[ik], pos, rot);
			}
			if (k == n_samples) break;
			const OracleClip* c = &clips[clip[k]];
			const uint32_t length = (uint32_t)(((float)c->frame_count / c->fps) * (1 << 15));
			const uint32_t t = looped[k] ? time_ticks[k] % length : (time_ticks[k] < length ? time_ticks[k] : length);
			sample(&rc[clip[k]], t, weight[k], pos, rot);
		}
		oracle_pose_compute_absolute(sk, pos, rot);
	}
	for (uint32_t c = 0; c < n_clips; ++c) {
		free(rc[c].pose_t);
		free(rc[c].pose_r);
	}
	free(rc);
	return status;
}

/* element-wise shims of normalize(Quat) and Animation::getRotation above */
void oracle_quat_normalize(const OQuat* q, OQuat* out, uint32_t n) { for (uint32_t i = 0; i < n; ++i) out[i] = oquat_normalize(q[i]); }
void oracle_rotation_d(const OracleClip* c, uint32_t track, const uint32_t* frames, OQuat* out, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) out[i] = packed_rotation_d(c, frames[i], &c->rotations[track]);
}
