/* TEST INFRASTRUCTURE — CPU restatement of the IK instructions of an animator's blend stack (see oracle_math.h for the rules of use),
 * built into oracle/liboracle_ik.so by oracle/Makefile on top of the pose restatement of oracle_anim.c (liboracle_lumix.so):
 *
 *   src/animation/controller.cpp:159-164        getAbsolutePosition (ik_absolute)
 *   src/animation/controller.cpp:166-265        evalIK (oracle_eval_ik)
 *   src/animation/controller.cpp:267-293        evalBlendStack: the SAMPLE and IK instructions in order (oracle_pose_stack_ik)
 *   src/animation/controller.cpp:142-157        getPose: time % getLength() when looped, minimum(time, getLength()) otherwise
 *   src/core/math.cpp:392, 395, 570-606         length, squaredLength, Quat(axis, angle), Quat::vec3ToVec3
 */
#include "oracle.h"

/* math.cpp:395 squaredLength(Vec3) */
static float ik_squared_length(OVec3 v) { return v.x * v.x + v.y * v.y + v.z * v.z; }

/* math.cpp:570-578 Quat(axis, angle) with the host libm's sinf / cosf */
static OQuat ik_axis_angle(OVec3 axis, float angle) {
	const float half_angle = angle * 0.5f;
	const float s = sinf(half_angle);
	return oquat(axis.x * s, axis.y * s, axis.z * s, cosf(half_angle));
}

/* math.cpp:581-606 Quat::vec3ToVec3 */
static OQuat oracle_vec3_to_vec3(OVec3 v0, OVec3 v1) {
	const OVec3 from = ov3_normalize(v0);
	const OVec3 to = ov3_normalize(v1);
	const float cos_angle = ov3_dot(from, to);
	if (cos_angle > -1.0005f && cos_angle < -0.9995f) {
		OVec3 n = ov3(0, from.z, -from.y);
		if (ik_squared_length(n) < 0.01) n = ov3(from.y, -from.x, 0); /* float promoted to double */
		n = ov3_normalize(n);
		return ik_axis_angle(n, 3.14159265f); /* math.h:404 PI */
	}
	const OVec3 half = ov3_normalize(ov3_add(from, to));
	return oquat(from.y * half.z - from.z * half.y, from.z * half.x - from.x * half.z, from.x * half.y - from.y * half.x, ov3_dot(from, half));
}

/* controller.cpp:159-164 getAbsolutePosition: recursive over Model::getBoneParent */
static OLocalRigidTransform ik_absolute(const OracleSkeleton* sk, const OVec3* pos, const OQuat* rot, int bone) {
	const int parent = sk->parents[bone];
	OLocalRigidTransform t;
	t.pos = pos[bone];
	t.rot = rot[bone];
	if (parent < 0) return t;
	return olrt_mul(ik_absolute(sk, pos, rot, parent), t);
}

/* controller.cpp:166-265 evalIK on a relative pose; leaf is the bone index Model::getBoneIndex found */
void oracle_eval_ik(const OracleSkeleton* sk, float alpha, OVec3 target, uint32_t leaf, uint32_t bones_count, OVec3* pos, OQuat* rot) {
	enum { MAX_BONES_COUNT = 32 };
	if (alpha < 0.001f) return;
	uint32_t indices[MAX_BONES_COUNT];
	OLocalRigidTransform transforms[MAX_BONES_COUNT];
	OVec3 old_pos[MAX_BONES_COUNT];
	float len[MAX_BONES_COUNT - 1];
	float len_sum = 0;
	indices[bones_count - 1] = leaf;
	for (uint32_t i = 1; i < bones_count; ++i) indices[bones_count - 1 - i] = (uint32_t)sk->parents[indices[bones_count - i]];

	const int first_bone_parent = sk->parents[indices[0]];
	OLocalRigidTransform roots_parent;
	if (first_bone_parent >= 0) roots_parent = ik_absolute(sk, pos, rot, first_bone_parent);
	else { roots_parent.pos = ov3(0, 0, 0); roots_parent.rot = oquat(0, 0, 0, 1); }

	OLocalRigidTransform parent_tr = roots_parent;
	for (uint32_t i = 0; i < bones_count; ++i) {
		OLocalRigidTransform tr;
		tr.pos = pos[indices[i]];
		tr.rot = rot[indices[i]];
		transforms[i] = olrt_mul(parent_tr, tr);
		old_pos[i] = transforms[i].pos;
		if (i > 0) {
			len[i - 1] = sqrtf(ik_squared_length(ov3_sub(transforms[i].pos, transforms[i - 1].pos))); /* math.cpp:392 length */
			len_sum += len[i - 1];
		}
		parent_tr = transforms[i];
	}

	OVec3 to_target = ov3_sub(target, transforms[0].pos);
	if (len_sum * len_sum < ik_squared_length(to_target)) {
		to_target = ov3_normalize(to_target);
		target = ov3_add(transforms[0].pos, ov3_muls(to_target, len_sum));
	}

	for (uint32_t iteration = 0; iteration < 5; ++iteration) {
		transforms[bones_count - 1].pos = target;
		for (int i = (int)bones_count - 1; i > 1; --i) {
			const OVec3 dir = ov3_normalize(ov3_sub(transforms[i - 1].pos, transforms[i].pos));
			transforms[i - 1].pos = ov3_add(transforms[i].pos, ov3_muls(dir, len[i - 1]));
		}
		for (uint32_t i = 1; i < bones_count; ++i) {
			const OVec3 dir = ov3_normalize(ov3_sub(transforms[i].pos, transforms[i - 1].pos));
			transforms[i].pos = ov3_add(transforms[i - 1].pos, ov3_muls(dir, len[i - 1]));
		}
	}

	for (int i = (int)bones_count - 2; i >= 0; --i) {
		const OVec3 old_d = ov3_sub(old_pos[i + 1], old_pos[i]);
		const OVec3 new_d = ov3_sub(transforms[i + 1].pos, transforms[i].pos);
		transforms[i].rot = oquat_mul(oracle_vec3_to_vec3(old_d, new_d), transforms[i].rot);
	}

	OLocalRigidTransform ik_out[MAX_BONES_COUNT];
	for (int i = (int)bones_count - 1; i > 0; --i) {
		transforms[i] = olrt_mul(olrt_inverted(transforms[i - 1]), transforms[i]);
		ik_out[i].pos = transforms[i].pos;
	}
	for (int i = (int)bones_count - 2; i > 0; --i) ik_out[i].rot = transforms[i].rot;
	ik_out[bones_count - 1].rot = rot[indices[bones_count - 1]];
	if (first_bone_parent >= 0) ik_out[0].rot = oquat_mul(oquat_conjugated(roots_parent.rot), transforms[0].rot);
	else ik_out[0].rot = transforms[0].rot;
	ik_out[0].pos = pos[indices[0]];

	for (uint32_t i = 0; i < bones_count; ++i) {
		const uint32_t idx = indices[i];
		pos[idx] = ov3_lerp(pos[idx], ik_out[i].pos, alpha);
		rot[idx] = oquat_nlerp(rot[idx], ik_out[i].rot, alpha);
	}
}

/* oracle_pose_stack with IK instructions: evalBlendStack (controller.cpp:267-293) runs the stack in order, so IK op k (leaf, bone count,
 * alpha = instruction alpha * ctx.weight, target) runs on the relative pose after the first ik_after[k] samples; ops with the same
 * ik_after run in list order (ik_after non-decreasing). */
void oracle_pose_stack_ik(const OracleSkeleton* sk, const OracleClip* clips, const uint32_t* clip, const uint32_t* time_ticks, const float* weight,
	const uint32_t* looped, uint32_t n_samples, const uint32_t* ik_after, const uint32_t* ik_leaf, const uint32_t* ik_bones, const float* ik_alpha,
	const float* ik_target3, uint32_t n_ik, OVec3* pos, OQuat* rot)
{
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
		oracle_pose_sample_weighted(c, sk->bone_count, t, weight[k], pos, rot);
	}
	oracle_pose_compute_absolute(sk, pos, rot);
}
