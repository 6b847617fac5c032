/* TEST INFRASTRUCTURE — CPU restatement of the SAMPLE instructions of an animator's blend stack (see oracle_math.h for the rules of use),
 * built into oracle/liboracle_stack.so by oracle/Makefile on top of the pose restatement of oracle_anim.c
 * (liboracle_lumix.so):
 *
 *   src/animation/animation_module.cpp:623-625  updateAnimator: Model::getRelativePose, evalBlendStack, Pose::computeAbsolute
 *   src/animation/controller.cpp:142-157        getPose: time % getLength() when looped, minimum(time, getLength()) otherwise
 *   src/animation/controller.cpp:267-293        evalBlendStack: the SAMPLE instructions in order (IK stays host code)
 *   src/animation/animation.h:20-23, 128        Time::fromSeconds, Animation::getLength() = fromSeconds(frame_count / fps)
 */
#include "oracle.h"

void oracle_pose_stack(const OracleSkeleton* sk, const OracleClip* clips, const uint32_t* clip, const uint32_t* time_ticks, const float* weight,
	const uint32_t* looped, uint32_t n_samples, OVec3* pos, OQuat* rot)
{
	for (uint32_t i = 0; i < sk->bone_count; ++i) { /* model.cpp:226-237 */
		pos[i] = sk->bind_relative[i].pos;
		rot[i] = sk->bind_relative[i].rot;
	}
	for (uint32_t k = 0; k < n_samples; ++k) {
		const OracleClip* c = &clips[clip[k]];
		const uint32_t length = (uint32_t)(((float)c->frame_count / c->fps) * (1 << 15));
		const uint32_t t = looped[k] ? time_ticks[k] % length : (time_ticks[k] < length ? time_ticks[k] : length); /* minimum(), math.h */
		/* Animation::getRelativePose with the sample's weight (animation.cpp:117-204, 294-311) */
		oracle_pose_sample_weighted(c, sk->bone_count, t, weight[k], pos, rot);
	}
	oracle_pose_compute_absolute(sk, pos, rot);
}
