// GPU pose evaluation + skinning palette + vertex skinning: kernels + C-ABI (include/lumix_b200.h "Animation").
//
// pose_palette_kernel — one warp per skeletal instance, the pose lives in shared memory:
//   Model::getRelativePose (src/renderer/model.cpp:226-237)            bind pose -> smem
//   AnimationSampler::getRelativePose<false,false> (src/animation/animation.cpp:117-204): const tracks, bit-packed
//     translation tracks (unpackChannel through double, :313-334), smallest-three rotation tracks + simd_nlerp (:30-95)
//   Pose::computeAbsolute (src/renderer/pose.cpp:66-133)               level-synchronous inside the warp
//   computeSkeletonDualQuats (src/renderer/pipeline.cpp:2680-2745) / computeSkinMatrices (src/renderer/model.cpp:132-137)
//     palette[j] = toDualQuat / toMatrix ({pos[j], rot[j]} * inverse_bind[j]) written once, coalesced
//   time advance of updateAnimable (src/animation/animation_module.cpp:458-469)
// root_motion_tables_kernel — Animation::setRootMotionBone (src/animation/animation.cpp:214-270): the root-motion tracks' rows of the
//   decoded keyframes replaced by pose_translations / pose_rotations (lb200_animation_set_root_motion), which the pose kernels then sample
// skin_kernel — evaluateSkin (model.cpp:103-109): palette of each instance staged in shared memory as 3x4 rows,
//   one thread per vertex, vertex data kept in registers across the instances of a group.
// Clips, skeleton and mesh are shared by all instances (L2-resident); HBM traffic is the per-instance output.
#include "lb200_internal.h"
#include "lb200_math.cuh"

#include <algorithm>
#include <memory>
#include <new>
#include <vector>

namespace {

using namespace lb;

struct DevClip {
	float fps;
	uint32_t frame_count;
	uint32_t t_bits, r_bits;          // frame sizes in bits
	uint32_t n_t, n_ct, n_r, n_cr;
	uint32_t t_off, ct_off, r_off, cr_off; // first element in the flat track arrays
	uint32_t t_stream, r_stream;      // byte offsets of the bit streams inside the stream blob (multiples of 4)
	uint32_t length_ticks;            // Animation::getLength(), animation.h:128
	uint32_t key_off;                 // first float4 of this clip's decoded keyframes: [key_rows(frame_count)][Bp] entries
	uint32_t flag_off, pad[3];        // first byte of this clip's per-bone track flags
};

// device-internal forms of the track descriptors: two 128-bit loads per animated track, one per constant track
struct alignas(16) DevTrack {
	float min[3]; uint32_t bone_offset;  // bone_index | offset_bits << 16
	float to_range[3]; uint32_t bits;    // bitsizes[0] | [1] << 8 | [2] << 16 | skipped_channel << 24
};
static_assert(sizeof(DevTrack) == 32, "");

struct Track { // unpacked in registers
	float min[3], to_range[3];
	uint32_t bone_index, offset_bits, bitsizes[3], skipped_channel;
};

__device__ __forceinline__ Track load_track(const DevTrack* __restrict__ p) {
	const uint4 a = __ldg(reinterpret_cast<const uint4*>(p));
	const uint4 b = __ldg(reinterpret_cast<const uint4*>(p) + 1);
	Track t;
	t.min[0] = __uint_as_float(a.x); t.min[1] = __uint_as_float(a.y); t.min[2] = __uint_as_float(a.z);
	t.bone_index = a.w & 0xffffu; t.offset_bits = a.w >> 16;
	t.to_range[0] = __uint_as_float(b.x); t.to_range[1] = __uint_as_float(b.y); t.to_range[2] = __uint_as_float(b.z);
	t.bitsizes[0] = b.w & 0xffu; t.bitsizes[1] = (b.w >> 8) & 0xffu; t.bitsizes[2] = (b.w >> 16) & 0xffu; t.skipped_channel = b.w >> 24;
	return t;
}

// AnimSysParams::n_layers of a system in sample-list mode (set_layers allows at most 16 layers)
constexpr uint32_t SAMPLE_LISTS = 0xffffffffu;

// The device form of one lb200_ik, two 128-bit loads: {after, path_len, bone_count, alpha} {target xyz, path_off}.  path_off is the byte
// offset, from the start of the op table, of the root-to-leaf path of the leaf bone (path_len bone indices, one byte each, first the bone
// whose parent is -1): the chain is its last bone_count entries and getAbsolutePosition of the chain's first parent folds the entries
// before them.  lb200_animation_set_stacks resolves it from the skeleton, once per distinct leaf.
constexpr uint32_t IK_MAX_BONES = 32; // controller.cpp:171 MAX_BONES_COUNT

// evalIK (controller.cpp:166-265) of op `op` on one instance's relative pose in shared memory, run by one lane of the instance group.
// The chain's working arrays live in that lane's local memory (L1): 1.3 KB that only one lane in G ever touches, which would cost every
// block of the IK kernels that much shared memory per instance for a path most instances of a frame do not take.
__device__ __noinline__ void eval_ik(float4* s_pos, float4* s_rot, const uint4* __restrict__ iks, uint32_t op) {
	const uint4 a = __ldg(iks + 2 * op), b = __ldg(iks + 2 * op + 1);
	const float alpha = __uint_as_float(a.w);
	if (alpha < 0.001f) return;                                 // :167
	const uint32_t n = a.z, path_len = a.y, first = path_len - n; // chain = path[first .. path_len), :184-187
	const unsigned char* path = reinterpret_cast<const unsigned char*>(iks) + b.w;
	V3 target = v3(__uint_as_float(b.x), __uint_as_float(b.y), __uint_as_float(b.z));
	unsigned char idx[IK_MAX_BONES];
	Rigid tr[IK_MAX_BONES];
	V3 old_pos[IK_MAX_BONES];
	float len[IK_MAX_BONES - 1];
	for (uint32_t i = 0; i < n; ++i) idx[i] = __ldg(path + first + i);
	auto bone = [&](uint32_t j) {
		const float4 p = s_pos[j], r = s_rot[j];
		Rigid t;
		t.pos = v3(p.x, p.y, p.z);
		t.rot = q4(r.x, r.y, r.z, r.w);
		return t;
	};
	// :190-198 getAbsolutePosition of the first bone's parent (:159-164): the left fold of the relative transforms from the root down
	Rigid roots_parent;
	if (first > 0) {
		roots_parent = bone(__ldg(path));
		for (uint32_t j = 1; j < first; ++j) roots_parent = rmul(roots_parent, bone(__ldg(path + j)));
	}
	else {
		roots_parent.pos = v3(0, 0, 0);
		roots_parent.rot = q4(0, 0, 0, 1);
	}
	// :200-210 bone space -> object space, bone lengths
	float len_sum = 0;
	Rigid parent_tr = roots_parent;
	for (uint32_t i = 0; i < n; ++i) {
		tr[i] = rmul(parent_tr, bone(idx[i]));
		old_pos[i] = tr[i].pos;
		if (i > 0) {
			len[i - 1] = length(sub(tr[i].pos, tr[i - 1].pos));
			len_sum = LB_FADD(len_sum, len[i - 1]);
		}
		parent_tr = tr[i];
	}
	// :212-216 an unreachable target moves onto the sphere the chain reaches
	V3 to_target = sub(target, tr[0].pos);
	if (LB_FMUL(len_sum, len_sum) < squared_length(to_target)) {
		to_target = normalize(to_target);
		target = add(tr[0].pos, muls(to_target, len_sum));
	}
	// :218-230 five FABRIK sweeps
	for (uint32_t iteration = 0; iteration < 5; ++iteration) {
		tr[n - 1].pos = target;
		for (int i = (int)n - 1; i > 1; --i) {
			const V3 dir = normalize(sub(tr[i - 1].pos, tr[i].pos));
			tr[i - 1].pos = add(tr[i].pos, muls(dir, len[i - 1]));
		}
		for (uint32_t i = 1; i < n; ++i) {
			const V3 dir = normalize(sub(tr[i].pos, tr[i - 1].pos));
			tr[i].pos = add(tr[i - 1].pos, muls(dir, len[i - 1]));
		}
	}
	// :233-239 rotations from the new positions
	for (int i = (int)n - 2; i >= 0; --i) {
		const Q4 rel_rot = vec3_to_vec3(sub(old_pos[i + 1], old_pos[i]), sub(tr[i + 1].pos, tr[i].pos));
		tr[i].rot = qmul(rel_rot, tr[i].rot);
	}
	// :243-246 object space -> bone space; tr[i] then holds ik_out[i] for 0 < i < n (its rotation too for i < n - 1, :247-249)
	for (int i = (int)n - 1; i > 0; --i) tr[i] = rmul(rinverted(tr[i - 1]), tr[i]);
	// :250-264: ik_out[0] keeps the pose position, ik_out[n - 1] the pose rotation (with n == 1 the rotation of :253-257 wins); the pose
	// moves towards ik_out by lerp and the scalar nlerp
	for (uint32_t i = 0; i < n; ++i) {
		const uint32_t j = idx[i];
		const float4 p = s_pos[j], r = s_rot[j];
		const V3 pose_pos = v3(p.x, p.y, p.z);
		const Q4 pose_rot = q4(r.x, r.y, r.z, r.w);
		V3 out_pos;
		Q4 out_rot;
		if (i == 0) {
			out_pos = pose_pos;
			out_rot = first > 0 ? qmul(conjugated(roots_parent.rot), tr[0].rot) : tr[0].rot;
		}
		else {
			out_pos = tr[i].pos;
			out_rot = i == n - 1 ? pose_rot : tr[i].rot;
		}
		const V3 np = lerp(pose_pos, out_pos, alpha);
		const Q4 nr = nlerp(pose_rot, out_rot, alpha);
		s_pos[j] = make_float4(np.x, np.y, np.z, 0.f);
		s_rot[j] = make_float4(nr.x, nr.y, nr.z, nr.w);
	}
}

// the IK ops of the instance whose `after` is `at` (the number of its samples applied so far), in list order, [ik, ik_end) advancing:
// the group joins, one lane solves on the shared pose, the group joins again before any lane reads the pose
template <class SP>
__device__ __forceinline__ void run_ik_ops(const SP& P, float4* s_pos, float4* s_rot, uint32_t at, uint32_t& ik, uint32_t ik_end, int sub, unsigned gmask) {
	while (ik < ik_end && __ldg(reinterpret_cast<const uint32_t*>(P.iks + 2 * ik)) == at) {
		__syncwarp(gmask);
		if (sub == 0) eval_ik(s_pos, s_rot, P.iks, ik);
		__syncwarp(gmask);
		++ik;
	}
}

// unaligned little-endian u64 at byte address `byte` of a word-addressed stream (the reference memcpy's 8 bytes, animation.cpp:44)
__device__ __forceinline__ unsigned long long load_u64_unaligned(const uint32_t* __restrict__ words, uint32_t byte) {
	const uint32_t w = byte >> 2;
	const uint32_t sh = (byte & 3u) * 8u;
	const uint32_t a = __ldg(words + w), b = __ldg(words + w + 1), c = __ldg(words + w + 2);
	const uint32_t lo = __funnelshift_r(a, b, sh);
	const uint32_t hi = __funnelshift_r(b, c, sh);
	return ((unsigned long long)hi << 32) | lo;
}

// low 32 bits of (v >> s), 0 <= s <= 64: the third channel of a (32, 32, 32) track starts at bit 64, past the 8 bytes the reference
// reads, and comes out 0 as the reference's two shifts by 32 leave it
__device__ __forceinline__ uint32_t shr64_lo32(unsigned long long v, uint32_t s) {
	const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
	if (s >= 64u) return 0u;
	return s >= 32u ? (hi >> (s - 32u)) : __funnelshift_r(lo, hi, s);
}
__device__ __forceinline__ uint32_t mask32(uint32_t bits) { return bits >= 32u ? 0xffffffffu : ((1u << bits) - 1u); }

// unpack_channel (animation.cpp:313-316) of a field known to fit 32 bits
__device__ __forceinline__ float unpack_channel32(uint32_t field, float mn, float range) {
	return __double2float_rn(LB_DADD((double)mn, LB_DMUL((double)range, __uint2double_rn(field))));
}

// animation.cpp:318-334 Animation::getTranslation
__device__ __forceinline__ V3 get_translation(const uint32_t* __restrict__ stream, uint32_t frame_bits, uint32_t frame, const Track& tr) {
	const uint32_t offset = frame_bits * frame + tr.offset_bits;
	unsigned long long tmp = load_u64_unaligned(stream, offset >> 3);
	tmp >>= (offset & 7u);
	V3 r;
	if ((tr.bitsizes[0] | tr.bitsizes[1] | tr.bitsizes[2]) <= 32u) {
		// every channel fits 32 bits (always true for importer output): same values, 32-bit integer path
		const uint32_t s1 = tr.bitsizes[0], s2 = s1 + tr.bitsizes[1];
		r.x = unpack_channel32((uint32_t)tmp & mask32(tr.bitsizes[0]), tr.min[0], tr.to_range[0]);
		r.y = unpack_channel32(shr64_lo32(tmp, s1) & mask32(tr.bitsizes[1]), tr.min[1], tr.to_range[1]);
		r.z = unpack_channel32(shr64_lo32(tmp, s2) & mask32(tr.bitsizes[2]), tr.min[2], tr.to_range[2]);
		return r;
	}
	r.x = unpack_channel(tmp, tr.min[0], tr.to_range[0], tr.bitsizes[0]);
	tmp >>= tr.bitsizes[0];
	r.y = unpack_channel(tmp, tr.min[1], tr.to_range[1], tr.bitsizes[1]);
	tmp >>= tr.bitsizes[1];
	r.z = unpack_channel(tmp, tr.min[2], tr.to_range[2], tr.bitsizes[2]);
	return r;
}

// animation.cpp:51-77 one packed rotation sample -> quaternion (smallest-three)
__device__ __forceinline__ Q4 unpack_rotation(unsigned long long packed, const Track& tr) {
	const bool is_negative = (packed & 1ull) != 0;
	packed >>= 1;
	V3 v;
	if ((tr.bitsizes[0] | tr.bitsizes[1] | tr.bitsizes[2]) <= 32u) {
		const uint32_t s1 = tr.bitsizes[0], s2 = s1 + tr.bitsizes[1];
		v.x = LB_FADD(tr.min[0], LB_FMUL(tr.to_range[0], __uint2float_rn((uint32_t)packed & mask32(tr.bitsizes[0]))));
		v.y = LB_FADD(tr.min[1], LB_FMUL(tr.to_range[1], __uint2float_rn(shr64_lo32(packed, s1) & mask32(tr.bitsizes[1]))));
		v.z = LB_FADD(tr.min[2], LB_FMUL(tr.to_range[2], __uint2float_rn(shr64_lo32(packed, s2) & mask32(tr.bitsizes[2]))));
	}
	else {
		const unsigned long long mask_x = (1ull << tr.bitsizes[0]) - 1ull;
		const unsigned long long mask_y = (1ull << tr.bitsizes[1]) - 1ull;
		const unsigned long long mask_z = (1ull << tr.bitsizes[2]) - 1ull;
		const unsigned long long py = packed >> tr.bitsizes[0];
		const unsigned long long pz = py >> tr.bitsizes[1];
		v.x = LB_FADD(tr.min[0], LB_FMUL(tr.to_range[0], __ull2float_rn(packed & mask_x)));
		v.y = LB_FADD(tr.min[1], LB_FMUL(tr.to_range[1], __ull2float_rn(py & mask_y)));
		v.z = LB_FADD(tr.min[2], LB_FMUL(tr.to_range[2], __ull2float_rn(pz & mask_z)));
	}
	const float rem = LB_FSUB(1.0f, dot(v, v));
	const float skipped = LB_FMUL(LB_FSQRT(rem > 0.f ? rem : 0.f), is_negative ? -1.0f : 1.0f); // maximum(0.f, x): 0 > x ? 0 : x
	switch (tr.skipped_channel) {
		case 0: return q4(skipped, v.x, v.y, v.z);
		case 1: return q4(v.x, skipped, v.y, v.z);
		case 2: return q4(v.x, v.y, skipped, v.z);
		default: return q4(v.x, v.y, v.z, skipped);
	}
}

// Unpack every frame of every clip once (clips are shared by all instances): block = (clip, row), threads over bones / tracks.
// Same arithmetic as the per-sample path of the reference: Animation::getTranslation (animation.cpp:318-334, unpackChannel through
// double) and the smallest-three reconstruction of AnimationSampler::getRotation (animation.cpp:51-77).
//
// A clip has key_rows(frame_count) = frame_count + 2 rows: frames 0 .. frame_count, then frame_count again.  The pose kernels read
// rows sample_idx and sample_idx + 1, and sample_idx reaches frame_count itself at or past the clip's end once frame_count - 0.00001f
// rounds to frame_count (frame_count >= 257).  There t == 0, so lerp / simd_nlerp of the last frame with its copy give the last frame,
// which is what the reference's read of frame_count + 1 yields for any finite value; the extra row keeps that read inside the clip's own
// table.  That holds because frame_count is at most MAX_FRAME_COUNT (lb200_animation_create refuses more): exact in fp32, so the clamp
// never rounds above it and sample_idx <= frame_count.  From 2^24 on an odd frame_count can round up and sample_idx pass frame_count + 1.
inline size_t key_rows(uint32_t frame_count) { return (size_t)frame_count + 2u; }
constexpr uint32_t MAX_FRAME_COUNT = (1u << 24) - 1u;
struct DecodeParams {
	const DevClip* clips;
	const DevTrack* tracks;
	const float4* const_t; const float4* const_r_value; const uint32_t* const_r_bone;
	const uint32_t* stream;
	const float4* bind_pos; const float4* bind_rot;
	float4* key_pos; float4* key_rot; unsigned char* key_flags;
	const uint32_t* frame_clip;  // block -> clip
	const uint32_t* frame_index; // block -> frame inside the clip
	uint32_t bone_count;
};

__global__ void __launch_bounds__(256) decode_clips_kernel(const __grid_constant__ DecodeParams P) {
	const uint32_t B = P.bone_count, Bp = (B + 3u) & ~3u;
	const uint32_t c = P.frame_clip[blockIdx.x], row = P.frame_index[blockIdx.x];
	const DevClip clip = P.clips[c];
	const uint32_t frame = row < clip.frame_count ? row : clip.frame_count; // the last row repeats the last frame
	float4* kp = P.key_pos + clip.key_off + (size_t)row * Bp;
	float4* kr = P.key_rot + clip.key_off + (size_t)row * Bp;
	unsigned char* kf = P.key_flags + clip.flag_off;
	for (uint32_t b = threadIdx.x; b < Bp; b += blockDim.x) {
		kp[b] = b < B ? P.bind_pos[b] : make_float4(0, 0, 0, 0);
		kr[b] = b < B ? P.bind_rot[b] : make_float4(0, 0, 0, 1);
		if (frame == 0) kf[b] = 0;
	}
	__syncthreads();
	for (uint32_t i = threadIdx.x; i < clip.n_ct; i += blockDim.x) {
		const float4 ct = P.const_t[clip.ct_off + i];
		const uint32_t bone = __float_as_uint(ct.w);
		kp[bone] = make_float4(ct.x, ct.y, ct.z, 0.f);
		if (frame == 0) atomicOr(reinterpret_cast<unsigned int*>(kf + (bone & ~3u)), 4u << (8u * (bone & 3u)));
	}
	for (uint32_t i = threadIdx.x; i < clip.n_cr; i += blockDim.x) {
		const uint32_t bone = P.const_r_bone[clip.cr_off + i];
		kr[bone] = P.const_r_value[clip.cr_off + i];
		if (frame == 0) atomicOr(reinterpret_cast<unsigned int*>(kf + (bone & ~3u)), 8u << (8u * (bone & 3u)));
	}
	__syncthreads();
	const uint32_t* t_stream = P.stream + (clip.t_stream >> 2);
	for (uint32_t i = threadIdx.x; i < clip.n_t; i += blockDim.x) {
		const Track tr = load_track(P.tracks + clip.t_off + i);
		const V3 v = get_translation(t_stream, clip.t_bits, frame, tr);
		kp[tr.bone_index] = make_float4(v.x, v.y, v.z, 0.f);
		if (frame == 0) atomicOr(reinterpret_cast<unsigned int*>(kf + (tr.bone_index & ~3u)), 1u << (8u * (tr.bone_index & 3u)));
	}
	const uint32_t* r_stream = P.stream + (clip.r_stream >> 2);
	for (uint32_t i = threadIdx.x; i < clip.n_r; i += blockDim.x) {
		const Track tr = load_track(P.tracks + clip.r_off + i);
		const uint32_t offset = clip.r_bits * frame + tr.offset_bits;
		unsigned long long p = load_u64_unaligned(r_stream, offset >> 3);
		p >>= (offset & 7u);
		const Q4 q = unpack_rotation(p, tr);
		kr[tr.bone_index] = make_float4(q.x, q.y, q.z, q.w);
		if (frame == 0) atomicOr(reinterpret_cast<unsigned int*>(kf + (tr.bone_index & ~3u)), 2u << (8u * (tr.bone_index & 3u)));
	}
}

// Animation::setRootMotionBone (animation.cpp:214-270) for the clips with root motion, one thread per (clip, frame): the frame's
// pose_translations / pose_rotations entry replaces the decoded keyframe of the tracks' bones, which is what the sampler reads for those
// tracks (animation.cpp:33-37, 321).  Runs after decode_clips_kernel has decoded the clip's rows from its packed tracks.
struct RootMotionParams {
	const DevClip* clips;
	const DevTrack* tracks;
	const uint32_t* stream;
	const int4* root_motion;     // per clip: flags, translation track, rotation track (indices into the clip's tracks, or -1), unused
	const uint32_t* frame_clip;  // thread -> clip
	const uint32_t* frame_index; // thread -> frame inside the clip
	uint32_t n;
	uint32_t bone_count;
	float4* key_pos; float4* key_rot;
};

constexpr uint32_t RM_Y = 1u, RM_XZ = 2u, RM_ROT = 4u; // Animation::Flags, animation.h:73-78

__global__ void __launch_bounds__(128) root_motion_tables_kernel(const __grid_constant__ RootMotionParams P) {
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= P.n) return;
	const uint32_t c = P.frame_clip[i], row = P.frame_index[i];
	const DevClip clip = P.clips[c];
	const uint32_t frame = row < clip.frame_count ? row : clip.frame_count; // key_rows: the last row repeats the last frame
	const int4 rm = P.root_motion[c];
	const uint32_t flags = (uint32_t)rm.x;
	const bool has_t = rm.y >= 0, has_r = rm.z >= 0;
	Track tt = {}, rt = {};
	if (has_t) tt = load_track(P.tracks + clip.t_off + rm.y);
	if (has_r) rt = load_track(P.tracks + clip.r_off + rm.z);
	// :249-251 tmp: Animation::getTranslation / getRotation (unpackChannel through double) of the tracks, 0 / identity without one
	auto sample = [&](uint32_t f) {
		Rigid t;
		t.pos = has_t ? get_translation(P.stream + (clip.t_stream >> 2), clip.t_bits, f, tt) : v3(0, 0, 0);
		t.rot = q4(0, 0, 0, 1);
		if (has_r) {
			const uint32_t offset = clip.r_bits * f + rt.offset_bits;
			const unsigned long long p = load_u64_unaligned(P.stream + (clip.r_stream >> 2), offset >> 3) >> (offset & 7u);
			t.rot = unpack_rotation_d(p, rt.min, rt.to_range, rt.bitsizes, rt.skipped_channel);
		}
		return t;
	};
	// :97-115 maskRootMotion
	auto mask = [&](const Rigid& t) {
		Rigid m;
		m.pos = v3(0, 0, 0);
		m.rot = q4(0, 0, 0, 1);
		if (flags & RM_Y) m.pos.y = t.pos.y;
		if (flags & RM_XZ) { m.pos.x = t.pos.x; m.pos.z = t.pos.z; }
		if (flags & RM_ROT) {
			m.rot.y = t.rot.y;
			m.rot.w = t.rot.w;
			m.rot = normalize(m.rot);
		}
		return m;
	};
	const Rigid tmp = sample(frame);
	const Rigid rmf = mask(tmp);
	// :254-255 rm0: the masked frame 0 where m_root_motion.translations / rotations were filled (:240-246), else 0 / identity
	const Rigid m0 = mask(sample(0));
	Rigid rm0;
	rm0.pos = has_t && (flags & (RM_Y | RM_XZ)) ? m0.pos : v3(0, 0, 0);
	rm0.rot = has_r && (flags & RM_ROT) ? m0.rot : q4(0, 0, 0, 1);
	const Rigid out = rmul(rmul(rm0, rinverted(rmf)), tmp); // :257 rm0 * rm.inverted() * tmp
	const size_t at = clip.key_off + (size_t)row * ((P.bone_count + 3u) & ~3u);
	if (has_t) P.key_pos[at + tt.bone_index] = make_float4(out.pos.x, out.pos.y, out.pos.z, 0.f);
	if (has_r) P.key_rot[at + rt.bone_index] = make_float4(out.rot.x, out.rot.y, out.rot.z, out.rot.w);
}

constexpr int POSE_THREADS = 128;

// One system as every pose kernel reads it: the pose path reads no other table of a system (the bit streams and track descriptors
// are only read by decode_clips_kernel).  A system in sample-list mode (lb200_animation_set_samples) has n_layers == SAMPLE_LISTS, and
// the unions hold its lists, IK ops and bind pose over fields that only clip mode reads.
struct AnimSysParams {
	const DevClip* clips;
	const float4* key_pos; const float4* key_rot; // decoded keyframes (decode_clips_kernel)
	const unsigned char* key_flags;               // per (clip, bone): bit0 / bit1 translation / rotation animated, bit2 / bit3 constant track
	const float4* inv_bind_pos; const float4* inv_bind_rot; // inverse bind transforms
	const short* parents;
	const unsigned char* level_bones; // bones of depth >= 1 sorted by depth (bone_count <= 196 fits a byte)
	const uint32_t* level_start;      // [max_level + 2]: level l occupies level_bones[level_start[l] .. level_start[l + 1])
	uint32_t bone_count;
	uint32_t max_level;
	uint32_t n_instances;
	uint32_t n_layers; // blend layers on top of the base clip (lb200_animation_set_layers): [instance][n_layers], or SAMPLE_LISTS
	union { const uint32_t* clip_index; const uint32_t* sample_offsets; }; // sample lists: [n_instances + 1] CSR offsets
	union { uint32_t* time_ticks; const uint32_t* ik_offsets; };           // sample lists: [n_instances + 1] CSR offsets of the IK ops, or null
	float* out_dq; float* out_mtx; float* out_pos; float* out_rot; // null where the palette flags do not ask for the output
	union { const uint32_t* layer_clip; const uint4* samples; };     // sample lists: lb200_sample entries
	union { const uint32_t* layer_time; const float4* bind_pose; };  // sample lists: bind pos[B], then bind rot[B]
	union { const float* layer_weight; const uint4* iks; };          // sample lists: the IK ops (IkOp) and their bone paths
};
static_assert(sizeof(AnimSysParams) == 160, "");

// One time step for every system of an update
struct PoseStep {
	uint32_t dt_ticks; // |time_delta| in ticks
	int dt_negative;
	int advance;
};

// Systems per pose_palette_many_kernel launch (DESIGN.md §4.3): the parameter block is 16 + 164 x cap bytes, 10.5 KB at 64;
// longer lists run as consecutive launches on the context stream.
constexpr uint32_t POSE_MANY_CAP = 64;

struct AnimManyParams {
	PoseStep step;
	uint32_t n_systems;
	uint32_t block_end[POSE_MANY_CAP]; // inclusive prefix of block counts: system s owns blocks [block_end[s - 1], block_end[s])
	AnimSysParams sys[POSE_MANY_CAP];
};
static_assert(offsetof(AnimManyParams, n_systems) == 12 && offsetof(AnimManyParams, block_end) == 16 &&
	offsetof(AnimManyParams, sys) == 16 + 4 * POSE_MANY_CAP && sizeof(AnimManyParams) == 16 + 164 * POSE_MANY_CAP, "");

// One instance group of G lanes: sample, blend layers, computeAbsolute, palettes and the time advance of every instance of block
// `block` of a system.  P holds the system's tables, A the time step.
// pose_palette_kernel and pose_palette_many_kernel both run it, so the reference arithmetic exists once.
// Which start and sample source the body compiles: POSE_EITHER reads the mode of each system (pose_palette_many_kernel); the per-system
// kernel compiles one mode per instantiation, so that clip mode runs the code it ran before sample lists existed.  IK compiles the
// IK ops of sample lists in (pose_palette_ik_kernel, pose_palette_many_ik_kernel); the kernels without it run the code they ran before.
enum PoseMode { POSE_CLIPS, POSE_LISTS, POSE_EITHER };

template <int G, int MODE, bool IK = false>
__device__ __forceinline__ void pose_palette_body(const AnimSysParams& P, const PoseStep& A, const uint32_t block) {
	extern __shared__ float4 smem4[];
	constexpr int INST_PER_BLOCK = POSE_THREADS / G;
	const int lane = threadIdx.x & 31;
	const int sub = threadIdx.x % G;          // lane inside the instance group
	const int grp = threadIdx.x / G;          // instance slot inside the block
	const uint32_t B = P.bone_count;
	const uint32_t Bp = (B + 3u) & ~3u;
	// block-shared skeleton data first (read by every instance at every depth level: keep it out of the L2 round trips):
	//   inverse bind pos[Bp], rot[Bp] (float4) | level_start[max_level + 2] (u32) | parents[Bp] (i16) | level_bones[Bp] (u8)
	float4* s_ibp = smem4;
	float4* s_ibr = s_ibp + Bp;
	uint32_t* s_level_start = reinterpret_cast<uint32_t*>(s_ibr + Bp);
	const uint32_t n_ls = (P.max_level + 2u + 3u) & ~3u;
	short* s_parents = reinterpret_cast<short*>(s_level_start + n_ls);
	unsigned char* s_level_bones = reinterpret_cast<unsigned char*>(s_parents + Bp);
	float4* inst_base = reinterpret_cast<float4*>(smem4 + 2 * Bp + (n_ls * 4 + Bp * 2 + Bp + 15) / 16);
	for (uint32_t i = threadIdx.x; i < B; i += POSE_THREADS) {
		s_ibp[i] = __ldg(P.inv_bind_pos + i);
		s_ibr[i] = __ldg(P.inv_bind_rot + i);
		s_parents[i] = P.parents[i];
	}
	for (uint32_t i = threadIdx.x; i < P.max_level + 2u; i += POSE_THREADS) s_level_start[i] = P.level_start[i];
	for (uint32_t i = threadIdx.x; i < P.level_start[P.max_level + 1]; i += POSE_THREADS) s_level_bones[i] = P.level_bones[i];
	__syncthreads();
	// per instance: rot[Bp] (float4) then pos[Bp] (float4, w unused): 128-bit shared accesses, conflict-free per quarter warp
	float4* s_rot = inst_base + (size_t)grp * Bp * 2;
	float4* s_pos = s_rot + Bp;
	const uint32_t inst = block * INST_PER_BLOCK + grp;
	const bool valid = inst < P.n_instances;
	// the lanes of one group share a mask so that __syncwarp only joins what must be joined
	const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));

	if (valid) {
		// the instance's start pose, then its samples [k_begin, k_end): the layers after the base clip in clip mode, the instance's
		// list after the bind pose in sample-list mode
		const bool lists = MODE == POSE_EITHER ? P.n_layers == SAMPLE_LISTS : MODE == POSE_LISTS;
		size_t k_begin, k_end;
		uint32_t ticks = 0, length = 0; // clip mode: the base clip's time and length, for the time step
		if (lists) {
			k_begin = P.sample_offsets[inst];
			k_end = P.sample_offsets[inst + 1];
			for (uint32_t b = sub; b < B; b += G) { // Model::getRelativePose, model.cpp:226-237
				s_pos[b] = __ldg(P.bind_pose + b);
				s_rot[b] = __ldg(P.bind_pose + B + b);
			}
		}
		else {
			const DevClip clip = P.clips[P.clip_index[inst]];
			ticks = P.time_ticks[inst];
			length = clip.length_ticks;
			k_begin = (size_t)inst * P.n_layers;
			k_end = k_begin + P.n_layers;

			// animation.h:27 toFrame: float(value / double(ONE_SECOND) * fps); animation.cpp:131-133
			const float frame = __double2float_rn(LB_DMUL(__uint2double_rn(ticks) / 32768.0, (double)clip.fps));
			const float hi = LB_FSUB(__uint2float_rn(clip.frame_count), 0.00001f);
			float sample = frame > 0.f ? frame : 0.f; // maximum(value, min): value > min ? value : min
			sample = sample < hi ? sample : hi;       // minimum(x, max)
			const uint32_t sample_idx = (uint32_t)sample;
			const float t = LB_FSUB(sample, __uint2float_rn(sample_idx));

			// Model::getRelativePose (model.cpp:226-237) + Animation::getRelativePose (animation.cpp:117-204) from the decoded keyframes:
			// the two frames of a track do not depend on the instance, so they were unpacked once per clip (decode_clips_kernel) with the
			// reference's arithmetic; here only the per-instance part remains: lerp (math.cpp:194-201) / simd_nlerp (simd_math.h:107-123)
			// for animated tracks, plain copy for constant tracks and untracked bones (which keep the bind pose).
			const float4* k0p = P.key_pos + clip.key_off + (size_t)sample_idx * Bp;
			const float4* k0r = P.key_rot + clip.key_off + (size_t)sample_idx * Bp;
			const unsigned char* kf = P.key_flags + clip.flag_off;
			for (uint32_t b = sub; b < B; b += G) {
				const uint32_t fl = kf[b];
				float4 p = __ldg(k0p + b);
				float4 r = __ldg(k0r + b);
				if (fl & 1u) {
					const float4 p1 = __ldg(k0p + Bp + b);
					const V3 v = lerp(v3(p.x, p.y, p.z), v3(p1.x, p1.y, p1.z), t);
					p = make_float4(v.x, v.y, v.z, 0.f);
				}
				if (fl & 2u) {
					const float4 r1 = __ldg(k0r + Bp + b);
					const Q4 q = simd_nlerp(q4(r.x, r.y, r.z, r.w), q4(r1.x, r1.y, r1.z, r1.w), t);
					r = make_float4(q.x, q.y, q.z, q.w);
				}
				s_pos[b] = p;
				s_rot[b] = r;
			}
		}
		__syncwarp(gmask);

		// Blend layers and sample lists (the animator's stack of weighted samples, controller.cpp:267-292 -> Animation::getRelativePose
		// with ctx.weight): every bone the sample's clip has a track for — constant or animated — moves towards the sample, lerp
		// (math.cpp:194-201) for positions and simd_nlerp for rotations when weight < 0.9999 (animation.cpp:294-311), plain replacement
		// otherwise; bones without a track are left alone (animation.cpp:136-203).  Bones are independent: no sync inside.
		// With IK, the instance's IK ops run between the samples where their `after` puts them (evalBlendStack's instruction order).
		uint32_t ik = 0, ik_end = 0;
		if (IK && lists && P.ik_offsets) { ik = P.ik_offsets[inst]; ik_end = P.ik_offsets[inst + 1]; }
		for (size_t li = k_begin; li < k_end; ++li) {
			if (IK) run_ik_ops(P, s_pos, s_rot, (uint32_t)(li - k_begin), ik, ik_end, sub, gmask);
			uint32_t lc, ltime;
			float w;
			if (lists) {
				const uint4 e = __ldg(P.samples + li);
				lc = e.x; w = __uint_as_float(e.z);
				const uint32_t len = P.clips[lc].length_ticks;
				ltime = e.w ? e.y % len : (e.y < len ? e.y : len); // getPose, controller.cpp:148
			}
			else {
				lc = P.layer_clip[li]; ltime = P.layer_time[li]; w = P.layer_weight[li];
			}
			const DevClip lclip = P.clips[lc];
			const bool use_weight = w < 0.9999f;
			const float lframe = __double2float_rn(LB_DMUL(__uint2double_rn(ltime) / 32768.0, (double)lclip.fps));
			const float lhi = LB_FSUB(__uint2float_rn(lclip.frame_count), 0.00001f);
			float ls = lframe > 0.f ? lframe : 0.f;
			ls = ls < lhi ? ls : lhi;
			const uint32_t lidx = (uint32_t)ls;
			const float lt = LB_FSUB(ls, __uint2float_rn(lidx));
			const float4* l0p = P.key_pos + lclip.key_off + (size_t)lidx * Bp;
			const float4* l0r = P.key_rot + lclip.key_off + (size_t)lidx * Bp;
			const unsigned char* lf = P.key_flags + lclip.flag_off;
			for (uint32_t b = sub; b < B; b += G) {
				const uint32_t fl = lf[b];
				if (fl & 5u) {
					const float4 p0 = __ldg(l0p + b);
					V3 v = v3(p0.x, p0.y, p0.z);
					if (fl & 1u) {
						const float4 p1 = __ldg(l0p + Bp + b);
						v = lerp(v, v3(p1.x, p1.y, p1.z), lt);
					}
					if (use_weight) {
						const float4 cur = s_pos[b];
						v = lerp(v3(cur.x, cur.y, cur.z), v, w);
					}
					s_pos[b] = make_float4(v.x, v.y, v.z, 0.f);
				}
				if (fl & 10u) {
					const float4 r0 = __ldg(l0r + b);
					Q4 q = q4(r0.x, r0.y, r0.z, r0.w);
					if (fl & 2u) {
						const float4 r1 = __ldg(l0r + Bp + b);
						q = simd_nlerp(q, q4(r1.x, r1.y, r1.z, r1.w), lt);
					}
					if (use_weight) {
						const float4 cur = s_rot[b];
						q = simd_nlerp(q4(cur.x, cur.y, cur.z, cur.w), q, w);
					}
					s_rot[b] = make_float4(q.x, q.y, q.z, q.w);
				}
			}
		}
		if (IK) run_ik_ops(P, s_pos, s_rot, (uint32_t)(k_end - k_begin), ik, ik_end, sub, gmask);
		__syncwarp(gmask);

		// Pose::computeAbsolute, pose.cpp:66-133: bones of one depth level are independent (the reference's 4-wide path
		// relies on the same fact); levels run in order so every parent is absolute before its children.
		for (uint32_t lvl = 1; lvl <= P.max_level; ++lvl) {
			const uint32_t lb = s_level_start[lvl], le = s_level_start[lvl + 1];
			for (uint32_t k = lb + sub; k < le; k += G) {
				const uint32_t b = s_level_bones[k];
				const int p = s_parents[b];
				const float4 pr = s_rot[p], pp = s_pos[p], cr = s_rot[b], cp = s_pos[b];
				const Q4 prot = q4(pr.x, pr.y, pr.z, pr.w);
				const V3 pos = add(rotate(prot, v3(cp.x, cp.y, cp.z)), v3(pp.x, pp.y, pp.z)); // :129
				const Q4 rot = qmul(prot, q4(cr.x, cr.y, cr.z, cr.w));                          // :130
				s_pos[b] = make_float4(pos.x, pos.y, pos.z, 0.f);
				s_rot[b] = make_float4(rot.x, rot.y, rot.z, rot.w);
			}
			__syncwarp(gmask);
		}

		// palettes: pipeline.cpp:2680-2745 / model.cpp:132-137
		for (uint32_t b = sub; b < B; b += G) {
			const float4 cr = s_rot[b], cp = s_pos[b];
			Rigid pose;
			pose.pos = v3(cp.x, cp.y, cp.z);
			pose.rot = q4(cr.x, cr.y, cr.z, cr.w);
			const float4 ip = s_ibp[b], ir = s_ibr[b];
			Rigid inv;
			inv.pos = v3(ip.x, ip.y, ip.z);
			inv.rot = q4(ir.x, ir.y, ir.z, ir.w);
			const Rigid skin = rmul(pose, inv);
			const size_t idx = (size_t)inst * B + b;
			if (P.out_dq) {
				const DualQ dq = to_dual_quat(skin);
				float4* o = reinterpret_cast<float4*>(P.out_dq + idx * 8);
				o[0] = make_float4(dq.r.x, dq.r.y, dq.r.z, dq.r.w);
				o[1] = make_float4(dq.d.x, dq.d.y, dq.d.z, dq.d.w);
			}
			if (P.out_mtx) {
				float m[16];
				to_matrix(skin, m);
				float4* o = reinterpret_cast<float4*>(P.out_mtx + idx * 16);
				o[0] = make_float4(m[0], m[1], m[2], m[3]);
				o[1] = make_float4(m[4], m[5], m[6], m[7]);
				o[2] = make_float4(m[8], m[9], m[10], m[11]);
				o[3] = make_float4(m[12], m[13], m[14], m[15]);
			}
			if (P.out_pos) {
				P.out_pos[idx * 3] = pose.pos.x; P.out_pos[idx * 3 + 1] = pose.pos.y; P.out_pos[idx * 3 + 2] = pose.pos.z;
				reinterpret_cast<float4*>(P.out_rot)[idx] = cr;
			}
		}

		// animation_module.cpp:458-469
		if (A.advance && !lists && sub == 0) {
			const uint32_t l = length;
			uint32_t nt;
			if (!A.dt_negative) nt = (ticks + A.dt_ticks) % l;
			else nt = (ticks + l - (A.dt_ticks % l)) % l;
			P.time_ticks[inst] = nt;
		}
	}
}

// G lanes cooperate on one instance (32 / G instances per warp): per-bone phases stride the bones by G, the absolute pass
// walks depth levels with up to G bones of a level in flight.  G is 8 unless LB200_POSE_LANES or lb200_animation_set_launch asks
// for another (lb200_animation_update).
template <int G, bool LISTS>
__global__ void __launch_bounds__(POSE_THREADS) pose_palette_kernel(const __grid_constant__ AnimSysParams P, const __grid_constant__ PoseStep A) {
	pose_palette_body<G, LISTS ? POSE_LISTS : POSE_CLIPS>(P, A, blockIdx.x);
}

// The same for up to POSE_MANY_CAP systems in one grid (lb200_animation_update_many): each block finds its system by a binary search
// over the prefix of block counts (uniform across the block, once per block) and runs the system's block as pose_palette_kernel would.
// Dynamic shared memory is sized for the launch's largest skeleton.
template <int G, bool IK>
__device__ __forceinline__ void pose_many_block(const AnimManyParams& M) {
	uint32_t lo = 0, hi = M.n_systems - 1;
	while (lo < hi) {
		const uint32_t mid = (lo + hi) >> 1;
		if (blockIdx.x < M.block_end[mid]) hi = mid;
		else lo = mid + 1;
	}
	const uint32_t first_block = lo ? M.block_end[lo - 1] : 0u;
	pose_palette_body<G, POSE_EITHER, IK>(M.sys[lo], M.step, blockIdx.x - first_block);
}

template <int G>
__global__ void __launch_bounds__(POSE_THREADS) pose_palette_many_kernel(const __grid_constant__ AnimManyParams M) {
	pose_many_block<G, false>(M);
}

// pose_palette_kernel<G, true> with the IK ops of the lists (lb200_animation_set_stacks): chosen only for a system that has IK ops
template <int G>
__global__ void __launch_bounds__(POSE_THREADS) pose_palette_ik_kernel(const __grid_constant__ AnimSysParams P, const __grid_constant__ PoseStep A) {
	pose_palette_body<G, POSE_LISTS, true>(P, A, blockIdx.x);
}

// pose_palette_many_kernel<G> with the IK ops: chosen only for a launch in which some system has IK ops
template <int G>
__global__ void __launch_bounds__(POSE_THREADS) pose_palette_many_ik_kernel(const __grid_constant__ AnimManyParams M) {
	pose_many_block<G, true>(M);
}

// ---- skinning ------------------------------------------------------------------------------------------------
constexpr int SKIN_THREADS = 256;
// SKIN_GROUP = instances per block (template parameter): vertex data stays in registers across them

template <int SKIN_GROUP>
__global__ void __launch_bounds__(SKIN_THREADS) skin_kernel(const float* __restrict__ palette_mtx, const float* __restrict__ positions3,
	const float4* __restrict__ weights4, const short* __restrict__ indices4, uint32_t n_vertices, uint32_t bone_count, uint32_t n_instances,
	float* __restrict__ out)
{
	extern __shared__ float4 s_rows[]; // [group][bone][3] rows of the 3x4 upper part
	const uint32_t v = blockIdx.x * SKIN_THREADS + threadIdx.x;
	const uint32_t inst0 = blockIdx.y * SKIN_GROUP;
	const uint32_t n_inst = min((uint32_t)SKIN_GROUP, n_instances - inst0);

	// stage palettes: matrix e = 16 floats column-major -> rows r0 = (m0,m4,m8,m12) ...
	const uint32_t total = n_inst * bone_count;
	for (uint32_t e = threadIdx.x; e < total; e += SKIN_THREADS) {
		const float4* src = reinterpret_cast<const float4*>(palette_mtx + ((size_t)inst0 * bone_count + e) * 16);
		const float4 c0 = __ldg(src), c1 = __ldg(src + 1), c2 = __ldg(src + 2), c3 = __ldg(src + 3);
		s_rows[e * 3 + 0] = make_float4(c0.x, c1.x, c2.x, c3.x);
		s_rows[e * 3 + 1] = make_float4(c0.y, c1.y, c2.y, c3.y);
		s_rows[e * 3 + 2] = make_float4(c0.z, c1.z, c2.z, c3.z);
	}
	__syncthreads();
	if (v >= n_vertices) return;

	const float px = positions3[3 * (size_t)v], py = positions3[3 * (size_t)v + 1], pz = positions3[3 * (size_t)v + 2];
	const float4 w = weights4[v];
	const short4 idx = reinterpret_cast<const short4*>(indices4)[v];

	for (uint32_t g = 0; g < n_inst; ++g) {
		const float4* rows = s_rows + (size_t)g * bone_count * 3;
		float o[3];
#pragma unroll
		for (int r = 0; r < 3; ++r) {
			const float4 a = rows[idx.x * 3 + r], b = rows[idx.y * 3 + r], c = rows[idx.z * 3 + r], d = rows[idx.w * 3 + r];
			// model.cpp:105-106: m = m0*w.x + m1*w.y + m2*w.z + m3*w.w, elementwise, left to right (math.cpp:1022-1071)
			const float m0 = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(a.x, w.x), LB_FMUL(b.x, w.y)), LB_FMUL(c.x, w.z)), LB_FMUL(d.x, w.w));
			const float m1 = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(a.y, w.x), LB_FMUL(b.y, w.y)), LB_FMUL(c.y, w.z)), LB_FMUL(d.y, w.w));
			const float m2 = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(a.z, w.x), LB_FMUL(b.z, w.y)), LB_FMUL(c.z, w.z)), LB_FMUL(d.z, w.w));
			const float m3 = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(a.w, w.x), LB_FMUL(b.w, w.y)), LB_FMUL(c.w, w.z)), LB_FMUL(d.w, w.w));
			// math.cpp:1231-1235 transformPoint: c0.r*x + c1.r*y + c2.r*z + c3.r
			o[r] = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(m0, px), LB_FMUL(m1, py)), LB_FMUL(m2, pz)), m3);
		}
		float* dst = out + ((size_t)(inst0 + g) * n_vertices + v) * 3;
		dst[0] = o[0]; dst[1] = o[1]; dst[2] = o[2];
	}
}

// Each kernel family by launch shape, at shapeIndex(G) for G = 4, 8, 16, 32 lanes per instance (the skin kernel: 4, 8, 16 instances
// per block).  Launches index these tables, and lb200_animation_create sets every kernel's shared memory from them.
using PoseKernel = void (*)(AnimSysParams, PoseStep);
using PoseManyKernel = void (*)(AnimManyParams);
using SkinKernel = void (*)(const float*, const float*, const float4*, const short*, uint32_t, uint32_t, uint32_t, float*);
const PoseKernel POSE_CLIP_KERNELS[] = {pose_palette_kernel<4, false>, pose_palette_kernel<8, false>, pose_palette_kernel<16, false>, pose_palette_kernel<32, false>};
const PoseKernel POSE_LIST_KERNELS[] = {pose_palette_kernel<4, true>, pose_palette_kernel<8, true>, pose_palette_kernel<16, true>, pose_palette_kernel<32, true>};
const PoseKernel POSE_IK_KERNELS[] = {pose_palette_ik_kernel<4>, pose_palette_ik_kernel<8>, pose_palette_ik_kernel<16>, pose_palette_ik_kernel<32>};
const PoseManyKernel POSE_MANY_KERNELS[] = {pose_palette_many_kernel<4>, pose_palette_many_kernel<8>, pose_palette_many_kernel<16>, pose_palette_many_kernel<32>};
const PoseManyKernel POSE_MANY_IK_KERNELS[] = {pose_palette_many_ik_kernel<4>, pose_palette_many_ik_kernel<8>, pose_palette_many_ik_kernel<16>, pose_palette_many_ik_kernel<32>};
const SkinKernel SKIN_KERNELS[] = {skin_kernel<4>, skin_kernel<8>, skin_kernel<16>};
int shapeIndex(int n) { return __builtin_ctz((unsigned)n) - 2; }

__global__ void __launch_bounds__(256) checksum_kernel(const uint32_t* __restrict__ data, size_t n, unsigned long long* __restrict__ out) {
	unsigned long long acc = 0;
	for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) acc += data[i];
	for (int off = 16; off; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
	if ((threadIdx.x & 31) == 0) atomicAdd(out, acc);
}

// Pose::computeRelative (pose.cpp:136-146) for every instance: the reference walks the bones from the last one down, so a bone's
// parent (index < bone) is still absolute when the bone is converted — every bone only needs the ABSOLUTE pose of itself and of its
// parent, and all (instance, bone) pairs are independent.  Bones below first_nonroot keep their pose.
__global__ void __launch_bounds__(256) pose_relative_kernel(const float* __restrict__ abs_pos, const float* __restrict__ abs_rot,
	const short* __restrict__ parents, uint32_t bone_count, uint32_t first_nonroot, size_t n_bones_total, float* __restrict__ rel_pos, float* __restrict__ rel_rot)
{
	const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_bones_total) return;
	const uint32_t bone = (uint32_t)(i % bone_count);
	const size_t base = i - bone;
	V3 p = v3(abs_pos[3 * i], abs_pos[3 * i + 1], abs_pos[3 * i + 2]);
	Q4 r = q4(abs_rot[4 * i], abs_rot[4 * i + 1], abs_rot[4 * i + 2], abs_rot[4 * i + 3]);
	if (bone >= first_nonroot) {
		const size_t pi = base + (uint32_t)parents[bone];
		const Q4 c = q4(abs_rot[4 * pi], abs_rot[4 * pi + 1], abs_rot[4 * pi + 2], -abs_rot[4 * pi + 3]); // conjugated() = (x, y, z, -w), math.cpp:664-667
		const V3 pp = v3(abs_pos[3 * pi], abs_pos[3 * pi + 1], abs_pos[3 * pi + 2]);
		p = rotate(c, sub(p, pp));
		r = qmul(c, r);
	}
	rel_pos[3 * i] = p.x; rel_pos[3 * i + 1] = p.y; rel_pos[3 * i + 2] = p.z;
	rel_rot[4 * i] = r.x; rel_rot[4 * i + 1] = r.y; rel_rot[4 * i + 2] = r.z; rel_rot[4 * i + 3] = r.w;
}

// Pose::blend (pose.cpp:30-41) for every bone of every instance: positions a*inv + b*w, rotations scalar nlerp (math.cpp:677-692:
// dot summed ((x+y)+z)+w, sign flip of t, normalise with 1/sqrt).  weight is already clamped; the caller skips weight <= 0.001.
__global__ void __launch_bounds__(256) pose_blend_kernel(float* __restrict__ pos_a, float* __restrict__ rot_a, const float* __restrict__ pos_b,
	const float* __restrict__ rot_b, size_t n_bones_total, float weight)
{
	const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n_bones_total) return;
	const float inv = LB_FSUB(1.0f, weight);
#pragma unroll
	for (int k = 0; k < 3; ++k) pos_a[3 * i + k] = LB_FADD(LB_FMUL(pos_a[3 * i + k], inv), LB_FMUL(pos_b[3 * i + k], weight));
	const Q4 q1 = q4(rot_a[4 * i], rot_a[4 * i + 1], rot_a[4 * i + 2], rot_a[4 * i + 3]);
	const Q4 q2 = q4(rot_b[4 * i], rot_b[4 * i + 1], rot_b[4 * i + 2], rot_b[4 * i + 3]);
	float t = weight;
	const float d = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(q1.x, q2.x), LB_FMUL(q1.y, q2.y)), LB_FMUL(q1.z, q2.z)), LB_FMUL(q1.w, q2.w));
	if (d < 0) t = -t;
	Q4 q = q4(LB_FADD(LB_FMUL(q1.x, inv), LB_FMUL(q2.x, t)), LB_FADD(LB_FMUL(q1.y, inv), LB_FMUL(q2.y, t)),
		LB_FADD(LB_FMUL(q1.z, inv), LB_FMUL(q2.z, t)), LB_FADD(LB_FMUL(q1.w, inv), LB_FMUL(q2.w, t)));
	const float len2 = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(q.x, q.x), LB_FMUL(q.y, q.y)), LB_FMUL(q.z, q.z)), LB_FMUL(q.w, q.w));
	const float l = LB_FDIV(1.0f, LB_FSQRT(len2));
	rot_a[4 * i] = LB_FMUL(q.x, l); rot_a[4 * i + 1] = LB_FMUL(q.y, l); rot_a[4 * i + 2] = LB_FMUL(q.z, l); rot_a[4 * i + 3] = LB_FMUL(q.w, l);
}

// RenderModuleImpl::updateBoneAttachment (render_module.cpp:377-405) for a batch of attachments: the attached entity follows a bone of a
// posed model instance — world transform = parent_entity_transform.compose(bone_transform * relative_transform) (math.cpp:763, 859-861),
// scale replaced by the entity's own.  One thread per attachment; the bone comes from the absolute pose this system keeps in HBM.
__global__ void __launch_bounds__(256) bone_attachments_kernel(const float* __restrict__ abs_pos, const float* __restrict__ abs_rot, uint32_t bone_count,
	const uint32_t* __restrict__ instance, const uint32_t* __restrict__ bone, const float* __restrict__ relative7,
	const lb200_transform* __restrict__ parent_tr, const float* __restrict__ original_scale3, uint32_t n, lb200_transform* __restrict__ out)
{
	const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
	if (i >= n) return;
	const size_t bi = (size_t)instance[i] * bone_count + bone[i];
	Rigid b;
	b.pos = v3(abs_pos[3 * bi], abs_pos[3 * bi + 1], abs_pos[3 * bi + 2]);
	b.rot = q4(abs_rot[4 * bi], abs_rot[4 * bi + 1], abs_rot[4 * bi + 2], abs_rot[4 * bi + 3]);
	const float* r = relative7 + 7 * (size_t)i;
	Rigid rel;
	rel.pos = v3(r[0], r[1], r[2]);
	rel.rot = q4(r[3], r[4], r[5], r[6]);
	const Rigid local = rmul(b, rel); // LocalRigidTransform::operator*, math.cpp:859-861
	const lb200_transform p = parent_tr[i];
	D3 pos;
	Q4 rot;
	compose_rigid(d3(p.pos[0], p.pos[1], p.pos[2]), q4(p.rot[0], p.rot[1], p.rot[2], p.rot[3]), v3(p.scale[0], p.scale[1], p.scale[2]), local, pos, rot);
	lb200_transform o;
	o.pos[0] = pos.x; o.pos[1] = pos.y; o.pos[2] = pos.z;
	o.rot[0] = rot.x; o.rot[1] = rot.y; o.rot[2] = rot.z; o.rot[3] = rot.w;
	o.scale[0] = original_scale3[3 * (size_t)i]; o.scale[1] = original_scale3[3 * (size_t)i + 1]; o.scale[2] = original_scale3[3 * (size_t)i + 2];
	out[i] = o;
}

} // namespace

struct lb200_animation {
	lb200_ctx* ctx = nullptr;
	uint32_t bone_count = 0, max_level = 0, n_clips = 0, max_instances = 0, n_instances = 0, n_vertices = 0;
	// every table created with the system gets an address, 16 bytes when it has no entries (TABLE_MIN_BYTES)
	DeviceArray<DevClip> d_clips;
	DeviceArray<DevTrack> d_tracks;
	DeviceArray<float4> d_const_t;
	DeviceArray<float4> d_const_r_value;
	DeviceArray<uint32_t> d_const_r_bone;
	DeviceArray<uint32_t> d_stream;
	DeviceArray<float4> d_bind; // bind_pos[B], bind_rot[B], inv_bind_pos[B], inv_bind_rot[B]
	DeviceArray<float4> d_key_pos, d_key_rot; DeviceArray<unsigned char> d_key_flags;
	std::vector<DevClip> clips;                // host copy of d_clips
	std::vector<lb200_root_motion> root_motion; // per clip, lb200_animation_set_root_motion; flags 0 or both tracks -1: none
	DeviceArray<short> d_parents; DeviceArray<unsigned char> d_level_bones; DeviceArray<uint32_t> d_level_start;
	int lanes_per_instance = 8;
	// lb200_animation_set_launch (0 = environment switch, else the default) and what the last update / skin launched
	int pose_lanes = 0, skin_group = 0;
	int last_pose_lanes = 0, last_skin_group = 0;
	DeviceArray<uint32_t> d_clip_index, d_time;
	uint32_t n_layers = 0; DeviceArray<uint32_t> d_layer_clip, d_layer_time; DeviceArray<float> d_layer_weight; // all three or none
	// sample-list mode (lb200_animation_set_samples): CSR offsets [max_instances + 1] and the samples, grown to the largest list set
	bool sample_lists = false;
	DeviceArray<uint32_t> d_sample_offsets; DeviceArray<lb200_sample> d_samples;
	// IK ops of the lists (lb200_animation_set_stacks): CSR offsets [max_instances + 1], the op table (IkOp pairs, then the leaves' bone
	// paths) grown like the samples; n_ik = ops of the current lists (0: the IK-free kernels run)
	uint32_t n_ik = 0;
	DeviceArray<uint32_t> d_ik_offsets; DeviceArray<uint4> d_iks;
	std::vector<short> parents; // Model::getBoneParent, for resolving IK chains
	// palettes and poses, allocated by the first update that asks for them; d_pos / d_rot and d_rel_pos / d_rel_rot go in pairs
	DeviceArray<float> d_dq, d_mtx, d_pos, d_rot;
	DeviceArray<float> d_rel_pos, d_rel_rot; // Pose::computeRelative of d_pos / d_rot
	uint32_t first_nonroot = 0;
	DeviceArray<float> d_mesh_pos; DeviceArray<float4> d_mesh_w; DeviceArray<short> d_mesh_idx;
	DeviceArray<float> d_skinned;
	DeviceArray<unsigned long long> d_checksum;
	// lb200_animation_set_entities: EntityRef::index per instance [0, n_entities) (max_instances allocated by the first call), < 0 = none
	DeviceArray<int32_t> d_entity;
	uint32_t n_entities = 0;
};

namespace {
constexpr size_t TABLE_MIN_BYTES = 16;

// a pair of pose buffers (positions 3 floats, rotations 4 floats per bone and instance): both or neither
int allocPosePair(lb200_ctx* ctx, DeviceArray<float>& pos, DeviceArray<float>& rot, size_t nb) {
	DeviceArray<float> p, r;
	LB200_CUDA(ctx, p.alloc(3 * nb));
	LB200_CUDA(ctx, r.alloc(4 * nb));
	pos = std::move(p); rot = std::move(r);
	return LB200_OK;
}

bool hasRootMotion(const lb200_root_motion& rm) { return rm.flags && (rm.translation_track >= 0 || rm.rotation_track >= 0); }

// The decoded keyframes of the listed clips: decode_clips_kernel from the packed tracks, then root_motion_tables_kernel for those of them
// with root motion.  Waits for both, so that the frame lists can go.
int decodeClips(lb200_animation* a, const std::vector<uint32_t>& list) {
	lb200_ctx* ctx = a->ctx;
	std::vector<uint32_t> frame_clip, frame_index, rm_clip, rm_frame;
	for (uint32_t c : list) {
		const bool rm = hasRootMotion(a->root_motion[c]);
		for (uint32_t f = 0; f < key_rows(a->clips[c].frame_count); ++f) {
			frame_clip.push_back(c); frame_index.push_back(f);
			if (rm) { rm_clip.push_back(c); rm_frame.push_back(f); }
		}
	}
	if (frame_clip.empty()) return LB200_OK;
	cudaStream_t st = ctx->stream;
	const uint32_t B = a->bone_count;
	DeviceArray<uint32_t> d_fc, d_fi;
	LB200_CUDA(ctx, d_fc.alloc(frame_clip.size()));
	LB200_CUDA(ctx, d_fi.alloc(frame_index.size()));
	LB200_CUDA(ctx, cudaMemcpyAsync(d_fc, frame_clip.data(), sizeof(uint32_t) * frame_clip.size(), cudaMemcpyHostToDevice, st));
	LB200_CUDA(ctx, cudaMemcpyAsync(d_fi, frame_index.data(), sizeof(uint32_t) * frame_index.size(), cudaMemcpyHostToDevice, st));
	DeviceArray<uint32_t> d_rc, d_rf;
	DeviceArray<int4> d_rm;
	if (!rm_clip.empty()) {
		std::vector<int4> rm(a->n_clips);
		for (uint32_t c = 0; c < a->n_clips; ++c) {
			const lb200_root_motion& r = a->root_motion[c];
			rm[c] = make_int4((int)r.flags, r.translation_track, r.rotation_track, 0);
		}
		LB200_CUDA(ctx, d_rc.alloc(rm_clip.size()));
		LB200_CUDA(ctx, d_rf.alloc(rm_frame.size()));
		LB200_CUDA(ctx, d_rm.alloc(rm.size()));
		LB200_CUDA(ctx, cudaMemcpyAsync(d_rc, rm_clip.data(), sizeof(uint32_t) * rm_clip.size(), cudaMemcpyHostToDevice, st));
		LB200_CUDA(ctx, cudaMemcpyAsync(d_rf, rm_frame.data(), sizeof(uint32_t) * rm_frame.size(), cudaMemcpyHostToDevice, st));
		LB200_CUDA(ctx, cudaMemcpyAsync(d_rm, rm.data(), sizeof(int4) * rm.size(), cudaMemcpyHostToDevice, st));
	}
	DecodeParams D;
	D.clips = a->d_clips; D.tracks = a->d_tracks; D.const_t = a->d_const_t; D.const_r_value = a->d_const_r_value; D.const_r_bone = a->d_const_r_bone;
	D.stream = a->d_stream; D.bind_pos = a->d_bind; D.bind_rot = a->d_bind + B;
	D.key_pos = a->d_key_pos; D.key_rot = a->d_key_rot; D.key_flags = a->d_key_flags;
	D.frame_clip = d_fc; D.frame_index = d_fi; D.bone_count = B;
	decode_clips_kernel<<<(unsigned)frame_clip.size(), 256, 0, st>>>(D);
	LB200_CHECK_LAUNCH(ctx);
	if (!rm_clip.empty()) {
		RootMotionParams R;
		R.clips = a->d_clips; R.tracks = a->d_tracks; R.stream = a->d_stream; R.root_motion = d_rm;
		R.frame_clip = d_rc; R.frame_index = d_rf; R.n = (uint32_t)rm_clip.size(); R.bone_count = B;
		R.key_pos = a->d_key_pos; R.key_rot = a->d_key_rot;
		root_motion_tables_kernel<<<(R.n + 127) / 128, 128, 0, st>>>(R);
		LB200_CHECK_LAUNCH(ctx);
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(st)); // before the frame lists are freed
	return LB200_OK;
}
} // namespace

extern "C" {

int lb200_animation_create(lb200_ctx* ctx, const lb200_skeleton* sk, const lb200_clip* clips, uint32_t n_clips, const lb200_mesh* mesh,
	uint32_t max_instances, lb200_animation** out)
{
	if (!out || !sk || !clips || !n_clips || !max_instances) return LB200_ERR_INVALID;
	if (!ctx) return LB200_ERR_NO_DEVICE;
	*out = nullptr;
	const uint32_t B = sk->bone_count;
	if (!B || B > 196 || !sk->parents || !sk->bind_relative7 || !sk->inverse_bind7) { lb200_set_error(ctx, "bad skeleton (bone_count %u)", B); return LB200_ERR_INVALID; }
	// pose.cpp:68-69 starts at first_nonroot; every later bone must have an earlier parent (model.cpp:381-384)
	std::vector<unsigned char> levels(B, 0);
	uint32_t max_level = 0;
	const uint32_t first = sk->first_nonroot_bone_index < 0 ? B : (uint32_t)sk->first_nonroot_bone_index;
	for (uint32_t i = first; i < B; ++i) {
		const int p = sk->parents[i];
		if (p < 0 || (uint32_t)p >= i) { lb200_set_error(ctx, "bone %u: parent %d is not an earlier bone", i, p); return LB200_ERR_INVALID; }
		levels[i] = (unsigned char)(levels[p] + 1);
		if (levels[i] > max_level) max_level = levels[i];
	}
	// bones of depth >= 1 grouped by depth (stable in bone order)
	std::vector<unsigned char> level_bones;
	std::vector<uint32_t> level_start(max_level + 2, 0);
	for (uint32_t l = 1; l <= max_level; ++l) {
		level_start[l] = (uint32_t)level_bones.size();
		for (uint32_t i = first; i < B; ++i) if (levels[i] == l) level_bones.push_back((unsigned char)i);
	}
	level_start[max_level + 1] = (uint32_t)level_bones.size();
	// lanes per instance: the choice minimises the lane-steps of the absolute pass, G * sum_l ceil(width_l / G), over G >= 8 (fewer
	// lanes cost occupancy).  G * ceil(w / G) never falls as G doubles, and a tie keeps the smaller G, so that choice is always 8.
	// G = 4, 16 and 32 run only when asked for (LB200_POSE_LANES, lb200_animation_set_launch).
	const int best_g = 8;
	std::vector<DevClip> dc(n_clips);
	std::vector<DevTrack> tracks;
	std::vector<float4> cts, cr_values;
	std::vector<uint32_t> cr_bones;
	auto packTrack = [](const lb200_track& t) {
		DevTrack d;
		memcpy(d.min, t.min, sizeof(d.min));
		memcpy(d.to_range, t.to_range, sizeof(d.to_range));
		d.bone_offset = (uint32_t)t.bone_index | ((uint32_t)t.offset_bits << 16);
		d.bits = (uint32_t)t.bitsizes[0] | ((uint32_t)t.bitsizes[1] << 8) | ((uint32_t)t.bitsizes[2] << 16) | ((uint32_t)t.skipped_channel << 24);
		return d;
	};
	// unpackChannel's mask (1 << bitsize) - 1 is defined below 64 bits only (animation.cpp:315); the importer writes at most 31
	auto channelsFit = [](const lb200_track& t) { return t.bitsizes[0] < 64 && t.bitsizes[1] < 64 && t.bitsizes[2] < 64; };
	std::vector<uint32_t> stream;
	auto appendStream = [&](const uint8_t* data, uint32_t bytes) -> uint32_t {
		const uint32_t off = (uint32_t)stream.size() * 4;
		const size_t words = (bytes + 3) / 4 + 4; // + 16 zero bytes: the 3-word unaligned read never leaves the blob
		const size_t base = stream.size();
		stream.resize(base + words, 0u);
		if (bytes) memcpy(stream.data() + base, data, bytes);
		return off;
	};
	for (uint32_t c = 0; c < n_clips; ++c) {
		const lb200_clip& s = clips[c];
		DevClip& d = dc[c];
		if (!(s.fps > 0) || !s.frame_count) { lb200_set_error(ctx, "clip %u: fps/frame_count invalid", c); return LB200_ERR_INVALID; }
		// the sampler's clamp frame_count - 0.00001f stays at or below frame_count only while frame_count is exact in fp32 (key_rows)
		if (s.frame_count > MAX_FRAME_COUNT) { lb200_set_error(ctx, "clip %u: %u frames, 2^24 or more", c, s.frame_count); return LB200_ERR_INVALID; }
		d.fps = s.fps; d.frame_count = s.frame_count;
		d.t_bits = s.translations_frame_size_bits; d.r_bits = s.rotations_frame_size_bits;
		d.n_t = s.n_translations; d.n_ct = s.n_const_translations; d.n_r = s.n_rotations; d.n_cr = s.n_const_rotations;
		d.t_off = (uint32_t)tracks.size();
		for (uint32_t i = 0; i < s.n_translations; ++i) {
			if (s.translations[i].bone_index >= B || !channelsFit(s.translations[i])) { lb200_set_error(ctx, "clip %u: translation track %u: bone or channel width out of range", c, i); return LB200_ERR_INVALID; }
			tracks.push_back(packTrack(s.translations[i]));
		}
		d.r_off = (uint32_t)tracks.size();
		for (uint32_t i = 0; i < s.n_rotations; ++i) {
			if (s.rotations[i].bone_index >= B || s.rotations[i].skipped_channel > 3 || !channelsFit(s.rotations[i])) { lb200_set_error(ctx, "clip %u: rotation track %u: bone, skipped channel or channel width out of range", c, i); return LB200_ERR_INVALID; }
			tracks.push_back(packTrack(s.rotations[i]));
		}
		d.ct_off = (uint32_t)cts.size();
		for (uint32_t i = 0; i < s.n_const_translations; ++i) { if (s.const_translations[i].bone_index >= B) { lb200_set_error(ctx, "clip %u: constant translation %u: bone %u out of range", c, i, (unsigned)s.const_translations[i].bone_index); return LB200_ERR_INVALID; } const lb200_const_translation& c0 = s.const_translations[i]; cts.push_back(make_float4(c0.value[0], c0.value[1], c0.value[2], __builtin_bit_cast(float, (uint32_t)c0.bone_index))); }
		d.cr_off = (uint32_t)cr_values.size();
		for (uint32_t i = 0; i < s.n_const_rotations; ++i) { if (s.const_rotations[i].bone_index >= B) { lb200_set_error(ctx, "clip %u: constant rotation %u: bone %u out of range", c, i, (unsigned)s.const_rotations[i].bone_index); return LB200_ERR_INVALID; } const lb200_const_rotation& c0 = s.const_rotations[i]; cr_values.push_back(make_float4(c0.value[0], c0.value[1], c0.value[2], c0.value[3])); cr_bones.push_back(c0.bone_index); }
		// streams must hold (frame_count + 1) frames + the loader's 8-byte tail (animation.cpp:439)
		const uint64_t need_t = s.n_translations ? ((uint64_t)d.t_bits * ((uint64_t)s.frame_count + 1) + 7) / 8 : 0;
		const uint64_t need_r = s.n_rotations ? ((uint64_t)d.r_bits * ((uint64_t)s.frame_count + 1) + 7) / 8 : 0;
		if (s.translation_stream_bytes < need_t || s.rotation_stream_bytes < need_r) { lb200_set_error(ctx, "clip %u: bit stream shorter than (frame_count+1) frames", c); return LB200_ERR_INVALID; }
		d.t_stream = appendStream(s.translation_stream, s.translation_stream_bytes);
		d.r_stream = appendStream(s.rotation_stream, s.rotation_stream_bytes);
		// Time::fromSeconds(m_frame_count / m_fps): a length that does not fit the u32 ticks would be an undefined conversion
		const float length = ((float)s.frame_count / s.fps) * (float)(1 << 15);
		if (!(length < 4294967296.0f)) { lb200_set_error(ctx, "clip %u: %u frames at %g fps last 2^32 ticks or more", c, s.frame_count, (double)s.fps); return LB200_ERR_INVALID; }
		d.length_ticks = (uint32_t)length;
		if (!d.length_ticks) { lb200_set_error(ctx, "clip %u: %u frames at %g fps last less than one tick", c, s.frame_count, (double)s.fps); return LB200_ERR_INVALID; }
		d.pad[0] = d.pad[1] = d.pad[2] = 0;
	}
	// decoded keyframe tables: key_rows (frame_count + 2) rows x Bp bones per clip, refused before anything is allocated when their
	// offsets would not fit the u32 key_off
	const uint32_t Bp = (B + 3u) & ~3u;
	size_t key_entries = 0;
	for (uint32_t c = 0; c < n_clips; ++c) {
		dc[c].key_off = (uint32_t)key_entries;
		dc[c].flag_off = c * Bp;
		key_entries += (size_t)key_rows(dc[c].frame_count) * Bp;
		if (key_entries > 0x7fffffffull) { lb200_set_error(ctx, "decoded clips exceed 2^31 keyframe entries"); return LB200_ERR_INVALID; }
	}

	// any early return below (allocation or copy failure) releases what has been allocated so far
	std::unique_ptr<lb200_animation, decltype(&lb200_animation_destroy)> a(new (std::nothrow) lb200_animation, lb200_animation_destroy);
	if (!a) return LB200_ERR_CUDA;
	a->ctx = ctx; a->bone_count = B; a->max_level = max_level; a->n_clips = n_clips; a->max_instances = max_instances;
	a->first_nonroot = first;
	a->parents.assign(sk->parents, sk->parents + B);
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, a->d_clips.alloc(n_clips, TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_tracks.alloc(tracks.size(), TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_const_t.alloc(cts.size(), TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_const_r_value.alloc(cr_values.size(), TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_const_r_bone.alloc(cr_bones.size(), TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_stream.alloc(stream.size(), TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_bind.alloc(4 * B, TABLE_MIN_BYTES));
	std::vector<float4> bind(4 * (size_t)B);
	for (uint32_t i = 0; i < B; ++i) {
		const float* r = sk->bind_relative7 + 7 * (size_t)i;
		const float* v = sk->inverse_bind7 + 7 * (size_t)i;
		bind[i] = make_float4(r[0], r[1], r[2], 0.f);
		bind[B + i] = make_float4(r[3], r[4], r[5], r[6]);
		bind[2 * B + i] = make_float4(v[0], v[1], v[2], 0.f);
		bind[3 * B + i] = make_float4(v[3], v[4], v[5], v[6]);
	}
	LB200_CUDA(ctx, a->d_parents.alloc(B, TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_level_bones.alloc(level_bones.size(), TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_level_start.alloc(level_start.size(), TABLE_MIN_BYTES));
	a->lanes_per_instance = best_g;
	LB200_CUDA(ctx, a->d_clip_index.alloc(max_instances, TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_time.alloc(max_instances, TABLE_MIN_BYTES));
	LB200_CUDA(ctx, a->d_checksum.alloc(1, TABLE_MIN_BYTES));
	cudaStream_t st = ctx->stream;
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_clips, dc.data(), sizeof(DevClip) * n_clips, cudaMemcpyHostToDevice, st));
	if (!tracks.empty()) LB200_CUDA(ctx, cudaMemcpyAsync(a->d_tracks, tracks.data(), sizeof(DevTrack) * tracks.size(), cudaMemcpyHostToDevice, st));
	if (!cts.empty()) LB200_CUDA(ctx, cudaMemcpyAsync(a->d_const_t, cts.data(), sizeof(float4) * cts.size(), cudaMemcpyHostToDevice, st));
	if (!cr_values.empty()) LB200_CUDA(ctx, cudaMemcpyAsync(a->d_const_r_value, cr_values.data(), sizeof(float4) * cr_values.size(), cudaMemcpyHostToDevice, st));
	if (!cr_bones.empty()) LB200_CUDA(ctx, cudaMemcpyAsync(a->d_const_r_bone, cr_bones.data(), sizeof(uint32_t) * cr_bones.size(), cudaMemcpyHostToDevice, st));
	if (!stream.empty()) LB200_CUDA(ctx, cudaMemcpyAsync(a->d_stream, stream.data(), sizeof(uint32_t) * stream.size(), cudaMemcpyHostToDevice, st));
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_bind, bind.data(), sizeof(float4) * bind.size(), cudaMemcpyHostToDevice, st));
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_parents, sk->parents, sizeof(short) * B, cudaMemcpyHostToDevice, st));
	if (!level_bones.empty()) LB200_CUDA(ctx, cudaMemcpyAsync(a->d_level_bones, level_bones.data(), level_bones.size(), cudaMemcpyHostToDevice, st));
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_level_start, level_start.data(), sizeof(uint32_t) * level_start.size(), cudaMemcpyHostToDevice, st));
	if (mesh && mesh->n_vertices) {
		a->n_vertices = mesh->n_vertices;
		for (uint32_t v = 0; v < mesh->n_vertices * 4; ++v) if (mesh->indices4[v] < 0 || (uint32_t)mesh->indices4[v] >= B) return LB200_ERR_INVALID;
		LB200_CUDA(ctx, a->d_mesh_pos.alloc(3 * mesh->n_vertices, TABLE_MIN_BYTES));
		LB200_CUDA(ctx, a->d_mesh_w.alloc(mesh->n_vertices, TABLE_MIN_BYTES));
		LB200_CUDA(ctx, a->d_mesh_idx.alloc(4 * mesh->n_vertices, TABLE_MIN_BYTES));
		LB200_CUDA(ctx, cudaMemcpyAsync(a->d_mesh_pos, mesh->positions3, sizeof(float) * 3 * mesh->n_vertices, cudaMemcpyHostToDevice, st));
		LB200_CUDA(ctx, cudaMemcpyAsync(a->d_mesh_w, mesh->weights4, sizeof(float4) * mesh->n_vertices, cudaMemcpyHostToDevice, st));
		LB200_CUDA(ctx, cudaMemcpyAsync(a->d_mesh_idx, mesh->indices4, sizeof(short) * 4 * mesh->n_vertices, cudaMemcpyHostToDevice, st));
	}
	{
		LB200_CUDA(ctx, a->d_key_pos.alloc(key_entries, TABLE_MIN_BYTES));
		LB200_CUDA(ctx, a->d_key_rot.alloc(key_entries, TABLE_MIN_BYTES));
		LB200_CUDA(ctx, a->d_key_flags.alloc((size_t)n_clips * Bp, TABLE_MIN_BYTES));
		a->clips = dc;
		a->root_motion.assign(n_clips, lb200_root_motion{0u, -1, -1});
		std::vector<uint32_t> all(n_clips);
		for (uint32_t c = 0; c < n_clips; ++c) all[c] = c;
		const int rc = decodeClips(a.get(), all);
		if (rc) return rc;
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(st));
	const int smem_max = (int)(sizeof(float4) * (2 * 196 * (POSE_THREADS / 8) + 2 * 196 + 128));
	const int smem_max4 = (int)std::min<size_t>(220 * 1024, sizeof(float4) * (2 * 196 * (POSE_THREADS / 4) + 2 * 196 + 128));
	for (int i = 0; i < 4; ++i) {
		const int smem = i == shapeIndex(4) ? smem_max4 : smem_max;
		for (PoseKernel k : {POSE_CLIP_KERNELS[i], POSE_LIST_KERNELS[i], POSE_IK_KERNELS[i]}) LB200_CUDA(ctx, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
		for (PoseManyKernel k : {POSE_MANY_KERNELS[i], POSE_MANY_IK_KERNELS[i]}) LB200_CUDA(ctx, cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
	}
	for (int i = 0; i < 3; ++i) LB200_CUDA(ctx, cudaFuncSetAttribute(SKIN_KERNELS[i], cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((4 << i) * 196 * 3 * sizeof(float4))));
	*out = a.release();
	return LB200_OK;
}

void lb200_animation_destroy(lb200_animation* a) {
	if (!a) return;
	cudaSetDevice(a->ctx->device);
	cudaStreamSynchronize(a->ctx->stream);
	delete a;
}

int lb200_animation_set_instances(lb200_animation* a, const uint32_t* clip_index, const uint32_t* time_ticks, uint32_t n) {
	if (!a || !clip_index || !time_ticks || n > a->max_instances) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	for (uint32_t i = 0; i < n; ++i) if (clip_index[i] >= a->n_clips) { lb200_set_error(ctx, "instance %u: clip %u out of range", i, clip_index[i]); return LB200_ERR_INVALID; }
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_clip_index, clip_index, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_time, time_ticks, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	a->n_instances = n;
	a->n_layers = 0; // layer tables are per instance: set them again after changing the instances
	a->sample_lists = false;
	a->n_ik = 0;
	return LB200_OK;
}

int lb200_animation_set_stacks(lb200_animation* a, uint32_t n_instances, const uint32_t* offsets, const lb200_sample* samples,
	const uint32_t* ik_offsets, const lb200_ik* iks)
{
	if (!a || !offsets || n_instances > a->max_instances) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (offsets[0] != 0) { lb200_set_error(ctx, "set_samples: offsets[0] is %u, not 0", offsets[0]); return LB200_ERR_INVALID; }
	for (uint32_t i = 0; i < n_instances; ++i) {
		if (offsets[i + 1] < offsets[i]) { lb200_set_error(ctx, "set_samples: offsets decrease at instance %u", i); return LB200_ERR_INVALID; }
	}
	const uint32_t total = offsets[n_instances];
	if (total && !samples) return LB200_ERR_INVALID;
	for (uint32_t k = 0; k < total; ++k) {
		if (samples[k].clip >= a->n_clips) { lb200_set_error(ctx, "set_samples: sample %u: clip %u out of range", k, samples[k].clip); return LB200_ERR_INVALID; }
	}
	// IK ops: validated, then put in their device form (IkOp) with the root-to-leaf path of each distinct leaf after the ops
	const uint32_t n_ik = ik_offsets ? ik_offsets[n_instances] : 0;
	std::vector<uint4> table;
	if (ik_offsets) {
		if (ik_offsets[0] != 0) { lb200_set_error(ctx, "set_stacks: ik_offsets[0] is %u, not 0", ik_offsets[0]); return LB200_ERR_INVALID; }
		for (uint32_t i = 0; i < n_instances; ++i) {
			if (ik_offsets[i + 1] < ik_offsets[i]) { lb200_set_error(ctx, "set_stacks: ik_offsets decrease at instance %u", i); return LB200_ERR_INVALID; }
		}
		if (n_ik && !iks) return LB200_ERR_INVALID;
		const uint32_t B = a->bone_count;
		std::vector<unsigned char> paths;
		std::vector<int64_t> leaf_path(B, -1); // byte offset of the leaf's path inside `paths`
		std::vector<uint32_t> path_len(B, 0);
		table.resize(2 * (size_t)n_ik);
		for (uint32_t i = 0; i < n_instances; ++i) {
			const uint32_t list_len = offsets[i + 1] - offsets[i];
			for (uint32_t k = ik_offsets[i]; k < ik_offsets[i + 1]; ++k) {
				const lb200_ik& op = iks[k];
				if (op.after > list_len || (k > ik_offsets[i] && op.after < iks[k - 1].after)) {
					lb200_set_error(ctx, "set_stacks: IK op %u: after %u is past the instance's %u samples or before the op it follows", k, op.after, list_len);
					return LB200_ERR_INVALID;
				}
				if (op.leaf_bone >= B || op.bone_count == 0 || op.bone_count > IK_MAX_BONES) {
					lb200_set_error(ctx, "set_stacks: IK op %u: leaf bone %u / bone count %u out of range", k, op.leaf_bone, op.bone_count);
					return LB200_ERR_INVALID;
				}
				if (leaf_path[op.leaf_bone] < 0) { // Model::getBoneParent walk from the leaf to the bone whose parent is -1
					std::vector<unsigned char> up;
					for (int b = (int)op.leaf_bone; b >= 0; b = a->parents[b]) {
						if ((uint32_t)b >= B || up.size() == B) { lb200_set_error(ctx, "set_stacks: bone %u: its parents leave the skeleton or loop", op.leaf_bone); return LB200_ERR_INVALID; }
						up.push_back((unsigned char)b);
					}
					leaf_path[op.leaf_bone] = (int64_t)paths.size();
					path_len[op.leaf_bone] = (uint32_t)up.size();
					paths.insert(paths.end(), up.rbegin(), up.rend());
				}
				if (op.bone_count > path_len[op.leaf_bone]) { // controller.cpp:185-186 would read bone -1
					lb200_set_error(ctx, "set_stacks: IK op %u: a chain of %u bones from bone %u leaves the skeleton", k, op.bone_count, op.leaf_bone);
					return LB200_ERR_INVALID;
				}
				table[2 * (size_t)k] = make_uint4(op.after, path_len[op.leaf_bone], op.bone_count, __builtin_bit_cast(uint32_t, op.alpha));
				table[2 * (size_t)k + 1] = make_uint4(__builtin_bit_cast(uint32_t, op.target[0]), __builtin_bit_cast(uint32_t, op.target[1]),
					__builtin_bit_cast(uint32_t, op.target[2]), (uint32_t)(sizeof(uint4) * table.size() + leaf_path[op.leaf_bone]));
			}
		}
		const size_t ops_words = table.size();
		table.resize(ops_words + (paths.size() + 15) / 16, make_uint4(0, 0, 0, 0));
		if (!paths.empty()) memcpy(table.data() + ops_words, paths.data(), paths.size());
	}
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	// every allocation before anything is replaced, so that a failed one leaves the system as it was
	if (!a->d_sample_offsets) LB200_CUDA(ctx, a->d_sample_offsets.alloc((size_t)a->max_instances + 1));
	if (n_ik && !a->d_ik_offsets) LB200_CUDA(ctx, a->d_ik_offsets.alloc((size_t)a->max_instances + 1));
	DeviceArray<lb200_sample> grown;
	DeviceArray<uint4> grown_iks;
	if (a->d_samples.size() < total) LB200_CUDA(ctx, grown.alloc(std::max<size_t>(total, 2 * a->d_samples.size())));
	if (a->d_iks.size() < table.size()) LB200_CUDA(ctx, grown_iks.alloc(std::max<size_t>(table.size(), 2 * a->d_iks.size())));
	if (grown || grown_iks) {
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // an update still reading the old lists
		if (grown) a->d_samples = std::move(grown);
		if (grown_iks) a->d_iks = std::move(grown_iks);
	}
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_sample_offsets, offsets, sizeof(uint32_t) * ((size_t)n_instances + 1), cudaMemcpyHostToDevice, ctx->stream));
	if (total) LB200_CUDA(ctx, cudaMemcpyAsync(a->d_samples, samples, sizeof(lb200_sample) * total, cudaMemcpyHostToDevice, ctx->stream));
	if (n_ik) {
		LB200_CUDA(ctx, cudaMemcpyAsync(a->d_ik_offsets, ik_offsets, sizeof(uint32_t) * ((size_t)n_instances + 1), cudaMemcpyHostToDevice, ctx->stream));
		LB200_CUDA(ctx, cudaMemcpyAsync(a->d_iks, table.data(), sizeof(uint4) * table.size(), cudaMemcpyHostToDevice, ctx->stream));
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	a->n_instances = n_instances;
	a->n_layers = 0;
	a->sample_lists = true;
	a->n_ik = n_ik;
	return LB200_OK;
}

int lb200_animation_set_samples(lb200_animation* a, uint32_t n_instances, const uint32_t* offsets, const lb200_sample* samples) {
	return lb200_animation_set_stacks(a, n_instances, offsets, samples, nullptr, nullptr);
}

int lb200_animation_set_entities(lb200_animation* a, const int32_t* entity_of_instance, uint32_t n) {
	if (!a) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (n > a->max_instances || (n && !entity_of_instance)) { lb200_set_error(ctx, "set_entities: %u ids for %u instances at most, or no array", n, a->max_instances); return LB200_ERR_INVALID; }
	{
		std::vector<int32_t> ids(entity_of_instance, entity_of_instance + n);
		std::sort(ids.begin(), ids.end());
		for (uint32_t i = 1; i < n; ++i) {
			if (ids[i] >= 0 && ids[i] == ids[i - 1]) { lb200_set_error(ctx, "set_entities: entity %d is listed twice", ids[i]); return LB200_ERR_INVALID; }
		}
	}
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!a->d_entity) LB200_CUDA(ctx, a->d_entity.alloc(a->max_instances));
	if (n) {
		LB200_CUDA(ctx, cudaMemcpyAsync(a->d_entity, entity_of_instance, sizeof(int32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
		LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // a build still reading the old ids, and the caller's array
	}
	a->n_entities = n;
	return LB200_OK;
}

int lb200_animation_set_root_motion(lb200_animation* a, uint32_t n_clips, const lb200_root_motion* per_clip) {
	if (!a || (n_clips && !per_clip)) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (n_clips != a->n_clips) { lb200_set_error(ctx, "set_root_motion: %u entries for %u clips", n_clips, a->n_clips); return LB200_ERR_INVALID; }
	for (uint32_t c = 0; c < n_clips; ++c) {
		const lb200_root_motion& r = per_clip[c];
		if (r.flags & ~(RM_Y | RM_XZ | RM_ROT)) { lb200_set_error(ctx, "set_root_motion: clip %u: flags 0x%x outside ANY_ROOT_MOTION", c, r.flags); return LB200_ERR_INVALID; }
		if (r.translation_track < -1 || r.translation_track >= (int64_t)a->clips[c].n_t || r.rotation_track < -1 || r.rotation_track >= (int64_t)a->clips[c].n_r) {
			lb200_set_error(ctx, "set_root_motion: clip %u: track %d / %d out of range", c, r.translation_track, r.rotation_track);
			return LB200_ERR_INVALID;
		}
	}
	// clips with root motion before or after: decoded again, then given their new tables
	std::vector<uint32_t> list;
	for (uint32_t c = 0; c < n_clips; ++c) {
		if (hasRootMotion(a->root_motion[c]) || hasRootMotion(per_clip[c])) list.push_back(c);
		a->root_motion[c] = per_clip[c];
	}
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	return decodeClips(a, list);
}

} // extern "C"

namespace {
// the palette and pose buffers `flags` asks for, allocated once per system at max_instances
int allocOutputs(lb200_animation* a, uint32_t flags) {
	lb200_ctx* ctx = a->ctx;
	const size_t nb = (size_t)a->max_instances * a->bone_count;
	if ((flags & LB200_PALETTE_DUAL_QUAT) && !a->d_dq) LB200_CUDA(ctx, a->d_dq.alloc(8 * nb));
	if ((flags & LB200_PALETTE_MATRIX) && !a->d_mtx) LB200_CUDA(ctx, a->d_mtx.alloc(16 * nb));
	if ((flags & LB200_PALETTE_POSE) && (!a->d_pos || !a->d_rot)) {
		const int rc = allocPosePair(ctx, a->d_pos, a->d_rot, nb);
		if (rc) return rc;
	}
	return LB200_OK;
}

// lanes per instance a system asks for: its set_launch value, then LB200_POSE_LANES, then its default (8)
int requestedLanes(const lb200_animation* a) {
	static const int g_env = [] { const char* e = getenv("LB200_POSE_LANES"); const int v = e ? atoi(e) : 0; return (v == 4 || v == 8 || v == 16 || v == 32) ? v : 0; }();
	return a->pose_lanes ? a->pose_lanes : g_env ? g_env : a->lanes_per_instance;
}

// 4 lanes = 32 instances per block: only while their poses of the largest skeleton fit in shared memory
int fitLanes(int G, uint32_t bone_count) {
	if (G == 4) {
		const uint32_t bp = (bone_count + 3u) & ~3u;
		if (sizeof(float4) * (2 * (size_t)bp * (POSE_THREADS / 4) + 2 * bp + 128) > 200 * 1024) G = 8;
	}
	return G;
}

// dynamic shared memory of one block of the pose kernel: inverse bind + topology, then per_block poses
size_t poseSmemBytes(const lb200_animation* a, unsigned per_block) {
	const uint32_t Bp_ = (a->bone_count + 3u) & ~3u;
	const uint32_t n_ls_ = (a->max_level + 2u + 3u) & ~3u;
	const size_t shared_words16 = 2 * Bp_ + (n_ls_ * 4 + Bp_ * 2 + Bp_ + 15) / 16; // in float4 units
	return sizeof(float4) * (shared_words16 + 2 * (size_t)Bp_ * per_block);
}

// Time::fromSeconds: u32(time * ONE_SECOND), animation.h:21-24 (:462 uses -time_delta for rewinds)
// animation_module.cpp:458 `if (time_delta > 0) ... else ...`: zero takes the rewind branch too, which leaves a time below the clip
// length alone and wraps one at or beyond it (time % length), exactly as the reference does on every update
PoseStep timeStep(float time_delta) {
	PoseStep A;
	A.dt_negative = !(time_delta > 0);
	A.dt_ticks = (uint32_t)((A.dt_negative ? -time_delta : time_delta) * (float)(1 << 15));
	A.advance = 1;
	return A;
}
// A system's tables for the pose kernels, with the outputs `flags` asks for.  The pose body samples the base clips and layers of clip
// mode, or the sample lists and the bind pose, whose fields share the unions.
AnimSysParams sysParams(const lb200_animation* a, uint32_t flags) {
	AnimSysParams S;
	S.clips = a->d_clips; S.key_pos = a->d_key_pos; S.key_rot = a->d_key_rot; S.key_flags = a->d_key_flags;
	S.inv_bind_pos = a->d_bind + 2 * a->bone_count; S.inv_bind_rot = a->d_bind + 3 * a->bone_count;
	S.parents = a->d_parents; S.level_bones = a->d_level_bones; S.level_start = a->d_level_start;
	S.bone_count = a->bone_count; S.max_level = a->max_level; S.n_instances = a->n_instances;
	S.time_ticks = a->d_time;
	S.layer_weight = a->d_layer_weight;
	if (a->sample_lists) {
		S.n_layers = SAMPLE_LISTS;
		S.sample_offsets = a->d_sample_offsets; S.samples = reinterpret_cast<const uint4*>(a->d_samples.get()); S.bind_pose = a->d_bind;
		S.ik_offsets = a->n_ik ? a->d_ik_offsets.get() : nullptr; S.iks = a->d_iks; // over time_ticks and layer_weight, which lists do not read
	}
	else {
		S.n_layers = a->n_layers;
		S.clip_index = a->d_clip_index; S.layer_clip = a->d_layer_clip; S.layer_time = a->d_layer_time;
	}
	S.out_dq = (flags & LB200_PALETTE_DUAL_QUAT) ? a->d_dq.get() : nullptr;
	S.out_mtx = (flags & LB200_PALETTE_MATRIX) ? a->d_mtx.get() : nullptr;
	S.out_pos = (flags & LB200_PALETTE_POSE) ? a->d_pos.get() : nullptr;
	S.out_rot = (flags & LB200_PALETTE_POSE) ? a->d_rot.get() : nullptr;
	return S;
}
// whether a system runs the IK kernels: sample lists with IK ops
bool hasIk(const lb200_animation* a) { return a->sample_lists && a->n_ik; }
} // namespace

extern "C" {

int lb200_animation_update(lb200_animation* a, float time_delta, uint32_t flags) {
	return lb200_animation_update_many(&a, 1, time_delta, flags);
}

int lb200_animation_update_many(lb200_animation* const* systems, uint32_t n, float time_delta, uint32_t flags) {
	lb200_range range("update animables"); // animation_module.cpp:743, one range for the frame's systems
	if (!n) return LB200_OK;
	if (!systems) return LB200_ERR_INVALID;
	for (uint32_t k = 0; k < n; ++k) if (!systems[k]) return LB200_ERR_INVALID;
	lb200_ctx* ctx = systems[0]->ctx;
	for (uint32_t k = 1; k < n; ++k) {
		if (systems[k]->ctx != ctx) { lb200_set_error(ctx, "update_many: system %u belongs to another context", k); return LB200_ERR_INVALID; }
	}
	{
		std::vector<const lb200_animation*> sorted(systems, systems + n);
		std::sort(sorted.begin(), sorted.end());
		if (std::adjacent_find(sorted.begin(), sorted.end()) != sorted.end()) { lb200_set_error(ctx, "update_many: a system is listed twice"); return LB200_ERR_INVALID; }
	}
	// systems without instances are skipped; the others agree on one G or run 8
	std::vector<lb200_animation*> run;
	run.reserve(n);
	uint32_t max_bones = 0;
	int G = 0;
	for (uint32_t k = 0; k < n; ++k) {
		lb200_animation* a = systems[k];
		if (!a->n_instances) continue;
		const int g = requestedLanes(a);
		G = run.empty() ? g : (G == g ? G : 8);
		max_bones = std::max(max_bones, a->bone_count);
		run.push_back(a);
	}
	if (run.empty()) return LB200_OK;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	for (lb200_animation* a : run) { // every buffer before the first launch
		const int rc = allocOutputs(a, flags);
		if (rc) return rc;
	}
	G = fitLanes(G, max_bones);
	const int lanes = shapeIndex(G);
	const unsigned per_block = POSE_THREADS / G;
	AnimManyParams M;
	M.step = timeStep(time_delta);
	for (size_t first = 0; first < run.size(); first += POSE_MANY_CAP) {
		const uint32_t count = (uint32_t)std::min<size_t>(POSE_MANY_CAP, run.size() - first);
		M.n_systems = count;
		uint32_t blocks = 0;
		size_t smem = 0;
		bool ik = false; // some system of the launch has IK ops: the IK kernels
		for (uint32_t s = 0; s < count; ++s) {
			const lb200_animation* a = run[first + s];
			ik = ik || hasIk(a);
			M.sys[s] = sysParams(a, flags);
			blocks += (a->n_instances + per_block - 1) / per_block;
			M.block_end[s] = blocks;
			smem = std::max(smem, poseSmemBytes(a, per_block));
		}
		if (count == 1) { // a launch of one system is the per-system kernel: no search, parameters read at fixed offsets
			const PoseKernel* family = ik ? POSE_IK_KERNELS : run[first]->sample_lists ? POSE_LIST_KERNELS : POSE_CLIP_KERNELS;
			family[lanes]<<<blocks, POSE_THREADS, smem, ctx->stream>>>(M.sys[0], M.step);
		}
		else (ik ? POSE_MANY_IK_KERNELS : POSE_MANY_KERNELS)[lanes]<<<blocks, POSE_THREADS, smem, ctx->stream>>>(M);
		LB200_CHECK_LAUNCH(ctx);
	}
	for (lb200_animation* a : run) a->last_pose_lanes = G;
	return LB200_OK;
}

int lb200_animation_skin(lb200_animation* a) {
	lb200_range range("skin");
	if (!a) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (!a->n_vertices || !a->d_mtx) { lb200_set_error(ctx, "skin needs a mesh and a matrix palette (update with LB200_PALETTE_MATRIX first)"); return LB200_ERR_STATE; }
	if (!a->n_instances) return LB200_OK;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (!a->d_skinned) LB200_CUDA(ctx, a->d_skinned.alloc(3 * (size_t)a->max_instances * a->n_vertices));
	static const int g_env = [] { const char* e = getenv("LB200_SKIN_GROUP"); const int v = e ? atoi(e) : 8; return (v == 4 || v == 16) ? v : 8; }();
	const int group = a->skin_group ? a->skin_group : g_env;
	const dim3 grid((a->n_vertices + SKIN_THREADS - 1) / SKIN_THREADS, (a->n_instances + group - 1) / group);
	if (grid.y > 65535) { lb200_set_error(ctx, "too many instances for one skin launch"); return LB200_ERR_INVALID; }
	const size_t smem = sizeof(float4) * 3 * a->bone_count * group;
	SKIN_KERNELS[shapeIndex(group)]<<<grid, SKIN_THREADS, smem, ctx->stream>>>(a->d_mtx, a->d_mesh_pos, a->d_mesh_w, a->d_mesh_idx, a->n_vertices,
		a->bone_count, a->n_instances, a->d_skinned);
	LB200_CHECK_LAUNCH(ctx);
	a->last_skin_group = group;
	return LB200_OK;
}

int lb200_animation_set_launch(lb200_animation* a, int pose_lanes, int skin_group) {
	if (!a) return LB200_ERR_INVALID;
	if (pose_lanes != 0 && pose_lanes != 4 && pose_lanes != 8 && pose_lanes != 16 && pose_lanes != 32) {
		lb200_set_error(a->ctx, "set_launch: pose_lanes %d is not 0, 4, 8, 16 or 32", pose_lanes);
		return LB200_ERR_INVALID;
	}
	if (skin_group != 0 && skin_group != 4 && skin_group != 8 && skin_group != 16) {
		lb200_set_error(a->ctx, "set_launch: skin_group %d is not 0, 4, 8 or 16", skin_group);
		return LB200_ERR_INVALID;
	}
	a->pose_lanes = pose_lanes;
	a->skin_group = skin_group;
	return LB200_OK;
}

int lb200_animation_get_launch(lb200_animation* a, int* pose_lanes, int* skin_group) {
	if (!a) return LB200_ERR_INVALID;
	if (pose_lanes) *pose_lanes = a->last_pose_lanes;
	if (skin_group) *skin_group = a->last_skin_group;
	return LB200_OK;
}

static int readBack(lb200_animation* a, const void* dev, size_t elem_bytes, uint32_t first, uint32_t count, void* out) {
	if (!a || !out || first + count > a->n_instances) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (!dev) { lb200_set_error(ctx, "requested buffer was never produced"); return LB200_ERR_STATE; }
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(out, (const char*)dev + elem_bytes * first, elem_bytes * count, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

int lb200_animation_get_dual_quats(lb200_animation* a, uint32_t first, uint32_t count, float* out8) {
	return readBack(a, a ? a->d_dq.get() : nullptr, sizeof(float) * 8 * (a ? a->bone_count : 0), first, count, out8);
}
int lb200_animation_get_matrices(lb200_animation* a, uint32_t first, uint32_t count, float* out16) {
	return readBack(a, a ? a->d_mtx.get() : nullptr, sizeof(float) * 16 * (a ? a->bone_count : 0), first, count, out16);
}
int lb200_animation_get_pose(lb200_animation* a, uint32_t first, uint32_t count, float* out_pos3, float* out_rot4) {
	int rc = readBack(a, a ? a->d_pos.get() : nullptr, sizeof(float) * 3 * (a ? a->bone_count : 0), first, count, out_pos3);
	if (rc) return rc;
	return readBack(a, a->d_rot, sizeof(float) * 4 * a->bone_count, first, count, out_rot4);
}
int lb200_animation_set_layers(lb200_animation* a, uint32_t n_layers, const uint32_t* clip_index, const uint32_t* time_ticks, const float* weight) {
	if (!a || n_layers > 16) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (a->sample_lists) { lb200_set_error(ctx, "set_layers: the system is in sample-list mode"); return LB200_ERR_INVALID; }
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	if (n_layers == 0) { a->n_layers = 0; return LB200_OK; }
	if (!clip_index || !time_ticks || !weight || !a->n_instances) return LB200_ERR_INVALID;
	const size_t n = (size_t)a->n_instances * n_layers;
	for (size_t i = 0; i < n; ++i) if (clip_index[i] >= a->n_clips) { lb200_set_error(ctx, "layer entry %zu: clip %u out of range", i, clip_index[i]); return LB200_ERR_INVALID; }
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	a->d_layer_clip.reset(); a->d_layer_time.reset(); a->d_layer_weight.reset(); // all three go before any is allocated again
	a->n_layers = 0;
	DeviceArray<uint32_t> layer_clip, layer_time; DeviceArray<float> layer_weight;
	LB200_CUDA(ctx, layer_clip.alloc(n));
	LB200_CUDA(ctx, layer_time.alloc(n));
	LB200_CUDA(ctx, layer_weight.alloc(n));
	a->d_layer_clip = std::move(layer_clip); a->d_layer_time = std::move(layer_time); a->d_layer_weight = std::move(layer_weight);
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_layer_clip, clip_index, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_layer_time, time_ticks, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(a->d_layer_weight, weight, sizeof(float) * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	a->n_layers = n_layers;
	return LB200_OK;
}

int lb200_animation_bone_attachments(lb200_animation* a, uint32_t n, const uint32_t* instance, const uint32_t* bone, const float* relative7,
	const lb200_transform* parent_transforms, const float* original_scale3, lb200_transform* out_transforms)
{
	if (!a || !n || !instance || !bone || !relative7 || !parent_transforms || !original_scale3 || !out_transforms) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (!a->d_pos || !a->n_instances) { lb200_set_error(ctx, "bone_attachments needs absolute poses (update with LB200_PALETTE_POSE)"); return LB200_ERR_STATE; }
	for (uint32_t i = 0; i < n; ++i) {
		if (instance[i] >= a->n_instances || bone[i] >= a->bone_count) { lb200_set_error(ctx, "attachment %u: instance %u / bone %u out of range", i, instance[i], bone[i]); return LB200_ERR_INVALID; }
	}
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	// one staging allocation per call: [instance n][bone n][relative 7n][scale 3n] u32/f32, [parent n][out n] transforms
	const size_t words = (size_t)n * (1 + 1 + 7 + 3);
	DeviceArray<uint32_t> d_words;
	DeviceArray<lb200_transform> d_tr;
	LB200_CUDA(ctx, d_words.alloc(words));
	LB200_CUDA(ctx, d_tr.alloc(2 * (size_t)n));
	LB200_CUDA(ctx, cudaMemcpyAsync(d_words, instance, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(d_words + n, bone, sizeof(uint32_t) * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(d_words + 2 * (size_t)n, relative7, sizeof(float) * 7 * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(d_words + 9 * (size_t)n, original_scale3, sizeof(float) * 3 * n, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaMemcpyAsync(d_tr, parent_transforms, sizeof(lb200_transform) * n, cudaMemcpyHostToDevice, ctx->stream));
	bone_attachments_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(a->d_pos, a->d_rot, a->bone_count, d_words, d_words + n,
		reinterpret_cast<const float*>(d_words + 2 * (size_t)n), d_tr, reinterpret_cast<const float*>(d_words + 9 * (size_t)n), n, d_tr + n);
	LB200_CHECK_LAUNCH(ctx);
	LB200_CUDA(ctx, cudaMemcpyAsync(out_transforms, d_tr + n, sizeof(lb200_transform) * n, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream)); // before the staging is freed
	return LB200_OK;
}

// The same with every table already in HBM and the result left there (SURVEY 8f N4: pose -> entity transform -> re-binning -> cull without the
// host in between): out feeds lb200_sortkeys_move_device / lb200_culling_set_many_device.  Indices are the caller's responsibility here.
int lb200_animation_bone_attachments_device(lb200_animation* a, uint32_t n, const uint32_t* dev_instance, const uint32_t* dev_bone, const float* dev_relative7,
	const lb200_transform* dev_parent_transforms, const float* dev_original_scale3, lb200_transform* dev_out_transforms)
{
	if (!a || !dev_instance || !dev_bone || !dev_relative7 || !dev_parent_transforms || !dev_original_scale3 || !dev_out_transforms) return LB200_ERR_INVALID;
	if (!n) return LB200_OK;
	lb200_ctx* ctx = a->ctx;
	if (!a->d_pos || !a->n_instances) { lb200_set_error(ctx, "bone_attachments needs absolute poses (update with LB200_PALETTE_POSE)"); return LB200_ERR_STATE; }
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	bone_attachments_kernel<<<(n + 255) / 256, 256, 0, ctx->stream>>>(a->d_pos, a->d_rot, a->bone_count, dev_instance, dev_bone, dev_relative7, dev_parent_transforms, dev_original_scale3, n, dev_out_transforms);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

} // extern "C"

int lb200_animation_internal_poses(const lb200_animation* a, AnimationPoses* out) {
	if (!a->d_pos || !a->n_instances) return LB200_ERR_STATE;
	*out = AnimationPoses{a->ctx, a->d_pos, a->d_rot, a->bone_count, a->n_instances};
	return LB200_OK;
}

void lb200_animation_internal_palette_source(const lb200_animation* a, AnimationPaletteSource* out) {
	*out = AnimationPaletteSource{a->ctx, a->d_pos, a->d_rot, a->d_bind + 2 * a->bone_count, a->d_bind + 3 * a->bone_count, a->d_entity, a->bone_count,
		std::min(a->n_instances, a->n_entities)};
}

extern "C" {

int lb200_animation_compute_relative(lb200_animation* a) {
	if (!a) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (!a->d_pos || !a->n_instances) { lb200_set_error(ctx, "compute_relative needs absolute poses (update with LB200_PALETTE_POSE)"); return LB200_ERR_STATE; }
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const size_t nb = (size_t)a->max_instances * a->bone_count;
	if (!a->d_rel_pos || !a->d_rel_rot) {
		const int rc = allocPosePair(ctx, a->d_rel_pos, a->d_rel_rot, nb);
		if (rc) return rc;
	}
	const size_t n = (size_t)a->n_instances * a->bone_count;
	pose_relative_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(a->d_pos, a->d_rot, a->d_parents, a->bone_count, a->first_nonroot, n, a->d_rel_pos, a->d_rel_rot);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

int lb200_animation_get_relative_pose(lb200_animation* a, uint32_t first, uint32_t count, float* out_pos3, float* out_rot4) {
	int rc = readBack(a, a ? a->d_rel_pos.get() : nullptr, sizeof(float) * 3 * (a ? a->bone_count : 0), first, count, out_pos3);
	if (rc) return rc;
	return readBack(a, a->d_rel_rot, sizeof(float) * 4 * a->bone_count, first, count, out_rot4);
}

int lb200_animation_blend_pose(lb200_animation* a, const lb200_animation* b, float weight, int relative) {
	if (!a || !b) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (b->ctx != ctx || a->bone_count != b->bone_count || a->n_instances != b->n_instances) { lb200_set_error(ctx, "blend_pose: the two systems differ in context, bone count or instance count"); return LB200_ERR_INVALID; }
	float* pa = relative ? a->d_rel_pos : a->d_pos; float* ra = relative ? a->d_rel_rot : a->d_rot;
	const float* pb = relative ? b->d_rel_pos : b->d_pos; const float* rb = relative ? b->d_rel_rot : b->d_rot;
	if (!pa || !pb || !a->n_instances) { lb200_set_error(ctx, "blend_pose: a pose buffer was never produced"); return LB200_ERR_STATE; }
	if (weight <= 0.001f) return LB200_OK;                           // pose.cpp:33
	weight = weight < 0.0f ? 0.0f : (weight > 1.0f ? 1.0f : weight); // pose.cpp:34
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const size_t n = (size_t)a->n_instances * a->bone_count;
	pose_blend_kernel<<<(unsigned)((n + 255) / 256), 256, 0, ctx->stream>>>(pa, ra, pb, rb, n, weight);
	LB200_CHECK_LAUNCH(ctx);
	return LB200_OK;
}

int lb200_animation_get_times(lb200_animation* a, uint32_t first, uint32_t count, uint32_t* out_ticks) {
	if (a && a->sample_lists) { lb200_set_error(a->ctx, "get_times: the system is in sample-list mode, its times are the caller's"); return LB200_ERR_INVALID; }
	return readBack(a, a ? a->d_time.get() : nullptr, sizeof(uint32_t), first, count, out_ticks);
}
int lb200_animation_get_skinned(lb200_animation* a, uint32_t first, uint32_t count, float* out_pos3) {
	return readBack(a, a ? a->d_skinned.get() : nullptr, sizeof(float) * 3 * (a ? a->n_vertices : 0), first, count, out_pos3);
}

int lb200_animation_skinned_checksum(lb200_animation* a, uint64_t* out) {
	if (!a || !out) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (!a->d_skinned) return LB200_ERR_STATE;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemsetAsync(a->d_checksum, 0, sizeof(unsigned long long), ctx->stream));
	const size_t n = (size_t)a->n_instances * a->n_vertices * 3;
	checksum_kernel<<<ctx->sm_count * 8, 256, 0, ctx->stream>>>(reinterpret_cast<const uint32_t*>(a->d_skinned.get()), n, a->d_checksum);
	LB200_CHECK_LAUNCH(ctx);
	unsigned long long v = 0;
	LB200_CUDA(ctx, cudaMemcpyAsync(&v, a->d_checksum, sizeof(v), cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	*out = v;
	return LB200_OK;
}

uint64_t lb200_animation_algorithmic_bytes(const lb200_animation* a, uint32_t flags, int skin) {
	if (!a) return 0;
	const uint64_t nb = (uint64_t)a->n_instances * a->bone_count;
	uint64_t bytes = 0;
	if (skin) {
		// 12 B written per vertex-instance + the instance's matrix palette read once
		bytes += (uint64_t)a->n_instances * a->n_vertices * 12 + nb * 64;
	}
	else {
		if (flags & LB200_PALETTE_DUAL_QUAT) bytes += nb * 32;
		if (flags & LB200_PALETTE_MATRIX) bytes += nb * 64;
		if (flags & LB200_PALETTE_POSE) bytes += nb * 28;
		bytes += (uint64_t)a->n_instances * 12; // clip index + time read + time write
	}
	return bytes;
}

} // extern "C"
