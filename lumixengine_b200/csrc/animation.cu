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
// skin_kernel — evaluateSkin (model.cpp:103-109): palette of each instance staged in shared memory as 3x4 rows,
//   one thread per vertex, vertex data kept in registers across the instances of a group.
// Clips, skeleton and mesh are shared by all instances (L2-resident); HBM traffic is the per-instance output.
#include "lb200_internal.h"
#include "lb200_math.cuh"

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
	uint32_t key_off;                 // first float4 of this clip's decoded keyframes: [(frame_count + 1)][Bp] entries
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

struct AnimParams {
	const DevClip* clips;
	const DevTrack* tracks;
	const float4* const_t;        // xyz value, w = bone index bits
	const float4* const_r_value;  // quaternion
	const uint32_t* const_r_bone;
	const uint32_t* stream; // all bit streams, word-addressed
	const float4* key_pos; const float4* key_rot; // decoded keyframes (decode_clips_kernel)
	const unsigned char* key_flags;               // per (clip, bone): bit0 / bit1 translation / rotation animated, bit2 / bit3 constant track
	const float4* bind_pos; const float4* bind_rot;         // Bone::relative_transform
	const float4* inv_bind_pos; const float4* inv_bind_rot; // inverse bind transforms
	const short* parents;
	const unsigned char* level_bones; // bones of depth >= 1 sorted by depth (bone_count <= 196 fits a byte)
	const uint32_t* level_start;      // [max_level + 2]: level l occupies level_bones[level_start[l] .. level_start[l + 1])
	uint32_t bone_count;
	uint32_t max_level;
	uint32_t n_instances;
	const uint32_t* clip_index;
	uint32_t* time_ticks;
	float* out_dq;    // n * B * 8 or null
	float* out_mtx;   // n * B * 16 or null
	float* out_pos;   // n * B * 3 or null
	float* out_rot;   // n * B * 4 or null
	uint32_t dt_ticks;   // |time_delta| in ticks
	int dt_negative;
	int advance;
	// blend layers on top of the base clip (lb200_animation_set_layers): [instance][n_layers]
	uint32_t n_layers;
	const uint32_t* layer_clip;
	const uint32_t* layer_time;
	const float* layer_weight;
};

// unaligned little-endian u64 at byte address `byte` of a word-addressed stream (the reference memcpy's 8 bytes, animation.cpp:44)
__device__ __forceinline__ unsigned long long load_u64_unaligned(const uint32_t* __restrict__ words, uint32_t byte) {
	const uint32_t w = byte >> 2;
	const uint32_t sh = (byte & 3u) * 8u;
	const uint32_t a = __ldg(words + w), b = __ldg(words + w + 1), c = __ldg(words + w + 2);
	const uint32_t lo = __funnelshift_r(a, b, sh);
	const uint32_t hi = __funnelshift_r(b, c, sh);
	return ((unsigned long long)hi << 32) | lo;
}

// low 32 bits of (v >> s), 0 <= s < 64
__device__ __forceinline__ uint32_t shr64_lo32(unsigned long long v, uint32_t s) {
	const uint32_t lo = (uint32_t)v, hi = (uint32_t)(v >> 32);
	return s >= 32u ? (hi >> (s - 32u)) : __funnelshift_r(lo, hi, s);
}
__device__ __forceinline__ uint32_t mask32(uint32_t bits) { return bits >= 32u ? 0xffffffffu : ((1u << bits) - 1u); }

// animation.cpp:313-316 unpackChannel: float(min + to_float_range * double(val & mask))
__device__ __forceinline__ float unpack_channel(unsigned long long val, float mn, float range, uint32_t bits) {
	const unsigned long long mask = (1ull << bits) - 1ull;
	return __double2float_rn(LB_DADD((double)mn, LB_DMUL((double)range, __ull2double_rn(val & mask))));
}
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

// Unpack every frame of every clip once (clips are shared by all instances): block = (clip, frame), threads over bones / tracks.
// Same arithmetic as the per-sample path of the reference: Animation::getTranslation (animation.cpp:318-334, unpackChannel through
// double) and the smallest-three reconstruction of AnimationSampler::getRotation (animation.cpp:51-77).
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
	const uint32_t c = P.frame_clip[blockIdx.x], frame = P.frame_index[blockIdx.x];
	const DevClip clip = P.clips[c];
	float4* kp = P.key_pos + clip.key_off + (size_t)frame * Bp;
	float4* kr = P.key_rot + clip.key_off + (size_t)frame * Bp;
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

constexpr int POSE_THREADS = 128;

// G lanes cooperate on one instance (32 / G instances per warp): per-bone phases stride the bones by G, the absolute pass
// walks depth levels with up to G bones of a level in flight.  G is 8 unless LB200_POSE_LANES or lb200_animation_set_launch asks
// for another (lb200_animation_update).
template <int G>
__global__ void __launch_bounds__(POSE_THREADS) pose_palette_kernel(const __grid_constant__ AnimParams P) {
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
	const uint32_t inst = blockIdx.x * INST_PER_BLOCK + grp;
	const bool valid = inst < P.n_instances;
	// the lanes of one group share a mask so that __syncwarp only joins what must be joined
	const unsigned gmask = (G == 32) ? 0xffffffffu : (((1u << G) - 1u) << (lane & ~(G - 1)));

	if (valid) {
		const DevClip clip = P.clips[P.clip_index[inst]];
		const uint32_t ticks = P.time_ticks[inst];

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
		__syncwarp(gmask);

		// Blend layers (the animator's stack of weighted samples, controller.cpp:267-292 -> Animation::getRelativePose with
		// ctx.weight): every bone the layer's clip has a track for — constant or animated — moves towards the layer's sample,
		// lerp (math.cpp:194-201) for positions and simd_nlerp for rotations when weight < 0.9999 (animation.cpp:294-311), plain
		// replacement otherwise; bones without a track are left alone (animation.cpp:136-203).  Bones are independent: no sync inside.
		for (uint32_t layer = 0; layer < P.n_layers; ++layer) {
			const size_t li = (size_t)inst * P.n_layers + layer;
			const DevClip lclip = P.clips[P.layer_clip[li]];
			const float w = P.layer_weight[li];
			const bool use_weight = w < 0.9999f;
			const float lframe = __double2float_rn(LB_DMUL(__uint2double_rn(P.layer_time[li]) / 32768.0, (double)lclip.fps));
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
		if (P.advance && sub == 0) {
			const uint32_t l = clip.length_ticks;
			uint32_t nt;
			if (!P.dt_negative) nt = (ticks + P.dt_ticks) % l;
			else nt = (ticks + l - (P.dt_ticks % l)) % l;
			P.time_ticks[inst] = nt;
		}
	}
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
	const Q4 prot = q4(p.rot[0], p.rot[1], p.rot[2], p.rot[3]);
	// Transform::compose(const LocalRigidTransform&), math.cpp:763: pos + rot.rotate(rhs.pos * scale) in fp32, added to the fp64 position
	const V3 rotated = rotate(prot, mul(local.pos, v3(p.scale[0], p.scale[1], p.scale[2])));
	const Q4 rot = qmul(prot, local.rot);
	lb200_transform o;
	o.pos[0] = LB_DADD(p.pos[0], (double)rotated.x); o.pos[1] = LB_DADD(p.pos[1], (double)rotated.y); o.pos[2] = LB_DADD(p.pos[2], (double)rotated.z);
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
	DeviceArray<short> d_parents; DeviceArray<unsigned char> d_level_bones; DeviceArray<uint32_t> d_level_start;
	int lanes_per_instance = 8;
	// lb200_animation_set_launch (0 = environment switch, else the default) and what the last update / skin launched
	int pose_lanes = 0, skin_group = 0;
	int last_pose_lanes = 0, last_skin_group = 0;
	DeviceArray<uint32_t> d_clip_index, d_time;
	uint32_t n_layers = 0; DeviceArray<uint32_t> d_layer_clip, d_layer_time; DeviceArray<float> d_layer_weight; // all three or none
	// palettes and poses, allocated by the first update that asks for them; d_pos / d_rot and d_rel_pos / d_rel_rot go in pairs
	DeviceArray<float> d_dq, d_mtx, d_pos, d_rot;
	DeviceArray<float> d_rel_pos, d_rel_rot; // Pose::computeRelative of d_pos / d_rot
	uint32_t first_nonroot = 0;
	DeviceArray<float> d_mesh_pos; DeviceArray<float4> d_mesh_w; DeviceArray<short> d_mesh_idx;
	DeviceArray<float> d_skinned;
	DeviceArray<unsigned long long> d_checksum;
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
		d.fps = s.fps; d.frame_count = s.frame_count;
		d.t_bits = s.translations_frame_size_bits; d.r_bits = s.rotations_frame_size_bits;
		d.n_t = s.n_translations; d.n_ct = s.n_const_translations; d.n_r = s.n_rotations; d.n_cr = s.n_const_rotations;
		d.t_off = (uint32_t)tracks.size();
		for (uint32_t i = 0; i < s.n_translations; ++i) { if (s.translations[i].bone_index >= B) return LB200_ERR_INVALID; tracks.push_back(packTrack(s.translations[i])); }
		d.r_off = (uint32_t)tracks.size();
		for (uint32_t i = 0; i < s.n_rotations; ++i) { if (s.rotations[i].bone_index >= B || s.rotations[i].skipped_channel > 3) return LB200_ERR_INVALID; tracks.push_back(packTrack(s.rotations[i])); }
		d.ct_off = (uint32_t)cts.size();
		for (uint32_t i = 0; i < s.n_const_translations; ++i) { if (s.const_translations[i].bone_index >= B) return LB200_ERR_INVALID; const lb200_const_translation& c0 = s.const_translations[i]; cts.push_back(make_float4(c0.value[0], c0.value[1], c0.value[2], __builtin_bit_cast(float, (uint32_t)c0.bone_index))); }
		d.cr_off = (uint32_t)cr_values.size();
		for (uint32_t i = 0; i < s.n_const_rotations; ++i) { if (s.const_rotations[i].bone_index >= B) return LB200_ERR_INVALID; const lb200_const_rotation& c0 = s.const_rotations[i]; cr_values.push_back(make_float4(c0.value[0], c0.value[1], c0.value[2], c0.value[3])); cr_bones.push_back(c0.bone_index); }
		// streams must hold (frame_count + 1) frames + the loader's 8-byte tail (animation.cpp:439)
		const uint64_t need_t = s.n_translations ? ((uint64_t)d.t_bits * (s.frame_count + 1) + 7) / 8 : 0;
		const uint64_t need_r = s.n_rotations ? ((uint64_t)d.r_bits * (s.frame_count + 1) + 7) / 8 : 0;
		if (s.translation_stream_bytes < need_t || s.rotation_stream_bytes < need_r) { lb200_set_error(ctx, "clip %u: bit stream shorter than (frame_count+1) frames", c); return LB200_ERR_INVALID; }
		d.t_stream = appendStream(s.translation_stream, s.translation_stream_bytes);
		d.r_stream = appendStream(s.rotation_stream, s.rotation_stream_bytes);
		d.length_ticks = (uint32_t)(((float)s.frame_count / s.fps) * (float)(1 << 15)); // Time::fromSeconds(m_frame_count / m_fps)
		if (!d.length_ticks) return LB200_ERR_INVALID;
		d.pad[0] = d.pad[1] = d.pad[2] = 0;
	}
	// decoded keyframe tables: (frame_count + 1) frames x Bp bones per clip
	const uint32_t Bp = (B + 3u) & ~3u;
	std::vector<uint32_t> frame_clip, frame_index;
	size_t key_entries = 0;
	for (uint32_t c = 0; c < n_clips; ++c) {
		dc[c].key_off = (uint32_t)key_entries;
		dc[c].flag_off = c * Bp;
		for (uint32_t f = 0; f <= dc[c].frame_count; ++f) { frame_clip.push_back(c); frame_index.push_back(f); }
		key_entries += (size_t)(dc[c].frame_count + 1) * Bp;
		if (key_entries > 0x7fffffffull) { lb200_set_error(ctx, "decoded clips exceed 2^31 keyframe entries"); return LB200_ERR_INVALID; }
	}

	// any early return below (allocation or copy failure) releases what has been allocated so far
	std::unique_ptr<lb200_animation, decltype(&lb200_animation_destroy)> a(new (std::nothrow) lb200_animation, lb200_animation_destroy);
	if (!a) return LB200_ERR_CUDA;
	a->ctx = ctx; a->bone_count = B; a->max_level = max_level; a->n_clips = n_clips; a->max_instances = max_instances;
	a->first_nonroot = first;
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
		DeviceArray<uint32_t> d_fc, d_fi;
		LB200_CUDA(ctx, d_fc.alloc(frame_clip.size(), TABLE_MIN_BYTES));
		LB200_CUDA(ctx, d_fi.alloc(frame_index.size(), TABLE_MIN_BYTES));
		LB200_CUDA(ctx, cudaMemcpyAsync(d_fc, frame_clip.data(), sizeof(uint32_t) * frame_clip.size(), cudaMemcpyHostToDevice, st));
		LB200_CUDA(ctx, cudaMemcpyAsync(d_fi, frame_index.data(), sizeof(uint32_t) * frame_index.size(), cudaMemcpyHostToDevice, st));
		DecodeParams D;
		D.clips = a->d_clips; D.tracks = a->d_tracks; D.const_t = a->d_const_t; D.const_r_value = a->d_const_r_value; D.const_r_bone = a->d_const_r_bone;
		D.stream = a->d_stream; D.bind_pos = a->d_bind; D.bind_rot = a->d_bind + B;
		D.key_pos = a->d_key_pos; D.key_rot = a->d_key_rot; D.key_flags = a->d_key_flags;
		D.frame_clip = d_fc; D.frame_index = d_fi; D.bone_count = B;
		decode_clips_kernel<<<(unsigned)frame_clip.size(), 256, 0, st>>>(D);
		LB200_CHECK_LAUNCH(ctx);
		LB200_CUDA(ctx, cudaStreamSynchronize(st)); // before d_fc / d_fi are freed
	}
	LB200_CUDA(ctx, cudaStreamSynchronize(st));
	{
		const int smem_max = (int)(sizeof(float4) * (2 * 196 * (POSE_THREADS / 8) + 2 * 196 + 128));
		const int smem_max4 = (int)std::min<size_t>(220 * 1024, sizeof(float4) * (2 * 196 * (POSE_THREADS / 4) + 2 * 196 + 128));
		LB200_CUDA(ctx, cudaFuncSetAttribute(pose_palette_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max4));
		LB200_CUDA(ctx, cudaFuncSetAttribute(pose_palette_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
		LB200_CUDA(ctx, cudaFuncSetAttribute(pose_palette_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
		LB200_CUDA(ctx, cudaFuncSetAttribute(pose_palette_kernel<32>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_max));
	}
	LB200_CUDA(ctx, cudaFuncSetAttribute(skin_kernel<4>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(4 * 196 * 3 * sizeof(float4))));
	LB200_CUDA(ctx, cudaFuncSetAttribute(skin_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(8 * 196 * 3 * sizeof(float4))));
	LB200_CUDA(ctx, cudaFuncSetAttribute(skin_kernel<16>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(16 * 196 * 3 * sizeof(float4))));
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
	return LB200_OK;
}

int lb200_animation_update(lb200_animation* a, float time_delta, uint32_t flags) {
	lb200_range range("update animables"); // animation_module.cpp:743
	if (!a) return LB200_ERR_INVALID;
	lb200_ctx* ctx = a->ctx;
	if (!a->n_instances) return LB200_OK;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	const size_t nb = (size_t)a->max_instances * a->bone_count;
	if ((flags & LB200_PALETTE_DUAL_QUAT) && !a->d_dq) LB200_CUDA(ctx, a->d_dq.alloc(8 * nb));
	if ((flags & LB200_PALETTE_MATRIX) && !a->d_mtx) LB200_CUDA(ctx, a->d_mtx.alloc(16 * nb));
	if ((flags & LB200_PALETTE_POSE) && (!a->d_pos || !a->d_rot)) {
		const int rc = allocPosePair(ctx, a->d_pos, a->d_rot, nb);
		if (rc) return rc;
	}
	AnimParams P;
	P.clips = a->d_clips; P.tracks = a->d_tracks; P.const_t = a->d_const_t; P.const_r_value = a->d_const_r_value; P.const_r_bone = a->d_const_r_bone; P.stream = a->d_stream;
	P.key_pos = a->d_key_pos; P.key_rot = a->d_key_rot; P.key_flags = a->d_key_flags;
	P.bind_pos = a->d_bind; P.bind_rot = a->d_bind + a->bone_count; P.inv_bind_pos = a->d_bind + 2 * a->bone_count; P.inv_bind_rot = a->d_bind + 3 * a->bone_count; P.parents = a->d_parents; P.level_bones = a->d_level_bones; P.level_start = a->d_level_start;
	P.bone_count = a->bone_count; P.max_level = a->max_level; P.n_instances = a->n_instances;
	P.clip_index = a->d_clip_index; P.time_ticks = a->d_time;
	P.n_layers = a->n_layers; P.layer_clip = a->d_layer_clip; P.layer_time = a->d_layer_time; P.layer_weight = a->d_layer_weight;
	P.out_dq = (flags & LB200_PALETTE_DUAL_QUAT) ? a->d_dq.get() : nullptr;
	P.out_mtx = (flags & LB200_PALETTE_MATRIX) ? a->d_mtx.get() : nullptr;
	P.out_pos = (flags & LB200_PALETTE_POSE) ? a->d_pos.get() : nullptr;
	P.out_rot = (flags & LB200_PALETTE_POSE) ? a->d_rot.get() : nullptr;
	// Time::fromSeconds: u32(time * ONE_SECOND), animation.h:21-24 (:462 uses -time_delta for rewinds)
	// animation_module.cpp:458 `if (time_delta > 0) ... else ...`: zero takes the rewind branch too, which leaves a time below the clip
	// length alone and wraps one at or beyond it (time % length), exactly as the reference does on every update
	P.dt_negative = !(time_delta > 0);
	P.dt_ticks = (uint32_t)((P.dt_negative ? -time_delta : time_delta) * (float)(1 << 15));
	P.advance = 1;
	static const int g_env = [] { const char* e = getenv("LB200_POSE_LANES"); const int v = e ? atoi(e) : 0; return (v == 4 || v == 8 || v == 16 || v == 32) ? v : 0; }();
	int G = a->pose_lanes ? a->pose_lanes : g_env ? g_env : a->lanes_per_instance;
	if (G == 4) { // 32 instances per block: only while their poses fit in shared memory
		const uint32_t bp = (a->bone_count + 3u) & ~3u;
		if (sizeof(float4) * (2 * (size_t)bp * (POSE_THREADS / 4) + 2 * bp + 128) > 200 * 1024) G = 8;
	}
	const unsigned per_block = POSE_THREADS / G;
	const unsigned blocks = (a->n_instances + per_block - 1) / per_block;
	const uint32_t Bp_ = (a->bone_count + 3u) & ~3u;
	const uint32_t n_ls_ = (a->max_level + 2u + 3u) & ~3u;
	const size_t shared_words16 = 2 * Bp_ + (n_ls_ * 4 + Bp_ * 2 + Bp_ + 15) / 16; // inverse bind + topology, in float4 units
	const size_t smem = sizeof(float4) * (shared_words16 + 2 * (size_t)Bp_ * per_block);
	if (G == 4) pose_palette_kernel<4><<<blocks, POSE_THREADS, smem, ctx->stream>>>(P);
	else if (G == 8) pose_palette_kernel<8><<<blocks, POSE_THREADS, smem, ctx->stream>>>(P);
	else if (G == 16) pose_palette_kernel<16><<<blocks, POSE_THREADS, smem, ctx->stream>>>(P);
	else pose_palette_kernel<32><<<blocks, POSE_THREADS, smem, ctx->stream>>>(P);
	LB200_CHECK_LAUNCH(ctx);
	a->last_pose_lanes = G;
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
#define LB200_SKIN_LAUNCH(G) skin_kernel<G><<<grid, SKIN_THREADS, smem, ctx->stream>>>(a->d_mtx, a->d_mesh_pos, a->d_mesh_w, a->d_mesh_idx, a->n_vertices, a->bone_count, a->n_instances, a->d_skinned)
	if (group == 4) LB200_SKIN_LAUNCH(4); else if (group == 16) LB200_SKIN_LAUNCH(16); else LB200_SKIN_LAUNCH(8);
#undef LB200_SKIN_LAUNCH
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
