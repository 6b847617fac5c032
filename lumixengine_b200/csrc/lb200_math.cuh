// Device (and host) arithmetic with the reference's exact operation order.
//
// The reference ships without FMA (MSVC /fp:precise + SSE2, scripts/genie.lua:144-147,301-315): every product and
// sum rounds separately.  All fp ops below go through *_rn intrinsics on the device so that no flag can fuse them
// (the library is additionally built with -fmad=false -prec-div=true -prec-sqrt=true -ftz=false).
// Each function names the reference lines it mirrors.
#pragma once

#include <cuda_runtime.h>
#include <math.h>
#include <stdint.h>

#if defined(__CUDA_ARCH__)
#define LB_HD __host__ __device__ __forceinline__
#define LB_FMUL(a, b) __fmul_rn((a), (b))
#define LB_FADD(a, b) __fadd_rn((a), (b))
#define LB_FSUB(a, b) __fsub_rn((a), (b))
#define LB_DMUL(a, b) __dmul_rn((a), (b))
#define LB_DADD(a, b) __dadd_rn((a), (b))
#define LB_DSUB(a, b) __dsub_rn((a), (b))
#define LB_DDIV(a, b) __ddiv_rn((a), (b))
#define LB_FSQRT(a) __fsqrt_rn((a))
#define LB_FDIV(a, b) __fdiv_rn((a), (b))
#define LB_U64_TO_D(a) __ull2double_rn((a))
#else
#define LB_HD inline
#define LB_FMUL(a, b) ((a) * (b))
#define LB_FADD(a, b) ((a) + (b))
#define LB_FSUB(a, b) ((a) - (b))
#define LB_DMUL(a, b) ((a) * (b))
#define LB_DADD(a, b) ((a) + (b))
#define LB_DSUB(a, b) ((a) - (b))
#define LB_DDIV(a, b) ((a) / (b))
#define LB_FSQRT(a) sqrtf((a))
#define LB_FDIV(a, b) ((a) / (b))
#define LB_U64_TO_D(a) ((double)(a))
#endif

namespace lb {

struct V3 { float x, y, z; };
struct D3 { double x, y, z; };
struct Q4 { float x, y, z, w; };
struct Rigid { V3 pos; Q4 rot; }; // LocalRigidTransform, math.h:266-274

LB_HD V3 v3(float x, float y, float z) { V3 r; r.x = x; r.y = y; r.z = z; return r; }
LB_HD D3 d3(double x, double y, double z) { D3 r; r.x = x; r.y = y; r.z = z; return r; }
LB_HD Q4 q4(float x, float y, float z, float w) { Q4 r; r.x = x; r.y = y; r.z = z; r.w = w; return r; }

LB_HD V3 add(V3 a, V3 b) { return v3(LB_FADD(a.x, b.x), LB_FADD(a.y, b.y), LB_FADD(a.z, b.z)); }
LB_HD V3 sub(V3 a, V3 b) { return v3(LB_FSUB(a.x, b.x), LB_FSUB(a.y, b.y), LB_FSUB(a.z, b.z)); }
LB_HD V3 neg(V3 a) { return v3(-a.x, -a.y, -a.z); }
LB_HD V3 muls(V3 a, float s) { return v3(LB_FMUL(a.x, s), LB_FMUL(a.y, s), LB_FMUL(a.z, s)); }
LB_HD V3 mul(V3 a, V3 b) { return v3(LB_FMUL(a.x, b.x), LB_FMUL(a.y, b.y), LB_FMUL(a.z, b.z)); } // math.cpp:459
LB_HD D3 add(D3 a, D3 b) { return d3(LB_DADD(a.x, b.x), LB_DADD(a.y, b.y), LB_DADD(a.z, b.z)); } // math.cpp:508
LB_HD D3 sub(D3 a, D3 b) { return d3(LB_DSUB(a.x, b.x), LB_DSUB(a.y, b.y), LB_DSUB(a.z, b.z)); } // math.cpp:506
// math.cpp:526-530 Vec3(const DVec3&)
LB_HD V3 tofloat(D3 a) { return v3((float)a.x, (float)a.y, (float)a.z); }

// math.cpp:1266-1268 dot(Vec3,Vec3): (x*x' + y*y') + z*z'
LB_HD float dot(V3 a, V3 b) { return LB_FADD(LB_FADD(LB_FMUL(a.x, b.x), LB_FMUL(a.y, b.y)), LB_FMUL(a.z, b.z)); }
// math.cpp:1274-1276
LB_HD V3 cross(V3 a, V3 b) {
	return v3(LB_FSUB(LB_FMUL(a.y, b.z), LB_FMUL(a.z, b.y)), LB_FSUB(LB_FMUL(a.z, b.x), LB_FMUL(a.x, b.z)), LB_FSUB(LB_FMUL(a.x, b.y), LB_FMUL(a.y, b.x)));
}
// math.cpp:1278-1280
LB_HD D3 cross(D3 a, D3 b) {
	return d3(LB_DSUB(LB_DMUL(a.y, b.z), LB_DMUL(a.z, b.y)), LB_DSUB(LB_DMUL(a.z, b.x), LB_DMUL(a.x, b.z)), LB_DSUB(LB_DMUL(a.x, b.y), LB_DMUL(a.y, b.x)));
}
// math.cpp:367-376
LB_HD V3 normalize(V3 v) {
	const float len2 = LB_FADD(LB_FADD(LB_FMUL(v.x, v.x), LB_FMUL(v.y, v.y)), LB_FMUL(v.z, v.z));
	const float inv_len = LB_FDIV(1.0f, LB_FSQRT(len2));
	return v3(LB_FMUL(v.x, inv_len), LB_FMUL(v.y, inv_len), LB_FMUL(v.z, inv_len));
}

// math.cpp:164-175 Quat::rotate(Vec3)
LB_HD V3 rotate(Q4 q, V3 v) {
	const V3 qvec = v3(q.x, q.y, q.z);
	V3 uv = cross(qvec, v);
	V3 uuv = cross(qvec, uv);
	uv = muls(uv, LB_FMUL(2.0f, q.w));
	uuv = muls(uuv, 2.0f);
	return add(add(v, uv), uuv);
}

// math.cpp:177-188 Quat::rotate(const DVec3&): all fp64, uv *= (2.0 * w)
LB_HD D3 rotate(Q4 q, D3 v) {
	const D3 qvec = d3((double)q.x, (double)q.y, (double)q.z);
	D3 uv = cross(qvec, v);
	D3 uuv = cross(qvec, uv);
	const double s = LB_DMUL(2.0, (double)q.w);
	uv = d3(LB_DMUL(uv.x, s), LB_DMUL(uv.y, s), LB_DMUL(uv.z, s));
	uuv = d3(LB_DMUL(uuv.x, 2.0), LB_DMUL(uuv.y, 2.0), LB_DMUL(uuv.z, 2.0));
	return add(add(v, uv), uuv);
}

// math.cpp:694-701 Quat::operator*(Quat): ((a + b) + c) - d per component
LB_HD Q4 qmul(Q4 a, Q4 r) {
	return q4(
		LB_FSUB(LB_FADD(LB_FADD(LB_FMUL(a.w, r.x), LB_FMUL(r.w, a.x)), LB_FMUL(a.y, r.z)), LB_FMUL(r.y, a.z)),
		LB_FSUB(LB_FADD(LB_FADD(LB_FMUL(a.w, r.y), LB_FMUL(r.w, a.y)), LB_FMUL(a.z, r.x)), LB_FMUL(r.z, a.x)),
		LB_FSUB(LB_FADD(LB_FADD(LB_FMUL(a.w, r.z), LB_FMUL(r.w, a.z)), LB_FMUL(a.x, r.y)), LB_FMUL(r.x, a.y)),
		LB_FSUB(LB_FSUB(LB_FSUB(LB_FMUL(a.w, r.w), LB_FMUL(a.x, r.x)), LB_FMUL(a.y, r.y)), LB_FMUL(a.z, r.z)));
}

// math.cpp:194-201 lerp(Vec3,Vec3,float)
LB_HD V3 lerp(V3 a, V3 b, float t) {
	const float invt = LB_FSUB(1.0f, t);
	return v3(LB_FADD(LB_FMUL(a.x, invt), LB_FMUL(b.x, t)), LB_FADD(LB_FMUL(a.y, invt), LB_FMUL(b.y, t)), LB_FADD(LB_FMUL(a.z, invt), LB_FMUL(b.z, t)));
}

// simd_math.h:107-123 simd_nlerp: horizontal sums are hadd(hadd()) = (x+y)+(z+w)
LB_HD Q4 simd_nlerp(Q4 q1, Q4 q2, float t) {
	const float inv = LB_FSUB(1.0f, t);
	const float d = LB_FADD(LB_FADD(LB_FMUL(q1.x, q2.x), LB_FMUL(q1.y, q2.y)), LB_FADD(LB_FMUL(q1.z, q2.z), LB_FMUL(q1.w, q2.w)));
	if (d < 0) t = -t;
	Q4 q = q4(LB_FADD(LB_FMUL(q1.x, inv), LB_FMUL(q2.x, t)), LB_FADD(LB_FMUL(q1.y, inv), LB_FMUL(q2.y, t)),
		LB_FADD(LB_FMUL(q1.z, inv), LB_FMUL(q2.z, t)), LB_FADD(LB_FMUL(q1.w, inv), LB_FMUL(q2.w, t)));
	const float len2 = LB_FADD(LB_FADD(LB_FMUL(q.x, q.x), LB_FMUL(q.y, q.y)), LB_FADD(LB_FMUL(q.z, q.z), LB_FMUL(q.w, q.w)));
	const float l = LB_FDIV(1.0f, LB_FSQRT(len2));
	return q4(LB_FMUL(q.x, l), LB_FMUL(q.y, l), LB_FMUL(q.z, l), LB_FMUL(q.w, l));
}

// math.cpp:859-861 LocalRigidTransform::operator*
LB_HD Rigid rmul(Rigid a, Rigid b) {
	Rigid r;
	r.pos = add(rotate(a.rot, b.pos), a.pos);
	r.rot = qmul(a.rot, b.rot);
	return r;
}

// math.cpp:395 squaredLength(Vec3): (x*x + y*y) + z*z
LB_HD float squared_length(V3 v) { return LB_FADD(LB_FADD(LB_FMUL(v.x, v.x), LB_FMUL(v.y, v.y)), LB_FMUL(v.z, v.z)); }
// math.cpp:392 length(Vec3): sqrtf of the same sum
LB_HD float length(V3 v) { return LB_FSQRT(squared_length(v)); }

// math.cpp:664-667 Quat::conjugated
LB_HD Q4 conjugated(Q4 q) { return q4(q.x, q.y, q.z, -q.w); }

// math.cpp:836-841 LocalRigidTransform::inverted: rot' = rot.conjugated(), pos' = rot'.rotate(-pos)
LB_HD Rigid rinverted(Rigid a) {
	Rigid r;
	r.rot = conjugated(a.rot);
	r.pos = rotate(r.rot, neg(a.pos));
	return r;
}

// math.cpp:677-691 nlerp(Quat, Quat, float), the scalar form: dot and length summed ((x+y)+z)+w, t negated for a negative dot,
// normalised with 1 / sqrtf
LB_HD Q4 nlerp(Q4 q1, Q4 q2, float t) {
	const float inv = LB_FSUB(1.0f, t);
	const float d = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(q1.x, q2.x), LB_FMUL(q1.y, q2.y)), LB_FMUL(q1.z, q2.z)), LB_FMUL(q1.w, q2.w));
	if (d < 0) t = -t;
	const Q4 q = q4(LB_FADD(LB_FMUL(q1.x, inv), LB_FMUL(q2.x, t)), LB_FADD(LB_FMUL(q1.y, inv), LB_FMUL(q2.y, t)),
		LB_FADD(LB_FMUL(q1.z, inv), LB_FMUL(q2.z, t)), LB_FADD(LB_FMUL(q1.w, inv), LB_FMUL(q2.w, t)));
	const float len2 = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(q.x, q.x), LB_FMUL(q.y, q.y)), LB_FMUL(q.z, q.z)), LB_FMUL(q.w, q.w));
	const float l = LB_FDIV(1.0f, LB_FSQRT(len2));
	return q4(LB_FMUL(q.x, l), LB_FMUL(q.y, l), LB_FMUL(q.z, l), LB_FMUL(q.w, l));
}

// Quat(axis, PI) (math.cpp:570-578): sinf / cosf of PI * 0.5f (math.h:404) as the reference's x86 libm returns them, 1 and
// -4.37113883e-08 (tests/golden/ik_kat.npz pins them)
constexpr float IK_SIN_HALF_PI = 1.0f;
constexpr float IK_COS_HALF_PI = -0x1.777a5cp-25f;

// math.cpp:581-606 Quat::vec3ToVec3.  The antiparallel branch's squaredLength(n) < 0.01 compares a float with a double.
LB_HD Q4 vec3_to_vec3(V3 v0, V3 v1) {
	const V3 from = normalize(v0);
	const V3 to = normalize(v1);
	const float cos_angle = dot(from, to);
	if (cos_angle > -1.0005f && cos_angle < -0.9995f) {
		V3 n = v3(0, from.z, -from.y);
		if ((double)squared_length(n) < 0.01) n = v3(from.y, -from.x, 0);
		n = normalize(n);
		return q4(LB_FMUL(n.x, IK_SIN_HALF_PI), LB_FMUL(n.y, IK_SIN_HALF_PI), LB_FMUL(n.z, IK_SIN_HALF_PI), IK_COS_HALF_PI);
	}
	const V3 half = normalize(add(from, to));
	return q4(LB_FSUB(LB_FMUL(from.y, half.z), LB_FMUL(from.z, half.y)), LB_FSUB(LB_FMUL(from.z, half.x), LB_FMUL(from.x, half.z)),
		LB_FSUB(LB_FMUL(from.x, half.y), LB_FMUL(from.y, half.x)), dot(from, half));
}

// math.cpp:378-389 normalize(Quat): 1 / sqrtf of the sum ((x*x + y*y) + z*z) + w*w, then four products
LB_HD Q4 normalize(Q4 q) {
	const float len2 = LB_FADD(LB_FADD(LB_FADD(LB_FMUL(q.x, q.x), LB_FMUL(q.y, q.y)), LB_FMUL(q.z, q.z)), LB_FMUL(q.w, q.w));
	const float inv_len = LB_FDIV(1.0f, LB_FSQRT(len2));
	return q4(LB_FMUL(q.x, inv_len), LB_FMUL(q.y, inv_len), LB_FMUL(q.z, inv_len), LB_FMUL(q.w, inv_len));
}

// animation.cpp:313-316 unpackChannel: float(min + to_float_range * double(val & mask))
LB_HD float unpack_channel(unsigned long long val, float mn, float range, uint32_t bits) {
	const unsigned long long mask = (1ull << bits) - 1ull;
	return (float)LB_DADD((double)mn, LB_DMUL((double)range, LB_U64_TO_D(val & mask)));
}

// animation.cpp:336-364 Animation::getRotation of one packed sample (already shifted to its first bit): the three channels through
// unpackChannel (double), unlike the float form of AnimationSampler::getRotation (:71-77), then the smallest-three reconstruction
LB_HD Q4 unpack_rotation_d(unsigned long long packed, const float* mn, const float* range, const uint32_t* bits, uint32_t skipped_channel) {
	const bool is_negative = (packed & 1ull) != 0;
	packed >>= 1;
	V3 v;
	v.x = unpack_channel(packed, mn[0], range[0], bits[0]);
	packed >>= bits[0];
	v.y = unpack_channel(packed, mn[1], range[1], bits[1]);
	packed >>= bits[1];
	v.z = unpack_channel(packed, mn[2], range[2], bits[2]);
	const float rem = LB_FSUB(1.0f, dot(v, v));
	const float skipped = LB_FMUL(LB_FSQRT(0.f > rem ? 0.f : rem), is_negative ? -1.0f : 1.0f); // maximum(0.f, x), math.h
	switch (skipped_channel) {
		case 0: return q4(skipped, v.x, v.y, v.z);
		case 1: return q4(v.x, skipped, v.y, v.z);
		case 2: return q4(v.x, v.y, skipped, v.z);
		default: return q4(v.x, v.y, v.z, skipped);
	}
}

// Transform::compose(const LocalRigidTransform&), math.cpp:763: pos + rot.rotate(rhs.pos * scale) in fp32, added to the fp64 position;
// rotation rot * rhs.rot.  RenderModuleImpl::updateBoneAttachment (render_module.cpp:399-403) composes the parent entity's transform with
// bone * relative this way and keeps the attached entity's own scale.
LB_HD void compose_rigid(D3 ppos, Q4 prot, V3 pscale, Rigid local, D3& pos, Q4& rot) {
	const V3 rotated = rotate(prot, mul(local.pos, pscale));
	rot = qmul(prot, local.rot);
	pos = d3(LB_DADD(ppos.x, (double)rotated.x), LB_DADD(ppos.y, (double)rotated.y), LB_DADD(ppos.z, (double)rotated.z));
}

} // namespace lb

namespace lb {

struct DualQ { Q4 r, d; };

// math.cpp:843-853 LocalRigidTransform::toDualQuat
LB_HD DualQ to_dual_quat(Rigid t) {
	const V3 p = t.pos;
	const Q4 r = t.rot;
	DualQ o;
	o.r = r;
	o.d.x = LB_FMUL(0.5f, LB_FSUB(LB_FADD(LB_FMUL(p.x, r.w), LB_FMUL(p.y, r.z)), LB_FMUL(p.z, r.y)));
	o.d.y = LB_FMUL(0.5f, LB_FADD(LB_FADD(LB_FMUL(-p.x, r.z), LB_FMUL(p.y, r.w)), LB_FMUL(p.z, r.x)));
	o.d.z = LB_FMUL(0.5f, LB_FADD(LB_FSUB(LB_FMUL(p.x, r.y), LB_FMUL(p.y, r.x)), LB_FMUL(p.z, r.w)));
	o.d.w = LB_FMUL(-0.5f, LB_FADD(LB_FADD(LB_FMUL(p.x, r.x), LB_FMUL(p.y, r.y)), LB_FMUL(p.z, r.z)));
	return o;
}

// math.cpp:727-756 Quat::toMatrix + :887-890 Matrix(pos, rot); m[col * 4 + row]
LB_HD void to_matrix(Rigid t, float* m) {
	const Q4 q = t.rot;
	const float fx = LB_FADD(q.x, q.x), fy = LB_FADD(q.y, q.y), fz = LB_FADD(q.z, q.z);
	const float fwx = LB_FMUL(fx, q.w), fwy = LB_FMUL(fy, q.w), fwz = LB_FMUL(fz, q.w);
	const float fxx = LB_FMUL(fx, q.x), fxy = LB_FMUL(fy, q.x), fxz = LB_FMUL(fz, q.x);
	const float fyy = LB_FMUL(fy, q.y), fyz = LB_FMUL(fz, q.y), fzz = LB_FMUL(fz, q.z);
	m[0] = LB_FSUB(1.0f, LB_FADD(fyy, fzz)); m[4] = LB_FSUB(fxy, fwz);                 m[8] = LB_FADD(fxz, fwy);
	m[1] = LB_FADD(fxy, fwz);                 m[5] = LB_FSUB(1.0f, LB_FADD(fxx, fzz)); m[9] = LB_FSUB(fyz, fwx);
	m[2] = LB_FSUB(fxz, fwy);                 m[6] = LB_FADD(fyz, fwx);                 m[10] = LB_FSUB(1.0f, LB_FADD(fxx, fyy));
	m[3] = 0; m[7] = 0; m[11] = 0;
	m[12] = t.pos.x; m[13] = t.pos.y; m[14] = t.pos.z; m[15] = 1;
}

} // namespace lb
