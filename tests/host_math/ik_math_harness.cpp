// TEST INFRASTRUCTURE.  The IK arithmetic of lumixengine_b200/csrc/lb200_math.cuh (vec3_to_vec3, nlerp, rinverted, length, conjugated)
// compiled for the host with a C ABI, so that tests/test_animation_ik_cpu.py can check it without a GPU against the reference-run vectors
// of tests/golden/ik_kat.npz bit for bit.
#include "lb200_math.cuh"

using namespace lb;

extern "C" {

void ikm_vec3_to_vec3(const float* a, const float* b, float* out, unsigned n) {
	for (unsigned i = 0; i < n; ++i) {
		const Q4 r = vec3_to_vec3(v3(a[3 * i], a[3 * i + 1], a[3 * i + 2]), v3(b[3 * i], b[3 * i + 1], b[3 * i + 2]));
		out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
	}
}

void ikm_nlerp(const float* a, const float* b, const float* t, float* out, unsigned n) {
	for (unsigned i = 0; i < n; ++i) {
		const Q4 r = nlerp(q4(a[4 * i], a[4 * i + 1], a[4 * i + 2], a[4 * i + 3]), q4(b[4 * i], b[4 * i + 1], b[4 * i + 2], b[4 * i + 3]), t[i]);
		out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
	}
}

void ikm_inverted(const float* a, float* out7, unsigned n) {
	for (unsigned i = 0; i < n; ++i) {
		const float* p = a + 7 * i;
		Rigid t;
		t.pos = v3(p[0], p[1], p[2]);
		t.rot = q4(p[3], p[4], p[5], p[6]);
		const Rigid r = rinverted(t);
		float* o = out7 + 7 * i;
		o[0] = r.pos.x; o[1] = r.pos.y; o[2] = r.pos.z; o[3] = r.rot.x; o[4] = r.rot.y; o[5] = r.rot.z; o[6] = r.rot.w;
	}
}

void ikm_length(const float* a, float* out, unsigned n) {
	for (unsigned i = 0; i < n; ++i) out[i] = length(v3(a[3 * i], a[3 * i + 1], a[3 * i + 2]));
}

void ikm_conjugated(const float* a, float* out, unsigned n) {
	for (unsigned i = 0; i < n; ++i) {
		const Q4 r = conjugated(q4(a[4 * i], a[4 * i + 1], a[4 * i + 2], a[4 * i + 3]));
		out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
	}
}

} // extern "C"
