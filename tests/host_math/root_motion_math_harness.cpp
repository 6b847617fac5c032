// The root-motion helpers of lumixengine_b200/csrc/lb200_math.cuh compiled for the host (tests/test_animation_root_motion_cpu.py):
// normalize(Quat) and Animation::getRotation's double-path unpack on arrays.
#include "lb200_math.cuh"

#include <string.h>

extern "C" {

void rm_normalize(const float* q4in, float* q4out, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) {
		const float* a = q4in + 4 * i;
		const lb::Q4 r = lb::normalize(lb::q4(a[0], a[1], a[2], a[3]));
		float* o = q4out + 4 * i;
		o[0] = r.x; o[1] = r.y; o[2] = r.z; o[3] = r.w;
	}
}

// frames[i] of the rotation track at bit offset offset_bits of a stream with frame_bits bits per frame
void rm_rotation_d(const uint8_t* stream, uint32_t frame_bits, uint32_t offset_bits, const float* mn, const float* range, const uint32_t* bits,
	uint32_t skipped_channel, const uint32_t* frames, float* q4out, uint32_t n)
{
	for (uint32_t i = 0; i < n; ++i) {
		const uint32_t offset = frame_bits * frames[i] + offset_bits;
		unsigned long long packed;
		memcpy(&packed, stream + offset / 8, sizeof(packed));
		packed >>= offset & 7;
		const lb::Q4 r = lb::unpack_rotation_d(packed, mn, range, bits, skipped_channel);
		float* o = q4out + 4 * i;
		o[0] = r.x; o[1] = r.y; o[2] = r.z; o[3] = r.w;
	}
}

} // extern "C"
