// TEST INFRASTRUCTURE — not product code.  Runs the REFERENCE'S OWN PipelineImpl::computeSkeletonDualQuats
// (src/renderer/pipeline.cpp:2680-2745: 4-wide SIMD batches through simd_math.h + the scalar tail) to pin
// oracle_palette_dual_quats as a whole, not only its primitives.
//
// pipeline.cpp cannot be compiled here (DX12 renderer), so oracle/build_ref.py cuts that one member function out of the
// reference file AT BUILD TIME into the temporary overlay (renderer/extracted_compute_skeleton_dual_quats.inl, deleted with
// the overlay; never stored in this repository) and this file includes it into a holder struct.  Model / Pose are filled
// through `#define private public` as in ref_anim_harness.cpp; only data members are read.
#define private public
#define protected public
#include "renderer/model.h"
#include "renderer/pose.h"
#undef private
#undef protected
#include "renderer/render_module.h"
#include "core/default_allocator.h"
#include "core/simd.h"
#include "core/simd_math.h"

#include <new>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

using namespace Lumix;

#define REF_API extern "C" __attribute__((visibility("default")))

namespace Lumix {

struct ExtractedPipeline {
#include "renderer/extracted_compute_skeleton_dual_quats.inl"
};

// file-static helpers of model.cpp, cut out the same way: evaluateSkin (model.cpp:103-109), computeSkinMatrices (model.cpp:132-137)
namespace extracted_model {
#include "renderer/extracted_model_statics.inl"
}

// model.cpp is not part of this library (it pulls in the whole renderer); the extracted function calls this accessor for the
// scalar tail.  It only gathers bone `i` out of the SoA inverse bind arrays.
LocalRigidTransform Model::getInverseBindTransform(i32 i) const {
	const SOATransform& s = m_inverse_bind;
	return {Vec3(s.px[i], s.py[i], s.pz[i]), Quat(s.rx[i], s.ry[i], s.rz[i], s.rw[i])};
}

} // namespace Lumix

struct RefSkeletonP { // same layout as RefSkeleton in ref_anim_harness.cpp
	uint32_t bone_count; int32_t first_nonroot;
	const int16_t* parents; const float* bind_relative7; const float* inverse_bind7;
};

template <typename T> struct RawStorageP {
	RawStorageP() { memset(mem, 0, sizeof(mem)); }
	T* get() { return reinterpret_cast<T*>(mem); }
	alignas(alignof(T)) unsigned char mem[sizeof(T)];
};

// pos3 / rot4: one absolute pose (bone_count bones); out8: bone_count dual quaternions {r.xyzw, d.xyzw}
REF_API int ref_skeleton_dual_quats(const RefSkeletonP* sk, const float* pos3, const float* rot4, float* out8) {
	static DefaultAllocator allocator;
	const uint32_t n = sk->bone_count;
	const uint32_t padded = (n + 3u) & ~3u;
	float* soa = (float*)aligned_alloc(16, sizeof(float) * 7 * padded);
	unsigned char* out = (unsigned char*)aligned_alloc(16, 32 * (size_t)padded);
	if (!soa || !out) return -1;
	memset(soa, 0, sizeof(float) * 7 * padded);

	RawStorageP<Model> model_mem;
	Model* model = model_mem.get();
	new (&model->m_bones) Array<Model::Bone>(allocator);
	for (uint32_t i = 0; i < n; ++i) model->m_bones.emplace(allocator);
	float** lanes[7] = {&model->m_inverse_bind.px, &model->m_inverse_bind.py, &model->m_inverse_bind.pz,
		&model->m_inverse_bind.rx, &model->m_inverse_bind.ry, &model->m_inverse_bind.rz, &model->m_inverse_bind.rw};
	for (int k = 0; k < 7; ++k) {
		*lanes[k] = soa + (size_t)k * padded;
		for (uint32_t i = 0; i < n; ++i) (*lanes[k])[i] = sk->inverse_bind7[7 * i + k];
	}
	{
		Pose pose(allocator);
		pose.resize((int)n);
		for (uint32_t i = 0; i < n; ++i) {
			pose.positions[i] = Vec3(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]);
			pose.rotations[i] = Quat(rot4[4 * i], rot4[4 * i + 1], rot4[4 * i + 2], rot4[4 * i + 3]);
		}
		pose.is_absolute = true;
		pose.slice.ptr = out;
		ModelInstance mi;
		mi.model = model;
		mi.pose = &pose;
		ExtractedPipeline holder;
		holder.computeSkeletonDualQuats(&mi);
		memcpy(out8, out, 32 * (size_t)n);
	}
	model->m_bones.~Array();
	free(soa);
	free(out);
	return 0;
}

// computeSkinMatrices (model.cpp:132-137) on one absolute pose: out16 = bone_count column-major matrices
REF_API int ref_skin_matrices(const RefSkeletonP* sk, const float* pos3, const float* rot4, float* out16) {
	static DefaultAllocator allocator;
	const uint32_t n = sk->bone_count;
	float* soa = (float*)malloc(sizeof(float) * 7 * (n ? n : 1));
	if (!soa) return -1;
	RawStorageP<Model> model_mem;
	Model* model = model_mem.get();
	float** lanes[7] = {&model->m_inverse_bind.px, &model->m_inverse_bind.py, &model->m_inverse_bind.pz,
		&model->m_inverse_bind.rx, &model->m_inverse_bind.ry, &model->m_inverse_bind.rz, &model->m_inverse_bind.rw};
	for (int k = 0; k < 7; ++k) {
		*lanes[k] = soa + (size_t)k * n;
		for (uint32_t i = 0; i < n; ++i) (*lanes[k])[i] = sk->inverse_bind7[7 * i + k];
	}
	{
		Pose pose(allocator);
		pose.resize((int)n);
		for (uint32_t i = 0; i < n; ++i) {
			pose.positions[i] = Vec3(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]);
			pose.rotations[i] = Quat(rot4[4 * i], rot4[4 * i + 1], rot4[4 * i + 2], rot4[4 * i + 3]);
		}
		static_assert(sizeof(Matrix) == 64, "");
		extracted_model::computeSkinMatrices(pose, *model, (Matrix*)out16);
	}
	free(soa);
	return 0;
}

// evaluateSkin (model.cpp:103-109) for n vertices against one matrix palette
REF_API void ref_evaluate_skin(const float* matrices16, const float* pos3, const float* weights4, const int16_t* indices4, float* out3, uint32_t n) {
	const Matrix* m = (const Matrix*)matrices16;
	for (uint32_t i = 0; i < n; ++i) {
		Mesh::Skin s;
		s.weights = Vec4(weights4[4 * i], weights4[4 * i + 1], weights4[4 * i + 2], weights4[4 * i + 3]);
		for (int k = 0; k < 4; ++k) s.indices[k] = indices4[4 * i + k];
		Vec3 p(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]);
		const Vec3 r = extracted_model::evaluateSkin(p, s, m);
		out3[3 * i] = r.x; out3[3 * i + 1] = r.y; out3[3 * i + 2] = r.z;
	}
}
