// TEST INFRASTRUCTURE — not product code.  Runs the REFERENCE'S OWN sort-key packers (src/renderer/pipeline.cpp:41-143: DrawCommandTypes,
// floatFlip, make*SortKey / make*SortValue), its Histogram + PipelineImpl::radixSort (:4020-4144) and Model::getLODMeshIndices
// (model.h:173-179) to pin oracle_sortkeys.c.
//
// pipeline.cpp cannot be compiled here (DX12 renderer), so oracle/build_ref.py cuts those two regions out of the reference file AT BUILD
// TIME into the temporary overlay (renderer/extracted_sort_key_packers.inl, renderer/extracted_radix_sort.inl; deleted with the overlay,
// never stored in this repository) and this file includes them.
#define private public
#define protected public
#include "renderer/model.h"
#include "renderer/material.h"
#undef private
#undef protected
#include "core/array.h"
#include "core/atomic.h"
#include "core/default_allocator.h"
#include "core/job_system.h"
#include "core/math.h"
#include "core/profiler.h"
#include "core/simd.h"
#include "core/sync.h"

#include <stdint.h>
#include <string.h>

using namespace Lumix;

#define REF_API extern "C" __attribute__((visibility("default")))

namespace Lumix {
namespace extracted_keys {
#include "renderer/extracted_sort_key_packers.inl"
}

struct ExtractedSorter {
	explicit ExtractedSorter(IAllocator& a) : m_allocator(a) {}
	IAllocator& m_allocator;
#include "renderer/extracted_radix_sort.inl"
};
} // namespace Lumix

template <typename T> struct RawStorageS {
	RawStorageS() { memset(mem, 0, sizeof(mem)); }
	T* get() { return reinterpret_cast<T*>(mem); }
	alignas(alignof(T)) unsigned char mem[sizeof(T)];
};

REF_API uint32_t ref_float_flip(uint32_t bits) { return extracted_keys::floatFlip(bits); }
REF_API uint64_t ref_make_mesh_sort_key(uint32_t sort_key, uint8_t bucket) {
	MeshMaterial mm = {};
	mm.sort_key = sort_key;
	return (uint64_t)extracted_keys::makeMeshSortKey(mm, bucket);
}
REF_API uint64_t ref_make_depth_sort_key(float depth_squared, uint8_t bucket) { return (uint64_t)extracted_keys::makeDepthSortKey(depth_squared, bucket); }
REF_API uint64_t ref_make_autoinstanced_sort_key(int32_t instancer_index, uint8_t bucket) { return (uint64_t)extracted_keys::makeAutoInstancedSortKey(instancer_index, bucket); }
REF_API uint64_t ref_make_decal_sort_key(uint32_t material_sort_key, uint8_t bucket) {
	RawStorageS<Material> mem; // only m_sort_key is read (Material::getSortKey)
	mem.get()->m_sort_key = material_sort_key;
	return (uint64_t)extracted_keys::makeDecalSortKey(mem.get(), bucket);
}
REF_API uint64_t ref_make_decal_sort_value(int32_t e) { return (uint64_t)extracted_keys::makeDecalSortValue(EntityPtr{e}); }
REF_API uint64_t ref_make_curve_decal_sort_value(int32_t e) { return (uint64_t)extracted_keys::makeCurveDecalSortValue(EntityPtr{e}); }
REF_API uint64_t ref_make_skinned_sort_value(int32_t e, uint32_t mesh_idx) { return (uint64_t)extracted_keys::makeSkinnedSortValue(EntityPtr{e}, mesh_idx); }
REF_API uint64_t ref_make_mesh_sort_value(int32_t e, uint32_t mesh_idx) { return (uint64_t)extracted_keys::makeMeshSortValue(EntityPtr{e}, mesh_idx); }
REF_API uint64_t ref_make_autoinstanced_sort_value(uint32_t batch_idx, uint32_t instancer_idx) { return (uint64_t)extracted_keys::makeAutoInstancedSortValue(batch_idx, instancer_idx); }

REF_API uint32_t ref_lod_mesh_indices(const float* lod_distances4, float squared_distance) {
	RawStorageS<Model> mem; // only m_lod_distances is read
	for (int i = 0; i < 4; ++i) mem.get()->m_lod_distances[i] = lod_distances4[i];
	return mem.get()->getLODMeshIndices(squared_distance);
}

// needs ref_jobs_init.  Runs inside a job like the engine does (sizes >= 512 build their histograms with jobs::runOnWorkers, which
// has to be called from a job-system fiber); the calling thread waits on a condition variable.
#include <pthread.h>
struct SortCall {
	uint64_t* keys; uint64_t* values; int size;
	pthread_mutex_t mutex; pthread_cond_t cond; bool done;
};
static void sortJob(void* p) {
	SortCall& c = *(SortCall*)p;
	static DefaultAllocator allocator;
	ExtractedSorter s(allocator);
	s.radixSort(c.keys, c.values, c.size);
	pthread_mutex_lock(&c.mutex);
	c.done = true;
	pthread_cond_signal(&c.cond);
	pthread_mutex_unlock(&c.mutex);
}
REF_API void ref_radix_sort(uint64_t* keys, uint64_t* values, int size) {
	SortCall c;
	c.keys = keys; c.values = values; c.size = size; c.done = false;
	pthread_mutex_init(&c.mutex, nullptr);
	pthread_cond_init(&c.cond, nullptr);
	jobs::run(&c, sortJob, nullptr);
	pthread_mutex_lock(&c.mutex);
	while (!c.done) pthread_cond_wait(&c.cond, &c.mutex);
	pthread_mutex_unlock(&c.mutex);
}
