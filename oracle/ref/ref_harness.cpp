// TEST INFRASTRUCTURE — not product code.  Built only where /root/reference exists (this container);
// the resulting oracle/_ref/libref_lumix.so travels to the GPU box as a prebuilt binary.
//
// A flat C API over the REFERENCE'S OWN compiled code:
//   * unmodified src/core/math.cpp + src/core/geometry.cpp  (arithmetic pins for oracle/ restatement)
//   * overlay build of src/renderer/culling_system.cpp on src/core/job_system.cpp
//     (SURVEY.md §8(c): 3 header/source edits + ref_stubs.cpp) — the stronger cull oracle and the
//     "reference" CPU baseline of bench.py.
// No reference source is copied into this repository; oracle/build_ref.py compiles it from where it lies.
#include "core/allocator.h"
#include "core/default_allocator.h"
#include "core/geometry.h"
#include "core/job_system.h"
#include "core/math.h"
#include "core/page_allocator.h"
#include "core/simd.h"
#include "core/simd_math.h"
#include "core/sync.h"
#include "renderer/culling_system.h"

#include <algorithm>
#include <pthread.h>
#include <stdint.h>
#include <string.h>
#include <time.h>
#include <vector>

using namespace Lumix;

#define REF_API extern "C" __attribute__((visibility("default")))

static double nowSeconds() {
	timespec ts;
	clock_gettime(CLOCK_MONOTONIC, &ts);
	return double(ts.tv_sec) + double(ts.tv_nsec) * 1e-9;
}

// ------------------------------------------------------------------------------------------------
// struct sizes (SURVEY.md §8a header line) — pinned by tests/test_oracle_ref.py
// ------------------------------------------------------------------------------------------------
REF_API int ref_sizeof(const char* what) {
	if (!strcmp(what, "Sphere")) return (int)sizeof(Sphere);
	if (!strcmp(what, "Frustum")) return (int)sizeof(Frustum);
	if (!strcmp(what, "ShiftedFrustum")) return (int)sizeof(ShiftedFrustum);
	if (!strcmp(what, "ShiftedFrustum.origin")) return (int)offsetof(ShiftedFrustum, origin);
	if (!strcmp(what, "Transform")) return (int)sizeof(Transform);
	if (!strcmp(what, "CullResult")) return (int)sizeof(CullResult);
	if (!strcmp(what, "CullResult.entities")) return (int)offsetof(CullResult, entities);
	if (!strcmp(what, "LocalRigidTransform")) return (int)sizeof(LocalRigidTransform);
	if (!strcmp(what, "DualQuat")) return (int)sizeof(DualQuat);
	if (!strcmp(what, "Matrix")) return (int)sizeof(Matrix);
	return -1;
}

// ------------------------------------------------------------------------------------------------
// RNG (math.cpp:1333-1378)
// ------------------------------------------------------------------------------------------------
REF_API void ref_rng_floats(uint32_t u, uint32_t v, uint32_t n, float* out, uint32_t* state_out) {
	RandomGenerator rg(u, v);
	for (uint32_t i = 0; i < n; ++i) out[i] = rg.randFloat();
	if (state_out) {
		// advance-equivalent state is not exposed; emit two more raw draws so callers can chain
		state_out[0] = rg.rand();
		state_out[1] = rg.rand();
	}
}

REF_API void ref_rng_range(uint32_t u, uint32_t v, uint32_t n, float from, float to, float* out) {
	RandomGenerator rg(u, v);
	for (uint32_t i = 0; i < n; ++i) out[i] = rg.randFloat(from, to);
}

// ------------------------------------------------------------------------------------------------
// geometry.cpp
// ------------------------------------------------------------------------------------------------
REF_API void ref_frustum_perspective(const double* pos, const float* dir, const float* up, float fov, float ratio, float near_d, float far_d, void* out256) {
	ShiftedFrustum f;
	memset(&f, 0, sizeof(f));
	f.computePerspective(DVec3(pos[0], pos[1], pos[2]), Vec3(dir[0], dir[1], dir[2]), Vec3(up[0], up[1], up[2]), fov, ratio, near_d, far_d);
	memcpy(out256, &f, sizeof(f));
}

REF_API void ref_frustum_ortho(const double* pos, const float* dir, const float* up, float width, float height, float near_d, float far_d, void* out256) {
	ShiftedFrustum f;
	memset(&f, 0, sizeof(f));
	f.computeOrtho(DVec3(pos[0], pos[1], pos[2]), Vec3(dir[0], dir[1], dir[2]), Vec3(up[0], up[1], up[2]), width, height, near_d, far_d);
	memcpy(out256, &f, sizeof(f));
}

REF_API void ref_viewport_frustum(int is_ortho, float fov, float ortho_size, int w, int h, const double* pos, const float* rot4, float near_d, float far_d, void* out256) {
	Viewport vp;
	vp.is_ortho = is_ortho != 0; vp.fov = fov; vp.ortho_size = ortho_size; vp.w = w; vp.h = h;
	vp.pos = DVec3(pos[0], pos[1], pos[2]);
	vp.rot = Quat(rot4[0], rot4[1], rot4[2], rot4[3]);
	vp.near = near_d; vp.far = far_d;
	ShiftedFrustum f;
	memset(&f, 0, sizeof(f));
	f = vp.getFrustum();
	memcpy(out256, &f, sizeof(f));
}

REF_API void ref_frustum_get_relative(const void* sf256, const double* origin, void* out224) {
	const ShiftedFrustum& f = *(const ShiftedFrustum*)sf256;
	Frustum r = f.getRelative(DVec3(origin[0], origin[1], origin[2]));
	memcpy(out224, &r, sizeof(r));
}

REF_API int ref_frustum_contains_aabb(const void* sf256, const double* pos, const float* size) {
	const ShiftedFrustum& f = *(const ShiftedFrustum*)sf256;
	return f.containsAABB(DVec3(pos[0], pos[1], pos[2]), Vec3(size[0], size[1], size[2])) ? 1 : 0;
}

REF_API int ref_frustum_intersects_aabb(const void* sf256, const double* pos, const float* size) {
	const ShiftedFrustum& f = *(const ShiftedFrustum*)sf256;
	return f.intersectsAABB(DVec3(pos[0], pos[1], pos[2]), Vec3(size[0], size[1], size[2])) ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// math.cpp
// ------------------------------------------------------------------------------------------------
REF_API void ref_cell_indices(const double* pos, float cell_size, int* out3) {
	// culling_system.cpp:27 : IVec3(pos * (1 / cell_size))
	const DVec3 p(pos[0], pos[1], pos[2]);
	const IVec3 i(p * (1 / cell_size));
	out3[0] = i.x; out3[1] = i.y; out3[2] = i.z;
}

REF_API void ref_transform_compose(const void* parent56, const void* local56, void* out56, uint32_t n) {
	const Transform* a = (const Transform*)parent56;
	const Transform* b = (const Transform*)local56;
	Transform* o = (Transform*)out56;
	for (uint32_t i = 0; i < n; ++i) o[i] = a[i].compose(b[i]);
}

// World::getRelativeMatrix (world.cpp:370-377) needs a World; its body is these three reference calls on m_transforms[entity]
REF_API void ref_relative_matrix(const void* tr56, const double* base_pos, float* out16, uint32_t n) {
	const Transform* t = (const Transform*)tr56;
	const DVec3 base(base_pos[0], base_pos[1], base_pos[2]);
	for (uint32_t i = 0; i < n; ++i) {
		Matrix mtx = t[i].rot.toMatrix();
		mtx.setTranslation(Vec3(t[i].pos - base));
		mtx.multiply3x3(t[i].scale);
		memcpy(out16 + 16 * (size_t)i, &mtx, sizeof(mtx));
	}
}

// the radius RenderModuleImpl::onModelInstanceMoved hands to CullingSystem::set (render_module.cpp:1554), with the reference's own
// variadic maximum (math.h:468-475)
REF_API void ref_sphere_radius(const void* tr56, const float* bounding_radius, float* out, uint32_t n) {
	const Transform* t = (const Transform*)tr56;
	for (uint32_t i = 0; i < n; ++i) out[i] = bounding_radius[i] * maximum(t[i].scale.x, t[i].scale.y, t[i].scale.z);
}

// the three reference calls of RenderModuleImpl::updateBoneAttachment (render_module.cpp:399-403) on caller-supplied data
REF_API void ref_bone_attachments(const void* parent56, const float* bone7, const float* relative7, const float* original_scale3, void* out56, uint32_t n) {
	const Transform* parent = (const Transform*)parent56;
	Transform* out = (Transform*)out56;
	for (uint32_t i = 0; i < n; ++i) {
		const float* b = bone7 + 7 * (size_t)i;
		const float* r = relative7 + 7 * (size_t)i;
		const LocalRigidTransform bone_transform = {Vec3(b[0], b[1], b[2]), Quat(b[3], b[4], b[5], b[6])};
		const LocalRigidTransform relative_transform = {Vec3(r[0], r[1], r[2]), Quat(r[3], r[4], r[5], r[6])};
		Transform result = parent[i].compose(bone_transform * relative_transform);
		result.scale = Vec3(original_scale3[3 * i], original_scale3[3 * i + 1], original_scale3[3 * i + 2]);
		out[i] = result;
	}
}

REF_API void ref_transform_compute_local(const void* parent56, const void* child56, void* out56, uint32_t n) {
	const Transform* p = (const Transform*)parent56;
	const Transform* c = (const Transform*)child56;
	Transform* o = (Transform*)out56;
	for (uint32_t i = 0; i < n; ++i) o[i] = Transform::computeLocal(p[i], c[i]);
}

REF_API void ref_quat_mul(const float* a, const float* b, float* out, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) {
		const Quat r = Quat(a[4 * i], a[4 * i + 1], a[4 * i + 2], a[4 * i + 3]) * Quat(b[4 * i], b[4 * i + 1], b[4 * i + 2], b[4 * i + 3]);
		out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
	}
}

REF_API void ref_quat_rotate(const float* q, const float* v, float* out, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) {
		const Vec3 r = Quat(q[4 * i], q[4 * i + 1], q[4 * i + 2], q[4 * i + 3]).rotate(Vec3(v[3 * i], v[3 * i + 1], v[3 * i + 2]));
		out[3 * i] = r.x; out[3 * i + 1] = r.y; out[3 * i + 2] = r.z;
	}
}

REF_API void ref_nlerp(const float* a, const float* b, const float* t, float* out, uint32_t n, int simd) {
	for (uint32_t i = 0; i < n; ++i) {
		const Quat qa(a[4 * i], a[4 * i + 1], a[4 * i + 2], a[4 * i + 3]);
		const Quat qb(b[4 * i], b[4 * i + 1], b[4 * i + 2], b[4 * i + 3]);
		const Quat r = simd ? simd_nlerp(qa, qb, t[i]) : nlerp(qa, qb, t[i]);
		out[4 * i] = r.x; out[4 * i + 1] = r.y; out[4 * i + 2] = r.z; out[4 * i + 3] = r.w;
	}
}

REF_API void ref_lerp_vec3(const float* a, const float* b, const float* t, float* out, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) {
		const Vec3 r = lerp(Vec3(a[3 * i], a[3 * i + 1], a[3 * i + 2]), Vec3(b[3 * i], b[3 * i + 1], b[3 * i + 2]), t[i]);
		out[3 * i] = r.x; out[3 * i + 1] = r.y; out[3 * i + 2] = r.z;
	}
}

static LocalRigidTransform lrt(const float* p) { return {Vec3(p[0], p[1], p[2]), Quat(p[3], p[4], p[5], p[6])}; }

// a, b, out: 7 floats each (pos xyz, rot xyzw)
REF_API void ref_lrt_mul(const float* a, const float* b, float* out, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) {
		const LocalRigidTransform r = lrt(a + 7 * i) * lrt(b + 7 * i);
		float* o = out + 7 * i;
		o[0] = r.pos.x; o[1] = r.pos.y; o[2] = r.pos.z; o[3] = r.rot.x; o[4] = r.rot.y; o[5] = r.rot.z; o[6] = r.rot.w;
	}
}

REF_API void ref_lrt_inverted(const float* a, float* out, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) {
		const LocalRigidTransform r = lrt(a + 7 * i).inverted();
		float* o = out + 7 * i;
		o[0] = r.pos.x; o[1] = r.pos.y; o[2] = r.pos.z; o[3] = r.rot.x; o[4] = r.rot.y; o[5] = r.rot.z; o[6] = r.rot.w;
	}
}

REF_API void ref_lrt_to_dual_quat(const float* a, float* out8, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) {
		const DualQuat dq = lrt(a + 7 * i).toDualQuat();
		memcpy(out8 + 8 * i, &dq, sizeof(dq));
	}
}

REF_API void ref_lrt_to_matrix(const float* a, float* out16, uint32_t n) {
	for (uint32_t i = 0; i < n; ++i) {
		const Matrix m = lrt(a + 7 * i).toMatrix();
		memcpy(out16 + 16 * i, &m, sizeof(m));
	}
}

// model.cpp:103-109 restated with the reference's own Matrix operators (evaluateSkin is file-static there)
REF_API void ref_skin_vertex(const float* matrices16, const float* pos3, const float* weights4, const int16_t* indices4, float* out3, uint32_t n) {
	const Matrix* m = (const Matrix*)matrices16;
	for (uint32_t i = 0; i < n; ++i) {
		const int16_t* idx = indices4 + 4 * i;
		const float* w = weights4 + 4 * i;
		const Matrix s = m[idx[0]] * w[0] + m[idx[1]] * w[1] + m[idx[2]] * w[2] + m[idx[3]] * w[3];
		const Vec3 r = s.transformPoint(Vec3(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]));
		out3[3 * i] = r.x; out3[3 * i + 1] = r.y; out3[3 * i + 2] = r.z;
	}
}

// ------------------------------------------------------------------------------------------------
// CullingSystem on the reference job system
// ------------------------------------------------------------------------------------------------
struct RefCulling {
	RefCulling() : page_allocator(allocator), system(CullingSystem::create(allocator, page_allocator)) {}
	DefaultAllocator allocator;
	PageAllocator page_allocator;
	UniquePtr<CullingSystem> system;
};

static DefaultAllocator* g_jobs_allocator = nullptr;
static int g_workers = 0;

REF_API int ref_jobs_init(int workers) {
	if (g_workers) return g_workers;
	if (workers < 1) workers = 1;
	if (workers > 64) workers = 64; // studio's own cap, studio_app.cpp:583
	g_jobs_allocator = new DefaultAllocator;
	if (!jobs::init((u8)workers, *g_jobs_allocator)) return 0;
	g_workers = workers;
	return g_workers;
}

REF_API int ref_jobs_workers() { return g_workers; }

REF_API void* ref_culling_create() { return new RefCulling; }

REF_API void ref_culling_destroy(void* h) { delete (RefCulling*)h; }

REF_API void ref_culling_add(void* h, const int32_t* entities, const uint8_t* types, const double* pos3, const float* radius, uint32_t n) {
	CullingSystem& cs = *((RefCulling*)h)->system;
	for (uint32_t i = 0; i < n; ++i) cs.add(EntityRef{entities[i]}, types[i], DVec3(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]), radius[i]);
}

REF_API void ref_culling_remove(void* h, const int32_t* entities, uint32_t n) {
	CullingSystem& cs = *((RefCulling*)h)->system;
	for (uint32_t i = 0; i < n; ++i) cs.remove(EntityRef{entities[i]});
}

REF_API void ref_culling_set(void* h, const int32_t* entities, const double* pos3, const float* radius, uint32_t n) {
	CullingSystem& cs = *((RefCulling*)h)->system;
	for (uint32_t i = 0; i < n; ++i) cs.set(EntityRef{entities[i]}, DVec3(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]), radius[i]);
}

REF_API void ref_culling_set_position(void* h, const int32_t* entities, const double* pos3, uint32_t n) {
	CullingSystem& cs = *((RefCulling*)h)->system;
	for (uint32_t i = 0; i < n; ++i) cs.setPosition(EntityRef{entities[i]}, DVec3(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]));
}

REF_API void ref_culling_set_radius(void* h, const int32_t* entities, const float* radius, uint32_t n) {
	CullingSystem& cs = *((RefCulling*)h)->system;
	for (uint32_t i = 0; i < n; ++i) cs.setRadius(EntityRef{entities[i]}, radius[i]);
}

REF_API float ref_culling_get_radius(void* h, int32_t entity) { return ((RefCulling*)h)->system->getRadius(EntityRef{entity}); }
REF_API int ref_culling_is_added(void* h, int32_t entity) { return ((RefCulling*)h)->system->isAdded(EntityRef{entity}) ? 1 : 0; }

struct CullCall {
	RefCulling* rc;
	const ShiftedFrustum* frustum;
	int type; // -1 = all
	uint32_t* out_ids;
	uint8_t* out_types;
	uint32_t cap;
	int iters;
	std::vector<double> times;
	uint32_t count = 0;
	uint32_t pages = 0;
	pthread_mutex_t mutex = PTHREAD_MUTEX_INITIALIZER;
	pthread_cond_t cond = PTHREAD_COND_INITIALIZER;
	bool done = false;
};

static void cullJob(void* ptr) {
	CullCall& c = *(CullCall*)ptr;
	CullingSystem& cs = *c.rc->system;
	for (int it = 0; it < c.iters; ++it) {
		const double t0 = nowSeconds();
		CullResult* res = c.type < 0 ? cs.cull(*c.frustum) : cs.cull(*c.frustum, (u8)c.type);
		const double t1 = nowSeconds();
		c.times.push_back(t1 - t0);
		if (it == c.iters - 1) {
			uint32_t n = 0, pages = 0;
			for (const CullResult* j = res; j; j = j->header.next) {
				++pages;
				for (u32 i = 0; i < j->header.count; ++i) {
					if (n < c.cap) {
						if (c.out_ids) c.out_ids[n] = (uint32_t)j->entities[i].index;
						if (c.out_types) c.out_types[n] = j->header.type;
					}
					++n;
				}
			}
			c.count = n;
			c.pages = pages;
		}
		if (res) res->free(c.rc->page_allocator); // as the caller does, pipeline.cpp:1045
	}
	pthread_mutex_lock(&c.mutex);
	c.done = true;
	pthread_cond_signal(&c.cond);
	pthread_mutex_unlock(&c.mutex);
}

// Runs `iters` culls on a job-system fiber (all engine code runs on fibers, app/main.cpp:308-327) and
// returns the visible count of the last one; ids are in the reference's (nondeterministic) order.
// times3 = {best, median, first} seconds of cull() alone (result walk + free excluded).
REF_API uint32_t ref_culling_cull(void* h, const void* sf256, int type, uint32_t* out_ids, uint8_t* out_types, uint32_t cap, int iters, double* times3, uint32_t* out_pages) {
	if (!g_workers) return 0xffffffffu;
	CullCall c;
	c.rc = (RefCulling*)h;
	// ShiftedFrustum is alignas(16); copy to an aligned local
	alignas(16) ShiftedFrustum f;
	memcpy(&f, sf256, sizeof(f));
	c.frustum = &f;
	c.type = type;
	c.out_ids = out_ids;
	c.out_types = out_types;
	c.cap = cap;
	c.iters = iters < 1 ? 1 : iters;
	jobs::run(&c, cullJob, nullptr);
	pthread_mutex_lock(&c.mutex);
	while (!c.done) pthread_cond_wait(&c.cond, &c.mutex);
	pthread_mutex_unlock(&c.mutex);
	if (times3) {
		std::vector<double> s = c.times;
		std::sort(s.begin(), s.end());
		times3[0] = s.front();
		times3[1] = s[s.size() / 2];
		times3[2] = c.times.front();
	}
	if (out_pages) *out_pages = c.pages;
	return c.count;
}
