// TEST INFRASTRUCTURE — not product code.  Drives the GPU cull THROUGH THE ENGINE'S OWN C++ INTERFACE: the reference's job system, allocators
// and PageAllocator (compiled from /root/reference by oracle/build_ref.py) linked with lumixengine_b200/host/culling_system_b200.cpp, which
// supplies CullingSystem::create (the single construction site is render_module.cpp:3569) and CullResult::free.  Everything below talks to
// the abstract CullingSystem (culling_system.h:58-77) exactly as the renderer does: cull() from job-system fibers for several views at once
// (pipeline.cpp:1036-1041), CullResult page chains from the engine's PageAllocator, CullResult::free by the caller (pipeline.cpp:1045).
#define private public
#include "core/page_allocator.h"
#undef private
#include "core/default_allocator.h"
#include "core/geometry.h"
#include "core/job_system.h"
#include "core/log_callback.h"
#include "renderer/culling_system.h"

#include <execinfo.h>
#include <signal.h>
#include <stdio.h>
#include <unistd.h>

#include <pthread.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

using namespace Lumix;

#define SHIM_API extern "C" __attribute__((visibility("default")))

struct ShimWorld {
	DefaultAllocator allocator;
	PageAllocator page_allocator;
	UniquePtr<CullingSystem> system;
	ShimWorld() : page_allocator(allocator), system(CullingSystem::create(allocator, page_allocator)) {}
};

static DefaultAllocator* g_jobs_allocator = nullptr;
static int g_workers = 0;

static void crashHandler(int sig) { // test aid: a native backtrace when something dies on a worker fiber
	void* frames[48];
	const int n = backtrace(frames, 48);
	const char msg[] = "[engine shim] fatal signal, backtrace:\n";
	(void)!write(2, msg, sizeof(msg) - 1);
	backtrace_symbols_fd(frames, n, 2);
	_exit(128 + sig);
}

static void logToStderr(LogLevel level, const char* msg) { fprintf(stderr, "[engine log %d] %s\n", (int)level, msg); }

SHIM_API int shim_jobs_init(int workers) {
	if (g_workers) return g_workers;
	registerLogCallback<&logToStderr>();
	struct sigaction sa;
	memset(&sa, 0, sizeof(sa));
	sa.sa_handler = crashHandler;
	sa.sa_flags = SA_ONSTACK; // on the alternate stack each worker gets below: a backtrace even when a fiber stack overflowed
	sigaction(SIGFPE, &sa, nullptr);
	sigaction(SIGSEGV, &sa, nullptr);
	sigaction(SIGBUS, &sa, nullptr);
	sigaction(SIGILL, &sa, nullptr);
	sigaction(SIGABRT, &sa, nullptr);
	if (workers < 1) workers = 1;
	if (workers > 64) workers = 64;
	g_jobs_allocator = new DefaultAllocator;
	if (!jobs::init((u8)workers, *g_jobs_allocator)) return 0;
	g_workers = workers;
	for (int w = 0; w < workers; ++w) {
		jobs::run(nullptr, [](void*) {
			stack_t ss;
			ss.ss_sp = malloc(1 << 16); ss.ss_size = 1 << 16; ss.ss_flags = 0;
			sigaltstack(&ss, nullptr);
		}, nullptr, (u8)w);
	}
	usleep(20000);
	return g_workers;
}

SHIM_API void* shim_create() { return new ShimWorld; }
SHIM_API void shim_destroy(void* h) {
	ShimWorld* w = (ShimWorld*)h;
	const bool dbg = getenv("SHIM_DEBUG") != nullptr;
	if (dbg) fprintf(stderr, "[shim] destroy: culling system\n");
	w->system.reset();
	if (dbg) fprintf(stderr, "[shim] destroyed (%d pages still allocated)\n", (int)w->page_allocator.allocated_count);
	// the allocators themselves are left alone: DefaultAllocator / PageAllocator teardown goes through os.cpp paths the Linux overlay only stubs
}
SHIM_API int shim_allocated_pages(void* h) { return (int)((ShimWorld*)h)->page_allocator.allocated_count; }

SHIM_API void shim_add(void* h, const int32_t* entities, const uint8_t* types, const double* pos3, const float* radius, uint32_t n) {
	CullingSystem& cs = *((ShimWorld*)h)->system;
	for (uint32_t i = 0; i < n; ++i) cs.add(EntityRef{entities[i]}, types[i], DVec3(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]), radius[i]);
}
SHIM_API void shim_set(void* h, const int32_t* entities, const double* pos3, const float* radius, uint32_t n) {
	CullingSystem& cs = *((ShimWorld*)h)->system;
	for (uint32_t i = 0; i < n; ++i) cs.set(EntityRef{entities[i]}, DVec3(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]), radius[i]);
}
SHIM_API void shim_remove(void* h, const int32_t* entities, uint32_t n) {
	CullingSystem& cs = *((ShimWorld*)h)->system;
	for (uint32_t i = 0; i < n; ++i) cs.remove(EntityRef{entities[i]});
}
SHIM_API float shim_get_radius(void* h, int32_t entity) { return ((ShimWorld*)h)->system->getRadius(EntityRef{entity}); }
SHIM_API int shim_is_added(void* h, int32_t entity) { return ((ShimWorld*)h)->system->isAdded(EntityRef{entity}) ? 1 : 0; }

struct ViewCall {
	ShimWorld* world;
	const ShiftedFrustum* frustum;
	int type;
	uint32_t* out_ids; uint8_t* out_types; uint32_t cap;
	uint32_t count, pages, bad_pages, null_result;
};

struct ViewBatch {
	ViewCall* calls; uint32_t n;
	AtomicI32 left = 0;
	pthread_mutex_t mutex = PTHREAD_MUTEX_INITIALIZER;
	pthread_cond_t cond = PTHREAD_COND_INITIALIZER;
	bool done = false;
};
struct ViewJob { ViewBatch* batch; uint32_t idx; };

static void viewJob(void* ptr) {
	ViewJob* job = (ViewJob*)ptr;
	ViewCall& c = job->batch->calls[job->idx];
	CullingSystem& cs = *c.world->system;
	static const bool dbg = getenv("SHIM_DEBUG") != nullptr;
	if (dbg) fprintf(stderr, "[shim] view %u: cull\n", job->idx);
	CullResult* res = c.type < 0 ? cs.cull(*c.frustum) : cs.cull(*c.frustum, (u8)c.type);
	if (dbg) fprintf(stderr, "[shim] view %u: cull returned %p\n", job->idx, (void*)res);
	uint32_t n = 0, pages = 0, bad = 0;
	for (const CullResult* j = res; j; j = j->header.next) { // what PipelineImpl::createSortKeys does with it: one type per page, <= 1020 ids
		++pages;
		if (j->header.count > (u32)lengthOf(j->entities) || ((uintptr_t)j & (PageAllocator::PAGE_SIZE - 1))) ++bad;
		for (u32 i = 0; i < j->header.count; ++i) {
			if (n < c.cap) { c.out_ids[n] = (uint32_t)j->entities[i].index; c.out_types[n] = j->header.type; }
			++n;
		}
	}
	c.count = n; c.pages = pages; c.bad_pages = bad; c.null_result = res ? 0 : 1;
	if (res) res->free(c.world->page_allocator); // the caller frees, pipeline.cpp:1045
	if (dbg) fprintf(stderr, "[shim] view %u: %u ids in %u pages, freed\n", job->idx, n, pages);
	ViewBatch* b = job->batch;
	if (b->left.dec() == 1) {
		pthread_mutex_lock(&b->mutex);
		b->done = true;
		pthread_cond_signal(&b->cond);
		pthread_mutex_unlock(&b->mutex);
	}
}

// n_views culls issued as n_views jobs at once (main view, shadow cascades, lights: pipeline.cpp:996-1063 runs them concurrently).
// out_ids / out_types: n_views x cap; out_info: n_views x {count, pages, bad_pages, null_result}.
SHIM_API void shim_cull_views(void* h, const void* frusta256, uint32_t n_views, int type, uint32_t* out_ids, uint8_t* out_types, uint32_t cap, uint32_t* out_info) {
	ViewBatch batch;
	ViewCall* calls = new ViewCall[n_views];
	ViewJob* jobs_ = new ViewJob[n_views];
	batch.calls = calls; batch.n = n_views; batch.left = (i32)n_views;
	for (uint32_t v = 0; v < n_views; ++v) {
		calls[v] = {(ShimWorld*)h, (const ShiftedFrustum*)((const uint8_t*)frusta256 + 256 * (size_t)v), type, out_ids + (size_t)cap * v, out_types + (size_t)cap * v, cap, 0, 0, 0, 0};
		jobs_[v] = {&batch, v};
	}
	for (uint32_t v = 0; v < n_views; ++v) jobs::run(&jobs_[v], viewJob, nullptr);
	pthread_mutex_lock(&batch.mutex);
	while (!batch.done) pthread_cond_wait(&batch.cond, &batch.mutex);
	pthread_mutex_unlock(&batch.mutex);
	for (uint32_t v = 0; v < n_views; ++v) { out_info[4 * v] = calls[v].count; out_info[4 * v + 1] = calls[v].pages; out_info[4 * v + 2] = calls[v].bad_pages; out_info[4 * v + 3] = calls[v].null_result; }
	delete[] calls;
	delete[] jobs_;
}

// CPU-only self test of the wake-up path the shim uses (no GPU involved): a job parks on a jobs::Signal; a plain OS thread (standing in for
// the driver's callback thread) schedules the job that turns it green.  Returns the number of completed round trips.
struct SelfTest { jobs::Signal* signal; };
static void* selfTestThread(void* p) {
	usleep(200);
	jobs::run(p, [](void* s) { jobs::turnGreen((jobs::Signal*)s); }, nullptr);
	return nullptr;
}
struct SelfTestCall { int rounds; int done; pthread_mutex_t mutex; pthread_cond_t cond; bool finished; };
static void selfTestJob(void* p) {
	SelfTestCall& c = *(SelfTestCall*)p;
	for (int i = 0; i < c.rounds; ++i) {
		jobs::Signal sig;
		jobs::turnRed(&sig);
		pthread_t t;
		pthread_create(&t, nullptr, selfTestThread, &sig);
		jobs::wait(&sig);
		pthread_join(t, nullptr);
		++c.done;
	}
	pthread_mutex_lock(&c.mutex);
	c.finished = true;
	pthread_cond_signal(&c.cond);
	pthread_mutex_unlock(&c.mutex);
}
SHIM_API int shim_selftest_signal(int rounds, int parallel) {
	SelfTestCall* calls = new SelfTestCall[parallel];
	for (int k = 0; k < parallel; ++k) {
		calls[k].rounds = rounds; calls[k].done = 0; calls[k].finished = false;
		pthread_mutex_init(&calls[k].mutex, nullptr); pthread_cond_init(&calls[k].cond, nullptr);
		jobs::run(&calls[k], selfTestJob, nullptr);
	}
	int total = 0;
	for (int k = 0; k < parallel; ++k) {
		pthread_mutex_lock(&calls[k].mutex);
		while (!calls[k].finished) pthread_cond_wait(&calls[k].cond, &calls[k].mutex);
		pthread_mutex_unlock(&calls[k].mutex);
		total += calls[k].done;
	}
	delete[] calls;
	return total;
}
