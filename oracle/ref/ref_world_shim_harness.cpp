// TEST INFRASTRUCTURE — not product code.  Runs the World patch (lumixengine_b200/host/world_b200.inl appended to a temporary copy of the
// reference's own src/engine/world.cpp by oracle/build_ref.py) inside real Lumix::World objects: two worlds get the same entities, the same
// hierarchy (World::setParent, world.cpp:619-701) and the same local transforms; then the same root moves go
//   world A: World::setTransform per root — the reference recursion World::transformEntity (world.cpp:255-282)
//   world B: World::setTransformsDeferredB200 + World::propagateHierarchyB200 — one level-order pass on the GPU through liblumix_b200.so
// and every entity's Transform plus the number of `transformed` delegate calls per entity are handed back for comparison.
// The Engine / SystemManager a World needs at construction (world.cpp:122-153) are minimal stand-ins: no systems, the engine's allocator.
#include "core/default_allocator.h"
#include "core/log_callback.h"
#include "core/page_allocator.h"
#include "core/stream.h"
#include "engine/engine.h"
#include "engine/plugin.h"
#include "engine/reflection.h"
#include "engine/resource.h"
#include "engine/world.h"

#include "lumix_b200.h"

#include <stdint.h>
#include <stdio.h>
#include <string.h>
#include <time.h>

using namespace Lumix;

#define SHIM_API extern "C" __attribute__((visibility("default")))

namespace Lumix::reflection {
// world.cpp asks the reflection registry which component types a module owns (World::addModule, world.cpp:218-228); there are no modules here
Span<const RegisteredComponent> getComponents() { return {}; }
}

namespace {

struct StubSystems final : SystemManager {
	StubSystems(IAllocator& a) : systems(a), libraries(a), loaded(a) {}
	void initSystems() override {}
	void unload(ISystem*) override {}
	ISystem* load(const char*) override { return nullptr; }
	void addSystem(ISystem*, void*) override {}
	void update(float) override {}
	ISystem* getSystem(const char*) override { return nullptr; }
	const Array<ISystem*>& getSystems() const override { return systems; }
	const Array<void*>& getLibraries() const override { return libraries; }
	void* getLibrary(ISystem*) const override { return nullptr; }
	DelegateList<void(void*)>& libraryLoaded() override { return loaded; }
	Array<ISystem*> systems;
	Array<void*> libraries;
	DelegateList<void(void*)> loaded;
};

[[noreturn]] void notHere(const char* what) {
	fprintf(stderr, "[world shim] %s is not part of this harness\n", what);
	__builtin_trap();
}

struct StubEngine final : Engine {
	StubEngine() : page_allocator(allocator), systems(allocator) {}
	void init() override {}
	World& createWorld() override { notHere("createWorld"); }
	void destroyWorld(World&) override {}
	void setMainWindow(os::WindowHandle) override {}
	os::WindowHandle getMainWindow() override { return nullptr; }
	FileSystem& getFileSystem() override { notHere("FileSystem"); }
	InputSystem& getInputSystem() override { notHere("InputSystem"); }
	SystemManager& getSystemManager() override { return systems; }
	ResourceManagerHub& getResourceManager() override { notHere("ResourceManagerHub"); }
	PageAllocator& getPageAllocator() override { return page_allocator; }
	IAllocator& getAllocator() override { return allocator; }
	EntityPtr instantiatePrefab(World&, const PrefabResource&, const DVec3&, const Quat&, const Vec3&, EntityMap&) override { return INVALID_ENTITY; }
	void startGame(World&) override {}
	void stopGame(World&) override {}
	void update(World&) override {}
	DeserializeProjectResult deserializeProject(InputMemoryStream&, Path&) override { return DeserializeProjectResult::CORRUPTED_FILE; }
	void serializeProject(OutputMemoryStream&, const Path&) const override {}
	float getLastTimeDelta() const override { return 0; }
	void setTimeMultiplier(float) override {}
	void pause(bool) override {}
	bool isPaused() const override { return false; }
	void nextFrame() override {}
	bool decompress(Span<const u8>, Span<u8>) override { return false; }
	bool compress(Span<const u8>, OutputMemoryStream&) override { return false; }
	DefaultAllocator allocator;
	PageAllocator page_allocator;
	StubSystems systems;
};

const ComponentType MOVED_LISTENER = {7}; // any component type: the listener stands for RenderModule::onModelInstanceMoved & co.

struct Listener {
	uint32_t* calls = nullptr;
	void onMoved(EntityRef e) { ++calls[e.index]; }
};

struct Side {
	Side(StubEngine& engine, uint32_t n, uint32_t* calls) : world(engine) {
		listener.calls = calls;
		world.componentTransformed(MOVED_LISTENER).bind<&Listener::onMoved>(&listener);
		(void)n;
	}
	World world;
	Listener listener;
};

double now() {
	timespec ts;
	clock_gettime(CLOCK_MONOTONIC, &ts);
	return ts.tv_sec + ts.tv_nsec * 1e-9;
}

void build(World& w, const int32_t* parents, const Transform* locals, const Transform* globals_of_roots, uint32_t n, const uint8_t* listens) {
	for (uint32_t i = 0; i < n; ++i) {
		const EntityRef e = w.createEntity({0, 0, 0}, Quat::IDENTITY);
		if ((uint32_t)e.index != i) notHere("entity numbering other than creation order");
		if (listens[i]) w.onComponentCreated(e, MOVED_LISTENER, nullptr); // the entity's archetype now holds the type: transformEntity will fire it
	}
	for (uint32_t i = 0; i < n; ++i) {
		if (parents[i] < 0) w.setTransform(EntityRef{(i32)i}, globals_of_roots[i]);
	}
	for (uint32_t i = 0; i < n; ++i) { // parents come before their children in the input
		if (parents[i] < 0) continue;
		w.setParent(EntityPtr{parents[i]}, EntityRef{(i32)i});
		w.setLocalTransform(EntityRef{(i32)i}, locals[i]);
	}
}

} // namespace

// rounds x { move `n_moved` entities (roots or entities outside any hierarchy) to moved_values[round] }.
// out_* : n Transforms (56 B each) after the last round; calls_* : n counters of `transformed` invocations during the rounds;
// seconds[0] / [1]: host time of the rounds on the reference recursion / on the B200 path; out_locals_ref (optional): world A's local
// transforms at the end.  Returns 0, or a negative stage number.
SHIM_API int wshim_run(const int32_t* parents, const void* locals, const void* root_globals, uint32_t n, const uint8_t* listens,
	const uint32_t* moved, const void* moved_values, uint32_t n_moved, uint32_t rounds, int reparent_between_rounds,
	void* out_ref, void* out_b200, uint32_t* calls_ref, uint32_t* calls_b200, double* seconds, void* out_locals_ref)
{
	static_assert(sizeof(Transform) == 56);
	lb200_ctx* ctx = nullptr;
	if (lb200_init(0, &ctx) != LB200_OK) return -1;
	int rc = 0;
	{
		StubEngine engine;
		memset(calls_ref, 0, 4 * (size_t)n);
		memset(calls_b200, 0, 4 * (size_t)n);
		Side a(engine, n, calls_ref), b(engine, n, calls_b200);
		build(a.world, parents, (const Transform*)locals, (const Transform*)root_globals, n, listens);
		build(b.world, parents, (const Transform*)locals, (const Transform*)root_globals, n, listens);
		memset(calls_ref, 0, 4 * (size_t)n);
		memset(calls_b200, 0, 4 * (size_t)n);
		Array<EntityRef> ents(engine.allocator);
		for (uint32_t k = 0; k < n_moved; ++k) ents.push(EntityRef{(i32)moved[k]});
		seconds[0] = seconds[1] = 0;
		bool topology_changed = true;
		for (uint32_t r = 0; r < rounds && rc == 0; ++r) {
			const Transform* vals = (const Transform*)moved_values + (size_t)r * n_moved;
			double t0 = now();
			for (uint32_t k = 0; k < n_moved; ++k) a.world.setTransform(ents[k], vals[k]);
			seconds[0] += now() - t0;
			t0 = now();
			b.world.setTransformsDeferredB200(ents.begin(), vals, n_moved);
			if (!b.world.propagateHierarchyB200(ctx, topology_changed)) rc = -2;
			seconds[1] += now() - t0;
			topology_changed = false;
			if (reparent_between_rounds && r + 1 < rounds) {
				// World::setParent on both sides: the last entity that has a parent moves under entity 0 (world.cpp:619-701 recomputes its local
				// transform, may swap m_hierarchy slots) — the next propagate has to rebuild the device topology
				for (uint32_t i = n; i-- > 0;) {
					if (parents[i] <= 0) continue;
					a.world.setParent(EntityPtr{0}, EntityRef{(i32)i});
					b.world.setParent(EntityPtr{0}, EntityRef{(i32)i});
					break;
				}
				topology_changed = true;
			}
		}
		for (uint32_t i = 0; i < n; ++i) {
			((Transform*)out_ref)[i] = a.world.getTransform(EntityRef{(i32)i});
			((Transform*)out_b200)[i] = b.world.getTransform(EntityRef{(i32)i});
			// the local transforms as the reference World holds them: setLocalTransform -> updateGlobalTransform -> setTransform -> transformEntity(update_local)
			// recomputes them from the composed global (world.cpp:704-712, 267-270), so they are not bit for bit what the caller passed in
			if (out_locals_ref) ((Transform*)out_locals_ref)[i] = a.world.getLocalTransform(EntityRef{(i32)i});
		}
	}
	lb200_shutdown(ctx);
	return rc;
}
