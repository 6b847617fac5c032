// Host-side bookkeeping of the CullingSystem: the reference's cell grid / page chains / entity->slot map
// (src/renderer/culling_system.cpp:23-63, 98-258) kept in a struct-of-arrays form whose page arrays are
// byte-identical to what the GPU reads (DESIGN.md §3), plus dirty-page tracking for the HBM mirror.
//
// Pure C++ (no CUDA calls): allocation of the page arrays goes through two function pointers so the same
// code runs with pinned memory under a context and with malloc in the CPU-only tests.
#pragma once

#include "lb200_internal.h"

#include <stdlib.h>
#include <thread>
#include <unordered_map>
#include <vector>

namespace lb {

constexpr uint32_t PAGE_SLOTS = LB200_PAGE_SLOTS; // usable spheres per page: MAX_COUNT - 1 = 200, culling_system.cpp:61,103
constexpr uint32_t NO_SLOT = 0xffffffffu;
constexpr int32_t NO_PAGE = -1;

// CellIndices, culling_system.cpp:23-38
struct CellKey {
	int32_t x, y, z;
	uint8_t type;
	uint8_t is_big;
	bool operator==(const CellKey& r) const { return x == r.x && y == r.y && z == r.z && type == r.type && is_big == r.is_big; }
};

// CellIndicesHasher, culling_system.cpp:41-48 (type / is_big folded in: the reference leaves that as a TODO; only bucket spread differs)
struct CellKeyHasher {
	size_t operator()(const CellKey& k) const {
		return (uint32_t)k.x * 73856093u + (uint32_t)k.y * 19349663u + (uint32_t)k.z * 83492791u + (uint32_t)k.type * 2654435761u + k.is_big;
	}
};

struct CullingHost {
	typedef void* (*AllocFn)(size_t);
	typedef void (*FreeFn)(void*);

	CullingHost(AllocFn a, FreeFn f) : alloc_fn(a), free_fn(f) { memset(type_counts, 0, sizeof(type_counts)); }
	~CullingHost() {
		free_fn(spheres); free_fn(entities); free_fn(desc);
	}

	// ---- page arrays (index = page id; the GPU mirror uses the same ids) ----
	float* spheres = nullptr;        // cap * 200 * {x,y,z,radius}
	int32_t* entities = nullptr;     // cap * 200
	lb200_page_desc* desc = nullptr; // cap
	std::vector<int32_t> next, prev; // CellPage::header.next / prev as page ids
	std::vector<CellKey> keys;       // CellPage::header.indices
	std::vector<uint32_t> cell_pos;  // position of the page inside `cells`
	uint32_t cap = 0;
	uint32_t high_water = 0;         // pages [0, high_water) have been handed out at least once
	std::vector<uint32_t> free_pages;

	std::vector<uint32_t> cells;     // m_cells (culling_system.cpp:381): one entry per live page, same order as the reference
	std::unordered_map<CellKey, uint32_t, CellKeyHasher> cell_map; // m_cell_map: key -> head page of the chain
	std::vector<uint32_t> entity_to_slot; // m_entity_to_cell: page*200 + index, NO_SLOT = not added
	uint32_t type_counts[256];
	uint32_t n_entities = 0;
	uint32_t n_bad_radius = 0; // spheres with radius < 0 or NaN: the GPU's plane masking assumes radius >= 0 and is switched off while any exist

	static bool badRadius(float r) { return !(r >= 0.0f); }

	// ---- dirty tracking for the HBM mirror ----
	std::vector<uint8_t> dirty_flag;
	std::vector<uint32_t> dirty_list;
	bool all_dirty = false;

	AllocFn alloc_fn;
	FreeFn free_fn;

	uint64_t edit_gen = 0; // bumped by every edit: the device-side re-binning tables (culling_rebin.cu) are rebuilt when it moved

	void markDirty(uint32_t page) {
		++edit_gen;
		if (!dirty_flag[page]) { dirty_flag[page] = 1; dirty_list.push_back(page); }
	}

	void clearDirty() {
		for (uint32_t p : dirty_list) dirty_flag[p] = 0;
		dirty_list.clear();
		all_dirty = false;
	}

	bool grow(uint32_t min_cap) {
		uint32_t new_cap = cap ? cap : 64;
		while (new_cap < min_cap) new_cap *= 2;
		float* s = (float*)alloc_fn(sizeof(float) * 4 * PAGE_SLOTS * (size_t)new_cap);
		int32_t* e = (int32_t*)alloc_fn(sizeof(int32_t) * PAGE_SLOTS * (size_t)new_cap);
		lb200_page_desc* d = (lb200_page_desc*)alloc_fn(sizeof(lb200_page_desc) * (size_t)new_cap);
		if (!s || !e || !d) return false;
		if (cap) {
			memcpy(s, spheres, sizeof(float) * 4 * PAGE_SLOTS * (size_t)cap);
			memcpy(e, entities, sizeof(int32_t) * PAGE_SLOTS * (size_t)cap);
			memcpy(d, desc, sizeof(lb200_page_desc) * (size_t)cap);
		}
		memset(d + cap, 0, sizeof(lb200_page_desc) * (size_t)(new_cap - cap));
		free_fn(spheres); free_fn(entities); free_fn(desc);
		spheres = s; entities = e; desc = d;
		next.resize(new_cap, NO_PAGE); prev.resize(new_cap, NO_PAGE);
		keys.resize(new_cap); cell_pos.resize(new_cap, 0); dirty_flag.resize(new_cap, 0);
		cap = new_cap;
		return true;
	}

	// m_page_allocator.allocate() + placement new CellPage, culling_system.cpp:111-112,143-144
	int32_t allocPage() {
		uint32_t p;
		if (!free_pages.empty()) { p = free_pages.back(); free_pages.pop_back(); }
		else {
			if (high_water == cap && !grow(cap + 1)) return NO_PAGE;
			p = high_water++;
		}
		memset(&desc[p], 0, sizeof(desc[p]));
		next[p] = prev[p] = NO_PAGE;
		return (int32_t)p;
	}

	void cellsPush(uint32_t p) { cell_pos[p] = (uint32_t)cells.size(); cells.push_back(p); }

	// Array::swapAndPopItem, culling_system.cpp:174
	void cellsSwapAndPop(uint32_t p) {
		const uint32_t i = cell_pos[p];
		const uint32_t last = cells.back();
		cells[i] = last;
		cell_pos[last] = i;
		cells.pop_back();
	}

	static CellKey makeKey(const double pos[3], uint8_t type, bool is_big) {
		// culling_system.cpp:25-31: IVec3(pos * (1 / cell_size)) — DVec3*float (math.cpp:496), int(double) truncates toward zero (math.cpp:133-138)
		const float inv = 1 / LB200_CELL_SIZE;
		CellKey k;
		k.x = int(pos[0] * inv);
		k.y = int(pos[1] * inv);
		k.z = int(pos[2] * inv);
		k.type = type;
		k.is_big = is_big ? 1 : 0;
		return k;
	}

	void writeSlot(uint32_t page, uint32_t idx, int32_t entity, const double pos[3], float radius) {
		// culling_system.cpp:100: Vec3(pos - cell.header.origin)
		const lb200_page_desc& d = desc[page];
		float* s = spheres + 4 * ((size_t)page * PAGE_SLOTS + idx);
		s[0] = (float)(pos[0] - d.origin[0]);
		s[1] = (float)(pos[1] - d.origin[1]);
		s[2] = (float)(pos[2] - d.origin[2]);
		s[3] = radius;
		if (badRadius(radius)) ++n_bad_radius;
		entities[(size_t)page * PAGE_SLOTS + idx] = entity;
	}

	// culling_system.cpp:98-128 addToCell; returns slot or NO_SLOT on allocation failure
	uint32_t addToCell(uint32_t cell, int32_t entity, const double pos[3], float radius) {
		const uint32_t count = desc[cell].count;
		if (count < PAGE_SLOTS) { // count < MAX_COUNT - 1
			writeSlot(cell, count, entity, pos, radius);
			++desc[cell].count;
			markDirty(cell);
			return cell * PAGE_SLOTS + count;
		}
		const int32_t np = allocPage();
		if (np < 0) return NO_SLOT;
		const uint32_t n = (uint32_t)np;
		memcpy(desc[n].origin, desc[cell].origin, sizeof(desc[n].origin));
		desc[n].type = desc[cell].type;
		desc[n].is_big = desc[cell].is_big;
		keys[n] = keys[cell];
		next[n] = (int32_t)cell;
		prev[n] = prev[cell];
		prev[cell] = (int32_t)n;
		if (prev[n] != NO_PAGE) next[prev[n]] = (int32_t)n;
		cellsPush(n);
		if (prev[n] == NO_PAGE) cell_map[keys[n]] = n;
		writeSlot(n, 0, entity, pos, radius);
		desc[n].count = 1;
		markDirty(n);
		return n * PAGE_SLOTS;
	}

	// culling_system.cpp:131-157
	int add(int32_t entity, uint8_t type, const double pos[3], float radius) {
		if (entity < 0) return LB200_ERR_INVALID;
		if (entity_to_slot.size() <= (size_t)entity) entity_to_slot.resize((size_t)entity + 1, NO_SLOT);
		const CellKey key = makeKey(pos, type, radius > LB200_CELL_SIZE);
		auto iter = cell_map.find(key);
		if (iter == cell_map.end()) {
			const int32_t np = allocPage();
			if (np < 0) return LB200_ERR_CUDA;
			const uint32_t n = (uint32_t)np;
			// :146 i.pos * double(m_cell_size) (math.cpp:149-152: {i * x, i * y, i * z})
			const double cs = double(LB200_CELL_SIZE);
			desc[n].origin[0] = cs * key.x;
			desc[n].origin[1] = cs * key.y;
			desc[n].origin[2] = cs * key.z;
			desc[n].type = type;
			desc[n].is_big = key.is_big;
			keys[n] = key;
			iter = cell_map.emplace(key, n).first;
			cellsPush(n);
		}
		const uint32_t slot = addToCell(iter->second, entity, pos, radius);
		if (slot == NO_SLOT) return LB200_ERR_CUDA;
		entity_to_slot[entity] = slot;
		++type_counts[type];
		++n_entities;
		return LB200_OK;
	}

	// culling_system.cpp:160-187
	int remove(int32_t entity) {
		if (entity < 0 || entity_to_slot.size() <= (size_t)entity) return LB200_OK;
		const uint32_t slot = entity_to_slot[entity];
		if (slot == NO_SLOT) return LB200_OK;
		const uint32_t cell = slot / PAGE_SLOTS;
		--type_counts[desc[cell].type];
		--n_entities;
		if (badRadius(spheres[4 * (size_t)slot + 3])) --n_bad_radius;
		if (desc[cell].count == 1) {
			if (prev[cell] == NO_PAGE) {
				if (next[cell] == NO_PAGE) cell_map.erase(keys[cell]);
				else cell_map[keys[cell]] = (uint32_t)next[cell];
			}
			if (prev[cell] != NO_PAGE) next[prev[cell]] = next[cell];
			if (next[cell] != NO_PAGE) prev[next[cell]] = prev[cell];
			cellsSwapAndPop(cell);
			desc[cell].count = 0; // the GPU skips empty pages
			markDirty(cell);
			free_pages.push_back(cell);
		}
		else {
			const uint32_t idx = slot % PAGE_SLOTS;
			const uint32_t last_idx = desc[cell].count - 1;
			const size_t base = (size_t)cell * PAGE_SLOTS;
			const int32_t last = entities[base + last_idx];
			entities[base + idx] = last;
			memcpy(spheres + 4 * (base + idx), spheres + 4 * (base + last_idx), sizeof(float) * 4);
			entity_to_slot[last] = cell * PAGE_SLOTS + idx;
			--desc[cell].count;
			markDirty(cell);
		}
		entity_to_slot[entity] = NO_SLOT;
		return LB200_OK;
	}

	bool isAdded(int32_t entity) const { // culling_system.cpp:372-375
		return entity >= 0 && (size_t)entity < entity_to_slot.size() && entity_to_slot[entity] != NO_SLOT;
	}

	float getRadius(int32_t entity) const { return spheres[4 * (size_t)entity_to_slot[entity] + 3]; } // :217-220

	static bool sameCell(const CellKey& a, const CellKey& b) { return a.x == b.x && a.y == b.y && a.z == b.z; }

	// culling_system.cpp:198-214
	int setPosition(int32_t entity, const double pos[3]) {
		if (!isAdded(entity)) return LB200_ERR_INVALID;
		const uint32_t slot = entity_to_slot[entity];
		const uint32_t cell = slot / PAGE_SLOTS;
		const CellKey nk = makeKey(pos, 0, false);
		if (sameCell(nk, keys[cell])) {
			float* s = spheres + 4 * (size_t)slot;
			s[0] = (float)(pos[0] - desc[cell].origin[0]);
			s[1] = (float)(pos[1] - desc[cell].origin[1]);
			s[2] = (float)(pos[2] - desc[cell].origin[2]);
			markDirty(cell);
			return LB200_OK;
		}
		const float radius = spheres[4 * (size_t)slot + 3];
		const uint8_t type = desc[cell].type;
		remove(entity);
		return add(entity, type, pos, radius);
	}

	// culling_system.cpp:222-240
	int set(int32_t entity, const double pos[3], float radius) {
		if (!isAdded(entity)) return LB200_ERR_INVALID;
		const uint32_t slot = entity_to_slot[entity];
		const uint32_t cell = slot / PAGE_SLOTS;
		const CellKey nk = makeKey(pos, 0, false);
		const bool was_big = desc[cell].is_big != 0;
		const bool is_big = radius > LB200_CELL_SIZE;
		if (was_big == is_big && sameCell(nk, keys[cell])) {
			float* s = spheres + 4 * (size_t)slot;
			n_bad_radius += (badRadius(radius) ? 1 : 0) - (badRadius(s[3]) ? 1 : 0);
			s[3] = radius;
			s[0] = (float)(pos[0] - desc[cell].origin[0]);
			s[1] = (float)(pos[1] - desc[cell].origin[1]);
			s[2] = (float)(pos[2] - desc[cell].origin[2]);
			markDirty(cell);
			return LB200_OK;
		}
		const uint8_t type = desc[cell].type;
		remove(entity);
		return add(entity, type, pos, radius);
	}

	// Batch form of set() for DISTINCT entities (the sphere refresh after a hierarchy propagate, render_module.cpp:1544-1554, touches every
	// moved entity once).  Most movers stay inside their cell and on the same side of the is_big threshold: those are plain overwrites of
	// their own slot, independent of each other, and run on all host cores; the rest — cell or chain changes, which rewire pages — then
	// run one by one in their original order through set().  In-cell overwrites do not touch the page structure and carry their data
	// along when a later swap-with-last moves them, so the final state is the one the sequential loop produces (tests/test_culling_host.py).
	int setManyUnique(const int32_t* ents, const double* pos3, const float* radius, uint32_t n) {
		for (uint32_t i = 0; i < n; ++i) if (!isAdded(ents[i])) return LB200_ERR_INVALID;
		unsigned workers = std::thread::hardware_concurrency();
		workers = workers > 32 ? 32 : (workers < 1 ? 1 : workers);
		if (n < 32768) workers = 1;
		std::vector<std::vector<uint32_t>> dirty(workers), slow(workers);
		std::vector<long long> bad_delta(workers, 0);
		auto run = [&](unsigned w) {
			const uint32_t begin = (uint32_t)((uint64_t)n * w / workers), end = (uint32_t)((uint64_t)n * (w + 1) / workers);
			for (uint32_t i = begin; i < end; ++i) {
				const uint32_t slot = entity_to_slot[ents[i]];
				const uint32_t cell = slot / PAGE_SLOTS;
				const double* pos = pos3 + 3 * (size_t)i;
				const CellKey nk = makeKey(pos, 0, false);
				const bool was_big = desc[cell].is_big != 0;
				const bool is_big = radius[i] > LB200_CELL_SIZE;
				if (was_big != is_big || !sameCell(nk, keys[cell])) { slow[w].push_back(i); continue; }
				float* s = spheres + 4 * (size_t)slot;
				bad_delta[w] += (badRadius(radius[i]) ? 1 : 0) - (badRadius(s[3]) ? 1 : 0);
				s[3] = radius[i];
				s[0] = (float)(pos[0] - desc[cell].origin[0]);
				s[1] = (float)(pos[1] - desc[cell].origin[1]);
				s[2] = (float)(pos[2] - desc[cell].origin[2]);
				// read first: once a page is flagged its line stays shared between the cores instead of bouncing on every mover
				if (!__atomic_load_n(&dirty_flag[cell], __ATOMIC_RELAXED) && !__atomic_exchange_n(&dirty_flag[cell], (uint8_t)1, __ATOMIC_RELAXED)) dirty[w].push_back(cell);
			}
		};
		if (workers == 1) run(0);
		else {
			std::vector<std::thread> pool;
			for (unsigned w = 1; w < workers; ++w) pool.emplace_back(run, w);
			run(0);
			for (std::thread& t : pool) t.join();
		}
		++edit_gen;
		for (unsigned w = 0; w < workers; ++w) {
			dirty_list.insert(dirty_list.end(), dirty[w].begin(), dirty[w].end());
			n_bad_radius = (uint32_t)((long long)n_bad_radius + bad_delta[w]);
		}
		for (unsigned w = 0; w < workers; ++w) {
			for (uint32_t i : slow[w]) {
				const int rc = set(ents[i], pos3 + 3 * (size_t)i, radius[i]);
				if (rc) return rc;
			}
		}
		return LB200_OK;
	}

	// culling_system.cpp:242-258
	int setRadius(int32_t entity, float radius) {
		if (!isAdded(entity)) return LB200_ERR_INVALID;
		const uint32_t slot = entity_to_slot[entity];
		const uint32_t cell = slot / PAGE_SLOTS;
		const bool was_big = desc[cell].is_big != 0;
		const bool is_big = radius > LB200_CELL_SIZE;
		float* s = spheres + 4 * (size_t)slot;
		if (was_big == is_big) {
			n_bad_radius += (badRadius(radius) ? 1 : 0) - (badRadius(s[3]) ? 1 : 0);
			s[3] = radius;
			markDirty(cell);
			return LB200_OK;
		}
		const uint8_t type = desc[cell].type;
		// :254 cell.header.origin + sphere->position (DVec3 + Vec3, math.cpp:512)
		const double pos[3] = {desc[cell].origin[0] + s[0], desc[cell].origin[1] + s[1], desc[cell].origin[2] + s[2]};
		remove(entity);
		return add(entity, type, pos, radius);
	}
};

} // namespace lb
