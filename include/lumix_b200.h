/* lumix_b200.h — C-ABI of the H100-native LumixEngine hot path (cull / hierarchy propagate / pose + skin palette).
 *
 * Plain C: pointers and sizes only, no C++/torch types.  Every entry point returns LB200_OK (0) or a negative
 * lb200_status; lb200_last_error() gives the text.  There is no CPU fallback: without a CUDA device every compute
 * entry point fails with LB200_ERR_NO_DEVICE.
 *
 * Each block cites the reference interface it replaces (paths relative to the LumixEngine tree).
 * INTEGRATION.md shows the engine-side C++ that binds these (CullingSystem::create body, World, AnimationModule).
 */
#ifndef LUMIX_B200_H
#define LUMIX_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define LB200_API __attribute__((visibility("default")))

typedef enum {
	LB200_OK = 0,
	LB200_ERR_NO_DEVICE = -1,   /* no CUDA device / driver: the product has no CPU path */
	LB200_ERR_CUDA = -2,        /* a CUDA runtime call failed; see lb200_last_error */
	LB200_ERR_INVALID = -3,     /* bad argument (null pointer, type == 0xff where reserved, index out of range) */
	LB200_ERR_CAPACITY = -4,    /* caller-provided output buffer too small */
	LB200_ERR_NCCL = -5,        /* NCCL not loadable or a collective failed */
	LB200_ERR_STATE = -6        /* call order violated (e.g. cull before any page was uploaded) */
} lb200_status;

typedef struct lb200_ctx lb200_ctx;

/* ------------------------------------------------------------------------------------------------------------
 * Context = one GPU, one stream.  Replaces nothing in the reference (it has no device); owned by the ISystem
 * the plugin entry creates (src/engine/plugin.h:64-96).
 * ---------------------------------------------------------------------------------------------------------- */
LB200_API int lb200_init(int device_ordinal, lb200_ctx** out_ctx);
/* A further context of the device whose stream has the lowest priority: its kernels fill the SMs only where the other contexts' streams
 * (which get the highest priority) leave room — e.g. the animation update next to the culling / exchange of the same frame. */
LB200_API int lb200_init_background(int device_ordinal, lb200_ctx** out_ctx);
LB200_API void lb200_shutdown(lb200_ctx* ctx);
LB200_API const char* lb200_last_error(const lb200_ctx* ctx); /* ctx may be NULL: last init error */
LB200_API int lb200_device_count(void);
LB200_API int lb200_synchronize(lb200_ctx* ctx);
/* Calls fn(user) from a driver thread once everything enqueued on the context stream so far has finished (cudaLaunchHostFunc).  For callers
 * that must not block their thread — the engine calls cull from job-system fibers (pipeline.cpp:1036-1041): fn schedules a job that turns a
 * jobs::Signal green and the fiber parks on that signal meanwhile.  fn must not call into this library. */
LB200_API int lb200_host_callback(lb200_ctx* ctx, void (*fn)(void*), void* user);
/* Kernels this library launched on ctx since init (bench.py's gpu_launches). */
LB200_API uint64_t lb200_launch_count(const lb200_ctx* ctx);
/* cudaStream_t of the context as an integer (for CUDA-event timing on the launching stream). */
LB200_API uint64_t lb200_stream_handle(const lb200_ctx* ctx);
/* Page-locked host memory for result buffers (the engine would pass memory from its own allocators, registered once). */
LB200_API void* lb200_host_alloc(lb200_ctx* ctx, size_t bytes);
LB200_API void lb200_host_free(lb200_ctx* ctx, void* p);
/* Copy `bytes` from a device pointer handed out by this library (e.g. *out_dev_ids) to host memory, ordered after the context stream. */
/* Device buffers for the entry points that take device pointers (lb200_culling_set_many_device, lb200_sortkeys_set_transforms_device). */
LB200_API void* lb200_device_alloc(lb200_ctx* ctx, size_t bytes);
LB200_API void lb200_device_free(lb200_ctx* ctx, void* device_ptr);
LB200_API int lb200_copy_to_device(lb200_ctx* ctx, void* dst_device, const void* src_host, size_t bytes);
LB200_API int lb200_copy_to_host(lb200_ctx* ctx, void* dst_host, const void* src_device, size_t bytes);
/* Device-time helpers: record a timestamp on the context stream / milliseconds between two of them (CUDA events). */
LB200_API int lb200_event_create(lb200_ctx* ctx, void** out_event);
LB200_API int lb200_event_record(lb200_ctx* ctx, void* event);
LB200_API int lb200_event_elapsed_ms(lb200_ctx* ctx, void* start, void* stop, float* out_ms);
LB200_API void lb200_event_destroy(lb200_ctx* ctx, void* event);

/* ------------------------------------------------------------------------------------------------------------
 * POD images of reference structs that cross the boundary (layouts verified against the reference build,
 * SURVEY.md §8a).
 * ---------------------------------------------------------------------------------------------------------- */
/* ShiftedFrustum, src/core/geometry.h:99-149 — 256 bytes: xs[8] ys[8] zs[8] ds[8] (planes NEAR,FAR,LEFT,RIGHT,TOP,
 * BOTTOM,EXTRA0,EXTRA1), Vec3 points[8], DVec3 origin at +224.  Built on the host by the engine's own
 * ShiftedFrustum::computePerspective/computeOrtho (geometry.cpp:390-409,470-499) or by lb200_frustum_* below. */
typedef struct {
	float xs[8], ys[8], zs[8], ds[8];
	float points[8][3];
	double origin[3];
	uint64_t pad_; /* the reference struct is alignas(16): sizeof == 256 */
} lb200_shifted_frustum;

/* Transform, src/core/math.h:306-327 — 56 bytes: DVec3 pos, Quat rot (xyzw), Vec3 scale. */
typedef struct {
	double pos[3];
	float rot[4];
	float scale[3];
} lb200_transform;

/* Host-side frustum construction, same arithmetic as geometry.cpp:390-409,470-499 (viewport {-1,-1}..{1,1}). */
LB200_API void lb200_frustum_perspective(lb200_shifted_frustum* out, const double position[3], const float direction[3], const float up[3],
	float fov, float ratio, float near_distance, float far_distance);
LB200_API void lb200_frustum_ortho(lb200_shifted_frustum* out, const double position[3], const float direction[3], const float up[3],
	float width, float height, float near_distance, float far_distance);
/* Viewport::getFrustum() (src/core/geometry.cpp:793-818): camera position + rotation quaternion (xyzw), vertical fov or ortho size,
 * viewport size in pixels (ratio = h > 0 ? w / (float)h : 1). */
LB200_API void lb200_frustum_from_viewport(lb200_shifted_frustum* out, int is_ortho, float fov, float ortho_size, int w, int h,
                                           const double pos[3], const float rot[4], float near_distance, float far_distance);

/* ------------------------------------------------------------------------------------------------------------
 * CullingSystem — replaces struct CullingSystem, src/renderer/culling_system.h:58-77 (one C function per virtual,
 * same argument meaning), implementation src/renderer/culling_system.cpp:67-403.
 *
 * The host keeps the reference's bookkeeping (300 m cell grid, pages of <=200 spheres, entity->slot map,
 * culling_system.cpp:98-258) and mirrors dirty pages to HBM before the next cull; cull itself runs on the GPU.
 * entity = EntityRef::index (src/engine/lumix.h:10-44).  type = RenderableTypes value (render_module.h:293-301);
 * 0xff is reserved for "all types" exactly as culling_system.cpp:310-319.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct lb200_culling lb200_culling;

#define LB200_TYPE_ALL 0xff
#define LB200_PAGE_SLOTS 200u   /* CellPage::MAX_COUNT - 1, culling_system.cpp:61,103 */
#define LB200_CELL_SIZE 300.0f  /* culling_system.cpp:75 */

/* CullingSystem::create, culling_system.cpp:399-402 */
LB200_API int lb200_culling_create(lb200_ctx* ctx, lb200_culling** out);
LB200_API void lb200_culling_destroy(lb200_culling* cs);
/* culling_system.cpp:131-157 / 160-187 / 198-214 / 242-258 / 222-240 / 217-220 / 372-375 */
LB200_API int lb200_culling_add(lb200_culling* cs, int32_t entity, uint8_t type, const double pos[3], float radius);
LB200_API int lb200_culling_remove(lb200_culling* cs, int32_t entity);
LB200_API int lb200_culling_set_position(lb200_culling* cs, int32_t entity, const double pos[3]);
LB200_API int lb200_culling_set_radius(lb200_culling* cs, int32_t entity, float radius);
LB200_API int lb200_culling_set(lb200_culling* cs, int32_t entity, const double pos[3], float radius);
LB200_API float lb200_culling_get_radius(const lb200_culling* cs, int32_t entity);
LB200_API int lb200_culling_is_added(const lb200_culling* cs, int32_t entity);
/* batch forms of the same calls (one FFI crossing for n entities) */
LB200_API int lb200_culling_add_many(lb200_culling* cs, const int32_t* entities, const uint8_t* types, const double* pos3, const float* radius, uint32_t n);
LB200_API int lb200_culling_set_many(lb200_culling* cs, const int32_t* entities, const double* pos3, const float* radius, uint32_t n);
/* set() for n DISTINCT entities, e.g. the sphere refresh after a hierarchy propagate (render_module.cpp:1544-1554): movers that stay in
 * their cell are overwritten in place on all host cores, the others go through set() one by one in the given order.  Same final state
 * as lb200_culling_set_many; an entity listed twice is undefined behaviour here. */
LB200_API int lb200_culling_set_many_unique(lb200_culling* cs, const int32_t* entities, const double* pos3, const float* radius, uint32_t n);
LB200_API int lb200_culling_set_position_many(lb200_culling* cs, const int32_t* entities, const double* pos3, uint32_t n);
LB200_API int lb200_culling_set_radius_many(lb200_culling* cs, const int32_t* entities, const float* radius, uint32_t n);
LB200_API int lb200_culling_remove_many(lb200_culling* cs, const int32_t* entities, uint32_t n);

/* Bookkeeping introspection (tests compare it with the reference's m_cells state). */
LB200_API uint32_t lb200_culling_page_count(const lb200_culling* cs);
LB200_API uint32_t lb200_culling_entity_count(const lb200_culling* cs);
LB200_API int lb200_culling_get_page(const lb200_culling* cs, uint32_t page, double origin[3], int32_t indices[3], uint8_t* type, uint8_t* is_big,
	uint32_t* count, float* spheres4 /* count*4 or NULL */, int32_t* entities /* count or NULL */);
/* Device page id (row index of the page in the HBM arrays and in the visibility bitmask) of the page-th entry of m_cells; -1 if out of range. */
LB200_API int32_t lb200_culling_page_id(const lb200_culling* cs, uint32_t page);

/* Result of one cull: visible entity ids grouped by renderable type.  ids[type_offset[t] .. type_offset[t]+type_count[t])
 * are the visible entities of type t (order inside a type is unspecified, as in the reference: SURVEY.md F4).
 * This is the flat form of the CullResult page chain (culling_system.h:17-56): one chain page = <=1020 ids of one type. */
typedef struct {
	uint32_t total;            /* sum of type_count */
	uint32_t n_types;          /* highest type with entities + 1 */
	uint32_t type_count[256];
	uint32_t type_offset[256];
	/* counters of the last cull (pages by classification, culling_system.cpp:342-363) */
	uint32_t pages_tested, pages_inside, pages_outside, pages_filtered;
	uint32_t entities_tested, entities_inside;
} lb200_cull_result;

/* CullingSystem::cull(frustum, type) / cull(frustum), culling_system.cpp:310-369.
 * Uploads dirty pages + the frustum, runs the cull kernel, delivers the visible ids in `out_ids` (host, capacity in ids) packed
 * type after type (result->type_offset).  A page-locked destination (lb200_host_alloc, cudaHostAlloc, cudaHostRegister) is written
 * by the device itself right behind the cull — one synchronisation, no count round trip, copy engine idle; pageable memory takes
 * cudaMemcpyAsync per type.  type == LB200_TYPE_ALL culls every type.  Returns LB200_ERR_CAPACITY if `capacity` < visible count
 * (result->total still holds the needed size; the content of out_ids is then unspecified).  With zero pages: total = 0 (the reference
 * returns nullptr, culling_system.cpp:322). */
LB200_API int lb200_culling_cull(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t* out_ids, uint32_t capacity,
	lb200_cull_result* result);

/* The same delivery without blocking the calling thread — the engine calls cull from job-system fibers, possibly for several views
 * (src/renderer/pipeline.cpp:1036-1041), and a fiber must not sit in an OS wait (docs/job_system.md):
 *   lb200_culling_cull_begin  uploads pending edits, enqueues the cull and the device-side write of ids + counts into `out_ids`
 *                             (page-locked memory only: lb200_host_alloc) and returns at once;
 *   lb200_culling_cull_poll   1 = finished, 0 = still running (jobs::yield() and ask again), < 0 = error;
 *   lb200_culling_cull_end    waits if it still has to, fills `result` like lb200_culling_cull (LB200_ERR_CAPACITY as there).
 * One begin may be outstanding per culling system. */
LB200_API int lb200_culling_cull_begin(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t* out_ids, uint32_t capacity);
LB200_API int lb200_culling_cull_poll(lb200_culling* cs);
LB200_API int lb200_culling_cull_end(lb200_culling* cs, lb200_cull_result* result);

/* Device-resident form: the same cull, result left in HBM (no D2H of ids).  *out_dev_ids receives the device pointer of the
 * id buffer: per-type segments, ids of type t at [type_offset[t], type_offset[t] + type_count[t]).  The buffer belongs to one of the
 * object's output lanes (2 by default, LB200_CULL_LANES): it stays valid through the next lanes - 1 culls, the cull after that reuses
 * it.  Counts land in `result` (a 2 KB D2H).  With want_counts = 0 nothing is
 * read back and the call is fully asynchronous on the context stream (result may be NULL). */
LB200_API int lb200_culling_cull_device(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, const uint32_t** out_dev_ids,
	lb200_cull_result* result, int want_counts);
/* n asynchronous culls issued from one call (a frame culls several views — main, shadow cascades, lights, pipeline.cpp:996-1063,3380,
 * which the engine runs concurrently from jobs — and a benchmark wants device time without per-call host overhead).  Consecutive culls
 * are independent: they go to different internal streams and output lanes, so the device overlaps them; the call forks from and joins
 * back into the context stream.  Results of the last one stay in HBM: lb200_culling_last_result / lb200_culling_read_bitmask. */
LB200_API int lb200_culling_cull_device_n(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t n);
/* Device id list (per-type segments) and counts of the cull issued last, whichever entry point issued it.  Synchronises the stream. */
LB200_API int lb200_culling_last_result(lb200_culling* cs, const uint32_t** out_dev_ids, lb200_cull_result* result);
/* Push pending page edits to HBM now (otherwise done lazily by the next cull). */
LB200_API int lb200_culling_flush(lb200_culling* cs);
/* Visibility bitmask of the last cull: bit (page*256 + slot); 8 words per page.  Copies page_count*8 words. */
LB200_API int lb200_culling_read_bitmask(lb200_culling* cs, uint32_t* out_words, uint32_t capacity_words);
/* Bench support: keep `replicas` identical copies of the page arrays in HBM and rotate through them on successive culls so that
 * back-to-back timed culls never re-read an L2-resident scene (B200_PROFILING.md "Timing hygiene"). */
LB200_API int lb200_culling_set_replicas(lb200_culling* cs, uint32_t replicas);
/* Algorithmic HBM bytes of the last cull (DESIGN.md §4): page descriptors + 16 B per tested sphere + 4 B per id read + 4 B per id written + mask. */
/* Device-side re-binning (SURVEY.md 8f N3): CullingSystem::set (culling_system.cpp:222-240) for n DISTINCT entities whose new world spheres lie
 * in device memory — the sphere refresh behind a hierarchy propagate (render_module.cpp:1544-1554; lb200_hierarchy_refresh_spheres) — without
 * the host's cell map in the loop: in-cell movers are overwritten in place, cell / big-ness changers leave their pages (tombstone + per-page
 * compaction, empty pages to a free list) and are re-inserted sorted by target chain (open page first, new pages from the free list).
 * dev_entities: n entity ids in device memory, or NULL for the identity (mover i = entity i); max_entity: largest entity id that can appear.
 * The host mirror is refreshed lazily: the next host-side accessor / mutator (add, remove, set*, get_page, ...) pulls the device state back
 * first (or call lb200_culling_sync_host).  Visible sets of later culls are the reference's; slots / pages inside a chain may differ from
 * a sequential replay of the same edits (as they do between two edit orders).  Needs set_replicas(1).
 * Cell range: the device keys a chain by 18 bits per cell axis, so it holds cells [-131072, 131071] on every axis (about +-39 321 km).  A
 * batch that computes a cell outside that range, and every device edit while the host holds such a chain, is applied by the host
 * bookkeeping instead (device state pulled back, batch copied to the host): same results, host speed.  The same holds for
 * lb200_culling_add_many_device and lb200_culling_remove_many_device.  lb200_culling_last_rebin_changers: the movers of the last
 * batch whose cell or big-ness changed. */
LB200_API int lb200_culling_set_many_device(lb200_culling* cs, const int32_t* dev_entities, const double* dev_pos3, const float* dev_radius, uint32_t n, uint32_t max_entity);
LB200_API int lb200_culling_sync_host(lb200_culling* cs);
LB200_API uint32_t lb200_culling_last_rebin_changers(const lb200_culling* cs);
/* CullingSystem::add (culling_system.cpp:131-157) for n entities whose spheres and types lie in device memory (spawn lists built on the
 * device).  dev_entities NULL = identity.  Every id must be in [0, max_entity], not added yet, listed once, and have a type other than
 * LB200_TYPE_ALL; otherwise the call returns LB200_ERR_INVALID and changes nothing.  Like lb200_culling_set_many_device the device stays
 * authoritative (the host mirror follows lazily), two synchronisations per call, and slots / pages may differ from a sequential replay
 * while visible sets do not.  Needs set_replicas(1). */
LB200_API int lb200_culling_add_many_device(lb200_culling* cs, const int32_t* dev_entities, const uint8_t* dev_types, const double* dev_pos3,
                                            const float* dev_radius, uint32_t n, uint32_t max_entity);
/* CullingSystem::remove (culling_system.cpp:160-187) for n entity ids in device memory.  Ids that are not added are skipped, as in the
 * reference; an id listed twice is removed once.  One synchronisation per call.  Needs set_replicas(1). */
LB200_API int lb200_culling_remove_many_device(lb200_culling* cs, const int32_t* dev_entities, uint32_t n);
/* Measurement helper: device time (ms) of `iters` single culls, each with the device to itself and its launch already queued when the
 * device reaches it (no host launch latency inside the interval, nothing overlapping the cull).  mode 0 = the cull, 1 = nothing between
 * the two event records, 2 = one empty kernel of the cull's grid (the fixed costs the first number contains). */
LB200_API int lb200_culling_time_lone_cull(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t iters, int mode, float* out_ms);
LB200_API uint64_t lb200_culling_last_algorithmic_bytes(const lb200_culling* cs);
/* Launch shape of later culls of this object, every entry point (cull, begin / end, cull_device[_n], cull_gather, cull_exchange[_n]).
 * blocks: 0 = the default rule (every co-resident block, LB200_CULL_BLOCKS_PER_SM per SM on the internal lanes, at most one block per
 * chunk of pages), -1 = every block that is co-resident when the cull has the device to itself (on the lanes too), 1..LB200_CULL_MAX_BLOCKS
 * = exactly that many, whatever fits and whatever the work (the cap keeps the kernel's 32-bit page index from overflowing).  chunk: pages per block per round, 0 = the default (ceil(pages / blocks) within
 * 32..256), 1..256 = exactly that many.  plane_masking: -1 = automatic (on unless some radius is negative or NaN), 0 = off.  Any other
 * value is LB200_ERR_INVALID.  The visible sets, statistics and mask rows do not depend on the shape.  get_launch reports the last cull:
 * blocks, chunk, rounds = ceil(pages / (blocks x chunk)), whether it was launched with programmatic dependent launch (no upload since the
 * cull before it) and whether plane masking was on (all 0 before the first cull; for a batch, its last cull). */
#define LB200_CULL_MAX_BLOCKS (1 << 20)
LB200_API int lb200_culling_set_launch(lb200_culling* cs, int blocks, int chunk, int plane_masking);
LB200_API int lb200_culling_get_launch(lb200_culling* cs, uint32_t* blocks, uint32_t* chunk, uint32_t* rounds, int* pdl, int* plane_masking);

/* Several views of one frame in one pass over the pages (the main camera and the shadow cascades, pipeline.cpp:734-827,1254-1258).
 * n_views culls of the same scene (1 <= n_views <= LB200_CULL_MAX_VIEWS): view v = frusta[v] with type filter types[v] (types may be
 * NULL = LB200_TYPE_ALL for every view).  Each view's visible set per type, statistics and mask rows equal those of a lone
 * lb200_culling_cull_device(frusta[v], types[v]).  Results stay in HBM, one id buffer / counter set / mask per view, owned by the culling
 * system apart from the output lanes; dev_ids (may be NULL) receives each view's id pointer (per-type segments as in
 * lb200_culling_cull_device).  want_counts != 0: results[v] filled (may be NULL; one read-back, one synchronisation) and
 * lb200_culling_last_algorithmic_bytes reports the whole call; 0: fully asynchronous, results may be NULL.
 * The view buffers stay valid until the next cull_views call; plain culls neither touch them nor are touched by them.  n_views = 1 runs
 * the single cull kernel; two or more run one fused kernel, whose pages per block per round are at most
 * min(256, 512 / n_views) (a larger chunk forced by lb200_culling_set_launch is capped; lb200_culling_get_launch reports the launch).
 * With no entity added every result is zero and nothing is launched.  Exchange mode is not part of this call. */
#define LB200_CULL_MAX_VIEWS 8
LB200_API int lb200_culling_cull_views(lb200_culling* cs, const lb200_shifted_frustum* frusta, const uint8_t* types, uint32_t n_views,
                                       const uint32_t** dev_ids, lb200_cull_result* results, int want_counts);
/* Make view k of the latest cull_views call "the last cull" for lb200_culling_last_result, lb200_culling_read_bitmask and
 * lb200_sortkeys_create_keys, with the per-type segment bases that view was culled with.  Any time after that call, plain culls in between
 * included.  LB200_ERR_INVALID for k >= its n_views; LB200_ERR_STATE if no cull_views was issued, if it culled an empty system, or if the
 * view buffers were released since (a growth of the page arrays, lb200_culling_set_replicas). */
LB200_API int lb200_culling_select_view(lb200_culling* cs, uint32_t k);

/* ------------------------------------------------------------------------------------------------------------
 * Sort keys — the consumer of the visible list (SURVEY.md 8f N1): PipelineImpl::createSortKeys (src/renderer/pipeline.cpp:3789-4018:
 * LOD selection + smoothing, sort keys / values :53-143, auto-instancing :452-523 and its instance data :3958-4016) and
 * PipelineImpl::radixSort (:4020-4144), on the device.  It reads the ids of the last cull where they lie in HBM; sorted keys / values
 * and the per-group instance data stay in HBM for the draw-command stage; the host reads back four counters.
 * One-instancer form of the reference (it runs one AutoInstancer per job worker and splits a mesh's instances over them): instancer
 * index 0 in the group values, every mesh's instances in one group.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct lb200_sortkeys lb200_sortkeys;
typedef struct lb200_sk_model {   /* per Model (src/renderer/model.h) */
	float lod_distances[4];       /* m_lod_distances (squared), model.h:234 */
	int32_t lod_from[5];          /* m_lod_indices[].from / .to, model.h:129-133,233 */
	int32_t lod_to[5];
	uint32_t mesh_base;           /* first entry of this model in the mesh table */
	uint32_t mesh_count;
} lb200_sk_model;
typedef struct lb200_sk_mesh {    /* per (model, mesh): MeshMaterial + Mesh + Material fields createSortKeys reads */
	uint32_t sort_key;            /* MeshMaterial::sort_key (model.h:65, RenderModule::computeSortKey): also the auto-instancer group */
	uint32_t material_index;      /* MeshMaterial::material_index */
	float lod;                    /* Mesh::lod (model.h:120) */
	uint8_t layer;                /* Material::getLayer() */
	uint8_t skinned;              /* Mesh::type == SKINNED */
	uint16_t pad;
} lb200_sk_mesh;
typedef struct lb200_sk_view {
	double camera_pos[3];         /* view.cp.pos */
	double lod_ref_point[3];      /* m_viewport.pos */
	float time_delta;             /* Engine::getLastTimeDelta() */
	float lod_multiplier;         /* Renderer::getLODMultiplier() */
	uint32_t frame_number;        /* Renderer::frameNumber() % 0xffffffff */
	uint32_t is_shadow;           /* view.cp.is_shadow */
	uint32_t max_sort_key;        /* Renderer::getMaxSortKey(); needs < max_groups */
	uint32_t pad;
	uint32_t bucket_map[256];     /* as built at pipeline.cpp:3803-3812: bucket | 0x100 if depth-sorted, 0xffffffff if the layer is not in the view */
	uint8_t layer_to_bucket[256]; /* View::layer_to_bucket */
} lb200_sk_view;
typedef struct lb200_sk_result { uint32_t n_keys, n_instances, n_pose, n_dirty, n_groups; } lb200_sk_result;
typedef struct lb200_sk_outputs { /* device pointers, valid until the next create_keys (create_keys_views for a view's) */
	const uint64_t* keys;              /* n_keys sort keys (sorted if asked), pipeline.cpp:62-71 layout */
	const uint64_t* values;            /* their sort values */
	const uint32_t* group_count;       /* per mesh sort key g in [0, n_groups): instances of the group */
	const uint32_t* group_offset;      /* ... and where they start in group_renderables / instance_data */
	const uint64_t* group_renderables; /* entity | mesh_idx << 40 */
	const void* instance_data;         /* 48 B per instance: rot (16), camera-relative pos (12), lod - mesh.lod (4), scale (12), material index (4) */
	const uint32_t* pose_list;         /* n_pose skinned instances whose palette is due this frame */
	const uint32_t* dirty_list;        /* n_dirty instances with ModelInstance::dirty set (material override refresh) */
	const float* lod;                  /* ModelInstance::lod per entity, updated by the pass (unpacked from the entity records by device_outputs) */
	const uint32_t* pose_frame;        /* Pose::frame per entity */
} lb200_sk_outputs;
#define LB200_SK_MOVED 1u /* ModelInstance::MOVED */
#define LB200_SK_DIRTY 2u /* ModelInstance::dirty */
LB200_API int lb200_sortkeys_create(lb200_ctx* ctx, uint32_t max_entities, uint32_t max_groups, uint32_t max_keys, uint32_t max_instances, lb200_sortkeys** out);
LB200_API void lb200_sortkeys_destroy(lb200_sortkeys* sk);
/* Replaces both tables.  LB200_ERR_INVALID for a mesh sort key >= max_groups or a non-empty LOD range outside [0, mesh_count) of its model.
 * A model whose meshes [mesh_base, mesh_base + mesh_count) leave the mesh table is stored, but create_keys refuses to launch
 * (LB200_ERR_INVALID) until set_models is called with tables that fit. */
LB200_API int lb200_sortkeys_set_models(lb200_sortkeys* sk, const lb200_sk_model* models, uint32_t n_models, const lb200_sk_mesh* meshes, uint32_t n_meshes);
/* Per-entity state, arrays indexed by entity id; a null pointer leaves that array as it is. */
LB200_API int lb200_sortkeys_set_instances(lb200_sortkeys* sk, uint32_t n, const uint32_t* model_of, const float* lod, const uint8_t* flags, const uint32_t* pose_frame,
                                           const uint32_t* decal_sort_key, const uint8_t* decal_layer);
/* World::getTransforms() (world.h:65), indexed by entity id: from the host, or from a device array (e.g. the hierarchy's globals).  Both
 * pack the transforms into the library's per-entity records when called (on the context stream): call again after the transforms changed. */
LB200_API int lb200_sortkeys_set_transforms(lb200_sortkeys* sk, const lb200_transform* transforms, uint32_t n);
LB200_API int lb200_sortkeys_set_transforms_device(lb200_sortkeys* sk, const lb200_transform* dev_transforms, uint32_t n);
/* createSortKeys (+ radixSort if `sort`) for the last cull of `cs` on the context stream.  Asynchronous unless `want_counts`. */
LB200_API int lb200_sortkeys_create_keys(lb200_sortkeys* sk, lb200_culling* cs, const lb200_sk_view* view, int sort, int want_counts, lb200_sk_result* result);
/* createSortKeys (+ radixSort if `sort`) for every view of the latest lb200_culling_cull_views call on `cs`, in one launch on the context
 * stream.  View v reads the ids, per-type segments and counters of view v of that call (never "the last cull"); n_views must equal its
 * view count.  The call does exactly what n_views calls of lb200_culling_select_view(cs, v) + lb200_sortkeys_create_keys(sk, cs,
 * &views[v], sort, ...) do in the order v = 0, 1, ...: a later view sees the ModelInstance::lod and Pose::frame that the earlier views
 * left, so a skinned instance joins the pose list of the first view that draws it and of no other.  The reference runs a frame's views
 * as concurrent jobs in no fixed order; view order is one of the orders it can produce.
 * Each view has its own outputs (keys, values, groups, instance data, pose and dirty lists; capacities max_keys / max_instances per
 * view), apart from those of lb200_sortkeys_create_keys: neither call touches the other's.  They stay valid until the next
 * create_keys_views on `sk` or its destroy; lb200_sortkeys_view_outputs hands them out.  The first call allocates them, a call with more
 * views than any before it reallocates them.  want_counts != 0: one read-back of every view's counters and one synchronisation fill
 * results[0, n_views); if a view exceeds a capacity the call returns LB200_ERR_CAPACITY with every results[v] still holding the sizes
 * needed.  want_counts = 0: fully asynchronous, results may be NULL.
 * LB200_ERR_STATE where lb200_culling_select_view refuses (no cull_views yet, an empty culling system, view buffers released by a growth
 * of the page arrays or lb200_culling_set_replicas) and before set_models / set_transforms.  LB200_ERR_INVALID for n_views 0, above
 * LB200_CULL_MAX_VIEWS or different from the cull's, for views whose max_sort_key differ (Renderer::getMaxSortKey() is renderer-wide),
 * and for everything lb200_sortkeys_create_keys refuses.  A refused call leaves the earlier outputs as they were. */
LB200_API int lb200_sortkeys_create_keys_views(lb200_sortkeys* sk, lb200_culling* cs, const lb200_sk_view* views, uint32_t n_views,
                                               int sort, int want_counts, lb200_sk_result* results /* n_views */);
/* Launch shape of later create_keys / create_keys_views calls.  blocks: 0 = the default (LB200_SK_BLOCKS_PER_SM per SM, else 2, and at most one block per 256
 * renderables the cull can emit), -1 = every block that is co-resident, n > 0 = min(n, co-resident blocks); only 0 caps the grid by the
 * work.  prefetch_ahead: 0..4 grid strides of L2 prefetch, -1 = the default (LB200_SK_PREFETCH, else 0).  Any other value is
 * LB200_ERR_INVALID.  get_launch reports the last launch of either call: blocks, whether the group counters lived in shared memory
 * (max_sort_key < 8192) and the prefetch distance (all 0 before the first). */
LB200_API int lb200_sortkeys_set_launch(lb200_sortkeys* sk, int blocks, int prefetch_ahead);
LB200_API int lb200_sortkeys_get_launch(lb200_sortkeys* sk, uint32_t* grid, int* groups_in_smem, uint32_t* prefetch_ahead);
LB200_API int lb200_sortkeys_device_outputs(lb200_sortkeys* sk, lb200_sk_outputs* out);
/* Device pointers of view k of the latest create_keys_views call (layout as lb200_sortkeys_device_outputs; lod / pose_frame are the
 * shared per-entity state).  LB200_ERR_STATE before any create_keys_views, LB200_ERR_INVALID for k >= its n_views. */
LB200_API int lb200_sortkeys_view_outputs(lb200_sortkeys* sk, uint32_t k, lb200_sk_outputs* out);
/* RenderModuleImpl::onModelInstanceMoved (src/renderer/render_module.cpp:1544-1554) for n instances whose new transforms lie in device memory:
 * the transforms go into the entity records, ModelInstance::MOVED is set (createSortKeys then draws the instance as DRAW_MESH, pipeline.cpp
 * :3904-3909) and the instance joins m_moved_instances once.  With dev_bounding_radius (per moved instance: Model::getOriginBoundingRadius)
 * the spheres CullingSystem::set needs are written to dev_out_pos3 (3 doubles each) / dev_out_radius for lb200_culling_set_many_device. */
LB200_API int lb200_sortkeys_move_device(lb200_sortkeys* sk, const int32_t* dev_entities, const lb200_transform* dev_transforms, uint32_t n, const float* dev_bounding_radius,
                                         double* dev_out_pos3, float* dev_out_radius);
/* RenderModuleImpl::endFrame (render_module.cpp:526-534): MOVED cleared and ModelInstance::prev_frame_transform taken for every instance moved
 * since the last call; lb200_sortkeys_prev_transforms hands out the per-entity device array of those transforms. */
LB200_API int lb200_sortkeys_end_frame(lb200_sortkeys* sk);
LB200_API int lb200_sortkeys_prev_transforms(lb200_sortkeys* sk, const lb200_transform** dev_prev);
/* m_moved_instances as it stands: *dev_list (device memory, NULL before the first move or spawn) holds *n entity ids, each at most once
 * (what end_frame will take prev_frame_transform of).  Reads the count back: synchronises the stream. */
LB200_API int lb200_sortkeys_moved_list(lb200_sortkeys* sk, const uint32_t** dev_list, uint32_t* n);
/* The entity ids the per-entity arrays hold, [0, max_entities): max_entities of create, or what a spawn call grew it to. */
LB200_API uint32_t lb200_sortkeys_max_entities(const lb200_sortkeys* sk);
/* Spawns on the device (the spawn lists of lb200_culling_add_many_device, for the stage behind the cull).
 * lb200_sortkeys_spawn_instances_device: RenderModuleImpl::createModelInstance + setModel + modelLoaded (render_module.cpp:3284-3292,
 * :3107-3148, :2911-2951) for n new model instances whose data lies in device memory.  For e = dev_entities[i] the entity's record ends as
 * the reference leaves ModelInstance and its Pose: transform dev_transforms[i] (what createSortKeys reads of World::getTransforms()),
 * model dev_model_of[i], lod = the highest l in 3 .. 0 whose lod_to[l] != -1 in that model (4 if none), MOVED off (VALID | ENABLED),
 * dirty = dev_dirty[i] != 0 (the instance has a material override; dev_dirty NULL = none has), Pose::frame 0xffffffff,
 * prev_frame_transform = dev_transforms[i] (the moved-list arrays are allocated if they do not exist yet).  An entity already in this
 * frame's moved list stays in it once: a later move in the same frame does not list it again, and end_frame takes its
 * prev_frame_transform as for any listed entity.
 * lb200_sortkeys_spawn_decals_device: createDecal / createCurveDecal + updateDecalInfo: the material sort key and layer createSortKeys
 * reads for DECAL / CURVE_DECAL renderables (pipeline.cpp:3841-3867).
 * Both: n = 0 returns LB200_OK and launches nothing, before any other check.  Otherwise LB200_ERR_INVALID for a NULL required pointer,
 * max_entity above INT32_MAX, an id outside [0, max_entity], an id listed twice or (instances) a model index at or above the current
 * model table's count; LB200_ERR_STATE (instances) before set_models.  A refused call changes nothing, capacity included.  The ids are
 * checked on the device, in one pass ahead of the writes, with one read-back and one synchronisation per call (two for a call that
 * grows).  A spawn of instances counts as set_transforms for create_keys, which reads only the records of culled ids.
 * Growth: max_entity >= max_entities grows every per-entity array (records, decal arrays, moved list, prev_frame_transform, the pose and
 * dirty lists of both output sets, scratch) to the next doubling of max_entities that holds max_entity, waiting for the stream first,
 * once the batch has been checked without refusals.  Everything keeps its contents (ModelInstance::lod, Pose::frame, the moved list,
 * prev_frame_transform, the latest create_keys / create_keys_views outputs), new ids start as create leaves them, max_keys and
 * max_instances keep the values create fixed, and set_instances / set_transforms take n up to the new max_entities.  A failed
 * allocation returns LB200_ERR_CUDA and leaves the object as it was.  Device pointers handed out before a call that grows (device_outputs,
 * view_outputs, prev_transforms, moved_list) are stale after it: ask again.
 * Despawn needs no call here: an id removed with lb200_culling_remove_many_device is in no visible list, so createSortKeys never reads
 * its record, and a later spawn of the id rewrites all of it (destroyModelInstance / destroyDecal reach createSortKeys only through the
 * cull). */
LB200_API int lb200_sortkeys_spawn_instances_device(lb200_sortkeys* sk, const int32_t* dev_entities, const uint32_t* dev_model_of,
                                                    const lb200_transform* dev_transforms, const uint8_t* dev_dirty, uint32_t n, uint32_t max_entity);
LB200_API int lb200_sortkeys_spawn_decals_device(lb200_sortkeys* sk, const int32_t* dev_entities, const uint32_t* dev_sort_key, const uint8_t* dev_layer,
                                                 uint32_t n, uint32_t max_entity);
/* mi.dirty = false of PipelineImpl::refreshMaterialOverrides (pipeline.cpp:3685-3721) for n instances whose refresh finished (device ids):
 * only the dirty bit changes, MOVED and the rest of the record stay.  Ids outside [0, max_entities) are skipped.  n = 0 returns LB200_OK
 * before any other check; otherwise a NULL dev_entities is LB200_ERR_INVALID.  Asynchronous. */
LB200_API int lb200_sortkeys_clear_dirty_device(lb200_sortkeys* sk, const int32_t* dev_entities, uint32_t n);
/* The stable LSD radix sort create_keys and the device re-binning use, on caller device buffers, on the context stream: sorts
 * n = min(*dev_count, cap) (u64 key, u64 value) pairs in place (the count is read on the device, like the two callers do).
 * max_blocks caps the cooperative grid (0 = as many as are co-resident; the grid is also at most ceil(cap / 2048)); force_tiled != 0 takes
 * the tiled path at any n.  The register path is taken iff !force_tiled && n <= grid * 512 * 16.  *out_grid (may be NULL) = blocks launched.
 * Entries [n, cap) are left untouched.  The scratch is kept in the context, grows to the largest cap (waiting for the stream when it
 * does) and is freed by lb200_shutdown. */
LB200_API int lb200_radix_sort_device(lb200_ctx* ctx, uint64_t* dev_keys, uint64_t* dev_values, const uint32_t* dev_count, uint32_t cap, uint32_t max_blocks,
                                      int force_tiled, uint32_t* out_grid);

/* ------------------------------------------------------------------------------------------------------------
 * Multi-GPU (one process per GPU; SURVEY.md §8e).  NCCL is dlopen()ed; the unique id travels through the caller
 * (torch.distributed store / any out-of-band channel).
 * ---------------------------------------------------------------------------------------------------------- */
LB200_API int lb200_comm_get_unique_id(lb200_ctx* ctx, uint8_t out_id[128]);
LB200_API int lb200_comm_init(lb200_ctx* ctx, int n_ranks, int rank, const uint8_t unique_id[128]);
LB200_API void lb200_comm_destroy(lb200_ctx* ctx);
/* Optional, collective (every rank, same argument): map every rank's gather buffers into every process over NVLink peer access
 * (CUDA IPC).  After it lb200_culling_cull_gather pushes each rank's slab straight into its peers' memory from one fused kernel
 * and synchronises with per-epoch flags instead of calling NCCL on the per-frame path.  Up to 8 ranks (one NVSwitch box). */
LB200_API int lb200_comm_enable_p2p(lb200_ctx* ctx, uint32_t max_slab_ids);
/* LB200_OK, or LB200_ERR_NCCL (once; the condition is reset) if a device-side wait for a peer's slab gave up since the last check. */
LB200_API int lb200_comm_status(lb200_ctx* ctx);
/* Slab layout of the exchange: every rank contributes `256 + slab_ids` u32 words = [256 per-type counts][its visible ids packed type after
 * type]; the gathered buffer holds n_ranks such slabs back to back (rank r at word r * (256 + slab_ids)).
 *
 * lb200_culling_cull_gather: the per-frame multi-GPU step — cull, pack on the device (no host round trip), ONE ncclAllGather of the slabs.
 * Fully asynchronous on the context stream.  *out_dev_slabs = device pointer of the gathered buffer.
 * lb200_culling_allgather: the same exchange for the cull that was just issued, plus a read-back of the counts
 * (out_counts[r*256 + t] = rank r's count of type t) and a stream synchronisation. */
LB200_API int lb200_culling_cull_gather(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t slab_ids, const uint32_t** out_dev_slabs);
LB200_API int lb200_culling_allgather(lb200_culling* cs, uint32_t slab_ids, const uint32_t** out_dev_slabs, uint32_t* out_counts /* n_ranks*256 */);
/* Distance in u32 words between consecutive ranks' slabs inside the buffer lb200_culling_cull_gather returns for this slab_ids
 * (256 + slab_ids on the NCCL path, the fixed peer-buffer stride after lb200_comm_enable_p2p). */
LB200_API uint32_t lb200_culling_gather_stride_words(const lb200_culling* cs, uint32_t slab_ids);

/* Bitmask exchange (SURVEY 8e): the cull kernel itself stores the 32-byte visibility row of every page it worked on — together
 * with the page id — straight into EVERY rank's memory over NVLink (no separate pack / collective launch; rows of pages outside the
 * frustum are all zero and never cross the links); a one-block kernel behind it sends the per-type counts and raises the epoch flags.
 * The visible ids stay sharded on the rank that owns the entities (*out_dev_ids, per-type segments as in lb200_culling_cull_device).
 * Needs lb200_comm_enable_p2p(ctx, max over ranks of lb200_culling_exchange_slab_words(cs) - 256).  Asynchronous on the context
 * stream; when the stream reaches the end of this call every rank's slab of this step is complete in *out_dev_slabs.
 * Slab of rank r = words [r * stride, (r + 1) * stride):
 *   [0,256)            visible count per renderable type
 *   [256,264)          n_pages, n_records, 0, cap, 0, 0, 0, 0
 *   [264, 264 + cap)   page id of record i < n_records (page ids of rank r)
 *   [264 + cap, ..)    8 words per record: bit s of the 256-bit row = slot s of the page is visible (slots >= 200 are 0)
 *   every page without a record has an all-zero row.
 * A peer that does not publish within ~4 s makes the next lb200_synchronize / exchange call return LB200_ERR_NCCL (lb200_comm_status). */
LB200_API int lb200_culling_cull_exchange(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, const uint32_t** out_dev_ids,
                                          const uint32_t** out_dev_slabs, uint32_t* out_slab_stride_words);
/* n independent exchange steps issued from one call: step (epoch) e runs on internal stream e % lanes on every rank, so the remote
 * stores, fences and flag round trip of one step overlap the culls of its neighbours (3 x lanes exchange buffers per rank).  Forks
 * from and joins back into the context stream; the out parameters describe the LAST step. */
LB200_API int lb200_culling_cull_exchange_n(lb200_culling* cs, const lb200_shifted_frustum* frustum, uint8_t type, uint32_t n,
                                            const uint32_t** out_dev_ids, const uint32_t** out_dev_slabs, uint32_t* out_slab_stride_words);
LB200_API uint32_t lb200_culling_exchange_slab_words(lb200_culling* cs);

/* ------------------------------------------------------------------------------------------------------------
 * Hierarchy — replaces the recursion World::transformEntity, src/engine/world.cpp:255-282 (child.global =
 * parent.global.compose(child.local), math.cpp:801-807) with a batched level-order pass.
 * Nodes are given in any order with parent indices (-1 = root); the library orders them by depth once.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct lb200_hierarchy lb200_hierarchy;
typedef struct lb200_animation lb200_animation; /* the Animation section below; bone attachments of a hierarchy take its systems */

LB200_API int lb200_hierarchy_create(lb200_ctx* ctx, const int32_t* parents, uint32_t n, lb200_hierarchy** out);
LB200_API void lb200_hierarchy_destroy(lb200_hierarchy* h);
LB200_API uint32_t lb200_hierarchy_depth(const lb200_hierarchy* h);
/* World::setParent (world.cpp:619-701) for any number of nodes at once, and nodes entering / leaving: replace the whole parent array.
 * parents[i] = parent node index, negative = root (as lb200_hierarchy_create); n may differ from the current node count.  The hierarchy then
 * holds exactly the level order lb200_hierarchy_create(parents, n) builds (roots in ascending index, then level by level each node's
 * children in ascending index).  Node i < min(old n, n) keeps its local and global transform; nodes >= old n start as the identity.  Locals
 * are not recomputed: for setParent's keep-the-global behaviour call set_subset, or set_globals + compute_locals, afterwards.  When n changes
 * the bounding radii are released (the next get_spheres / refresh_spheres must pass them) and the sphere pointers may change.
 * A parent >= n, a cycle or n = 0 returns LB200_ERR_INVALID (create's error texts) and leaves the hierarchy as it was.
 * The device form reads the parents from device memory and reads back only the build's counters and the depth + 1 level starts;
 * max_blocks caps the grid of the cooperative kernels (0 = as many as are co-resident).  Both launch the same kernels at any depth. */
LB200_API int lb200_hierarchy_set_parents(lb200_hierarchy* h, const int32_t* parents, uint32_t n);
LB200_API int lb200_hierarchy_set_parents_device(lb200_hierarchy* h, const int32_t* dev_parents, uint32_t n, uint32_t max_blocks);
/* Introspection: order[k] = node at level position k (n), parent_pos[k] = its parent's level position (n, -1 for roots),
 * level_start = the first position of every level and n (depth + 1). */
LB200_API int lb200_hierarchy_get_level_order(lb200_hierarchy* h, uint32_t* order, int32_t* parent_pos, uint32_t* level_start);
/* World::setLocalTransform for all nodes (world.h:98-123): upload locals (n Transforms, caller's node order). */
LB200_API int lb200_hierarchy_set_locals(lb200_hierarchy* h, const lb200_transform* locals);
/* Root world transforms (entries of non-root nodes are ignored). */
LB200_API int lb200_hierarchy_set_root_globals(lb200_hierarchy* h, const lb200_transform* globals);
/* World::setLocalTransform / World::setTransform for SOME nodes (world.h:98-123): `count` node indices with their new local transforms
 * (globals = 0) or world transforms (globals = 1; meaningful for roots).  Only count x 60 bytes cross PCIe. */
LB200_API int lb200_hierarchy_set_subset(lb200_hierarchy* h, const uint32_t* nodes, const lb200_transform* values, uint32_t count, int globals);
/* Run the propagation on the GPU; globals stay in HBM. */
LB200_API int lb200_hierarchy_propagate(lb200_hierarchy* h);
/* World::getTransforms (world.h:65): copy globals back in the caller's node order. */
LB200_API int lb200_hierarchy_get_globals(lb200_hierarchy* h, lb200_transform* out_globals);
/* RenderModuleImpl::onModelInstanceMoved, render_module.cpp:1544-1554: world sphere per node =
 * (global.pos, bounding_radius * max(scale)); out_pos3 n*3 doubles, out_radius n floats (host). */
LB200_API int lb200_hierarchy_get_spheres(lb200_hierarchy* h, const float* bounding_radius, double* out_pos3, float* out_radius);
/* The same refresh left in device memory (bounding_radius may be NULL after the first call: the radii uploaded last are kept): *dev_pos3 = n x 3
 * doubles, *dev_radius = n floats, both indexed like `parents`; input of lb200_culling_set_many_device when node index = entity id. */
LB200_API int lb200_hierarchy_refresh_spheres(lb200_hierarchy* h, const float* bounding_radius, const double** dev_pos3, const float** dev_radius);
/* The other direction, World::transformEntity(entity, update_local = true) (world.cpp:267-270) / World::setParent (world.cpp:619-701):
 * world transforms are authoritative (physics, editor gizmo, re-parenting) and the local transforms follow:
 * local = Transform::computeLocal(parent global, own global) (math.cpp:809-816) for every non-root node, one launch.
 * set_globals uploads all n world transforms (caller's node order); get_locals copies the locals back (roots: as uploaded). */
LB200_API int lb200_hierarchy_set_globals(lb200_hierarchy* h, const lb200_transform* globals);
LB200_API int lb200_hierarchy_compute_locals(lb200_hierarchy* h);
LB200_API int lb200_hierarchy_get_locals(lb200_hierarchy* h, lb200_transform* out_locals);
/* World::getRelativeMatrix (src/engine/world.cpp:370-377) of every node against one base position (the camera): out_matrices = n x 16
 * floats, column-major like Matrix (math.h:329-392), indexed like `parents`.  Consumers of the propagated transforms
 * (pipeline.cpp instance setup) take these instead of calling getRelativeMatrix per entity. */
LB200_API int lb200_hierarchy_get_relative_matrices(lb200_hierarchy* h, const double base_pos[3], float* out_matrices);
LB200_API uint64_t lb200_hierarchy_algorithmic_bytes(const lb200_hierarchy* h);
/* Which entities a propagate moved: the entities whose `transformed` delegates World::transformEntity (world.cpp:255-282) fires, i.e. every
 * entity set through setTransform / setLocalTransform and every descendant of one, each once — the set RenderModuleImpl::onModelInstanceMoved
 * (render_module.cpp:1544-1566) hands to MOVED, m_moved_instances and CullingSystem::set.
 * Marks: set_subset marks the nodes it lists (both forms); mark_moved marks nodes directly (a node >= n: LB200_ERR_INVALID, nothing marked).
 * set_locals, set_root_globals, set_globals and compute_locals mark nothing, and plain propagate neither reads nor clears marks.
 * set_entities: entity id per node (caller's node order, n entries); a negative id keeps the node out of every moved list (no component
 * listens: onModelInstanceMoved's isAdded early-out, render_module.cpp:1545).  Default: node i = entity i.
 * set_parents[_device] keeps the marks and entity ids of nodes i < min(old n, n); new nodes start unmarked with entity i. */
LB200_API int lb200_hierarchy_set_entities(lb200_hierarchy* h, const int32_t* entity_of_node);
LB200_API int lb200_hierarchy_mark_moved(lb200_hierarchy* h, const uint32_t* nodes, uint32_t count);
typedef struct {
	const int32_t* entities;          /* k entity ids, in ascending node index */
	const lb200_transform* transforms; /* their new world transforms */
	const double* pos3;               /* their world spheres (3 doubles each) and radii, as refresh_spheres computes them; NULL when no */
	const float* radius;              /*   bounding radii are held */
	const uint32_t* count;            /* k, in device memory */
} lb200_hierarchy_moved;
/* lb200_hierarchy_propagate (the same globals, byte for byte) + the moved list: every node that is marked or has a marked ancestor in the
 * current topology and whose entity id is not negative, once, in ascending node index; then every mark is cleared.  bounding_radius (n, or
 * NULL) is taken as refresh_spheres takes it: uploaded if given, otherwise the radii held are used, otherwise pos3 / radius are NULL.  The
 * buffers belong to the hierarchy (capacity n) and stay valid until the next propagate_moved, set_parents[_device] or destroy.  With
 * out_count, k is read back (4 bytes, one synchronisation); without it the call does not wait for the device. */
LB200_API int lb200_hierarchy_propagate_moved(lb200_hierarchy* h, const float* bounding_radius, lb200_hierarchy_moved* out, uint32_t* out_count);
/* Bone attachments held by the hierarchy (RenderModuleImpl::m_bone_attachments, render_module.cpp:377-405): attachment k moves node
 * attached[k] to bone bone[k] of instance instance[k] of animation system slot system[k] (the slot indexes the systems array of
 * propagate_attached), parent node parent[k], relative7[k] = BoneAttachment::relative_transform (pos xyz, rot xyzw).  n = 0 removes the
 * table.  Host arrays; copied.  A node >= n, attached[k] == parent[k] or the same attached node twice (an entity has one BoneAttachment):
 * LB200_ERR_INVALID, the table left as it was.  set_parents[_device] keeps the table (node indices), and the rounds are rebuilt. */
LB200_API int lb200_hierarchy_set_attachments(lb200_hierarchy* h, uint32_t n, const uint32_t* attached, const uint32_t* parent,
                                              const uint32_t* system, const uint32_t* instance, const uint32_t* bone, const float* relative7);
/* propagate_moved + every attachment round, one moved list (the same buffers, lifetime and count read-back as propagate_moved's).  The
 * frame World::setTransform (world.cpp:255-282, 337-342) and onModelInstanceMoved (render_module.cpp:1544-1566) make of it:
 *  1. the marked edits propagate; an attached non-root node is recomposed only when it is marked or an ancestor moved in this pass, so the
 *     global an attachment set stays bit for bit (compose o computeLocal is not exact);
 *  2. the attachments run in rounds: X after Y when Y's attached node is an ancestor-or-self of X's parent node or a strict ancestor of
 *     X's attached node.  X is active when posed[system] != 0 (posed == NULL: every system was updated this frame) or its parent node has
 *     moved so far in this call and has an entity id >= 0.  An active X sets its node's global to parent.compose(bone * relative) with the
 *     node's current global scale, and its local to computeLocal(world parent, global) (roots: no local); then the round's active nodes'
 *     subtrees are recomposed.  Inactive attachments leave their node alone.
 * Every system needs absolute poses (an update with LB200_PALETTE_POSE).  Refused, with globals, locals, marks and the table unchanged:
 * LB200_ERR_INVALID for a slot >= n_systems, an instance >= its system's instance count or a bone >= its bone count, or a cycle (an
 * attached node that is an ancestor-or-self of its own parent node, directly or through other attachments); LB200_ERR_STATE for a NULL
 * system, one of another context or one without absolute poses, and for a table whose nodes set_parents has shrunk away (until the next
 * set_attachments).  The rounds are built on the device at the first call after set_attachments or set_parents[_device] (a few
 * read-backs); later calls read nothing back unless out_count is asked for.  A slot is only checked here (set_attachments cannot know
 * n_systems).  An empty table is propagate_moved: the systems are not looked at. */
LB200_API int lb200_hierarchy_propagate_attached(lb200_hierarchy* h, lb200_animation* const* systems, const uint8_t* posed, uint32_t n_systems,
                                                 const float* bounding_radius, lb200_hierarchy_moved* out, uint32_t* out_count);
/* Introspection: rounds[k] = the round of attachment k (1-based, table order) and *n_rounds as the last round build made them
 * (LB200_ERR_STATE before one); rounds may be NULL. */
LB200_API int lb200_hierarchy_get_attachment_rounds(lb200_hierarchy* h, uint32_t* rounds, uint32_t* n_rounds);

/* ------------------------------------------------------------------------------------------------------------
 * Animation — replaces AnimationModuleImpl::updateAnimable (src/animation/animation_module.cpp:439-472):
 * Model::getRelativePose (model.cpp:226-237) -> Animation::getRelativePose (animation.cpp:117-204) ->
 * Pose::computeAbsolute (pose.cpp:66-133), then the palette builds computeSkeletonDualQuats
 * (src/renderer/pipeline.cpp:2680-2745) / computeSkinMatrices (src/renderer/model.cpp:132-137) and the CPU
 * skinning evaluateSkin (model.cpp:103-109).
 * ---------------------------------------------------------------------------------------------------------- */
/* Animation::TranslationTrack / RotationTrack, src/animation/animation.h:92-118, pointer-free */
typedef struct {
	uint16_t bone_index;
	uint16_t offset_bits;
	uint8_t bitsizes[3];
	uint8_t skipped_channel; /* rotation tracks only */
	float min[3];
	float to_range[3];
} lb200_track; /* 32 bytes */

typedef struct { uint16_t bone_index; uint16_t pad; float value[3]; } lb200_const_translation; /* animation.h:86-90 */
typedef struct { uint16_t bone_index; uint16_t pad; float value[4]; } lb200_const_rotation;    /* animation.h:100-104 */

/* struct Animation, animation.h:158-170 (in-memory form after Animation::load, animation.cpp:397-493).  Root motion is not part of this
 * struct: lb200_animation_set_root_motion gives a system's clips the flags and root-motion tracks Animation::setRootMotionBone resolved,
 * and the system then samples those tracks as the reference does (m_root_motion.pose_translations / pose_rotations, animation.cpp:33-37,
 * 321). */
typedef struct {
	float fps;
	uint32_t frame_count;
	uint32_t translations_frame_size_bits, rotations_frame_size_bits;
	uint32_t n_translations, n_const_translations, n_rotations, n_const_rotations;
	const lb200_track* translations;
	const lb200_const_translation* const_translations;
	const lb200_track* rotations;
	const lb200_const_rotation* const_rotations;
	const uint8_t* translation_stream; uint32_t translation_stream_bytes; /* incl. the 8-byte tail padding, animation.cpp:439 */
	const uint8_t* rotation_stream; uint32_t rotation_stream_bytes;
} lb200_clip;

/* Model skeleton, src/renderer/model.h:154-166,225-244: parents (parent < child, model.cpp:381-384), bind pose relative
 * transforms (Bone::relative_transform) and inverse bind transforms; each transform = 7 floats (pos xyz, rot xyzw). */
typedef struct {
	uint32_t bone_count;               /* <= 196, model.h:155 */
	int32_t first_nonroot_bone_index;  /* model.h getFirstNonrootBoneIndex */
	const int16_t* parents;
	const float* bind_relative7;
	const float* inverse_bind7;
} lb200_skeleton;

/* Mesh::Skin, model.h:81-84 + positions: n_vertices * {pos[3]}, {weights[4]}, {indices[4] i16} */
typedef struct {
	uint32_t n_vertices;
	const float* positions3;
	const float* weights4;
	const int16_t* indices4;
} lb200_mesh;


#define LB200_PALETTE_DUAL_QUAT 1u  /* 32 B/bone, pipeline.cpp:2680-2745 */
#define LB200_PALETTE_MATRIX 2u     /* 64 B/bone, model.cpp:132-137 */
#define LB200_PALETTE_POSE 4u       /* absolute pose write-back (pos 12 B + rot 16 B per bone) for lockPose consumers */

/* Refused with LB200_ERR_INVALID, before anything is allocated: a clip with fps <= 0, no frames or 2^24 frames or more (the sampler's
 * clamp to frame_count - 0.00001f is computed in fp32 and could pass the last frame from there on); one whose length
 * (frame_count / fps * 32768, in fp32 as Time::fromSeconds) is below one tick or 2^32 ticks or more; a track whose bone is outside the
 * skeleton (constant tracks too), with a channel of 64 bits or more (bitsizes[k] >= 64; unpackChannel's mask is undefined there, the importer writes at most 31),
 * or a rotation track with skipped_channel > 3; a bit stream shorter than (frame_count + 1) frames; clips whose decoded keyframe tables,
 * (frame_count + 2) rows of bone_count rounded up to 4 entries each, pass 2^31 entries together. */
LB200_API int lb200_animation_create(lb200_ctx* ctx, const lb200_skeleton* skeleton, const lb200_clip* clips, uint32_t n_clips,
	const lb200_mesh* mesh /* may be NULL */, uint32_t max_instances, lb200_animation** out);
LB200_API void lb200_animation_destroy(lb200_animation* a);
/* Per-instance state: Animable{time, animation}, animation_module.h:17-21.  time in Time ticks (1 s = 32768, animation.h:17-43). */
LB200_API int lb200_animation_set_instances(lb200_animation* a, const uint32_t* clip_index, const uint32_t* time_ticks, uint32_t n);
/* One updateAnimables pass (animation_module.cpp:737-749) for all instances: evaluate at the current time, build the requested
 * palettes in HBM, then step the time as :458-469 do: time_delta > 0: (time + dt) % length; otherwise (rewind, and zero):
 * (time + length - (-dt % length)) % length — a time already below the clip length is left alone by a zero step.  A system in
 * sample-list mode (lb200_animation_set_samples) evaluates its lists and steps no time. */
LB200_API int lb200_animation_update(lb200_animation* a, float time_delta, uint32_t palette_flags);
/* lb200_animation_update of every listed system in one device pass: the frame's updateAnimables over all its skeletons (one system per
 * Model), launched as one grid of up to 64 systems (longer lists run as consecutive launches on the context stream).
 * - Results: bit for bit what lb200_animation_update(systems[k], time_delta, palette_flags) gives for every k — dual quaternions,
 *   matrices, absolute poses and advanced times, in each system's own buffers.  Systems are independent, so the order does not
 *   matter.  A system with 0 instances is skipped, as update skips it.
 * - Execution: asynchronous on the context stream, no synchronisation and no read-back, inside the NVTX range "update animables".
 * - n = 0 returns LB200_OK before any other check and launches nothing.
 * - LB200_ERR_INVALID, with nothing changed and nothing launched: systems == NULL with n > 0, a NULL entry, a system listed twice
 *   (its time would advance twice), systems of different contexts.
 * - Palette and pose buffers are allocated per system, as update allocates them, before anything is launched; a failed allocation
 *   returns LB200_ERR_CUDA with nothing launched.
 * - Lanes per instance: one G serves the whole call.  If every listed system with instances would choose the same G on its own
 *   (its set_launch value, then LB200_POSE_LANES, then 8) that G runs, otherwise 8; 4 lanes fall back to 8 when the call's largest
 *   skeleton has more than 192 bones.  get_launch on each of these systems reports the G that ran.  Results do not depend on G. */
LB200_API int lb200_animation_update_many(lb200_animation* const* systems, uint32_t n, float time_delta, uint32_t palette_flags);
/* evaluateSkin (model.cpp:103-109) for every vertex of every instance from the matrix palette; output stays in HBM. */
LB200_API int lb200_animation_skin(lb200_animation* a);
/* Launch shape of later updates and skins, for tests and tuning.  pose_lanes = lanes per instance of the pose kernel (4, 8, 16 or 32);
 * with 4 lanes, a skeleton whose poses do not fit in shared memory (more than 192 bones) still runs on 8.  skin_group = instances per
 * skinning block (4, 8 or 16).  0 keeps the default: the LB200_POSE_LANES / LB200_SKIN_GROUP environment switch if set, else 8.
 * Any other value is LB200_ERR_INVALID.  get_launch reports what the last update and the last skin launched (0 before the first). */
LB200_API int lb200_animation_set_launch(lb200_animation* a, int pose_lanes, int skin_group);
LB200_API int lb200_animation_get_launch(lb200_animation* a, int* pose_lanes, int* skin_group);
/* Read-backs (host buffers).  Instances [first, first+count). */
LB200_API int lb200_animation_get_dual_quats(lb200_animation* a, uint32_t first, uint32_t count, float* out8);
LB200_API int lb200_animation_get_matrices(lb200_animation* a, uint32_t first, uint32_t count, float* out16);
LB200_API int lb200_animation_get_pose(lb200_animation* a, uint32_t first, uint32_t count, float* out_pos3, float* out_rot4);
/* Blend layers: the animator's stack of weighted samples (src/animation/controller.cpp:267-292, nodes.cpp) in a flat per-instance
 * form.  After the base clip of set_instances (sampled with weight 1 onto the bind pose) every instance applies n_layers further
 * samples in order, entry [instance * n_layers + k] = (clip, time in ticks, weight): Animation::getRelativePose with ctx.weight
 * (animation.cpp:117-204, 294-311) — bones the layer's clip tracks move towards its sample by lerp / simd_nlerp when weight < 0.9999,
 * are replaced otherwise; other bones keep their pose.  Layer times are the caller's (not advanced by update).  n_layers = 0 removes
 * the layers; lb200_animation_set_instances also does.  Up to 16 layers. */
LB200_API int lb200_animation_set_layers(lb200_animation* a, uint32_t n_layers, const uint32_t* clip_index, const uint32_t* time_ticks, const float* weight);
/* One SAMPLE instruction of an animator's blend stack (controller.cpp:267-293 -> getPose :142-157): clip index, time in ticks, weight,
 * looped (0 = clamped).  16 bytes, read by the pose kernel as one 128-bit load. */
typedef struct { uint32_t clip; uint32_t time_ticks; float weight; uint32_t looped; } lb200_sample;
/* Sample lists: the SAMPLE part of each animator's evalBlendStack, one list per instance (CSR: instance i owns
 * samples[offsets[i] .. offsets[i+1])).  Instance i starts from the bind pose (Model::getRelativePose, model.cpp:226-237) and applies its
 * samples in order, each with Animation::getRelativePose's arithmetic for its weight (animation.cpp:117-204, 294-311): bones the clip
 * tracks are replaced at weight >= 0.9999 and moved by lerp / simd_nlerp below it, other bones keep their pose.  A sample is taken at
 * time % length when looped and at min(time, length) otherwise, length = Animation::getLength().  Any count per instance, 0 included
 * (the bind pose).  Then computeAbsolute and the requested palettes / pose, as update always does.
 * - Mode: set_samples puts the system in sample-list mode with n_instances instances; set_instances puts it back in clip mode.  In
 *   sample-list mode update and update_many step no time (the animator's controller owns it), and get_times and set_layers return
 *   LB200_ERR_INVALID.  update_many takes clip-mode and sample-list systems in one call.
 * - LB200_ERR_INVALID, with nothing changed: n_instances > max_instances, NULL offsets, NULL samples with offsets[n_instances] > 0,
 *   offsets[0] != 0, decreasing offsets, a clip index out of range.  (Clips of length 0 are refused by create, so a looped sample never
 *   divides by 0.)
 * - The lists are copied before the call returns.
 * - set_samples(a, n, offsets, samples) is set_stacks(a, n, offsets, samples, NULL, NULL): it drops the IK ops of an earlier set_stacks. */
LB200_API int lb200_animation_set_samples(lb200_animation* a, uint32_t n_instances, const uint32_t* offsets, const lb200_sample* samples);
/* One IK instruction of an animator's blend stack (controller.cpp:275-281).  32 bytes, read by the pose kernel as two 128-bit loads. */
typedef struct {
	uint32_t after;      /* how many of the instance's samples run before it: 0 = on the bind pose, list length = after all of them */
	uint32_t leaf_bone;  /* bone index (Model::getBoneIndex of the instruction's BoneNameHash) */
	uint32_t bone_count; /* bones of the chain, 1 .. 32, the leaf and its bone_count - 1 nearest ancestors */
	float alpha;         /* what evalIK receives: the instruction's alpha * ctx.weight */
	float target[3];     /* model space */
	uint32_t reserved;
} lb200_ik;
/* Blend stacks: set_samples plus one CSR list of IK ops per instance (instance i owns iks[ik_offsets[i] .. ik_offsets[i+1])), each run
 * between the instance's samples where its `after` puts it, as evalBlendStack runs the stack's instructions in order.  Ops of one
 * instance have non-decreasing `after`; ops with the same `after` run in list order.  An op is evalIK (controller.cpp:166-265) on the
 * relative pose at that point: nothing below alpha 0.001, otherwise the chain from the leaf up goes to model space, an unreachable
 * target is pulled onto the chain's reach, 5 FABRIK iterations move the joints, Quat::vec3ToVec3 turns the moves into rotations, and
 * the pose moves towards the result by lerp and the scalar nlerp with alpha.  Bit for bit what the reference computes, except where
 * it computes a NaN (two coincident joints), whose payload may differ.
 * - ik_offsets == NULL: no IK ops (set_samples).  Systems with IK ops run their own kernels; the others run the same code as before.
 * - LB200_ERR_INVALID, with nothing changed: every refusal of set_samples, ik_offsets[0] != 0, decreasing ik_offsets, NULL iks with
 *   ik_offsets[n_instances] > 0, `after` greater than the instance's sample count or smaller than the op before it in the instance,
 *   leaf_bone >= the skeleton's bone count, bone_count 0 or above 32, a chain that leaves the skeleton (walking bone_count - 1
 *   parents from the leaf reaches -1), which the reference meets with an ASSERT or undefined behaviour.
 * - The ops are copied before the call returns; the chains are resolved from the skeleton then. */
LB200_API int lb200_animation_set_stacks(lb200_animation* a, uint32_t n_instances, const uint32_t* offsets, const lb200_sample* samples,
	const uint32_t* ik_offsets, const lb200_ik* iks);
/* Root motion of one clip, as Animation::setRootMotionBone (animation.cpp:214-270) resolved it for the skeleton's root-motion bone.
 * 12 bytes. */
typedef struct {
	uint32_t flags;            /* Animation::Flags (animation.h:73-78): Y_ROOT_TRANSLATION 1, XZ_ROOT_TRANSLATION 2, ROOT_ROTATION 4 */
	int32_t translation_track; /* index into the clip's lb200_clip.translations (the bone's first animated translation track), or -1 */
	int32_t rotation_track;    /* index into the clip's lb200_clip.rotations, or -1 */
} lb200_root_motion;
/* Root motion per clip (per_clip[c] for clip c of create): afterwards every pose, palette and consumer of the system samples clip c as the
 * reference samples an Animation on which setRootMotionBone ran once, freshly loaded, with those flags and tracks.  For every frame f of
 * 0 .. frame_count, the tracks' values tmp (Animation::getTranslation / getRotation; a missing track gives 0 / identity) are masked by
 * maskRootMotion (animation.cpp:97-115) to rm, rm0 is the masked value of frame 0 (0 / identity where the flags leave the translation /
 * rotation out), and the tracks sample rm0 * rm.inverted() * tmp in place of their packed values.  A track whose part of the motion the
 * flags leave out is replaced too, as the reference replaces it.
 * - An entry with flags 0, or with both tracks -1, leaves the clip as create decoded it.  A later call replaces an earlier one: clips
 *   with root motion before are decoded again from their packed tracks first, so an entry reset to flags 0 / tracks -1 samples bit for bit
 *   as a system that never had root motion.
 * - The tables are built on the device (one thread per clip and frame) and the call returns after they are; times, instances, layers
 *   and lists are kept.  Only the clips' decoded keyframes change: every update runs the same kernels as without root motion.
 * - The module's entity-transform step (animation_module.cpp:630-635, Animation::getRootMotion) is not part of this: the library keeps
 *   no root-motion deltas.
 * - LB200_ERR_INVALID, with nothing changed: NULL per_clip with n_clips > 0, n_clips other than the system's clip count, a track index
 *   below -1 or at / past the clip's track count, flag bits outside ANY_ROOT_MOTION (7). */
LB200_API int lb200_animation_set_root_motion(lb200_animation* a, uint32_t n_clips, const lb200_root_motion* per_clip);
/* Pose::computeRelative (src/renderer/pose.cpp:136-146) of every instance's absolute pose (needs an update with LB200_PALETTE_POSE):
 * the parent-relative poses IK / ragdoll consumers start from (controller.cpp).  Kept in HBM next to the absolute ones. */
LB200_API int lb200_animation_compute_relative(lb200_animation* a);
LB200_API int lb200_animation_get_relative_pose(lb200_animation* a, uint32_t first, uint32_t count, float* out_pos3, float* out_rot4);
/* Pose::blend (pose.cpp:30-41), instance by instance: a's poses move towards b's by `weight` (<= 0.001: untouched; clamped to [0,1]);
 * positions a*(1-w) + b*w, rotations scalar nlerp.  relative != 0 blends the parent-relative buffers of compute_relative, else the
 * absolute ones.  Both systems: same context, skeleton size and instance count. */
LB200_API int lb200_animation_blend_pose(lb200_animation* a, const lb200_animation* b, float weight, int relative);
/* RenderModuleImpl::updateBoneAttachment (src/renderer/render_module.cpp:377-405) for n attachments at once (SURVEY 8f N4): entity i
 * follows bone bone[i] of instance instance[i] (absolute poses of the last update with LB200_PALETTE_POSE):
 * out[i] = parent_transforms[i].compose(bone_transform * relative7[i]) (math.cpp:763, 859-861) with scale = original_scale3[i].
 * Host arrays in, host transforms out (the engine then feeds them to World::setTransform / the batched propagate). */
LB200_API int lb200_animation_bone_attachments(lb200_animation* a, uint32_t n, const uint32_t* instance, const uint32_t* bone, const float* relative7,
                                               const lb200_transform* parent_transforms, const float* original_scale3, lb200_transform* out_transforms);
/* The same with every table in device memory and the transforms left there: the device-side chain pose -> attached entity transform ->
 * lb200_sortkeys_move_device -> lb200_culling_set_many_device -> cull (SURVEY 8f N4).  No index validation.  Both forms move the attached
 * entities alone: for attachments inside a hierarchy (parent globals read from it, the attached subtrees and the locals following,
 * attachments of attachments) use lb200_hierarchy_set_attachments + lb200_hierarchy_propagate_attached. */
LB200_API int lb200_animation_bone_attachments_device(lb200_animation* a, uint32_t n, const uint32_t* dev_instance, const uint32_t* dev_bone, const float* dev_relative7,
                                                      const lb200_transform* dev_parent_transforms, const float* dev_original_scale3, lb200_transform* dev_out_transforms);
LB200_API int lb200_animation_get_times(lb200_animation* a, uint32_t first, uint32_t count, uint32_t* out_ticks);
LB200_API int lb200_animation_get_skinned(lb200_animation* a, uint32_t first, uint32_t count, float* out_pos3);
/* Checksum of the skinned vertex buffer computed on the device (sum of the raw u32 bit patterns, mod 2^64) —
 * a size-independent property for full-size parity runs. */
LB200_API int lb200_animation_skinned_checksum(lb200_animation* a, uint64_t* out);
LB200_API uint64_t lb200_animation_algorithmic_bytes(const lb200_animation* a, uint32_t palette_flags, int skin);

/* ------------------------------------------------------------------------------------------------------------
 * Skinning palettes of the instances createSortKeys claims — PoseProcessor::push + computeSkeletonDualQuats
 * (src/renderer/pipeline.cpp:3730-3787, 2680-2745) on the device, for the pose lists lb200_sortkeys_create_keys[_views] left in HBM.
 * ---------------------------------------------------------------------------------------------------------- */
/* The entity each instance poses: entity_of_instance[i] = EntityRef::index of the ModelInstance whose Pose instance i writes, negative =
 * none.  Host array, copied before the call returns; instances at or past n have no entity.  set_instances, set_samples and set_stacks
 * leave the table alone.  LB200_ERR_INVALID, with nothing changed: n > max_instances, NULL entity_of_instance with n > 0, a
 * non-negative id listed twice.  Precedent: lb200_hierarchy_set_entities. */
LB200_API int lb200_animation_set_entities(lb200_animation* a, const int32_t* entity_of_instance, uint32_t n);
typedef struct {
	const float* dual_quats;  /* DualQuat per bone (r xyzw, d xyzw: 32 B), the slices of every palette the build wrote */
	const uint32_t* offset;   /* per entity, max_entities long: first bone of its slice in dual_quats, 0xffffffff = listed, no instance */
	const uint32_t* n_bones;  /* bones written (one word) */
} lb200_sk_palettes;
/* For every entity e of the pose list of the latest create_keys (views == 0), or of every view's pose list of the latest create_keys_views
 * (views == 1), in one pass: the instance of `systems` whose entity id is e (lb200_animation_set_entities; if several are, one of them)
 * writes its bone_count dual quaternions to_dual_quat(pose_abs[b] * inv_bind[b]) into a slice of one palette buffer, and offset[e] = the
 * slice's first bone.  The draw stage reads the palette of a DRAW_SKINNED value's entity e at dual_quats + 8 * offset[e].
 * - Bits: exactly what lb200_animation_update(..., LB200_PALETTE_DUAL_QUAT) writes for that instance from the same poses.
 * - A listed entity no instance lists gets offset 0xffffffff and nothing is written: a skinned model without an animation component
 *   keeps Model::getPose's palette, which stays on the host.  Entities not listed keep the offset they had.
 * - Slices are disjoint and contiguous (32-byte aligned) and *n_bones is their sum; their order is not specified.  The buffer holds the
 *   bones of every instance with an entity id, so a build cannot run out of room.
 * - Execution: asynchronous on the context stream, no read-back; the list lengths are read on the device, clamped to the lists'
 *   capacity.  Host work grows with the number of systems, not of instances.  One launch maps entities to instances and one builds
 *   palettes per 64 systems (one build launch for an empty list).
 * - Buffers are allocated or grown before anything is launched (a build that grows the palette buffer waits for the stream first); a
 *   failed allocation returns LB200_ERR_CUDA with the earlier outputs intact.  The pointers stay valid until the next build_palettes;
 *   a spawn that grows max_entities grows `offset` too, keeping its contents, and makes pointers handed out before it stale.
 * - Refused, with the earlier outputs as they were: LB200_ERR_INVALID for NULL out, NULL systems with n_systems > 0, a NULL entry, a
 *   system listed twice, a system of another context, views other than 0 / 1; LB200_ERR_STATE for a system with instances that have
 *   entity ids but no absolute poses yet (no update with LB200_PALETTE_POSE), views == 1 before any create_keys_views and views == 0
 *   before any create_keys. */
LB200_API int lb200_sortkeys_build_palettes(lb200_sortkeys* sk, lb200_animation* const* systems, uint32_t n_systems, int views, lb200_sk_palettes* out);

/* ------------------------------------------------------------------------------------------------------------
 * Light clusters — PipelineImpl::fillClusters (src/renderer/pipeline.cpp:3327-3684) on the device, for the LOCAL_LIGHT ids a view's
 * cull left in HBM: the per-light ClusterLight records, the shadow-atlas candidates of AtlasSorter (:2375-2401) and the binning of
 * lights, environment probes and reflection probes into the 64 px x 64 px x 16 froxel grid (clusters[] and map[]).  The shadow atlas
 * (allocation, bakeShadow, shadow matrices) and the probe arrays stay with the host, as in the reference.
 * ---------------------------------------------------------------------------------------------------------- */
typedef struct lb200_clusters lb200_clusters;
#define LB200_LIGHT_CAST_SHADOWS 1u   /* PointLight::CAST_SHADOWS */
#define LB200_LIGHT_DYNAMIC 2u        /* PointLight::DYNAMIC */
#define LB200_CLUSTERS_LAST_CULL 0xffffffffu /* lb200_cluster_view.view: the last cull of the culling system (a lone cull, or select_view's) */
#define LB200_CLUSTERS_MAX_ATLAS 64   /* ShadowAtlas::inv_map (pipeline.cpp:267) and AtlasSorter::lights (:2399) hold 64 entries */
/* The PointLight fields fillClusters reads (render_module.h:156-171).  32 bytes. */
typedef struct {
	float color[3];
	float intensity;
	float fov;
	float attenuation_param;
	float range;
	uint32_t flags;               /* LB200_LIGHT_* */
} lb200_point_light;
/* fillClusters' ClusterLight (:3331-3341), 64 bytes; padding is written as zero. */
typedef struct {
	float pos[3];                 /* Vec3(transform.pos - cam_pos): the difference in fp64, each component then rounded to fp32 */
	float radius;                 /* range */
	float rot[4];                 /* the transform's rotation */
	float color[3];               /* color * intensity */
	float attenuation_param;
	uint32_t atlas_idx;           /* shadow-atlas entry, 0xffffffff = none */
	float fov;
	float padding[2];
} lb200_cluster_light;
/* Cluster (:3343-3348): the cluster's entries are map[offset, offset + lights_count + env_probes_count + refl_probes_count), lights
 * first, then environment probes, then reflection probes, each kind in increasing index. */
typedef struct { uint32_t offset, lights_count, env_probes_count, refl_probes_count; } lb200_cluster;
/* ClusterEnvProbe (:3350-3359, 208 bytes) and ClusterReflProbe (:3361-3367, 48 bytes) as the host fills and sorts them (:3497-3538).
 * The binning reads pos and outer_range / half_extents. */
typedef struct {
	float pos[3]; float pad0;
	float rot[4];
	float inner_range[3]; float pad1;
	float outer_range[3]; float pad2;
	float sh_coefs[9][4];
} lb200_cluster_env_probe;
typedef struct {
	float pos[3]; uint32_t layer;
	float rot[4];
	float half_extents[3]; float pad1;
} lb200_cluster_refl_probe;
typedef struct {
	double cam_pos[3];            /* CameraParams::pos */
	uint32_t w, h;                /* the pipeline's viewport in pixels, 1 .. 4096 each */
	uint32_t view;                /* view k of the latest lb200_culling_cull_views, or LB200_CLUSTERS_LAST_CULL */
	uint32_t pad;
	lb200_shifted_frustum frustum; /* CameraParams::frustum: the planes are built from its points */
} lb200_cluster_view;
/* One entry of AtlasSorter::lights. */
typedef struct { uint32_t light_idx; float priority; int32_t entity; } lb200_shadow_candidate;
typedef struct {
	uint32_t n_lights;            /* visible lights = entries of lights[] and light_entities[] */
	uint32_t n_clusters;          /* size[0] * size[1] * size[2] */
	uint32_t n_map;               /* entries of map[] */
	uint32_t size[3];             /* ((w + 63) / 64, (h + 63) / 64, 16) */
	uint32_t n_shadow;            /* AtlasSorter::count */
	lb200_shadow_candidate shadow[LB200_CLUSTERS_MAX_ATLAS];
	uint32_t n_uncast;            /* visible lights without CAST_SHADOWS whose entity has an atlas entry, in light order (:3405-3407) */
	int32_t uncast[LB200_CLUSTERS_MAX_ATLAS]; /* their entities */
} lb200_cluster_result;
typedef struct {                  /* device pointers, valid until the next lb200_clusters_fill */
	const lb200_cluster_light* lights;  /* n_lights */
	const lb200_cluster* clusters;      /* n_clusters */
	const int32_t* map;                 /* n_map */
	const int32_t* light_entities;      /* n_lights: the entity of light i, in the order of the cull's LOCAL_LIGHT segment */
} lb200_cluster_outputs;
/* Per-entity tables for entity ids [0, max_entities): point lights start as all zero, atlas entries as none. */
LB200_API int lb200_clusters_create(lb200_ctx* ctx, uint32_t max_entities, lb200_clusters** out);
LB200_API void lb200_clusters_destroy(lb200_clusters* cl);
/* RenderModule's point lights: records[i] for entity entities[i].  LB200_ERR_INVALID, nothing changed: NULL arrays with n > 0, an entity
 * outside [0, max_entities) or listed twice. */
LB200_API int lb200_clusters_set_point_lights(lb200_clusters* cl, const int32_t* entities, const lb200_point_light* records, uint32_t n);
/* ShadowAtlas::map: entity entities[i] gets entry atlas_idx[i], -1 removes its entry, in list order.  LB200_ERR_INVALID, nothing changed:
 * NULL arrays with n > 0, an entity outside [0, max_entities), an index outside -1 .. 63, more than LB200_CLUSTERS_MAX_ATLAS entities
 * with an entry afterwards. */
LB200_API int lb200_clusters_set_atlas(lb200_clusters* cl, const int32_t* entities, const int32_t* atlas_idx, uint32_t n);
/* fillClusters up to the host's atlas step, for the LOCAL_LIGHT segment of the chosen cull of cs, on the context stream:
 *  - lights[i] and light_entities[i] for the i-th id of the segment, transforms from sk's entity records (set_transforms[_device],
 *    move_device and spawns keep them current);
 *  - result->shadow: the list AtlasSorter::push leaves after the CAST_SHADOWS lights are pushed in light order with
 *    computeShadowPriority (:3322-3325), ties and NaN priorities included (a NaN fov gives the device's canonical NaN, bits
 *    0x7fffffff, as the priority, where x86 keeps the input's payload); result->uncast: what :3405-3407 removes from the atlas;
 *  - the planes of :3468-3495 (built on the host in fp32, as the reference builds them), range() per axis (:3540-3561) for every light
 *    (radius = range), env probe (length(outer_range)) and refl probe (length(half_extents)), and clusters[] / map[] exactly as the
 *    count, offset and scatter passes of :3628-3666 leave them.
 * Byte for byte the reference's output for the light order of the cull; for a fixed light order every run gives the same bytes.
 * Kernels: four launches whatever the number of lights (four more when map[] grows).  The call reads back `result` (one copy) and
 * waits for it.  map[] grows as needed and keeps its capacity; a growth re-runs the call's kernels once.
 * LB200_ERR_INVALID, with the earlier outputs as they were: NULL view / result, NULL probes with a count > 0, w or h of 0 or above 4096
 * (xplanes[65] of the reference holds 64 columns), a view index at or past the latest cull_views' count, a culling system whose entity
 * ids reach past sk's or cl's max_entities, an sk without transforms, an sk or cs of another context.  LB200_ERR_STATE where the chosen
 * cull does not exist. */
LB200_API int lb200_clusters_fill(lb200_clusters* cl, lb200_sortkeys* sk, lb200_culling* cs, const lb200_cluster_view* view,
                                  const lb200_cluster_env_probe* env_probes, uint32_t n_env, const lb200_cluster_refl_probe* refl_probes,
                                  uint32_t n_refl, lb200_cluster_result* result);
/* The atlas step's outcome (:3414-3437): lights[light_idx[i]].atlas_idx = atlas_idx[i] on the device, in list order (-1 is written as
 * 0xffffffff, no entry).  Asynchronous.  LB200_ERR_STATE before a fill; LB200_ERR_INVALID (nothing written) for NULL arrays with n > 0,
 * a light index at or past the last fill's n_lights or an atlas index outside -1 .. 63. */
LB200_API int lb200_clusters_patch_atlas(lb200_clusters* cl, const uint32_t* light_idx, const int32_t* atlas_idx, uint32_t n);
/* Device pointers of the last fill's lights, clusters, map and light entities (LB200_ERR_STATE before a fill). */
LB200_API int lb200_clusters_outputs(lb200_clusters* cl, lb200_cluster_outputs* out);
/* Grid of clusters_items_kernel in later fills.  blocks: 0 = the default (one block per 256 items the cull can emit plus the probes,
 * at most every co-resident block), -1 = every co-resident block, n > 0 = min(n, co-resident blocks); only 0 caps the grid by the work.
 * Any other value is LB200_ERR_INVALID, with nothing changed.  Outputs do not depend on the grid.  get_launch reports the last fill: its
 * items-kernel grid and the tiles of 256 items per block, ceil(ceil(n_items / grid) / 256) for the fill's lights and probes (both 0
 * before the first fill). */
LB200_API int lb200_clusters_set_launch(lb200_clusters* cl, int blocks);
LB200_API int lb200_clusters_get_launch(lb200_clusters* cl, uint32_t* grid, uint32_t* tiles_per_block);

#ifdef __cplusplus
}
#endif
#endif /* LUMIX_B200_H */
