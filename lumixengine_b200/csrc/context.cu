// Context lifecycle + host-side frustum construction of the C-ABI (include/lumix_b200.h).
#include "lb200_internal.h"
#include <stdlib.h>
#include "lb200_math.cuh"

static char g_init_error[512] = {0};

uint32_t lb200_cull_lanes() {
	static const uint32_t lanes = [] {
		const char* e = getenv("LB200_CULL_LANES");
		const int v = e ? atoi(e) : 2; // H100: 2 lanes x 2 blocks/SM beat 3 / 4 / 6 lanes (DESIGN.md 4.1)
		return (uint32_t)(v < 1 ? 1 : (v > LB200_MAX_LANES ? LB200_MAX_LANES : v));
	}();
	return lanes;
}

void lb200_set_error(lb200_ctx* ctx, const char* fmt, ...) {
	char* dst = ctx ? ctx->error : g_init_error;
	va_list args;
	va_start(args, fmt);
	vsnprintf(dst, 512, fmt, args);
	va_end(args);
}

int lb200_coop_grid_limit(lb200_ctx* ctx, const void* kernel, int threads, size_t smem, uint32_t* out) {
	int per_sm = 0;
	LB200_CUDA(ctx, cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, smem));
	if (per_sm < 1) { lb200_set_error(ctx, "cooperative kernel does not fit on an SM (%zu B of shared memory)", smem); return LB200_ERR_CUDA; }
	*out = (uint32_t)per_sm * (uint32_t)ctx->sm_count;
	return LB200_OK;
}

extern "C" {

int lb200_device_count(void) {
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) {
		cudaGetLastError();
		return 0;
	}
	return n;
}

static int initContext(int device_ordinal, int stream_priority_low, lb200_ctx** out_ctx);

int lb200_init(int device_ordinal, lb200_ctx** out_ctx) { return initContext(device_ordinal, 0, out_ctx); }

// A second context of a device whose stream yields to the others: for work that should fill the device only where latency-critical
// streams (cull, exchange) leave room — e.g. the animation update running next to the culling of the same frame.
int lb200_init_background(int device_ordinal, lb200_ctx** out_ctx) { return initContext(device_ordinal, 1, out_ctx); }

static int initContext(int device_ordinal, int stream_priority_low, lb200_ctx** out_ctx) {
	if (!out_ctx) return LB200_ERR_INVALID;
	*out_ctx = nullptr;
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess || n == 0) {
		cudaGetLastError();
		lb200_set_error(nullptr, "no CUDA device (%s): lumix_b200 has no CPU path", e == cudaSuccess ? "device count 0" : cudaGetErrorString(e));
		return LB200_ERR_NO_DEVICE;
	}
	if (device_ordinal < 0 || device_ordinal >= n) {
		lb200_set_error(nullptr, "device ordinal %d out of range [0,%d)", device_ordinal, n);
		return LB200_ERR_INVALID;
	}
	lb200_ctx* ctx = new lb200_ctx;
	ctx->device = device_ordinal;
	int prio_least = 0, prio_greatest = 0;
	if ((e = cudaSetDevice(device_ordinal)) != cudaSuccess
		|| (e = cudaDeviceGetStreamPriorityRange(&prio_least, &prio_greatest)) != cudaSuccess
		|| (e = cudaStreamCreateWithPriority(ctx->stream.create(), cudaStreamNonBlocking, stream_priority_low ? prio_least : prio_greatest)) != cudaSuccess
		|| (e = cudaStreamCreateWithFlags(ctx->copy_stream.create(), cudaStreamNonBlocking)) != cudaSuccess
		|| (e = cudaDeviceGetAttribute(&ctx->sm_count, cudaDevAttrMultiProcessorCount, device_ordinal)) != cudaSuccess) {
		lb200_set_error(nullptr, "context creation failed: %s", cudaGetErrorString(e));
		delete ctx;
		return LB200_ERR_CUDA;
	}
	*out_ctx = ctx;
	return LB200_OK;
}

void lb200_shutdown(lb200_ctx* ctx) {
	if (!ctx) return;
	lb200_comm_destroy(ctx);
	cudaSetDevice(ctx->device);
	if (ctx->stream) cudaStreamSynchronize(ctx->stream);
	if (ctx->copy_stream) cudaStreamSynchronize(ctx->copy_stream);
	delete ctx;
}

const char* lb200_last_error(const lb200_ctx* ctx) { return ctx ? ctx->error : g_init_error; }

int lb200_synchronize(lb200_ctx* ctx) {
	if (!ctx) return LB200_ERR_INVALID;
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return lb200_comm_check(ctx);
}

int lb200_host_callback(lb200_ctx* ctx, void (*fn)(void*), void* user) {
	if (!ctx || !fn) return LB200_ERR_INVALID;
	LB200_CUDA(ctx, cudaLaunchHostFunc(ctx->stream, fn, user));
	return LB200_OK;
}

// The C API's allocations and events belong to the caller, who frees them with the matching call below: raw, not handles.
void* lb200_host_alloc(lb200_ctx* ctx, size_t bytes) {
	if (!ctx) return nullptr;
	void* p = nullptr;
	cudaSetDevice(ctx->device);
	if (cudaHostAlloc(&p, bytes ? bytes : 1, cudaHostAllocPortable) != cudaSuccess) {
		lb200_set_error(ctx, "cudaHostAlloc(%zu) failed: %s", bytes, cudaGetErrorString(cudaGetLastError()));
		return nullptr;
	}
	return p;
}

void lb200_host_free(lb200_ctx* ctx, void* p) {
	(void)ctx;
	if (p) cudaFreeHost(p);
}

void* lb200_device_alloc(lb200_ctx* ctx, size_t bytes) {
	if (!ctx) return nullptr;
	void* p = nullptr;
	cudaSetDevice(ctx->device);
	if (cudaMalloc(&p, bytes ? bytes : 1) != cudaSuccess) {
		lb200_set_error(ctx, "cudaMalloc(%zu) failed: %s", bytes, cudaGetErrorString(cudaGetLastError()));
		return nullptr;
	}
	return p;
}

void lb200_device_free(lb200_ctx* ctx, void* p) {
	if (!ctx || !p) return;
	cudaSetDevice(ctx->device);
	cudaStreamSynchronize(ctx->stream);
	cudaFree(p);
}

int lb200_copy_to_device(lb200_ctx* ctx, void* dst_device, const void* src_host, size_t bytes) {
	if (!ctx || (bytes && (!dst_device || !src_host))) return LB200_ERR_INVALID;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(dst_device, src_host, bytes, cudaMemcpyHostToDevice, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

int lb200_copy_to_host(lb200_ctx* ctx, void* dst_host, const void* src_device, size_t bytes) {
	if (!ctx || (bytes && (!dst_host || !src_device))) return LB200_ERR_INVALID;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaMemcpyAsync(dst_host, src_device, bytes, cudaMemcpyDeviceToHost, ctx->stream));
	LB200_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
	return LB200_OK;
}

int lb200_event_create(lb200_ctx* ctx, void** out_event) {
	if (!ctx || !out_event) return LB200_ERR_INVALID;
	cudaEvent_t e;
	LB200_CUDA(ctx, cudaSetDevice(ctx->device));
	LB200_CUDA(ctx, cudaEventCreate(&e));
	*out_event = e;
	return LB200_OK;
}

int lb200_event_record(lb200_ctx* ctx, void* event) {
	if (!ctx || !event) return LB200_ERR_INVALID;
	LB200_CUDA(ctx, cudaEventRecord((cudaEvent_t)event, ctx->stream));
	return LB200_OK;
}

int lb200_event_elapsed_ms(lb200_ctx* ctx, void* start, void* stop, float* out_ms) {
	if (!ctx || !start || !stop || !out_ms) return LB200_ERR_INVALID;
	LB200_CUDA(ctx, cudaEventSynchronize((cudaEvent_t)stop));
	LB200_CUDA(ctx, cudaEventElapsedTime(out_ms, (cudaEvent_t)start, (cudaEvent_t)stop));
	return LB200_OK;
}

void lb200_event_destroy(lb200_ctx* ctx, void* event) {
	(void)ctx;
	if (event) cudaEventDestroy((cudaEvent_t)event);
}

uint64_t lb200_launch_count(const lb200_ctx* ctx) { return ctx ? ctx->launches.load() : 0; }
uint64_t lb200_stream_handle(const lb200_ctx* ctx) { return ctx ? (uint64_t)(uintptr_t)(cudaStream_t)ctx->stream : 0; }

// ---------------------------------------------------------------------------------------------------------------
// Frustum construction (host).  geometry.cpp:311-351 (setPoints / setPlanesFromPoints), :421-427 (setPlane),
// :390-409 (computeOrtho), :470-499 (computePerspective).  Kept on the host exactly as the engine does (SURVEY a8).
// ---------------------------------------------------------------------------------------------------------------
using namespace lb;

static void setPlane(lb200_shifted_frustum* f, int side, V3 normal, V3 point) {
	f->xs[side] = normal.x;
	f->ys[side] = normal.y;
	f->zs[side] = normal.z;
	f->ds[side] = -dot(point, normal);
}

static V3 pt(const lb200_shifted_frustum* f, int i) { return v3(f->points[i][0], f->points[i][1], f->points[i][2]); }

static void setPlanesFromPoints(lb200_shifted_frustum* f) {
	enum { NEAR_ = 0, FAR_, LEFT_, RIGHT_, TOP_, BOTTOM_, EXTRA0_, EXTRA1_ };
	const V3 normal_near = neg(normalize(cross(sub(pt(f, 0), pt(f, 1)), sub(pt(f, 0), pt(f, 2)))));
	const V3 normal_far = normalize(cross(sub(pt(f, 4), pt(f, 5)), sub(pt(f, 4), pt(f, 6))));
	setPlane(f, EXTRA0_, normal_near, pt(f, 0));
	setPlane(f, EXTRA1_, normal_near, pt(f, 0));
	setPlane(f, NEAR_, normal_near, pt(f, 0));
	setPlane(f, FAR_, normal_far, pt(f, 4));
	setPlane(f, LEFT_, normalize(cross(sub(pt(f, 1), pt(f, 2)), sub(pt(f, 1), pt(f, 5)))), pt(f, 1));
	setPlane(f, RIGHT_, neg(normalize(cross(sub(pt(f, 0), pt(f, 3)), sub(pt(f, 0), pt(f, 4))))), pt(f, 0));
	setPlane(f, TOP_, normalize(cross(sub(pt(f, 0), pt(f, 1)), sub(pt(f, 0), pt(f, 4)))), pt(f, 0));
	setPlane(f, BOTTOM_, normalize(cross(sub(pt(f, 2), pt(f, 3)), sub(pt(f, 2), pt(f, 6)))), pt(f, 2));
}

static void setPoints(lb200_shifted_frustum* f, V3 near_center, V3 far_center, V3 right_near, V3 up_near, V3 right_far, V3 up_far) {
	const float vmin = -1, vmax = 1;
	const V3 p[8] = {
		add(add(near_center, muls(right_near, vmax)), muls(up_near, vmax)),
		add(add(near_center, muls(right_near, vmin)), muls(up_near, vmax)),
		add(add(near_center, muls(right_near, vmin)), muls(up_near, vmin)),
		add(add(near_center, muls(right_near, vmax)), muls(up_near, vmin)),
		add(add(far_center, muls(right_far, vmax)), muls(up_far, vmax)),
		add(add(far_center, muls(right_far, vmin)), muls(up_far, vmax)),
		add(add(far_center, muls(right_far, vmin)), muls(up_far, vmin)),
		add(add(far_center, muls(right_far, vmax)), muls(up_far, vmin)),
	};
	for (int i = 0; i < 8; ++i) { f->points[i][0] = p[i].x; f->points[i][1] = p[i].y; f->points[i][2] = p[i].z; }
	setPlanesFromPoints(f);
}

void lb200_frustum_perspective(lb200_shifted_frustum* f, const double position[3], const float direction[3], const float up_[3],
	float fov, float ratio, float near_distance, float far_distance)
{
	memset(f, 0, sizeof(*f));
	const V3 dir = v3(direction[0], direction[1], direction[2]);
	const V3 up = v3(up_[0], up_[1], up_[2]);
	const float scale = tanf(fov * 0.5f);
	const V3 right = cross(dir, up);
	const V3 up_near = muls(muls(up, near_distance), scale);
	const V3 right_near = muls(right, near_distance * scale * ratio);
	const V3 up_far = muls(muls(up, far_distance), scale);
	const V3 right_far = muls(right, far_distance * scale * ratio);
	const V3 z = normalize(dir);
	const V3 near_center = muls(z, near_distance);
	const V3 far_center = muls(z, far_distance);
	f->origin[0] = position[0]; f->origin[1] = position[1]; f->origin[2] = position[2];
	setPoints(f, near_center, far_center, right_near, up_near, right_far, up_far);
}

void lb200_frustum_ortho(lb200_shifted_frustum* f, const double position[3], const float direction[3], const float up_[3],
	float width, float height, float near_distance, float far_distance)
{
	memset(f, 0, sizeof(*f));
	const V3 dir = v3(direction[0], direction[1], direction[2]);
	const V3 up = v3(up_[0], up_[1], up_[2]);
	const V3 z = normalize(dir);
	f->origin[0] = position[0]; f->origin[1] = position[1]; f->origin[2] = position[2];
	const V3 near_center = muls(neg(z), near_distance);
	const V3 far_center = muls(neg(z), far_distance);
	const V3 x = muls(normalize(cross(up, z)), width);
	const V3 y = muls(normalize(cross(z, x)), height);
	setPoints(f, near_center, far_center, x, y, x, y);
}

// Viewport::getFrustum(), geometry.cpp:793-818: direction / up from the camera rotation (Quat * Vec3 = rotate, math.cpp:721-724),
// ratio = h > 0 ? w / (float)h : 1; the reference builds at the origin and then stores pos, which gives the same bytes.
void lb200_frustum_from_viewport(lb200_shifted_frustum* f, int is_ortho, float fov, float ortho_size, int w, int h, const double pos[3],
	const float rot[4], float near_distance, float far_distance)
{
	const Q4 q = q4(rot[0], rot[1], rot[2], rot[3]);
	const float ratio = h > 0 ? w / (float)h : 1;
	const V3 up = rotate(q, v3(0, 1, 0));
	const float up3[3] = {up.x, up.y, up.z};
	if (is_ortho) {
		const V3 d = rotate(q, v3(0, 0, 1));
		const float d3_[3] = {d.x, d.y, d.z};
		lb200_frustum_ortho(f, pos, d3_, up3, ortho_size * ratio, ortho_size, near_distance, far_distance);
		return;
	}
	const V3 d = rotate(q, v3(0, 0, -1));
	const float d3_[3] = {d.x, d.y, d.z};
	lb200_frustum_perspective(f, pos, d3_, up3, fov, ratio, near_distance, far_distance);
}

} // extern "C"
