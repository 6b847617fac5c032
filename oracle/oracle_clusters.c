/* TEST INFRASTRUCTURE — C restatement of PipelineImpl::fillClusters (src/renderer/pipeline.cpp:3327-3684) up to the host's atlas step:
 * the ClusterLight records (:3388-3396), AtlasSorter::push (:2375-2401) with computeShadowPriority (:3322-3325), the lights the host
 * removes from the atlas (:3405-3407), the planes (:3468-3495), range() (:3540-3561) and the count / offset / map passes (:3563-3666).
 * Built by oracle/Makefile with the reference's flags (SSE2, no FMA, no fast-math); pinned to the reference's own code
 * (oracle/_ref/libclusters_shim_b200.so) and to tests/golden/clusters_kat.npz by tests/test_clusters_cpu.py.
 *
 * Inputs are per light, in light order: entity, world position (fp64), rotation, the PointLight fields (32 bytes, lb200_point_light) and
 * the entity's atlas entry (-1 = none).  Probes are ClusterEnvProbe (208 bytes) / ClusterReflProbe (48 bytes) as the host sorted them. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float x, y, z; } v3;
typedef struct { float x, y, z, w; } v4;
typedef struct { float color[3], intensity, fov, attenuation_param, range; uint32_t flags; } point_light;
typedef struct { float pos[3], radius, rot[4], color[3], attenuation_param; uint32_t atlas_idx; float fov, padding[2]; } cluster_light;
typedef struct { uint32_t offset, lights_count, env_probes_count, refl_probes_count; } cluster;
typedef struct { uint32_t idx; float priority; int32_t entity; } sorter_light;

static v3 sub3(v3 a, v3 b) { v3 r = {a.x - b.x, a.y - b.y, a.z - b.z}; return r; }
static v3 mul3(v3 a, float s) { v3 r = {a.x * s, a.y * s, a.z * s}; return r; }
static v3 cross3(v3 a, v3 b) { v3 r = {a.y * b.z - a.z * b.y, a.z * b.x - a.x * b.z, a.x * b.y - a.y * b.x}; return r; }
static float dot3(v3 a, v3 b) { return a.x * b.x + a.y * b.y + a.z * b.z; }
static v3 normalize3(v3 v) {
	const float inv_len = 1 / sqrtf(v.x * v.x + v.y * v.y + v.z * v.z);
	v3 r = {v.x * inv_len, v.y * inv_len, v.z * inv_len};
	return r;
}
static v3 lerp3(v3 a, v3 b, float t) {
	const float invt = 1.0f - t;
	v3 r = {a.x * invt + b.x * t, a.y * invt + b.y * t, a.z * invt + b.z * t};
	return r;
}
static v4 plane(v3 n, v3 p) { v4 r = {n.x, n.y, n.z, -dot3(n, p)}; return r; }
static float plane_dist(v4 pl, v3 p) { return pl.x * p.x + pl.y * p.y + pl.z * p.z + pl.w; }

/* xplanes[65], yplanes[65], zplanes[17] of the viewport w x h (:3468-3495); entries past size + 1 are zero */
void oc_cluster_planes(const float points[24], int w, int h, float xplanes[65 * 4], float yplanes[65 * 4], float zplanes[17 * 4]) {
	v3 pt[8];
	for (int i = 0; i < 8; ++i) { pt[i].x = points[3 * i]; pt[i].y = points[3 * i + 1]; pt[i].z = points[3 * i + 2]; }
	const int sx = (w + 63) / 64, sy = (h + 63) / 64, sz = 16;
	memset(xplanes, 0, sizeof(float) * 65 * 4);
	memset(yplanes, 0, sizeof(float) * 65 * 4);
	memset(zplanes, 0, sizeof(float) * 17 * 4);
	const v3 cam_dir = normalize3(cross3(sub3(pt[2], pt[0]), sub3(pt[1], pt[0])));
	for (int i = 0; i < sz + 1; ++i) {
		const float znear = 0.1f, zfar = 10000.0f;
		const float z = znear * powf(zfar / znear, i / (float)sz);
		const v4 p = plane(cam_dir, mul3(cam_dir, z));
		memcpy(zplanes + 4 * i, &p, sizeof(p));
	}
	for (int i = 0; i < sy + 1; ++i) {
		const float t = i / (float)sy;
		const v3 a = lerp3(pt[0], pt[3], t), b = lerp3(pt[1], pt[2], t), c = lerp3(pt[4], pt[7], t);
		const v4 p = plane(normalize3(cross3(sub3(b, a), sub3(c, a))), a);
		memcpy(yplanes + 4 * i, &p, sizeof(p));
	}
	for (int i = 0; i < sx + 1; ++i) {
		const float t = i / (float)sx;
		const v3 a = lerp3(pt[1], pt[0], t), b = lerp3(pt[2], pt[3], t), c = lerp3(pt[5], pt[4], t);
		const v4 p = plane(normalize3(cross3(sub3(b, a), sub3(c, a))), a);
		memcpy(xplanes + 4 * i, &p, sizeof(p));
	}
}

/* range() of :3540-3561: out[0] = first cluster, out[1] = one past the last, both -1 if none */
void oc_cluster_range(const float p3[3], float r, int size, const float* planes4, int out[2]) {
	const v3 p = {p3[0], p3[1], p3[2]};
	const v4* planes = (const v4*)planes4;
	out[0] = -1; out[1] = -1;
	if (plane_dist(planes[0], p) < -r) return;
	for (int i = 0; i < size; ++i) {
		const float dist = plane_dist(planes[i + 1], p);
		if (dist > r) continue;
		out[0] = i;
		for (int i2 = i + 1; i2 < size + 1; ++i2) {
			if (plane_dist(planes[i2], p) < -r) { out[1] = i2; return; }
		}
		out[1] = size;
		return;
	}
}

/* AtlasSorter::push */
static void sorter_push(sorter_light* lights, uint32_t* count, uint32_t light_idx, float priority, int32_t e) {
	uint32_t idx = 0;
	while (idx < *count) {
		if (lights[idx].priority < priority) break;
		++idx;
	}
	if (idx == 64) return;
	if (*count == 64) --*count;
	memmove(&lights[idx + 1], &lights[idx], sizeof(lights[0]) * (*count - idx));
	lights[idx].idx = light_idx;
	lights[idx].priority = priority;
	lights[idx].entity = e;
	++*count;
}

/* Returns the entries map[] needs; map is written up to map_cap.  clusters: ((w+63)/64) ((h+63)/64) 16 entries.  shadow: 64 entries,
 * uncast: n_lights entries. */
uint32_t oc_clusters_fill(const float points[24], int w, int h, const double cam[3], uint32_t n_lights, const int32_t* entities, const double* pos3,
	const float* rot4, const void* point_lights, const int32_t* atlas, uint32_t n_env, const void* env_probes, uint32_t n_refl, const void* refl_probes,
	void* lights_out, void* clusters_out, int32_t* map, uint32_t map_cap, uint32_t* n_shadow, void* shadow_out, uint32_t* n_uncast, int32_t* uncast)
{
	const point_light* pls = (const point_light*)point_lights;
	cluster_light* lights = (cluster_light*)lights_out;
	cluster* clusters = (cluster*)clusters_out;
	sorter_light* sorter = (sorter_light*)shadow_out;
	uint32_t count = 0, uncast_count = 0;
	memset(lights, 0, sizeof(cluster_light) * n_lights);
	for (uint32_t i = 0; i < n_lights; ++i) {
		const point_light* pl = &pls[i];
		cluster_light* light = &lights[i];
		light->radius = pl->range;
		for (int c = 0; c < 3; ++c) light->pos[c] = (float)(pos3[3 * i + c] - cam[c]);
		memcpy(light->rot, rot4 + 4 * i, sizeof(light->rot));
		light->fov = pl->fov;
		for (int c = 0; c < 3; ++c) light->color[c] = pl->color[c] * pl->intensity;
		light->attenuation_param = pl->attenuation_param;
		if (pl->flags & 1u) {
			light->atlas_idx = atlas[i] >= 0 ? (uint32_t)atlas[i] : 0xffffffffu;
			const float lr3 = light->radius * light->radius * light->radius;
			const double dx = cam[0] - pos3[3 * i], dy = cam[1] - pos3[3 * i + 1], dz = cam[2] - pos3[3 * i + 2];
			sorter_push(sorter, &count, i, (float)(light->fov * lr3 / sqrt(dx * dx + dy * dy + dz * dz)), entities[i]);
		} else {
			light->atlas_idx = 0xffffffffu;
			if (atlas[i] >= 0) uncast[uncast_count++] = entities[i];
		}
	}
	*n_shadow = count;
	*n_uncast = uncast_count;

	const int sx = (w + 63) / 64, sy = (h + 63) / 64, sz = 16;
	const uint32_t n_clusters = (uint32_t)(sx * sy * sz);
	float xplanes[65 * 4], yplanes[65 * 4], zplanes[17 * 4];
	oc_cluster_planes(points, w, h, xplanes, yplanes, zplanes);
	const uint32_t n_items = n_lights + n_env + n_refl;
	int* rng = (int*)malloc(sizeof(int) * 6 * (n_items ? n_items : 1));
	for (uint32_t g = 0; g < n_items; ++g) {
		float p[3], r;
		if (g < n_lights) {
			memcpy(p, lights[g].pos, sizeof(p));
			r = lights[g].radius;
		} else if (g < n_lights + n_env) {
			const float* e = (const float*)((const char*)env_probes + 208 * (size_t)(g - n_lights));
			memcpy(p, e, sizeof(p));
			const float* o = e + 12; /* outer_range */
			r = sqrtf(o[0] * o[0] + o[1] * o[1] + o[2] * o[2]);
		} else {
			const float* e = (const float*)((const char*)refl_probes + 48 * (size_t)(g - n_lights - n_env));
			memcpy(p, e, sizeof(p));
			const float* o = e + 8; /* half_extents */
			r = sqrtf(o[0] * o[0] + o[1] * o[1] + o[2] * o[2]);
		}
		oc_cluster_range(p, r, sx, xplanes, rng + 6 * g);
		oc_cluster_range(p, r, sy, yplanes, rng + 6 * g + 2);
		oc_cluster_range(p, r, sz, zplanes, rng + 6 * g + 4);
	}
	memset(clusters, 0, sizeof(cluster) * n_clusters);
	for (int pass = 0; pass < 2; ++pass) {
		if (pass == 1) {
			uint32_t offset = 0;
			for (uint32_t c = 0; c < n_clusters; ++c) {
				clusters[c].offset = offset;
				offset += clusters[c].lights_count + clusters[c].env_probes_count + clusters[c].refl_probes_count;
			}
		}
		for (uint32_t g = 0; g < n_items; ++g) {
			const int* q = rng + 6 * g;
			const int kind = g < n_lights ? 0 : g < n_lights + n_env ? 1 : 2;
			const int32_t index = (int32_t)(kind == 0 ? g : kind == 1 ? g - n_lights : g - n_lights - n_env);
			for (int z = q[4]; z < q[5]; ++z)
				for (int y = q[2]; y < q[3]; ++y)
					for (int x = q[0]; x < q[1]; ++x) {
						cluster* cl = &clusters[x + y * sx + z * sx * sy];
						if (pass == 0) {
							if (kind == 0) ++cl->lights_count; else if (kind == 1) ++cl->env_probes_count; else ++cl->refl_probes_count;
						} else {
							if (cl->offset < map_cap) map[cl->offset] = index;
							++cl->offset;
						}
					}
		}
	}
	uint32_t total = 0;
	for (uint32_t c = 0; c < n_clusters; ++c) {
		const uint32_t k = clusters[c].lights_count + clusters[c].env_probes_count + clusters[c].refl_probes_count;
		clusters[c].offset -= k;
		total += k;
	}
	free(rng);
	return total;
}
