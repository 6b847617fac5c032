// TEST INFRASTRUCTURE — runs the reference's own fillClusters code on plain inputs (oracle/build_ref.py compiles it into
// oracle/_ref/libclusters_shim_b200.so).  The build cuts AtlasSorter, computeShadowPriority, the Cluster* structs, the plane construction and
// range() + the for_each_*_pair lambdas + the count / offset / map passes out of the reference's pipeline.cpp into .inl files next to its
// sources; this file supplies the scope those pieces expect (lights, clusters, size, frustum, the probe arrays and a frame allocator).
// The light records and the atlas pushes are written out here as :3388-3408 does them, over the reference's own Vec3 / DVec3 / Quat
// operators.  Same entry point and arguments as oc_clusters_fill (oracle/oracle_clusters.c).
#include "core/geometry.h"
#include "core/math.h"
#include "engine/lumix.h"

#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

namespace Lumix {
#include "renderer/extracted_cluster_sorter.inl"
}

using namespace Lumix;

namespace {
struct PointLightIn { Vec3 color; float intensity; float fov; float attenuation_param; float range; u32 flags; };
static_assert(sizeof(PointLightIn) == 32, "lb200_point_light");
struct FrameAllocator {
	void* p = nullptr;
	void* allocate(size_t n, size_t) { p = malloc(n ? n : 1); return p; }
};
struct ModuleArray {
	u32 n;
	u32 length() const { return n; }
};
} // namespace

extern "C" __attribute__((visibility("default"))) uint32_t ref_clusters_fill(const float points[24], int w, int h, const double cam[3], uint32_t n_lights,
	const int32_t* entities, const double* pos3, const float* rot4, const void* point_lights, const int32_t* atlas, uint32_t n_env, const void* env_in,
	uint32_t n_refl, const void* refl_in, void* lights_out, void* clusters_out, int32_t* map_out, uint32_t map_cap, uint32_t* n_shadow, void* shadow_out,
	uint32_t* n_uncast, int32_t* uncast)
{
#include "renderer/extracted_cluster_types.inl"
	const IVec3 size((w + 63) / 64, (h + 63) / 64, 16);
	const u32 clusters_count = size.x * size.y * size.z;
	Cluster* clusters = (Cluster*)calloc(clusters_count, sizeof(Cluster));
	const u32 lights_count = n_lights;
	ClusterLight* lights = (ClusterLight*)calloc(n_lights ? n_lights : 1, sizeof(ClusterLight));
	const DVec3 cam_pos(cam[0], cam[1], cam[2]);
	const PointLightIn* pls = (const PointLightIn*)point_lights;
	AtlasSorter atlas_sorter;
	u32 uncast_count = 0;
	for (u32 i = 0; i < n_lights; ++i) {
		const PointLightIn& pl = pls[i];
		ClusterLight& light = lights[i];
		light.radius = pl.range;
		const DVec3 light_pos(pos3[3 * i], pos3[3 * i + 1], pos3[3 * i + 2]);
		light.pos = Vec3(light_pos - cam_pos);
		light.rot = Quat(rot4[4 * i], rot4[4 * i + 1], rot4[4 * i + 2], rot4[4 * i + 3]);
		light.fov = pl.fov;
		light.color = pl.color * pl.intensity;
		light.attenuation_param = pl.attenuation_param;
		if (pl.flags & 1) {
			light.atlas_idx = atlas[i] >= 0 ? (u32)atlas[i] : (u32)-1;
			EntityRef e;
			e.index = entities[i];
			atlas_sorter.push(i, computeShadowPriority(light.fov, light.radius, light_pos, cam_pos), e);
		} else {
			light.atlas_idx = -1;
			if (atlas[i] >= 0) uncast[uncast_count++] = entities[i];
		}
	}
	*n_shadow = atlas_sorter.count;
	*n_uncast = uncast_count;
	for (u32 i = 0; i < atlas_sorter.count; ++i) {
		uint32_t* s = (uint32_t*)shadow_out + 3 * i;
		s[0] = atlas_sorter.lights[i].idx;
		memcpy(s + 1, &atlas_sorter.lights[i].priority, 4);
		memcpy(s + 2, &atlas_sorter.lights[i].entity.index, 4);
	}

	ShiftedFrustum frustum;
	memcpy((void*)frustum.points, points, sizeof(float) * 24);
	const ModuleArray module_env_probes{n_env}, module_refl_probes{n_refl};
	ClusterEnvProbe* env_probes = (ClusterEnvProbe*)env_in;
	ClusterReflProbe* refl_probes = (ClusterReflProbe*)refl_in;
	FrameAllocator frame_allocator;
#include "renderer/extracted_cluster_planes.inl"
#include "renderer/extracted_cluster_binning.inl"
	memcpy(lights_out, lights, sizeof(ClusterLight) * n_lights);
	memcpy(clusters_out, clusters, sizeof(Cluster) * clusters_count);
	memcpy(map_out, map, sizeof(i32) * (offset < map_cap ? offset : map_cap));
	free(frame_allocator.p);
	free(lights);
	free(clusters);
	return offset;
}
