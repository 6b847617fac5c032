"""Host-side mirror of PipelineImpl::fillClusters (src/renderer/pipeline.cpp:3327-3684) on the device (csrc/clusters.cu,
include/lumix_b200.h "Light clusters"): ClusterLight records, the AtlasSorter list and the froxel binning of lights and probes for the
LOCAL_LIGHT ids a view's cull left in HBM."""
import ctypes as C

import numpy as np

from ._lib import ShiftedFrustum, check, ptr, vp

CAST_SHADOWS, DYNAMIC = 1, 2  # PointLight::Flags
LAST_CULL = 0xFFFFFFFF        # ClusterView.view: the last cull of the culling system
MAX_ATLAS = 64

POINT_LIGHT_DTYPE = np.dtype([("color", np.float32, 3), ("intensity", np.float32), ("fov", np.float32), ("attenuation_param", np.float32),
                              ("range", np.float32), ("flags", np.uint32)])
CLUSTER_LIGHT_DTYPE = np.dtype([("pos", np.float32, 3), ("radius", np.float32), ("rot", np.float32, 4), ("color", np.float32, 3),
                                ("attenuation_param", np.float32), ("atlas_idx", np.uint32), ("fov", np.float32), ("padding", np.float32, 2)])
CLUSTER_DTYPE = np.dtype([("offset", np.uint32), ("lights_count", np.uint32), ("env_probes_count", np.uint32), ("refl_probes_count", np.uint32)])
CLUSTER_ENV_PROBE_DTYPE = np.dtype([("pos", np.float32, 3), ("pad0", np.float32), ("rot", np.float32, 4), ("inner_range", np.float32, 3), ("pad1", np.float32),
                                    ("outer_range", np.float32, 3), ("pad2", np.float32), ("sh_coefs", np.float32, (9, 4))])
CLUSTER_REFL_PROBE_DTYPE = np.dtype([("pos", np.float32, 3), ("layer", np.uint32), ("rot", np.float32, 4), ("half_extents", np.float32, 3), ("pad1", np.float32)])
SHADOW_CANDIDATE_DTYPE = np.dtype([("light_idx", np.uint32), ("priority", np.float32), ("entity", np.int32)])
assert POINT_LIGHT_DTYPE.itemsize == 32 and CLUSTER_LIGHT_DTYPE.itemsize == 64 and CLUSTER_DTYPE.itemsize == 16
assert CLUSTER_ENV_PROBE_DTYPE.itemsize == 208 and CLUSTER_REFL_PROBE_DTYPE.itemsize == 48


class ClusterView(C.Structure):
    _fields_ = [("cam_pos", C.c_double * 3), ("w", C.c_uint32), ("h", C.c_uint32), ("view", C.c_uint32), ("pad", C.c_uint32), ("frustum", ShiftedFrustum)]


class ShadowCandidate(C.Structure):
    _fields_ = [("light_idx", C.c_uint32), ("priority", C.c_float), ("entity", C.c_int32)]


class ClusterResult(C.Structure):
    _fields_ = [("n_lights", C.c_uint32), ("n_clusters", C.c_uint32), ("n_map", C.c_uint32), ("size", C.c_uint32 * 3), ("n_shadow", C.c_uint32),
                ("shadow", ShadowCandidate * MAX_ATLAS), ("n_uncast", C.c_uint32), ("uncast", C.c_int32 * MAX_ATLAS)]


class ClusterOutputs(C.Structure):
    _fields_ = [(n, vp) for n in ("lights", "clusters", "map", "light_entities")]


def make_view(cam_pos, frustum, w, h, view=LAST_CULL):
    """lb200_cluster_view: camera position (fp64), the view's ShiftedFrustum, viewport size, and which cull (k of the latest cull_views
    or LAST_CULL)."""
    v = ClusterView()
    for c in range(3):
        v.cam_pos[c] = float(cam_pos[c])
    v.w, v.h, v.view = int(w), int(h), int(view)
    C.memmove(C.byref(v.frustum), C.byref(frustum), C.sizeof(ShiftedFrustum))
    return v


def shadow_list(res):
    """The AtlasSorter list of a ClusterResult as a SHADOW_CANDIDATE_DTYPE array."""
    return np.frombuffer(bytes(res.shadow), SHADOW_CANDIDATE_DTYPE)[:res.n_shadow].copy()


class Clusters:
    def __init__(self, ctx, max_entities):
        self.ctx, self.L = ctx, ctx.L
        self.h = vp()
        check(self.L.lb200_clusters_create(ctx.h, C.c_uint32(max_entities), C.byref(self.h)), ctx.h)
        self.max_entities = max_entities
        ctx._adopt(self)

    def _err(self, rc):
        check(rc, self.ctx.h)

    def close(self):
        if self.h:
            self.L.lb200_clusters_destroy(self.h)
            self.h = None

    def setPointLights(self, entities, records):
        """RenderModule's PointLights (POINT_LIGHT_DTYPE) of distinct entities."""
        e = np.ascontiguousarray(entities, np.int32)
        r = np.ascontiguousarray(records, POINT_LIGHT_DTYPE)
        assert len(e) == len(r)
        self._err(self.L.lb200_clusters_set_point_lights(self.h, ptr(e), ptr(r), C.c_uint32(len(e))))

    def setAtlas(self, entities, atlas_idx):
        """ShadowAtlas::map entries, in list order; -1 removes an entity's entry."""
        e = np.ascontiguousarray(entities, np.int32)
        a = np.ascontiguousarray(atlas_idx, np.int32)
        assert len(e) == len(a)
        self._err(self.L.lb200_clusters_set_atlas(self.h, ptr(e), ptr(a), C.c_uint32(len(e))))

    def fillClusters(self, sortkeys, culling, view, env_probes=None, refl_probes=None):
        """fillClusters up to the host's atlas step for the cull `view` names.  -> ClusterResult (the call waits for it)."""
        env = np.ascontiguousarray(env_probes if env_probes is not None else np.zeros(0, CLUSTER_ENV_PROBE_DTYPE), CLUSTER_ENV_PROBE_DTYPE)
        refl = np.ascontiguousarray(refl_probes if refl_probes is not None else np.zeros(0, CLUSTER_REFL_PROBE_DTYPE), CLUSTER_REFL_PROBE_DTYPE)
        res = ClusterResult()
        self._err(self.L.lb200_clusters_fill(self.h, sortkeys.h, culling.h, C.byref(view), ptr(env) if len(env) else None, C.c_uint32(len(env)),
                                             ptr(refl) if len(refl) else None, C.c_uint32(len(refl)), C.byref(res)))
        return res

    def patchAtlas(self, light_idx, atlas_idx):
        """The atlas step's atlas_idx values into lights[] on the device (asynchronous)."""
        li = np.ascontiguousarray(light_idx, np.uint32)
        a = np.ascontiguousarray(atlas_idx, np.int32)
        assert len(li) == len(a)
        self._err(self.L.lb200_clusters_patch_atlas(self.h, ptr(li), ptr(a), C.c_uint32(len(li))))

    def setLaunch(self, blocks=0):
        """Grid of the items kernel in later fills (lb200_clusters_set_launch): 0 = the default rule, -1 = every co-resident block,
        n > 0 = min(n, co-resident blocks)."""
        self._err(self.L.lb200_clusters_set_launch(self.h, C.c_int(blocks)))

    def lastLaunch(self):
        """(items-kernel grid, tiles of 256 items per block) of the last fill; (0, 0) before the first."""
        g, t = C.c_uint32(), C.c_uint32()
        self._err(self.L.lb200_clusters_get_launch(self.h, C.byref(g), C.byref(t)))
        return g.value, t.value

    def outputs(self):
        o = ClusterOutputs()
        self._err(self.L.lb200_clusters_outputs(self.h, C.byref(o)))
        return o

    def read(self, res):
        """Host copies of what the last fillClusters left in HBM (`res` = its ClusterResult)."""
        o = self.outputs()
        cp = self.ctx.copy_to_host
        return dict(lights=cp(o.lights, res.n_lights, CLUSTER_LIGHT_DTYPE), clusters=cp(o.clusters, res.n_clusters, CLUSTER_DTYPE),
                    map=cp(o.map, res.n_map, np.int32), light_entities=cp(o.light_entities, res.n_lights, np.int32))
