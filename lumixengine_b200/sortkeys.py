"""Host-side mirror of the stage right behind the cull: PipelineImpl::createSortKeys + radixSort (src/renderer/pipeline.cpp:3789-4144)
on the device (csrc/sortkeys.cu, include/lumix_b200.h "Sort keys")."""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import check, ptr, vp

SK_MODEL_DTYPE = np.dtype([("lod_distances", np.float32, 4), ("lod_from", np.int32, 5), ("lod_to", np.int32, 5), ("mesh_base", np.uint32), ("mesh_count", np.uint32)])
SK_MESH_DTYPE = np.dtype([("sort_key", np.uint32), ("material_index", np.uint32), ("lod", np.float32), ("layer", np.uint8), ("skinned", np.uint8), ("pad", np.uint16)])
SK_VIEW_DTYPE = np.dtype([("camera_pos", np.float64, 3), ("lod_ref_point", np.float64, 3), ("time_delta", np.float32), ("lod_multiplier", np.float32),
                          ("frame_number", np.uint32), ("is_shadow", np.uint32), ("max_sort_key", np.uint32), ("pad", np.uint32),
                          ("bucket_map", np.uint32, 256), ("layer_to_bucket", np.uint8, 256)])
MOVED, DIRTY = 1, 2  # ModelInstance::MOVED / ModelInstance::dirty


class SkResult(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in ("n_keys", "n_instances", "n_pose", "n_dirty", "n_groups")]


class SkOutputs(C.Structure):
    _fields_ = [(n, vp) for n in ("keys", "values", "group_count", "group_offset", "group_renderables", "instance_data", "pose_list", "dirty_list", "lod", "pose_frame")]


def make_view(camera_pos, lod_ref_point, time_delta, lod_multiplier, frame_number, is_shadow, max_sort_key, layer_to_bucket, depth_sorted_buckets=()):
    """lb200_sk_view from what PipelineImpl::View holds: layer_to_bucket[layer] (0xff = layer not in the view); buckets listed in
    `depth_sorted_buckets` sort by depth (BucketDesc::DEPTH).  bucket_map follows pipeline.cpp:3803-3812."""
    v = np.zeros(1, SK_VIEW_DTYPE)
    v["camera_pos"], v["lod_ref_point"] = camera_pos, lod_ref_point
    v["time_delta"], v["lod_multiplier"], v["frame_number"], v["is_shadow"], v["max_sort_key"] = time_delta, lod_multiplier, frame_number % 0xffffffff, int(is_shadow), max_sort_key
    l2b = np.full(256, 0xff, np.uint8)
    l2b[:len(layer_to_bucket)] = layer_to_bucket
    v["layer_to_bucket"][0] = l2b
    bm = l2b.astype(np.uint32)
    bm[l2b == 0xff] = 0xffffffff
    for b in depth_sorted_buckets:
        bm[l2b == b] |= 0x100
    v["bucket_map"][0] = bm
    return v


def radix_sort_device(ctx, dev_keys, dev_values, dev_count, cap, max_blocks=0, tiled=False):
    """lb200_radix_sort_device: enqueues the stable sort of min(*dev_count, cap) (u64 key, u64 value) pairs in place on the context stream
    (device pointers as ints) and returns the blocks launched.  Nothing waits unless the context's scratch has to grow to `cap`."""
    grid = C.c_uint32()
    check(ctx.L.lb200_radix_sort_device(ctx.h, vp(dev_keys), vp(dev_values), vp(dev_count), C.c_uint32(cap), C.c_uint32(max_blocks), C.c_int(1 if tiled else 0),
                                        C.byref(grid)), ctx.h)
    return int(grid.value)


def radix_sort(ctx, keys, values, count=None, max_blocks=0, tiled=False):
    """The device sort on host arrays of `cap = len(keys)` pairs: sorts the first min(count, cap) (count defaults to cap) and leaves the rest.
    -> (keys, values, grid): host copies of all cap pairs after the sort, and the blocks launched."""
    keys = np.ascontiguousarray(keys, np.uint64)
    values = np.ascontiguousarray(values, np.uint64)
    assert keys.shape == values.shape and keys.ndim == 1
    cap = len(keys)
    dev = [ctx.to_device(a) for a in (keys, values, np.array([cap if count is None else count], np.uint32))]
    try:
        grid = radix_sort_device(ctx, dev[0], dev[1], dev[2], cap, max_blocks, tiled)
        return ctx.copy_to_host(dev[0], cap, np.uint64), ctx.copy_to_host(dev[1], cap, np.uint64), grid
    finally:
        for p in dev:
            ctx.free_device(p)


class SortKeys:
    def __init__(self, ctx, max_entities, max_groups, max_keys=0, max_instances=0):
        self.ctx, self.L = ctx, ctx.L
        self.h = vp()
        check(self.L.lb200_sortkeys_create(ctx.h, C.c_uint32(max_entities), C.c_uint32(max_groups), C.c_uint32(max_keys), C.c_uint32(max_instances), C.byref(self.h)), ctx.h)
        self.max_entities = max_entities

    def _err(self, rc):
        check(rc, self.ctx.h)

    def close(self):
        if self.h:
            self.L.lb200_sortkeys_destroy(self.h)
            self.h = None

    def setModels(self, models, meshes):
        models = np.ascontiguousarray(models, SK_MODEL_DTYPE)
        meshes = np.ascontiguousarray(meshes, SK_MESH_DTYPE)
        self._err(self.L.lb200_sortkeys_set_models(self.h, ptr(models), C.c_uint32(len(models)), ptr(meshes), C.c_uint32(len(meshes))))

    def setInstances(self, model_of=None, lod=None, flags=None, pose_frame=None, decal_sort_key=None, decal_layer=None):
        arrs = [(model_of, np.uint32), (lod, np.float32), (flags, np.uint8), (pose_frame, np.uint32), (decal_sort_key, np.uint32), (decal_layer, np.uint8)]
        arrs = [None if a is None else np.ascontiguousarray(a, t) for a, t in arrs]
        n = max(len(a) for a in arrs if a is not None)
        assert all(a is None or len(a) == n for a in arrs)
        self._err(self.L.lb200_sortkeys_set_instances(self.h, C.c_uint32(n), *[ptr(a) if a is not None else None for a in arrs]))

    def setTransforms(self, transforms):
        t = np.ascontiguousarray(transforms)
        assert t.dtype.itemsize == 56
        self._err(self.L.lb200_sortkeys_set_transforms(self.h, ptr(t), C.c_uint32(len(t))))

    def createSortKeys(self, culling, view, sort=True, want_counts=True):
        """For the last cull issued on `culling`.  -> SkResult (None if not want_counts: nothing is read back, nothing waits)."""
        view = np.ascontiguousarray(view, SK_VIEW_DTYPE).reshape(1)
        res = SkResult()
        self._err(self.L.lb200_sortkeys_create_keys(self.h, culling.h, ptr(view), C.c_int(1 if sort else 0), C.c_int(1 if want_counts else 0), C.byref(res)))
        return res if want_counts else None

    def setLaunch(self, blocks=0, prefetch_ahead=-1):
        """Launch shape of later createSortKeys calls: blocks 0 = the default (environment switch, else 2 per SM, at most one per 256
        renderables), -1 = all co-resident, n > 0 = min(n, co-resident); prefetch_ahead 0..4 grid strides, -1 = the default."""
        self._err(self.L.lb200_sortkeys_set_launch(self.h, C.c_int(blocks), C.c_int(prefetch_ahead)))

    def lastLaunch(self):
        """(grid, group counters in shared memory, prefetch distance) of the last createSortKeys; zeros before the first."""
        g, s, p = C.c_uint32(), C.c_int(), C.c_uint32()
        self._err(self.L.lb200_sortkeys_get_launch(self.h, C.byref(g), C.byref(s), C.byref(p)))
        return int(g.value), bool(s.value), int(p.value)

    def moveDevice(self, dev_entities, dev_transforms, n, dev_bounding_radius=None, dev_out_pos3=None, dev_out_radius=None):
        """RenderModule::onModelInstanceMoved for n instances whose transforms lie in device memory (pointers as ints): records updated, MOVED set;
        with bounding radii also the spheres for CullingSystem.set_many_device."""
        self._err(self.L.lb200_sortkeys_move_device(self.h, vp(dev_entities), vp(dev_transforms), C.c_uint32(n), vp(dev_bounding_radius) if dev_bounding_radius else None,
                                                    vp(dev_out_pos3) if dev_out_pos3 else None, vp(dev_out_radius) if dev_out_radius else None))

    def endFrame(self):
        """RenderModule::endFrame: MOVED cleared, prev_frame_transform taken for the instances moved since the last call."""
        self._err(self.L.lb200_sortkeys_end_frame(self.h))

    def prevTransforms(self):
        """Host copy of ModelInstance::prev_frame_transform per entity (zeros until an instance went through moveDevice + endFrame)."""
        from .hierarchy import TRANSFORM_DTYPE
        p = vp()
        self._err(self.L.lb200_sortkeys_prev_transforms(self.h, C.byref(p)))
        if not p:
            return np.zeros(self.max_entities, TRANSFORM_DTYPE)
        return self.ctx.copy_to_host(p.value, self.max_entities, TRANSFORM_DTYPE)

    def read(self, res):
        """Host copies of everything the last createSortKeys left in HBM."""
        o = SkOutputs()
        self._err(self.L.lb200_sortkeys_device_outputs(self.h, C.byref(o)))
        cp = self.ctx.copy_to_host
        g = res.n_groups
        return dict(keys=cp(o.keys, res.n_keys, np.uint64), values=cp(o.values, res.n_keys, np.uint64), group_count=cp(o.group_count, g, np.uint32),
                    group_offset=cp(o.group_offset, g, np.uint32), group_renderables=cp(o.group_renderables, res.n_instances, np.uint64),
                    instance_data=cp(o.instance_data, res.n_instances * 48, np.uint8).reshape(-1, 48), pose_list=cp(o.pose_list, res.n_pose, np.uint32),
                    dirty_list=cp(o.dirty_list, res.n_dirty, np.uint32), lod=cp(o.lod, self.max_entities, np.float32), pose_frame=cp(o.pose_frame, self.max_entities, np.uint32))
