"""Batched World hierarchy propagation (replaces World::transformEntity, src/engine/world.cpp:255-282) over the C-ABI.

Transforms cross the boundary as the engine's 56-byte `Transform` (src/core/math.h:306-327): numpy structured dtype
TRANSFORM_DTYPE = {pos: 3 x f64, rot: 4 x f32 (xyzw), scale: 3 x f32}.
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import check, ptr, vp

TRANSFORM_DTYPE = np.dtype({"names": ["pos", "rot", "scale"], "formats": [(np.float64, 3), (np.float32, 4), (np.float32, 3)],
                            "offsets": [0, 24, 40], "itemsize": 56})
assert TRANSFORM_DTYPE.itemsize == 56


class Hierarchy:
    """parents[i] = parent node index or -1 (World::setParent, world.cpp:619-701)."""

    def __init__(self, ctx, parents):
        self.L = _lib.lib()
        self.ctx = ctx
        p = np.ascontiguousarray(parents, np.int32)
        self.n = len(p)
        h = vp()
        check(self.L.lb200_hierarchy_create(ctx.h, ptr(p), C.c_uint32(self.n), C.byref(h)), ctx.h)
        self.h = h
        ctx._adopt(self)

    def close(self):
        if self.h:
            self.L.lb200_hierarchy_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    @property
    def depth(self):
        return int(self.L.lb200_hierarchy_depth(self.h))

    def setParents(self, parents):
        """World::setParent for any number of nodes, and nodes entering or leaving: the whole parent array again (len may differ from n).
        The level order is rebuilt on the device as the constructor builds it; node i < min(old n, new n) keeps its transforms, new nodes
        start as the identity.  A parent >= n or a cycle raises and leaves the hierarchy as it was."""
        p = np.ascontiguousarray(parents, np.int32)
        check(self.L.lb200_hierarchy_set_parents(self.h, ptr(p), C.c_uint32(len(p))), self.ctx.h)
        self.n = len(p)

    def setParentsDevice(self, dev_parents, n, max_blocks=0):
        """setParents from n int32 parents in device memory (a device pointer); max_blocks caps the builder's cooperative grid (0 = all
        co-resident blocks)."""
        check(self.L.lb200_hierarchy_set_parents_device(self.h, vp(dev_parents), C.c_uint32(n), C.c_uint32(max_blocks)), self.ctx.h)
        self.n = int(n)

    def levelOrder(self):
        """(order u32[n]: level position -> node, parent_pos i32[n]: -> the parent's level position or -1, level_start u32[depth + 1])."""
        order = np.empty(self.n, np.uint32)
        parent_pos = np.empty(self.n, np.int32)
        level_start = np.empty(self.depth + 1, np.uint32)
        check(self.L.lb200_hierarchy_get_level_order(self.h, ptr(order), ptr(parent_pos), ptr(level_start)), self.ctx.h)
        return order, parent_pos, level_start

    def setLocalTransforms(self, locals_):
        a = np.ascontiguousarray(locals_, TRANSFORM_DTYPE)
        assert len(a) == self.n
        check(self.L.lb200_hierarchy_set_locals(self.h, ptr(a)), self.ctx.h)

    def setRootTransforms(self, globals_):
        a = np.ascontiguousarray(globals_, TRANSFORM_DTYPE)
        assert len(a) == self.n
        check(self.L.lb200_hierarchy_set_root_globals(self.h, ptr(a)), self.ctx.h)

    def setTransforms(self, globals_):
        """World transforms of ALL nodes (authoritative globals: physics, gizmo, re-parenting)."""
        a = np.ascontiguousarray(globals_, TRANSFORM_DTYPE)
        assert len(a) == self.n
        check(self.L.lb200_hierarchy_set_globals(self.h, ptr(a)), self.ctx.h)

    def computeLocalTransforms(self):
        """transformEntity(update_local=true) (world.cpp:267-270) for every non-root node: local = computeLocal(parent, own)."""
        check(self.L.lb200_hierarchy_compute_locals(self.h), self.ctx.h)

    def getLocalTransforms(self, out=None):
        if out is None:
            out = np.empty(self.n, TRANSFORM_DTYPE)
        check(self.L.lb200_hierarchy_get_locals(self.h, ptr(out)), self.ctx.h)
        return out

    def propagate(self):
        check(self.L.lb200_hierarchy_propagate(self.h), self.ctx.h)

    def getTransforms(self, out=None):
        """World::getTransforms (world.h:65) for every node, caller order."""
        if out is None:
            out = np.empty(self.n, TRANSFORM_DTYPE)
        check(self.L.lb200_hierarchy_get_globals(self.h, ptr(out)), self.ctx.h)
        return out

    def getSpheres(self, bounding_radius):
        """(pos f64[n,3], radius f32[n]) = what onModelInstanceMoved hands to CullingSystem::set (render_module.cpp:1544-1554)."""
        b = np.ascontiguousarray(bounding_radius, np.float32)
        pos = np.empty((self.n, 3), np.float64)
        rad = np.empty(self.n, np.float32)
        check(self.L.lb200_hierarchy_get_spheres(self.h, ptr(b), ptr(pos), ptr(rad)), self.ctx.h)
        return pos, rad

    def setSubset(self, nodes, transforms, globals_=False):
        """World::setLocalTransform (or setTransform with globals_=True, for roots) for some nodes: only those transforms are uploaded."""
        import ctypes as C
        nd = np.ascontiguousarray(nodes, np.uint32)
        tr = np.ascontiguousarray(transforms, TRANSFORM_DTYPE)
        assert len(nd) == len(tr)
        check(self.L.lb200_hierarchy_set_subset(self.h, ptr(nd), ptr(tr), C.c_uint32(len(nd)), C.c_int(1 if globals_ else 0)), self.ctx.h)

    def refreshSpheres(self, bounding_radius=None):
        """The same refresh left in HBM -> (device pointer of pos f64[n,3], device pointer of radius f32[n]); CullingSystem.set_many_device
        takes them when node index = entity id.  bounding_radius may be omitted after the first call."""
        import ctypes as C
        b = None if bounding_radius is None else np.ascontiguousarray(bounding_radius, np.float32)
        p, r = C.c_void_p(), C.c_void_p()
        check(self.L.lb200_hierarchy_refresh_spheres(self.h, ptr(b) if b is not None else None, C.byref(p), C.byref(r)), self.ctx.h)
        return p.value, r.value

    def getRelativeMatrices(self, base_pos):
        """World::getRelativeMatrix(entity, base_pos) (world.cpp:370-377) for every node: float32[n,16], column-major."""
        b = np.ascontiguousarray(base_pos, np.float64)
        out = np.empty((self.n, 16), np.float32)
        check(self.L.lb200_hierarchy_get_relative_matrices(self.h, ptr(b), ptr(out)), self.ctx.h)
        return out

    def algorithmic_bytes(self):
        return int(self.L.lb200_hierarchy_algorithmic_bytes(self.h))
