"""TEST INFRASTRUCTURE — ctypes bindings for the CPU oracle (oracle/liboracle_lumix.so, the restatement)
and, when present, the reference's own compiled code (oracle/_ref/libref_lumix.so).

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this
module.  The product (lumixengine_b200) never does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "liboracle_lumix.so")
REF_SO = os.path.join(HERE, "_ref", "libref_lumix.so")
# the reference's animation code next to the animation binding (oracle/ref/ref_root_motion_harness.cpp and the harnesses it includes)
ANIMATION_SHIM_SO = os.path.join(HERE, "_ref", "libanimation_shim_b200.so")

u8p = C.POINTER(C.c_uint8)
vp = C.c_void_p
_made = set()


def make(target):
    """Bring one restatement library of oracle/Makefile up to date, once per process; -> its path."""
    if target not in _made:
        subprocess.check_call(["make", "-s", "-C", HERE, target])
        _made.add(target)
    return os.path.join(HERE, target)


def build(force=False):
    """Compile the C restatements and, where the reference tree is, oracle/_ref (oracle/build_ref.py); each only when stale."""
    from . import build_ref
    subprocess.check_call(["make", "-s", "-C", HERE] + (["-B"] if force else []))
    build_ref.build(force)


def _ptr(a):
    return None if a is None else a.ctypes.data_as(vp)


class Stats(C.Structure):
    _fields_ = [(n, C.c_uint32) for n in (
        "pages_total", "pages_filtered", "pages_tested", "pages_inside", "pages_outside",
        "entities_total", "entities_tested", "entities_inside", "visible", "visible_tested")]

    def asdict(self):
        return {n: int(getattr(self, n)) for n, _ in self._fields_}


class Track(C.Structure):
    _fields_ = [("bone_index", C.c_uint16), ("offset_bits", C.c_uint16), ("bitsizes", C.c_uint8 * 3),
                ("skipped_channel", C.c_uint8), ("min", C.c_float * 3), ("to_range", C.c_float * 3)]


class ConstTranslation(C.Structure):
    _fields_ = [("bone_index", C.c_uint16), ("pad", C.c_uint16), ("value", C.c_float * 3)]


class ConstRotation(C.Structure):
    _fields_ = [("bone_index", C.c_uint16), ("pad", C.c_uint16), ("value", C.c_float * 4)]


class Clip(C.Structure):
    _fields_ = [("fps", C.c_float), ("frame_count", C.c_uint32),
                ("translations_frame_size_bits", C.c_uint32), ("rotations_frame_size_bits", C.c_uint32),
                ("n_translations", C.c_uint32), ("n_const_translations", C.c_uint32),
                ("n_rotations", C.c_uint32), ("n_const_rotations", C.c_uint32),
                ("translations", vp), ("const_translations", vp), ("rotations", vp), ("const_rotations", vp),
                ("translation_stream", vp), ("rotation_stream", vp)]


class Skeleton(C.Structure):
    _fields_ = [("bone_count", C.c_uint32), ("first_nonroot_bone_index", C.c_int32),
                ("parents", vp), ("bind_relative", vp), ("inverse_bind", vp)]


_lib = None


def lib():
    global _lib
    if _lib is None:
        L = C.CDLL(make("liboracle_lumix.so"))
        L.oracle_culling_create.restype = vp
        L.oracle_culling_cull.restype = C.c_uint32
        L.oracle_culling_page_count.restype = C.c_uint32
        L.oracle_culling_get_radius.restype = C.c_float
        L.oracle_time_advance.restype = C.c_uint32
        _lib = L
    return _lib


def frustum_perspective(pos, direction, up, fov, ratio, near, far):
    """-> 256-byte ShiftedFrustum image (np.uint8[256]); geometry.cpp:470-499."""
    out = np.zeros(256, np.uint8)
    lib().oracle_frustum_perspective(_ptr(out), (C.c_double * 3)(*pos), (C.c_float * 3)(*direction), (C.c_float * 3)(*up),
                                     C.c_float(fov), C.c_float(ratio), C.c_float(near), C.c_float(far))
    return out


def frustum_ortho(pos, direction, up, width, height, near, far):
    out = np.zeros(256, np.uint8)
    lib().oracle_frustum_ortho(_ptr(out), (C.c_double * 3)(*pos), (C.c_float * 3)(*direction), (C.c_float * 3)(*up),
                               C.c_float(width), C.c_float(height), C.c_float(near), C.c_float(far))
    return out


def rng_floats(u, v, n):
    uu, vv = C.c_uint32(u), C.c_uint32(v)
    out = np.empty(n, np.float32)
    lib().oracle_rng_floats(C.byref(uu), C.byref(vv), C.c_uint32(n), _ptr(out))
    return out, (uu.value, vv.value)


class OracleCulling:
    """Restated CullingSystemImpl (culling_system.cpp:67-383)."""

    def __init__(self):
        self.L = lib()
        self.h = vp(self.L.oracle_culling_create())

    def __del__(self):
        try:
            self.L.oracle_culling_destroy(self.h)
        except Exception:
            pass

    def add(self, entities, types, pos, radius):
        e = np.ascontiguousarray(entities, np.int32)
        t = np.ascontiguousarray(types, np.uint8)
        p = np.ascontiguousarray(pos, np.float64)
        r = np.ascontiguousarray(radius, np.float32)
        self.L.oracle_culling_add_many(self.h, _ptr(e), _ptr(t), _ptr(p), _ptr(r), C.c_uint32(len(e)))

    def set(self, entities, pos, radius):
        e = np.ascontiguousarray(entities, np.int32)
        p = np.ascontiguousarray(pos, np.float64)
        r = np.ascontiguousarray(radius, np.float32)
        self.L.oracle_culling_set_many(self.h, _ptr(e), _ptr(p), _ptr(r), C.c_uint32(len(e)))

    def set_position(self, entities, pos):
        e = np.ascontiguousarray(entities, np.int32)
        p = np.ascontiguousarray(pos, np.float64)
        self.L.oracle_culling_set_position_many(self.h, _ptr(e), _ptr(p), C.c_uint32(len(e)))

    def set_radius(self, entities, radius):
        e = np.ascontiguousarray(entities, np.int32)
        r = np.ascontiguousarray(radius, np.float32)
        self.L.oracle_culling_set_radius_many(self.h, _ptr(e), _ptr(r), C.c_uint32(len(e)))

    def remove(self, entities):
        e = np.ascontiguousarray(entities, np.int32)
        self.L.oracle_culling_remove_many(self.h, _ptr(e), C.c_uint32(len(e)))

    def get_radius(self, entity):
        return float(self.L.oracle_culling_get_radius(self.h, C.c_int32(entity)))

    def is_added(self, entity):
        return bool(self.L.oracle_culling_is_added(self.h, C.c_int32(entity)))

    def page_count(self):
        return int(self.L.oracle_culling_page_count(self.h))

    def cull(self, frustum256, type=-1, cap=None, want_ids=True):
        """-> (ids uint32[V], types uint8[V], stats dict); order = m_cells order (a legal order, SURVEY F4)."""
        st = Stats()
        f = np.ascontiguousarray(frustum256, np.uint8)
        if not want_ids:
            n = self.L.oracle_culling_cull(self.h, _ptr(f), C.c_int(type), None, None, C.c_uint32(0), C.byref(st))
            return None, None, st.asdict()
        if cap is None:
            cap = self.L.oracle_culling_cull(self.h, _ptr(f), C.c_int(type), None, None, C.c_uint32(0), C.byref(st))
        ids = np.empty(max(cap, 1), np.uint32)
        tys = np.empty(max(cap, 1), np.uint8)
        n = self.L.oracle_culling_cull(self.h, _ptr(f), C.c_int(type), _ptr(ids), _ptr(tys), C.c_uint32(cap), C.byref(st))
        n = min(n, cap)
        return ids[:n], tys[:n], st.asdict()

    def pages(self):
        """Dump of every page of m_cells: list of dicts (origin, indices, type, is_big, count, spheres, entities)."""
        out = []
        for i in range(self.page_count()):
            o = (C.c_double * 3)()
            ind = (C.c_int * 3)()
            ty, big, cnt = C.c_uint8(), C.c_uint8(), C.c_int()
            sph = np.empty((201, 4), np.float32)
            ent = np.empty(201, np.int32)
            self.L.oracle_culling_get_page(self.h, C.c_uint32(i), o, ind, C.byref(ty), C.byref(big), C.byref(cnt), _ptr(sph), _ptr(ent))
            c = cnt.value
            out.append(dict(origin=tuple(o), indices=tuple(ind), type=ty.value, is_big=big.value, count=c,
                            spheres=sph[:c].copy(), entities=ent[:c].copy()))
        return out


def propagate(parents, locals56, globals56):
    """world.cpp:255-282 over a forest. locals56/globals56: uint8[n,56] images of Transform. Returns new globals."""
    p = np.ascontiguousarray(parents, np.int32)
    l = np.ascontiguousarray(locals56, np.uint8)
    g = np.array(globals56, np.uint8, copy=True, order="C")
    lib().oracle_propagate(_ptr(p), _ptr(l), _ptr(g), C.c_uint32(len(p)))
    return g


def transform_compose(parent56, local56):
    """Element-wise Transform::compose (math.cpp:801-807)."""
    a = np.ascontiguousarray(parent56, np.uint8)
    b = np.ascontiguousarray(local56, np.uint8)
    out = np.zeros_like(a)
    lib().oracle_transform_compose(_ptr(a), _ptr(b), _ptr(out), C.c_uint32(len(a)))
    return out


def compute_locals(parents, globals56, locals56):
    """World::transformEntity(update_local) for every non-root node: local = Transform::computeLocal(parent global, own global)."""
    p = np.ascontiguousarray(parents, np.int32)
    g = np.ascontiguousarray(globals56, np.uint8)
    l = np.array(locals56, np.uint8, copy=True, order="C")
    lib().oracle_compute_locals(_ptr(p), _ptr(g), _ptr(l), C.c_uint32(len(p)))
    return l


def transform_compute_local(parent56, child56, use_ref=False):
    """Element-wise Transform::computeLocal (math.cpp:809-816); use_ref=True runs the reference's own function (oracle/_ref)."""
    a = np.ascontiguousarray(parent56, np.uint8)
    b = np.ascontiguousarray(child56, np.uint8)
    out = np.zeros_like(a)
    if use_ref:
        ref().ref_transform_compute_local(_ptr(a), _ptr(b), _ptr(out), C.c_uint32(len(a)))
    else:
        lib().oracle_transform_compute_local(_ptr(a), _ptr(b), _ptr(out), C.c_uint32(len(a)))
    return out


def bone_attachments(parent56, bone7, relative7, original_scale3, use_ref=False):
    """RenderModuleImpl::updateBoneAttachment (render_module.cpp:399-403) per attachment -> uint8[n,56] Transforms."""
    p = np.ascontiguousarray(parent56, np.uint8)
    b = np.ascontiguousarray(bone7, np.float32)
    r = np.ascontiguousarray(relative7, np.float32)
    sc = np.ascontiguousarray(original_scale3, np.float32)
    out = np.zeros_like(p)
    f = ref().ref_bone_attachments if use_ref else lib().oracle_bone_attachments
    f(_ptr(p), _ptr(b), _ptr(r), _ptr(sc), _ptr(out), C.c_uint32(len(p)))
    return out


def relative_matrices(globals56, base_pos):
    """World::getRelativeMatrix (world.cpp:370-377) for every transform: float32[n,16], column-major like Matrix."""
    g = np.ascontiguousarray(globals56, np.uint8)
    b = np.ascontiguousarray(base_pos, np.float64)
    out = np.empty((len(g), 16), np.float32)
    lib().oracle_relative_matrices(_ptr(g), _ptr(b), _ptr(out), C.c_uint32(len(g)))
    return out


def ref_relative_matrices(globals56, base_pos):
    """The same through the reference's own Quat::toMatrix / Matrix::setTranslation / multiply3x3 (oracle/_ref)."""
    g = np.ascontiguousarray(globals56, np.uint8)
    b = np.ascontiguousarray(base_pos, np.float64)
    out = np.empty((len(g), 16), np.float32)
    ref().ref_relative_matrix(_ptr(g), _ptr(b), _ptr(out), C.c_uint32(len(g)))
    return out


def sphere_radius(globals56, bounding_radius, use_ref=False):
    """render_module.cpp:1554: bounding_radius * maximum(scale.x, scale.y, scale.z); use_ref=True uses the reference's own maximum."""
    g = np.ascontiguousarray(globals56, np.uint8)
    b = np.ascontiguousarray(bounding_radius, np.float32)
    out = np.empty(len(b), np.float32)
    (ref().ref_sphere_radius if use_ref else lib().oracle_sphere_radius)(_ptr(g), _ptr(b), _ptr(out), C.c_uint32(len(b)))
    return out


# ---------------------------------------------------------------------------------------------------
# reference's own compiled code
# ---------------------------------------------------------------------------------------------------
_ref = None


def ref_available():
    return os.path.exists(REF_SO)


def ref():
    global _ref
    if _ref is None:
        L = C.CDLL(REF_SO)
        L.ref_culling_create.restype = vp
        L.ref_culling_cull.restype = C.c_uint32
        L.ref_culling_get_radius.restype = C.c_float
        _ref = L
    return _ref


def frustum_from_viewport(pos, rot, fov, w, h, near, far, is_ortho=False, ortho_size=100.0, use_ref=False):
    """Viewport::getFrustum() (geometry.cpp:793-818) -> 256-byte ShiftedFrustum image; use_ref=True runs the reference's own."""
    out = np.zeros(256, np.uint8)
    args = (C.c_int(1 if is_ortho else 0), C.c_float(fov), C.c_float(ortho_size), C.c_int(w), C.c_int(h), (C.c_double * 3)(*pos), (C.c_float * 4)(*rot),
            C.c_float(near), C.c_float(far))
    if use_ref:
        ref().ref_viewport_frustum(*args, _ptr(out))
    else:
        lib().oracle_frustum_from_viewport(_ptr(out), *args)
    return out


def ref_frustum_perspective(pos, direction, up, fov, ratio, near, far):
    out = np.zeros(256, np.uint8)
    ref().ref_frustum_perspective((C.c_double * 3)(*pos), (C.c_float * 3)(*direction), (C.c_float * 3)(*up),
                                  C.c_float(fov), C.c_float(ratio), C.c_float(near), C.c_float(far), _ptr(out))
    return out


def ref_frustum_ortho(pos, direction, up, width, height, near, far):
    out = np.zeros(256, np.uint8)
    ref().ref_frustum_ortho((C.c_double * 3)(*pos), (C.c_float * 3)(*direction), (C.c_float * 3)(*up),
                            C.c_float(width), C.c_float(height), C.c_float(near), C.c_float(far), _ptr(out))
    return out


class RefCulling:
    """The reference's CullingSystemImpl (overlay build) on the reference's job system."""

    def __init__(self, workers=1):
        self.L = ref()
        self.workers = self.L.ref_jobs_init(C.c_int(workers))
        if not self.workers:
            raise RuntimeError("reference job system failed to initialise")
        self.h = vp(self.L.ref_culling_create())

    def add(self, entities, types, pos, radius):
        e = np.ascontiguousarray(entities, np.int32)
        t = np.ascontiguousarray(types, np.uint8)
        p = np.ascontiguousarray(pos, np.float64)
        r = np.ascontiguousarray(radius, np.float32)
        self.L.ref_culling_add(self.h, _ptr(e), _ptr(t), _ptr(p), _ptr(r), C.c_uint32(len(e)))

    def set(self, entities, pos, radius):
        e = np.ascontiguousarray(entities, np.int32)
        p = np.ascontiguousarray(pos, np.float64)
        r = np.ascontiguousarray(radius, np.float32)
        self.L.ref_culling_set(self.h, _ptr(e), _ptr(p), _ptr(r), C.c_uint32(len(e)))

    def set_position(self, entities, pos):
        e = np.ascontiguousarray(entities, np.int32)
        p = np.ascontiguousarray(pos, np.float64)
        self.L.ref_culling_set_position(self.h, _ptr(e), _ptr(p), C.c_uint32(len(e)))

    def set_radius(self, entities, radius):
        e = np.ascontiguousarray(entities, np.int32)
        r = np.ascontiguousarray(radius, np.float32)
        self.L.ref_culling_set_radius(self.h, _ptr(e), _ptr(r), C.c_uint32(len(e)))

    def remove(self, entities):
        e = np.ascontiguousarray(entities, np.int32)
        self.L.ref_culling_remove(self.h, _ptr(e), C.c_uint32(len(e)))

    def cull(self, frustum256, type=-1, cap=0, iters=1):
        """-> (ids, types, dict(best_s, median_s, first_s, pages)); ids in the reference's job-completion order."""
        f = np.ascontiguousarray(frustum256, np.uint8)
        ids = np.empty(max(cap, 1), np.uint32)
        tys = np.empty(max(cap, 1), np.uint8)
        times = (C.c_double * 3)()
        pages = C.c_uint32()
        n = self.L.ref_culling_cull(self.h, _ptr(f), C.c_int(type), _ptr(ids), _ptr(tys), C.c_uint32(cap), C.c_int(iters), times, C.byref(pages))
        if n == 0xFFFFFFFF:
            raise RuntimeError("reference job system not initialised")
        k = min(n, cap)
        return ids[:k], tys[:k], dict(count=int(n), best_s=times[0], median_s=times[1], first_s=times[2], pages=int(pages.value))


# ---------------------------------------------------------------------------------------------------
# animation oracle (oracle_anim.c).  `skeleton` / `clips` are objects with .as_struct(cls) and numpy fields
# (the product's lumixengine_b200.animation.Skeleton / AnimationClip are plain data holders and fit).
# ---------------------------------------------------------------------------------------------------
def animate_instances(skeleton, clips, clip_index, time_ticks, want=("pos", "rot", "dq", "mtx")):
    """Model::getRelativePose -> Animation::getRelativePose -> Pose::computeAbsolute -> palettes, per instance."""
    sk = skeleton.as_struct(Skeleton)
    arr = (Clip * len(clips))(*[c.as_struct(Clip) for c in clips])
    ci = np.ascontiguousarray(clip_index, np.uint32)
    tt = np.ascontiguousarray(time_ticks, np.uint32)
    n, B = len(ci), skeleton.bone_count
    out = {}
    pos = np.empty((n, B, 3), np.float32) if "pos" in want else None
    rot = np.empty((n, B, 4), np.float32) if "rot" in want else None
    dq = np.empty((n, B, 8), np.float32) if "dq" in want else None
    mtx = np.empty((n, B, 16), np.float32) if "mtx" in want else None
    lib().oracle_animate_instances(C.byref(sk), arr, _ptr(ci), _ptr(tt), C.c_uint32(n), _ptr(pos), _ptr(rot), _ptr(dq), _ptr(mtx))
    out.update(pos=pos, rot=rot, dq=dq, mtx=mtx)
    return out


def skin_vertices(matrices, positions, weights, indices):
    m = np.ascontiguousarray(matrices, np.float32)
    p = np.ascontiguousarray(positions, np.float32)
    w = np.ascontiguousarray(weights, np.float32)
    i = np.ascontiguousarray(indices, np.int16)
    out = np.empty_like(p)
    lib().oracle_skin_vertices(_ptr(m), _ptr(p), _ptr(w), _ptr(i), _ptr(out), C.c_uint32(len(p)))
    return out


def time_advance(time_ticks, time_delta, fps, frame_count, use_ref=False):
    """Animable time after one update (animation_module.cpp:458-469), either sign of time_delta."""
    L = ref() if use_ref else lib()
    f = L.ref_time_advance if use_ref else L.oracle_time_advance
    f.restype = C.c_uint32
    return int(f(C.c_uint32(int(time_ticks)), C.c_float(time_delta), C.c_float(fps), C.c_uint32(frame_count)))


# ---------------------------------------------------------------------------------------------------
# element-wise pins: the same call on the restatement (oracle_math.h via small C shims) and on the reference build
# ---------------------------------------------------------------------------------------------------
class RefClip(C.Structure):
    _fields_ = Clip._fields_


class RefSkeleton(C.Structure):
    _fields_ = [("bone_count", C.c_uint32), ("first_nonroot", C.c_int32), ("parents", vp), ("bind_relative7", vp), ("inverse_bind7", vp)]


def _skeleton_struct(skeleton, cls):
    s = cls()
    s.bone_count = skeleton.bone_count
    if cls is RefSkeleton:
        s.first_nonroot = skeleton.first_nonroot_bone_index
        s.bind_relative7 = skeleton.bind_relative7.ctypes.data
        s.inverse_bind7 = skeleton.inverse_bind7.ctypes.data
    else:
        s.first_nonroot_bone_index = skeleton.first_nonroot_bone_index
        s.bind_relative = skeleton.bind_relative7.ctypes.data
        s.inverse_bind = skeleton.inverse_bind7.ctypes.data
    s.parents = skeleton.parents.ctypes.data
    return s


def ref_pose_evaluate(skeleton, clip, time_ticks, weight=1.0, start_from_bind=True, compute_absolute=True, pos=None, rot=None):
    """The reference's own Animation::getRelativePose (+ Pose::computeAbsolute) on one instance."""
    sk = _skeleton_struct(skeleton, RefSkeleton)
    c = clip.as_struct(RefClip)
    B = skeleton.bone_count
    p = np.zeros((B, 3), np.float32) if pos is None else np.array(pos, np.float32, copy=True)
    r = np.zeros((B, 4), np.float32) if rot is None else np.array(rot, np.float32, copy=True)
    ref().ref_pose_evaluate(C.byref(sk), C.byref(c), C.c_uint32(int(time_ticks)), C.c_float(weight), C.c_int(1 if start_from_bind else 0),
                            C.c_int(1 if compute_absolute else 0), _ptr(p), _ptr(r))
    return p, r


def pose_evaluate(skeleton, clip, time_ticks, weight=1.0, start_from_bind=True, compute_absolute=True, pos=None, rot=None):
    """Same call on the restatement (oracle_anim.c)."""
    sk = _skeleton_struct(skeleton, Skeleton)
    c = clip.as_struct(Clip)
    B = skeleton.bone_count
    if start_from_bind:
        p = np.ascontiguousarray(skeleton.bind_relative7[:, :3], np.float32).copy()
        r = np.ascontiguousarray(skeleton.bind_relative7[:, 3:], np.float32).copy()
    else:
        p = np.array(pos, np.float32, copy=True)
        r = np.array(rot, np.float32, copy=True)
    lib().oracle_pose_sample_weighted(C.byref(c), C.c_uint32(B), C.c_uint32(int(time_ticks)), C.c_float(weight), _ptr(p), _ptr(r))
    if compute_absolute:
        lib().oracle_pose_compute_absolute(C.byref(sk), _ptr(p), _ptr(r))
    return p, r


def ref_skeleton_dual_quats(skeleton, pos, rot):
    """The reference's own PipelineImpl::computeSkeletonDualQuats (pipeline.cpp:2680-2745, SIMD batches + scalar tail) on one absolute
    pose -> float32[bone_count, 8]; None when oracle/_ref was built without the palette harness."""
    L = ref()
    if not hasattr(L, "ref_skeleton_dual_quats"):
        return None
    sk = _skeleton_struct(skeleton, RefSkeleton)
    p = np.ascontiguousarray(pos, np.float32)
    r = np.ascontiguousarray(rot, np.float32)
    out = np.zeros((skeleton.bone_count, 8), np.float32)
    rc = L.ref_skeleton_dual_quats(C.byref(sk), _ptr(p), _ptr(r), _ptr(out))
    assert rc == 0
    return out


def ref_skin_matrices(skeleton, pos, rot):
    """The reference's own computeSkinMatrices (model.cpp:132-137) on one absolute pose -> float32[bone_count, 16] or None."""
    L = ref()
    if not hasattr(L, "ref_skin_matrices"):
        return None
    sk = _skeleton_struct(skeleton, RefSkeleton)
    p = np.ascontiguousarray(pos, np.float32)
    r = np.ascontiguousarray(rot, np.float32)
    out = np.zeros((skeleton.bone_count, 16), np.float32)
    assert L.ref_skin_matrices(C.byref(sk), _ptr(p), _ptr(r), _ptr(out)) == 0
    return out


def ref_evaluate_skin(matrices, vertices, weights, indices):
    """The reference's own evaluateSkin (model.cpp:103-109) per vertex -> float32[n, 3] or None."""
    L = ref()
    if not hasattr(L, "ref_evaluate_skin"):
        return None
    m = np.ascontiguousarray(matrices, np.float32)
    v = np.ascontiguousarray(vertices, np.float32)
    w = np.ascontiguousarray(weights, np.float32)
    i = np.ascontiguousarray(indices, np.int16)
    out = np.zeros((len(v), 3), np.float32)
    L.ref_evaluate_skin(_ptr(m), _ptr(v), _ptr(w), _ptr(i), _ptr(out), C.c_uint32(len(v)))
    return out


class RefLoaded(C.Structure):
    _fields_ = [("ok", C.c_int32), ("fps", C.c_float), ("frame_count", C.c_uint32), ("flags", C.c_uint32), ("t_bits", C.c_uint32), ("r_bits", C.c_uint32),
                ("n_t", C.c_uint32), ("n_ct", C.c_uint32), ("n_r", C.c_uint32), ("n_cr", C.c_uint32), ("t_stream_offset", C.c_uint32),
                ("r_stream_offset", C.c_uint32), ("mem_size", C.c_uint32)]


def ref_animation_load(image, cap=256):
    """The reference's own Animation::load (animation.cpp:397-493) on a compiled .ani image -> dict of everything it parsed."""
    from lumixengine_b200.animation import TRACK_DTYPE
    img = np.frombuffer(bytes(image), np.uint8).copy()
    out = RefLoaded()
    th, cth, rh, crh = (np.zeros(cap, np.uint64) for _ in range(4))
    t, r = np.zeros(cap, TRACK_DTYPE), np.zeros(cap, TRACK_DTYPE)
    ctv, crv = np.zeros((cap, 3), np.float32), np.zeros((cap, 4), np.float32)
    ref().ref_animation_load(_ptr(img), C.c_uint32(len(img)), C.byref(out), _ptr(th), _ptr(t), _ptr(cth), _ptr(ctv), _ptr(rh), _ptr(r), _ptr(crh), _ptr(crv),
                             C.c_uint32(cap))
    d = {k: getattr(out, k) for k, _ in RefLoaded._fields_}
    d.update(t_hash=th[:out.n_t], t=t[:out.n_t], ct_hash=cth[:out.n_ct], ct_value=ctv[:out.n_ct], r_hash=rh[:out.n_r], r=r[:out.n_r],
             cr_hash=crh[:out.n_cr], cr_value=crv[:out.n_cr])
    return d


def pose_compute_absolute(skeleton, pos, rot):
    """Pose::computeAbsolute (pose.cpp:66-133) on one relative pose -> (pos, rot)."""
    sk = _skeleton_struct(skeleton, Skeleton)
    p = np.array(pos, np.float32, copy=True)
    r = np.array(rot, np.float32, copy=True)
    lib().oracle_pose_compute_absolute(C.byref(sk), _ptr(p), _ptr(r))
    return p, r


def pose_compute_relative(skeleton, pos, rot, use_ref=False):
    """Pose::computeRelative (pose.cpp:136-146) on one absolute pose -> (pos, rot) relative to the parents."""
    p = np.array(pos, np.float32, copy=True)
    r = np.array(rot, np.float32, copy=True)
    if use_ref:
        sk = _skeleton_struct(skeleton, RefSkeleton)
        ref().ref_pose_compute_relative(C.byref(sk), _ptr(p), _ptr(r))
    else:
        sk = _skeleton_struct(skeleton, Skeleton)
        lib().oracle_pose_compute_relative(C.byref(sk), _ptr(p), _ptr(r))
    return p, r


def pose_blend(pos_a, rot_a, pos_b, rot_b, weight, use_ref=False):
    """Pose::blend (pose.cpp:30-41): a blended towards b by weight -> (pos, rot)."""
    p = np.array(pos_a, np.float32, copy=True)
    r = np.array(rot_a, np.float32, copy=True)
    pb = np.ascontiguousarray(pos_b, np.float32)
    rb = np.ascontiguousarray(rot_b, np.float32)
    f = ref().ref_pose_blend if use_ref else lib().oracle_pose_blend
    f(C.c_uint32(len(p)), _ptr(p), _ptr(r), _ptr(pb), _ptr(rb), C.c_float(weight))
    return p, r


def palettes(skeleton, pos, rot):
    sk = _skeleton_struct(skeleton, Skeleton)
    p = np.ascontiguousarray(pos, np.float32)
    r = np.ascontiguousarray(rot, np.float32)
    dq = np.empty((skeleton.bone_count, 8), np.float32)
    mtx = np.empty((skeleton.bone_count, 16), np.float32)
    lib().oracle_palette_dual_quats(C.byref(sk), _ptr(p), _ptr(r), _ptr(dq))
    lib().oracle_palette_matrices(C.byref(sk), _ptr(p), _ptr(r), _ptr(mtx))
    return dq, mtx


# ---- sort keys / LOD / auto-instancing / radix sort (oracle_sortkeys.c; pipeline.cpp:53-143, 452-523, 3789-4144) ----
SK_MODEL_DTYPE = np.dtype([("lod_distances", np.float32, 4), ("lod_from", np.int32, 5), ("lod_to", np.int32, 5), ("mesh_base", np.uint32), ("mesh_count", np.uint32)])
SK_MESH_DTYPE = np.dtype([("sort_key", np.uint32), ("material_index", np.uint32), ("lod", np.float32), ("layer", np.uint8), ("skinned", np.uint8), ("pad", np.uint16)])
SK_VIEW_DTYPE = np.dtype([("camera_pos", np.float64, 3), ("lod_ref_point", np.float64, 3), ("time_delta", np.float32), ("lod_multiplier", np.float32),
                          ("frame_number", np.uint32), ("is_shadow", np.uint32), ("max_sort_key", np.uint32), ("pad", np.uint32),
                          ("bucket_map", np.uint32, 256), ("layer_to_bucket", np.uint8, 256)])
assert SK_MODEL_DTYPE.itemsize == 64 and SK_MESH_DTYPE.itemsize == 16 and SK_VIEW_DTYPE.itemsize == 48 + 24 + 1024 + 256


def create_sort_keys(visible_ids, visible_types, transforms56, model_of, lod, flags, pose_frame, decal_sort_key, decal_layer, models, meshes, view,
                     sort=True):
    """PipelineImpl::createSortKeys (one worker) + radixSort on flat inputs.  `lod` and `pose_frame` are updated in place like the
    reference's ModelInstance::lod / Pose::frame.  -> dict(keys, values (sorted if `sort`), group_count, group_offset, group_renderables,
    instance_data[n, 48] bytes, pose_list, dirty_list)."""
    L = lib()
    ids = np.ascontiguousarray(visible_ids, np.uint32)
    tys = np.ascontiguousarray(visible_types, np.uint8)
    n = len(ids)
    view = np.ascontiguousarray(view, SK_VIEW_DTYPE).reshape(1)
    n_groups = int(view["max_sort_key"][0]) + 1
    cap_keys = 8 * n + n_groups + 16
    cap_inst = 8 * n + 16
    keys, values = np.zeros(cap_keys, np.uint64), np.zeros(cap_keys, np.uint64)
    gcount, goff = np.zeros(n_groups, np.uint32), np.zeros(n_groups, np.uint32)
    grend, idata = np.zeros(cap_inst, np.uint64), np.zeros((cap_inst, 48), np.uint8)
    pose_list, dirty_list = np.zeros(n + 1, np.uint32), np.zeros(n + 1, np.uint32)
    cnt = (C.c_uint32 * 4)()
    tr = np.ascontiguousarray(transforms56)
    assert tr.dtype.itemsize * (tr.shape[-1] if tr.ndim > 1 else 1) == 56 or tr.dtype.itemsize == 56
    models = np.ascontiguousarray(models, SK_MODEL_DTYPE)
    meshes = np.ascontiguousarray(meshes, SK_MESH_DTYPE)
    assert lod.dtype == np.float32 and lod.flags.c_contiguous and pose_frame.dtype == np.uint32 and pose_frame.flags.c_contiguous
    rc = L.oracle_create_sort_keys(_ptr(ids), _ptr(tys), C.c_uint32(n), _ptr(tr), _ptr(np.ascontiguousarray(model_of, np.uint32)), _ptr(lod),
                                   _ptr(np.ascontiguousarray(flags, np.uint8)), _ptr(pose_frame),
                                   _ptr(np.ascontiguousarray(decal_sort_key, np.uint32)), _ptr(np.ascontiguousarray(decal_layer, np.uint8)),
                                   _ptr(models), _ptr(meshes), _ptr(view), _ptr(keys), _ptr(values), C.c_uint32(cap_keys), C.byref(cnt, 0),
                                   _ptr(gcount), _ptr(goff), _ptr(grend), _ptr(idata), C.c_uint32(cap_inst), C.byref(cnt, 4),
                                   _ptr(pose_list), C.c_uint32(n + 1), C.byref(cnt, 8), _ptr(dirty_list), C.c_uint32(n + 1), C.byref(cnt, 12))
    assert rc == 0, "oracle_create_sort_keys: capacity"
    nk, ni, npose, nd = (int(c) for c in cnt)
    keys, values = keys[:nk].copy(), values[:nk].copy()
    if sort and nk:
        L.oracle_radix_sort(_ptr(keys), _ptr(values), C.c_uint32(nk))
    return dict(keys=keys, values=values, group_count=gcount, group_offset=goff, group_renderables=grend[:ni].copy(), instance_data=idata[:ni].copy(),
                pose_list=pose_list[:npose].copy(), dirty_list=dirty_list[:nd].copy())


def radix_sort(keys, values, reference_copy_back=False):
    """PipelineImpl::radixSort restated; reference_copy_back=True keeps the reference's literal last lines (see oracle_sortkeys.c)."""
    k, v = np.ascontiguousarray(keys, np.uint64).copy(), np.ascontiguousarray(values, np.uint64).copy()
    lib().oracle_radix_sort_ex(_ptr(k), _ptr(v), C.c_uint32(len(k)), C.c_int(1 if reference_copy_back else 0))
    return k, v


def sortkey_packers(which):
    """The oracle's ('oracle') or the reference's own ('ref') packers as a dict of callables with identical signatures."""
    L = lib() if which == "oracle" else ref()
    pre = "oracle_" if which == "oracle" else "ref_"
    sig = {"float_flip": (C.c_uint32, [C.c_uint32]), "make_mesh_sort_key": (C.c_uint64, [C.c_uint32, C.c_uint8]),
           "make_depth_sort_key": (C.c_uint64, [C.c_float, C.c_uint8]), "make_autoinstanced_sort_key": (C.c_uint64, [C.c_int32, C.c_uint8]),
           "make_decal_sort_key": (C.c_uint64, [C.c_uint32, C.c_uint8]), "make_decal_sort_value": (C.c_uint64, [C.c_int32]),
           "make_curve_decal_sort_value": (C.c_uint64, [C.c_int32]), "make_skinned_sort_value": (C.c_uint64, [C.c_int32, C.c_uint32]),
           "make_mesh_sort_value": (C.c_uint64, [C.c_int32, C.c_uint32]), "make_autoinstanced_sort_value": (C.c_uint64, [C.c_uint32, C.c_uint32]),
           "lod_mesh_indices": (C.c_uint32, [vp, C.c_float])}
    out = {}
    for name, (res, args) in sig.items():
        f = getattr(L, pre + name)
        f.restype, f.argtypes = res, args
        out[name] = f
    return out


def ref_radix_sort(keys, values, workers=2):
    """The reference's own PipelineImpl::radixSort (on its job system)."""
    R = ref()
    assert R.ref_jobs_init(C.c_int(workers))
    k, v = np.ascontiguousarray(keys, np.uint64).copy(), np.ascontiguousarray(values, np.uint64).copy()
    R.ref_radix_sort(_ptr(k), _ptr(v), C.c_int(len(k)))
    return k, v
