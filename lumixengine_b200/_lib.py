"""ctypes loader for liblumix_b200.so (the C-ABI of include/lumix_b200.h).

The CUDA library is the product: there is no Python or CPU fallback.  A missing .so raises at import of the first
compute object, a missing GPU raises NoDeviceError from Context().
"""
import ctypes as C
import os
import subprocess
import weakref

HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.path.join(HERE, "liblumix_b200.so")

OK = 0
ERR_NO_DEVICE = -1
ERR_CUDA = -2
ERR_INVALID = -3
ERR_CAPACITY = -4
ERR_NCCL = -5
ERR_STATE = -6
TYPE_ALL = 0xFF
PAGE_SLOTS = 200

PALETTE_DUAL_QUAT = 1
PALETTE_MATRIX = 2
PALETTE_POSE = 4

vp = C.c_void_p


class LumixB200Error(RuntimeError):
    def __init__(self, code, text=""):
        self.code = code
        names = {ERR_NO_DEVICE: "NO_DEVICE", ERR_CUDA: "CUDA", ERR_INVALID: "INVALID", ERR_CAPACITY: "CAPACITY", ERR_NCCL: "NCCL", ERR_STATE: "STATE"}
        super().__init__(f"lumix_b200 error {names.get(code, code)}: {text}")


class NoDeviceError(LumixB200Error):
    pass


class ShiftedFrustum(C.Structure):
    """ShiftedFrustum, src/core/geometry.h:99-149 (256 bytes)."""
    _fields_ = [("xs", C.c_float * 8), ("ys", C.c_float * 8), ("zs", C.c_float * 8), ("ds", C.c_float * 8),
                ("points", (C.c_float * 3) * 8), ("origin", C.c_double * 3), ("pad_", C.c_uint64)]


assert C.sizeof(ShiftedFrustum) == 256


class CullResult(C.Structure):
    _fields_ = [("total", C.c_uint32), ("n_types", C.c_uint32), ("type_count", C.c_uint32 * 256), ("type_offset", C.c_uint32 * 256),
                ("pages_tested", C.c_uint32), ("pages_inside", C.c_uint32), ("pages_outside", C.c_uint32), ("pages_filtered", C.c_uint32),
                ("entities_tested", C.c_uint32), ("entities_inside", C.c_uint32)]


class Track(C.Structure):
    _fields_ = [("bone_index", C.c_uint16), ("offset_bits", C.c_uint16), ("bitsizes", C.c_uint8 * 3), ("skipped_channel", C.c_uint8),
                ("min", C.c_float * 3), ("to_range", C.c_float * 3)]


class ConstTranslation(C.Structure):
    _fields_ = [("bone_index", C.c_uint16), ("pad", C.c_uint16), ("value", C.c_float * 3)]


class ConstRotation(C.Structure):
    _fields_ = [("bone_index", C.c_uint16), ("pad", C.c_uint16), ("value", C.c_float * 4)]


class Clip(C.Structure):
    _fields_ = [("fps", C.c_float), ("frame_count", C.c_uint32), ("translations_frame_size_bits", C.c_uint32), ("rotations_frame_size_bits", C.c_uint32),
                ("n_translations", C.c_uint32), ("n_const_translations", C.c_uint32), ("n_rotations", C.c_uint32), ("n_const_rotations", C.c_uint32),
                ("translations", vp), ("const_translations", vp), ("rotations", vp), ("const_rotations", vp),
                ("translation_stream", vp), ("translation_stream_bytes", C.c_uint32),
                ("rotation_stream", vp), ("rotation_stream_bytes", C.c_uint32)]


class Skeleton(C.Structure):
    _fields_ = [("bone_count", C.c_uint32), ("first_nonroot_bone_index", C.c_int32), ("parents", vp), ("bind_relative7", vp), ("inverse_bind7", vp)]


class SkPalettes(C.Structure):
    """lb200_sk_palettes: device pointers of the latest lb200_sortkeys_build_palettes."""
    _fields_ = [("dual_quats", vp), ("offset", vp), ("n_bones", vp)]


class Mesh(C.Structure):
    _fields_ = [("n_vertices", C.c_uint32), ("positions3", vp), ("weights4", vp), ("indices4", vp)]


# every symbol include/lumix_b200.h declares (tests/test_abi.py checks the header against this and the .so)
SYMBOLS = [
    "lb200_init", "lb200_shutdown", "lb200_last_error", "lb200_device_count", "lb200_synchronize", "lb200_host_callback", "lb200_launch_count", "lb200_stream_handle",
    "lb200_init_background", "lb200_host_alloc", "lb200_host_free", "lb200_copy_to_host", "lb200_device_alloc", "lb200_device_free", "lb200_copy_to_device", "lb200_event_create", "lb200_event_record", "lb200_event_elapsed_ms", "lb200_event_destroy",
    "lb200_frustum_perspective", "lb200_frustum_ortho", "lb200_frustum_from_viewport",
    "lb200_culling_create", "lb200_culling_destroy", "lb200_culling_add", "lb200_culling_remove", "lb200_culling_set_position",
    "lb200_culling_set_radius", "lb200_culling_set", "lb200_culling_get_radius", "lb200_culling_is_added",
    "lb200_culling_add_many", "lb200_culling_set_many", "lb200_culling_set_many_unique", "lb200_culling_set_position_many", "lb200_culling_set_radius_many", "lb200_culling_remove_many",
    "lb200_culling_page_count", "lb200_culling_entity_count", "lb200_culling_get_page",
    "lb200_culling_cull", "lb200_culling_cull_begin", "lb200_culling_cull_poll", "lb200_culling_cull_end", "lb200_culling_cull_device", "lb200_culling_cull_device_n", "lb200_culling_last_result", "lb200_culling_flush", "lb200_culling_read_bitmask", "lb200_culling_set_replicas",
    "lb200_culling_last_algorithmic_bytes", "lb200_culling_time_lone_cull", "lb200_culling_set_launch", "lb200_culling_get_launch", "lb200_culling_set_many_device", "lb200_culling_sync_host", "lb200_culling_last_rebin_changers",
    "lb200_culling_add_many_device", "lb200_culling_remove_many_device", "lb200_culling_cull_views", "lb200_culling_select_view",
    "lb200_comm_get_unique_id", "lb200_comm_init", "lb200_comm_destroy", "lb200_comm_enable_p2p", "lb200_comm_status", "lb200_culling_gather_stride_words", "lb200_culling_allgather", "lb200_culling_cull_gather",
    "lb200_culling_cull_exchange", "lb200_culling_cull_exchange_n", "lb200_culling_exchange_slab_words", "lb200_culling_page_id",
    "lb200_sortkeys_create", "lb200_sortkeys_destroy", "lb200_sortkeys_set_models", "lb200_sortkeys_set_instances", "lb200_sortkeys_set_transforms",
    "lb200_sortkeys_set_transforms_device", "lb200_sortkeys_create_keys", "lb200_sortkeys_create_keys_views", "lb200_sortkeys_set_launch", "lb200_sortkeys_get_launch", "lb200_sortkeys_device_outputs",
    "lb200_sortkeys_view_outputs",
    "lb200_sortkeys_move_device", "lb200_sortkeys_end_frame", "lb200_sortkeys_prev_transforms", "lb200_sortkeys_moved_list", "lb200_sortkeys_max_entities",
    "lb200_sortkeys_spawn_instances_device", "lb200_sortkeys_spawn_decals_device", "lb200_sortkeys_clear_dirty_device", "lb200_radix_sort_device", "lb200_animation_bone_attachments_device",
    "lb200_animation_set_entities", "lb200_sortkeys_build_palettes",
    "lb200_clusters_create", "lb200_clusters_destroy", "lb200_clusters_set_point_lights", "lb200_clusters_set_atlas", "lb200_clusters_fill",
    "lb200_clusters_patch_atlas", "lb200_clusters_outputs", "lb200_clusters_set_launch", "lb200_clusters_get_launch",
    "lb200_hierarchy_create", "lb200_hierarchy_destroy", "lb200_hierarchy_depth",
    "lb200_hierarchy_set_parents", "lb200_hierarchy_set_parents_device", "lb200_hierarchy_get_level_order", "lb200_hierarchy_set_locals", "lb200_hierarchy_set_root_globals", "lb200_hierarchy_set_subset",
    "lb200_hierarchy_propagate", "lb200_hierarchy_get_globals", "lb200_hierarchy_get_spheres", "lb200_hierarchy_refresh_spheres", "lb200_hierarchy_get_relative_matrices", "lb200_hierarchy_set_globals", "lb200_hierarchy_compute_locals", "lb200_hierarchy_get_locals", "lb200_hierarchy_algorithmic_bytes",
    "lb200_hierarchy_set_entities", "lb200_hierarchy_mark_moved", "lb200_hierarchy_propagate_moved",
    "lb200_hierarchy_set_attachments", "lb200_hierarchy_propagate_attached", "lb200_hierarchy_get_attachment_rounds",
    "lb200_animation_create", "lb200_animation_destroy", "lb200_animation_set_instances", "lb200_animation_update", "lb200_animation_update_many", "lb200_animation_skin",
    "lb200_animation_set_launch", "lb200_animation_get_launch",
    "lb200_animation_get_dual_quats", "lb200_animation_get_matrices", "lb200_animation_get_pose", "lb200_animation_get_times", "lb200_animation_set_layers", "lb200_animation_set_samples", "lb200_animation_set_stacks", "lb200_animation_set_root_motion", "lb200_animation_bone_attachments", "lb200_animation_compute_relative", "lb200_animation_get_relative_pose", "lb200_animation_blend_pose",
    "lb200_animation_get_skinned", "lb200_animation_skinned_checksum", "lb200_animation_algorithmic_bytes",
]

_lib = None


def source_hash():
    """sha256 over the sources liblumix_b200.so is built from (csrc/*, include/lumix_b200.h), in name order."""
    import glob
    import hashlib
    h = hashlib.sha256()
    files = sorted(glob.glob(os.path.join(HERE, "csrc", "*.cu")) + glob.glob(os.path.join(HERE, "csrc", "*.cuh")) + glob.glob(os.path.join(HERE, "csrc", "*.h"))
                   + glob.glob(os.path.join(HERE, "csrc", "*.hpp")) + [os.path.join(HERE, "csrc", "Makefile"), os.path.join(os.path.dirname(HERE), "include", "lumix_b200.h")])
    for f in files:
        h.update(os.path.basename(f).encode())
        h.update(open(f, "rb").read())
    return h.hexdigest()[:16]


def recorded_source_hash():
    p = SO_PATH + ".srchash"
    return open(p).read().strip() if os.path.exists(p) else None


def build():
    """Compile liblumix_b200.so for sm_90a (nvcc cross-compiles without a GPU) and record the hash of the sources next to it."""
    subprocess.check_call(["make", "-s", "-C", os.path.join(HERE, "csrc"), "-j8"])
    with open(SO_PATH + ".srchash", "w") as f:
        f.write(source_hash() + "\n")


def lib():
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise ImportError(f"{SO_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` (there is no CPU fallback)")
    L = C.CDLL(SO_PATH)
    L.lb200_last_error.restype = C.c_char_p
    L.lb200_last_error.argtypes = [vp]
    L.lb200_launch_count.restype = C.c_uint64
    L.lb200_launch_count.argtypes = [vp]
    L.lb200_stream_handle.restype = C.c_uint64
    L.lb200_stream_handle.argtypes = [vp]
    L.lb200_culling_get_radius.restype = C.c_float
    L.lb200_culling_page_count.restype = C.c_uint32
    L.lb200_culling_last_rebin_changers.restype = C.c_uint32
    L.lb200_culling_entity_count.restype = C.c_uint32
    L.lb200_culling_gather_stride_words.restype = C.c_uint32
    L.lb200_culling_exchange_slab_words.restype = C.c_uint32
    L.lb200_culling_page_id.restype = C.c_int32
    L.lb200_culling_last_algorithmic_bytes.restype = C.c_uint64
    L.lb200_sortkeys_max_entities.restype = C.c_uint32
    L.lb200_sortkeys_max_entities.argtypes = [vp]
    L.lb200_hierarchy_depth.restype = C.c_uint32
    L.lb200_hierarchy_algorithmic_bytes.restype = C.c_uint64
    L.lb200_animation_algorithmic_bytes.restype = C.c_uint64
    L.lb200_shutdown.restype = None
    L.lb200_sortkeys_destroy.restype = None
    L.lb200_clusters_destroy.restype = None
    L.lb200_clusters_destroy.argtypes = [vp]
    L.lb200_host_alloc.restype = vp
    L.lb200_host_alloc.argtypes = [vp, C.c_size_t]
    L.lb200_host_free.restype = None
    L.lb200_device_alloc.restype = vp
    L.lb200_device_alloc.argtypes = [vp, C.c_size_t]
    L.lb200_device_free.restype = None
    L.lb200_device_free.argtypes = [vp, vp]
    L.lb200_host_free.argtypes = [vp, vp]
    L.lb200_event_destroy.restype = None
    L.lb200_event_destroy.argtypes = [vp, vp]
    L.lb200_event_record.argtypes = [vp, vp]
    L.lb200_culling_destroy.restype = None
    L.lb200_hierarchy_destroy.restype = None
    L.lb200_animation_destroy.restype = None
    L.lb200_animation_update_many.argtypes = [C.POINTER(vp), C.c_uint32, C.c_float, C.c_uint32]
    L.lb200_animation_set_entities.argtypes = [vp, vp, C.c_uint32]
    L.lb200_sortkeys_build_palettes.argtypes = [vp, C.POINTER(vp), C.c_uint32, C.c_int, C.POINTER(SkPalettes)]
    L.lb200_comm_destroy.restype = None
    L.lb200_frustum_perspective.restype = None
    L.lb200_frustum_ortho.restype = None
    for name in ("lb200_shutdown", "lb200_culling_destroy", "lb200_hierarchy_destroy", "lb200_animation_destroy", "lb200_comm_destroy", "lb200_synchronize"):
        getattr(L, name).argtypes = [vp]
    _lib = L
    return L


def check(rc, ctx_handle=None):
    if rc == OK:
        return
    text = lib().lb200_last_error(ctx_handle)
    text = text.decode(errors="replace") if text else ""
    if rc == ERR_NO_DEVICE:
        raise NoDeviceError(rc, text)
    raise LumixB200Error(rc, text)


def ptr(a):
    return None if a is None else a.ctypes.data_as(vp)


LB200_ERR_CUDA_CODE = -2


class Context:
    """One GPU + one stream (lb200_ctx)."""

    def __init__(self, device=0, background=False):
        self.L = lib()
        h = vp()
        check((self.L.lb200_init_background if background else self.L.lb200_init)(C.c_int(device), C.byref(h)), None)
        self.h = h
        self.device = device
        self._children = weakref.WeakSet()  # objects that hold device memory of this context

    def _adopt(self, child):
        self._children.add(child)

    def synchronize(self):
        check(self.L.lb200_synchronize(self.h), self.h)

    @property
    def launches(self):
        return int(self.L.lb200_launch_count(self.h))

    @property
    def stream(self):
        return int(self.L.lb200_stream_handle(self.h))

    def close(self):
        if self.h:
            for child in list(self._children):
                child.close()
            self.L.lb200_shutdown(self.h)
            self.h = None

    def host_alloc(self, n, dtype):
        """Page-locked numpy array of n elements."""
        import numpy as np
        dt = np.dtype(dtype)
        p = self.L.lb200_host_alloc(self.h, C.c_size_t(max(n, 1) * dt.itemsize))
        if not p:
            check(ERR_CUDA, self.h)
        buf = (C.c_uint8 * (max(n, 1) * dt.itemsize)).from_address(p)
        return np.frombuffer(buf, dtype=dt, count=n)

    def to_device(self, array):
        """Device copy of a numpy array -> device pointer (int); free it with free_device."""
        import numpy as np
        a = np.ascontiguousarray(array)
        p = self.L.lb200_device_alloc(self.h, C.c_size_t(max(a.nbytes, 1)))
        if not p:
            check(LB200_ERR_CUDA_CODE, self.h)
        check(self.L.lb200_copy_to_device(self.h, vp(p), ptr(a), C.c_size_t(a.nbytes)), self.h)
        return p

    def free_device(self, dev_ptr):
        self.L.lb200_device_free(self.h, vp(dev_ptr))

    def copy_to_host(self, dev_ptr, n, dtype):
        """numpy array of n elements read from a device pointer this library handed out."""
        import numpy as np
        out = np.empty(n, dtype)
        check(self.L.lb200_copy_to_host(self.h, ptr(out), vp(dev_ptr), C.c_size_t(out.nbytes)), self.h)
        return out

    def event(self):
        e = vp()
        check(self.L.lb200_event_create(self.h, C.byref(e)), self.h)
        return e

    def record(self, e):
        check(self.L.lb200_event_record(self.h, e), self.h)

    def elapsed_ms(self, a, b):
        ms = C.c_float()
        check(self.L.lb200_event_elapsed_ms(self.h, a, b, C.byref(ms)), self.h)
        return float(ms.value)

    # multi-GPU
    def comm_unique_id(self):
        import numpy as np
        out = np.zeros(128, np.uint8)
        check(self.L.lb200_comm_get_unique_id(self.h, ptr(out)), self.h)
        return out

    def comm_init(self, n_ranks, rank, unique_id):
        import numpy as np
        uid = np.ascontiguousarray(unique_id, np.uint8)
        check(self.L.lb200_comm_init(self.h, C.c_int(n_ranks), C.c_int(rank), ptr(uid)), self.h)

    def comm_enable_p2p(self, max_slab_ids):
        """Collective: NVLink peer exchange for cull_gather (lb200_comm_enable_p2p)."""
        check(self.L.lb200_comm_enable_p2p(self.h, C.c_uint32(max_slab_ids)), self.h)


def device_count():
    return int(lib().lb200_device_count())
