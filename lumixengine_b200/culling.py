"""Host-side mirror of the reference's CullingSystem interface (src/renderer/culling_system.h:58-77) over the C-ABI.

Method names and argument meaning follow the reference (`add`, `remove`, `setPosition`, `setRadius`, `set`,
`getRadius`, `isAdded`, `cull(frustum[, type])`); array arguments are the batched form of the same calls.
`cull` returns a CullResult-like object (visible ids grouped per renderable type, culling_system.h:17-56).
"""
import ctypes as C

import numpy as np

from . import _lib
from ._lib import ShiftedFrustum, check, ptr, vp

TYPE_ALL = _lib.TYPE_ALL


def frustum_perspective(position, direction, up, fov, ratio, near, far):
    """ShiftedFrustum::computePerspective (src/core/geometry.cpp:470-499) -> ShiftedFrustum POD."""
    f = ShiftedFrustum()
    _lib.lib().lb200_frustum_perspective(C.byref(f), (C.c_double * 3)(*position), (C.c_float * 3)(*direction), (C.c_float * 3)(*up),
                                         C.c_float(fov), C.c_float(ratio), C.c_float(near), C.c_float(far))
    return f


def frustum_ortho(position, direction, up, width, height, near, far):
    """ShiftedFrustum::computeOrtho (src/core/geometry.cpp:390-409)."""
    f = ShiftedFrustum()
    _lib.lib().lb200_frustum_ortho(C.byref(f), (C.c_double * 3)(*position), (C.c_float * 3)(*direction), (C.c_float * 3)(*up),
                                   C.c_float(width), C.c_float(height), C.c_float(near), C.c_float(far))
    return f


def frustum_from_viewport(pos, rot, fov, w, h, near, far, is_ortho=False, ortho_size=100.0):
    """Viewport::getFrustum() (src/core/geometry.cpp:793-818): camera position, rotation quaternion (xyzw), viewport size in pixels."""
    f = ShiftedFrustum()
    _lib.lib().lb200_frustum_from_viewport(C.byref(f), C.c_int(1 if is_ortho else 0), C.c_float(fov), C.c_float(ortho_size), C.c_int(w), C.c_int(h),
                                           (C.c_double * 3)(*pos), (C.c_float * 4)(*rot), C.c_float(near), C.c_float(far))
    return f


def digest_ids(ids, types, n_types=4):
    """Order-independent digest of a visible set: per renderable type (count, sum of ids, xor of ids)."""
    ids = np.asarray(ids).astype(np.uint64)
    types = np.asarray(types)
    out = []
    for t in range(n_types):
        sel = ids[types == t]
        out.append([int(len(sel)), int(sel.sum(dtype=np.uint64)), int(np.bitwise_xor.reduce(sel)) if len(sel) else 0])
    return out


def frustum_bytes(f):
    return np.frombuffer(bytes(f), np.uint8).copy()


def frustum_from_bytes(b):
    return ShiftedFrustum.from_buffer_copy(np.ascontiguousarray(b, np.uint8).tobytes())


class CullResult:
    """Flat form of the CullResult page chain: ids grouped by type; `pages()` re-chunks into <=1020-id pages."""

    PAGE_IDS = 1020  # (4096 - 16) / 4, culling_system.h:55

    def __init__(self, ids, raw):
        self.ids = ids
        self.raw = raw
        self.total = int(raw.total)
        self.type_count = np.ctypeslib.as_array(raw.type_count).copy()
        self.type_offset = np.ctypeslib.as_array(raw.type_offset).copy()
        self.stats = dict(pages_tested=int(raw.pages_tested), pages_inside=int(raw.pages_inside), pages_outside=int(raw.pages_outside),
                          pages_filtered=int(raw.pages_filtered), entities_tested=int(raw.entities_tested), entities_inside=int(raw.entities_inside))

    def count(self):  # CullResult::count, culling_system.h:26-34
        return self.total

    def of_type(self, t):
        o, c = int(self.type_offset[t]), int(self.type_count[t])
        return self.ids[o:o + c]

    def types(self):
        """uint8 type of every id, aligned with `ids`."""
        out = np.empty(self.total, np.uint8)
        for t in np.nonzero(self.type_count)[0]:
            o, c = int(self.type_offset[t]), int(self.type_count[t])
            out[o:o + c] = t
        return out

    def pages(self):
        """[(type, ids<=1020)] — what the engine-side shim writes into PageAllocator pages (INTEGRATION.md)."""
        out = []
        for t in np.nonzero(self.type_count)[0]:
            seg = self.of_type(int(t))
            for s in range(0, len(seg), self.PAGE_IDS):
                out.append((int(t), seg[s:s + self.PAGE_IDS]))
        return out


class CullingSystem:
    """CullingSystem::create(allocator, page_allocator) -> here CullingSystem(ctx).  ctx=None gives the host bookkeeping only
    (no device; `cull` raises NoDeviceError)."""

    def __init__(self, ctx=None):
        self.L = _lib.lib()
        self.ctx = ctx
        h = vp()
        check(self.L.lb200_culling_create(ctx.h if ctx else None, C.byref(h)), ctx.h if ctx else None)
        self.h = h
        if ctx is not None:
            ctx._adopt(self)
        self._out = None
        self._out_pinned = None

    def close(self):
        if self.h:
            self.L.lb200_culling_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def _err(self, rc):
        check(rc, self.ctx.h if self.ctx else None)

    # ---- CullingSystem virtuals (scalar or array arguments) ----
    def add(self, entity, type, pos, radius):
        e = np.atleast_1d(np.asarray(entity, np.int32))
        t = np.ascontiguousarray(np.broadcast_to(np.asarray(type, np.uint8), e.shape))
        p = np.ascontiguousarray(np.asarray(pos, np.float64).reshape(-1, 3))
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, np.float32), e.shape))
        self._err(self.L.lb200_culling_add_many(self.h, ptr(e), ptr(t), ptr(p), ptr(r), C.c_uint32(len(e))))

    def remove(self, entity):
        e = np.atleast_1d(np.asarray(entity, np.int32))
        self._err(self.L.lb200_culling_remove_many(self.h, ptr(e), C.c_uint32(len(e))))

    def setPosition(self, entity, pos):
        e = np.atleast_1d(np.asarray(entity, np.int32))
        p = np.ascontiguousarray(np.asarray(pos, np.float64).reshape(-1, 3))
        self._err(self.L.lb200_culling_set_position_many(self.h, ptr(e), ptr(p), C.c_uint32(len(e))))

    def setRadius(self, entity, radius):
        e = np.atleast_1d(np.asarray(entity, np.int32))
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, np.float32), e.shape))
        self._err(self.L.lb200_culling_set_radius_many(self.h, ptr(e), ptr(r), C.c_uint32(len(e))))

    def set(self, entity, pos, radius, unique=False):
        """CullingSystem::set for one entity or a batch.  unique=True promises that no entity is listed twice (the sphere refresh after a
        propagate): in-cell movers are then overwritten in place on all host cores (lb200_culling_set_many_unique)."""
        e = np.atleast_1d(np.asarray(entity, np.int32))
        p = np.ascontiguousarray(np.asarray(pos, np.float64).reshape(-1, 3))
        r = np.ascontiguousarray(np.broadcast_to(np.asarray(radius, np.float32), e.shape))
        f = self.L.lb200_culling_set_many_unique if unique else self.L.lb200_culling_set_many
        self._err(f(self.h, ptr(e), ptr(p), ptr(r), C.c_uint32(len(e))))

    def getRadius(self, entity):
        return float(self.L.lb200_culling_get_radius(self.h, C.c_int32(entity)))

    def isAdded(self, entity):
        return bool(self.L.lb200_culling_is_added(self.h, C.c_int32(entity)))

    # ---- introspection ----
    def page_count(self):
        return int(self.L.lb200_culling_page_count(self.h))

    def entity_count(self):
        return int(self.L.lb200_culling_entity_count(self.h))

    def pages(self):
        out = []
        for i in range(self.page_count()):
            o = (C.c_double * 3)()
            ind = (C.c_int32 * 3)()
            ty, big, cnt = C.c_uint8(), C.c_uint8(), C.c_uint32()
            sph = np.empty((_lib.PAGE_SLOTS, 4), np.float32)
            ent = np.empty(_lib.PAGE_SLOTS, np.int32)
            self._err(self.L.lb200_culling_get_page(self.h, C.c_uint32(i), o, ind, C.byref(ty), C.byref(big), C.byref(cnt), ptr(sph), ptr(ent)))
            c = cnt.value
            out.append(dict(origin=tuple(o), indices=tuple(ind), type=ty.value, is_big=big.value, count=c, spheres=sph[:c].copy(), entities=ent[:c].copy()))
        return out

    # ---- cull ----
    def _out_buffer(self, n):
        if self._out is None or len(self._out) < n:
            cap = max(n, 1024)
            self._out = self.ctx.host_alloc(cap, np.uint32) if self.ctx else np.empty(cap, np.uint32)
        return self._out

    def cull(self, frustum, type=TYPE_ALL):
        """CullingSystem::cull(frustum[, type]) (culling_system.cpp:310-369): host frustum in, visible ids out (host)."""
        if type != TYPE_ALL and not 0 <= type < 0xFF:
            raise ValueError("type must be 0..254 (0xff is reserved for all types, culling_system.cpp:312)")
        out = self._out_buffer(self.entity_count())
        res = _lib.CullResult()
        rc = self.L.lb200_culling_cull(self.h, C.byref(frustum), C.c_uint8(type), ptr(out), C.c_uint32(len(out)), C.byref(res))
        self._err(rc)
        # a view of the page-locked result buffer, valid until the next cull on this object (the engine shim copies it into CullResult pages)
        return CullResult(out[:res.total], res)

    def cull_begin(self, frustum, type=TYPE_ALL):
        """Non-blocking form of cull(): enqueue the cull and the device-side write of the result into the page-locked buffer."""
        out = self._out_buffer(self.entity_count())
        self._err(self.L.lb200_culling_cull_begin(self.h, C.byref(frustum), C.c_uint8(type), ptr(out), C.c_uint32(len(out))))

    def cull_poll(self):
        """True once the cull started by cull_begin has finished (a job would yield and ask again)."""
        rc = self.L.lb200_culling_cull_poll(self.h)
        if rc < 0:
            self._err(rc)
        return rc == 1

    def cull_end(self):
        """Result of the cull started by cull_begin (waits if it still has to): the same CullResult view cull() returns."""
        res = _lib.CullResult()
        self._err(self.L.lb200_culling_cull_end(self.h, C.byref(res)))
        return CullResult(self._out[:res.total], res)

    def cull_device(self, frustum, type=TYPE_ALL, want_counts=True):
        """Same cull, ids stay in HBM: returns (device pointer int, lb200_cull_result or None)."""
        dev = vp()
        res = _lib.CullResult()
        rc = self.L.lb200_culling_cull_device(self.h, C.byref(frustum), C.c_uint8(type), C.byref(dev), C.byref(res) if want_counts else None,
                                              C.c_int(1 if want_counts else 0))
        self._err(rc)
        return (dev.value or 0), (res if want_counts else None)

    def cull_device_n(self, frustum, n, type=TYPE_ALL):
        """n independent asynchronous culls issued from C: consecutive ones run on different streams / output lanes and overlap."""
        self._err(self.L.lb200_culling_cull_device_n(self.h, C.byref(frustum), C.c_uint8(type), C.c_uint32(n)))

    def cull_views(self, frusta, types=None, want_counts=True):
        """Several views of the same scene culled in one pass over the pages (lb200_culling_cull_views): a frame's main camera and its shadow
        cascades.  frusta: 1..8 ShiftedFrustum; types: None (every view culls all types) or one type filter per view (0xff = all).  Returns
        [(device ids pointer, lb200_cull_result or None)] per view, each equal to a lone cull_device of that view.  The results stay valid
        until the next cull_views call; select_view(k) makes view k the last cull."""
        frusta = list(frusta)
        n = len(frusta)
        arr = (ShiftedFrustum * max(n, 1))(*frusta)
        ty = None
        if types is not None:
            ty = np.ascontiguousarray(types, np.uint8)
            if len(ty) != n:
                raise ValueError(f"{len(ty)} type filters for {n} views")
        dev = (vp * max(n, 1))()
        res = (_lib.CullResult * max(n, 1))()
        self._err(self.L.lb200_culling_cull_views(self.h, arr if n else None, ptr(ty), C.c_uint32(n), dev, res if want_counts else None,
                                                  C.c_int(1 if want_counts else 0)))
        return [((dev[v] or 0), (res[v] if want_counts else None)) for v in range(n)]

    def select_view(self, k):
        """Make view k of the latest cull_views call the last cull (last_result, read_bitmask, SortKeys.createSortKeys)."""
        self._err(self.L.lb200_culling_select_view(self.h, C.c_uint32(k)))

    def last_result(self):
        """(device ids pointer, lb200_cull_result) of the cull issued last (e.g. the last one of cull_device_n)."""
        dev = vp()
        res = _lib.CullResult()
        self._err(self.L.lb200_culling_last_result(self.h, C.byref(dev), C.byref(res)))
        return (dev.value or 0), res

    def flush(self):
        self._err(self.L.lb200_culling_flush(self.h))

    def set_replicas(self, n):
        self._err(self.L.lb200_culling_set_replicas(self.h, C.c_uint32(n)))

    def read_bitmask(self):
        n = self.page_count()
        out = np.zeros(max(n, 1) * 8, np.uint32)
        self._err(self.L.lb200_culling_read_bitmask(self.h, ptr(out), C.c_uint32(len(out))))
        return out[:n * 8].reshape(n, 8)

    def set_many_device(self, dev_pos3, dev_radius, n, dev_entities=None, max_entity=None):
        """CullingSystem::set for n distinct entities whose new spheres lie in device memory (pointers as ints); the host mirror follows lazily."""
        self._err(self.L.lb200_culling_set_many_device(self.h, vp(dev_entities) if dev_entities else None, vp(dev_pos3), vp(dev_radius), C.c_uint32(n),
                                                        C.c_uint32(n - 1 if max_entity is None else max_entity)))
        return int(self.L.lb200_culling_last_rebin_changers(self.h))

    def add_many_device(self, dev_pos3, dev_radius, dev_types, n, dev_entities=None, max_entity=None):
        """CullingSystem::add for n entities whose spheres (f64[n, 3], f32[n]) and types (u8[n]) lie in device memory (pointers as ints).
        Ids must lie in [0, max_entity], be new and distinct, types below 0xff; otherwise nothing changes and LumixB200Error is raised."""
        self._err(self.L.lb200_culling_add_many_device(self.h, vp(dev_entities) if dev_entities else None, vp(dev_types), vp(dev_pos3), vp(dev_radius),
                                                        C.c_uint32(n), C.c_uint32(n - 1 if max_entity is None else max_entity)))

    def remove_many_device(self, dev_entities, n):
        """CullingSystem::remove for n entity ids (i32[n]) in device memory; ids that are not added are skipped, duplicates removed once."""
        self._err(self.L.lb200_culling_remove_many_device(self.h, vp(dev_entities), C.c_uint32(n)))

    def sync_host(self):
        self._err(self.L.lb200_culling_sync_host(self.h))

    def time_lone_cull(self, frustum, iters=20, type=TYPE_ALL, mode=0):
        """Device time (ms, per iteration) of single culls that have the device to themselves, launch pre-queued (no host latency).
        mode 1 / 2: nothing / one empty kernel of the same grid between the events (the fixed costs inside the number)."""
        out = np.zeros(iters, np.float32)
        self._err(self.L.lb200_culling_time_lone_cull(self.h, C.byref(frustum), C.c_uint8(type), C.c_uint32(iters), C.c_int(mode), ptr(out)))
        return out

    def last_algorithmic_bytes(self):
        return int(self.L.lb200_culling_last_algorithmic_bytes(self.h))

    def setLaunch(self, blocks=0, chunk=0, plane_masking=-1):
        """Launch shape of later culls on this object (lb200_culling_set_launch): blocks 0 = the default rule, -1 = every co-resident
        block, n > 0 = exactly n; chunk 0 = the default, 1..256 pages per block per round; plane_masking -1 = automatic, 0 = off."""
        self._err(self.L.lb200_culling_set_launch(self.h, C.c_int(blocks), C.c_int(chunk), C.c_int(plane_masking)))

    def lastLaunch(self):
        """dict(blocks, chunk, rounds, pdl, plane_masking) of the last cull (the last of a batch); zeros before the first."""
        b, c, r, p, m = C.c_uint32(), C.c_uint32(), C.c_uint32(), C.c_int(), C.c_int()
        self._err(self.L.lb200_culling_get_launch(self.h, C.byref(b), C.byref(c), C.byref(r), C.byref(p), C.byref(m)))
        return dict(blocks=int(b.value), chunk=int(c.value), rounds=int(r.value), pdl=bool(p.value), plane_masking=bool(m.value))

    def allgather(self, slab_ids, n_ranks):
        """Exchange of the cull just issued: returns (device pointer of the gathered slabs, counts[n_ranks, 256])."""
        counts = np.zeros(n_ranks * 256, np.uint32)
        dev = vp()
        self._err(self.L.lb200_culling_allgather(self.h, C.c_uint32(slab_ids), C.byref(dev), ptr(counts)))
        return (dev.value or 0), counts.reshape(n_ranks, 256)

    def cull_gather(self, frustum, slab_ids, type=TYPE_ALL):
        """Per-frame multi-GPU step, asynchronous: cull + device-side pack + one NCCL all-gather.  Returns the device pointer."""
        dev = vp()
        self._err(self.L.lb200_culling_cull_gather(self.h, C.byref(frustum), C.c_uint8(type), C.c_uint32(slab_ids), C.byref(dev)))
        return dev.value or 0

    def page_ids(self):
        """Device page id of every m_cells entry (row of the page in the HBM arrays and the visibility bitmask)."""
        return np.array([self.L.lb200_culling_page_id(self.h, C.c_uint32(i)) for i in range(self.page_count())], np.int64)

    def exchange_slab_words(self):
        """u32 words one rank contributes to the bitmask exchange; pass max over ranks - 256 to Context.comm_enable_p2p."""
        return int(self.L.lb200_culling_exchange_slab_words(self.h))

    def cull_exchange(self, frustum, type=TYPE_ALL):
        """Per-frame multi-GPU step, asynchronous: the cull kernel stores visibility rows + per-type counts into every rank's memory
        (NVLink peer stores); ids stay sharded.  Returns (device ids pointer, device slabs pointer, slab stride in words)."""
        ids, slabs, stride = vp(), vp(), C.c_uint32()
        self._err(self.L.lb200_culling_cull_exchange(self.h, C.byref(frustum), C.c_uint8(type), C.byref(ids), C.byref(slabs), C.byref(stride)))
        return (ids.value or 0), (slabs.value or 0), int(stride.value)

    def cull_exchange_n(self, frustum, n, type=TYPE_ALL):
        """n independent exchange steps issued from C on the internal lanes; returns the (ids, slabs, stride) of the last step."""
        ids, slabs, stride = vp(), vp(), C.c_uint32()
        self._err(self.L.lb200_culling_cull_exchange_n(self.h, C.byref(frustum), C.c_uint8(type), C.c_uint32(n), C.byref(ids), C.byref(slabs), C.byref(stride)))
        return (ids.value or 0), (slabs.value or 0), int(stride.value)

    def read_exchanged(self, slabs_ptr, stride, n_ranks):
        """Host copy of the exchanged slabs -> per rank dict(counts[256], n_pages, n_records, mask[n_pages, 8] by page id).
        A slab holds one {page id, visibility row} record per page the rank worked on (cull_kernel.cuh); every other page's row is zero."""
        host = self.ctx.copy_to_host(slabs_ptr, stride * n_ranks, np.uint32).reshape(n_ranks, stride)
        out = []
        for r in range(n_ranks):
            n_pages, n_rec, _, cap = (int(v) for v in host[r, 256:260])
            pages = host[r, 264:264 + n_rec]
            rows = host[r, 264 + cap:264 + cap + 8 * n_rec].reshape(n_rec, 8)
            mask = np.zeros((n_pages, 8), np.uint32)
            mask[pages] = rows
            out.append(dict(counts=host[r, :256].copy(), n_pages=n_pages, n_records=n_rec, mask=mask))
        return out

    def read_gathered(self, dev_ptr, slab_ids, n_ranks, stride=None):
        """Host copy of the gathered buffer -> (slabs[r] = ids of rank r, counts[n_ranks, 256])."""
        stride = int(self.L.lb200_culling_gather_stride_words(self.h, C.c_uint32(slab_ids))) if stride is None else stride
        host = self.ctx.copy_to_host(dev_ptr, stride * n_ranks, np.uint32).reshape(n_ranks, stride)
        return [host[r, 256:256 + slab_ids] for r in range(n_ranks)], host[:, :256].copy()
