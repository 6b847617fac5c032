"""Spawns into the sort-key records on the device (SortKeys.spawnInstancesDevice / spawnDecalsDevice / clearDirtyDevice,
lb200_sortkeys_spawn_*_device), growth of the per-entity arrays, and the moved list across spawns.

The expected outputs come from oracle.create_sort_keys on flat per-entity arrays, which this module edits with the spawn rules of
RenderModuleImpl::createModelInstance + setModel + modelLoaded (render_module.cpp:3284-3292, :3107-3148, :2911-2951), createDecal +
updateDecalInfo, onModelInstanceMoved and endFrame (`World` below keeps that restatement to itself).  The culling side is a device-authoritative
CullingSystem edited with add_many_device / remove_many_device / set_many_device next to the oracle's, as a spawn frame issues them.
"""
import ctypes as C

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib, scenes, sortkeys
from lumixengine_b200._lib import LumixB200Error

pytestmark = pytest.mark.gpu

LIGHT = (0.3, -0.8, 0.2)
CASCADES = (40.0, 200.0, 900.0, 2500.0)
SHADOW_BUCKETS = [0, 0xff, 0xff, 1]
TIME_DELTA = 0.15
EXTENT = np.array([2500.0, 300.0, 2500.0])
MOVED, DIRTY = sortkeys.MOVED, sortkeys.DIRTY


def spawn_lod(models, m):
    """modelLoaded (render_module.cpp:2942-2948): the highest LOD 3 .. 0 whose `to` is not -1, else ModelInstance::lod's initial 4."""
    for l in range(3, -1, -1):
        if models["lod_to"][m][l] != -1:
            return np.float32(l)
    return np.float32(4.0)


def _canon(keys, values):
    o = np.lexsort((values, keys))
    return keys[o], values[o]


def _compare_view(got, exp, what):
    assert np.all(got["keys"][1:] >= got["keys"][:-1]), f"{what}: keys not sorted"
    gk, gv = _canon(got["keys"], got["values"])
    ek, ev = _canon(exp["keys"], exp["values"])
    assert np.array_equal(gk, ek) and np.array_equal(gv, ev), f"{what}: pairs differ ({len(gk)} against {len(ek)})"
    assert np.array_equal(got["group_count"], exp["group_count"]) and np.array_equal(got["group_offset"], exp["group_offset"]), what
    go, eo = np.argsort(got["group_renderables"], kind="stable"), np.argsort(exp["group_renderables"], kind="stable")
    assert np.array_equal(got["group_renderables"][go], exp["group_renderables"][eo]), what
    g_of = np.repeat(np.arange(len(exp["group_count"])), exp["group_count"])
    assert np.array_equal(g_of[go], g_of[eo]), what
    assert np.array_equal(got["instance_data"][go], exp["instance_data"][eo]), what
    assert np.array_equal(np.sort(got["pose_list"]), np.sort(exp["pose_list"])), f"{what}: pose list"
    assert np.array_equal(np.sort(got["dirty_list"]), np.sort(exp["dirty_list"])), f"{what}: dirty list"


def _drawn(got):
    """Model instances a view's outputs draw: the entity of every DRAW_MESH / DRAW_SKINNED value and of every auto-instanced instance (the
    low 32 bits; the type is bits 32-39 of a value)."""
    v = got["values"]
    t = (v >> np.uint64(32)) & np.uint64(0xff)
    mesh = v[(t == 0) | (t == 2)]  # DRAW_MESH, DRAW_SKINNED
    return set((mesh & np.uint64(0xffffffff)).tolist()) | set((got["group_renderables"] & np.uint64(0xffffffff)).tolist())


def _bits_equal(a, b, what):
    for f in ("pos", "rot", "scale"):
        assert np.ascontiguousarray(a[f]).tobytes() == np.ascontiguousarray(b[f]).tobytes(), f"{what}: {f} differs"


def _cams():
    a = dict(scenes.c1_frustum_args(), far=2500.0)
    return [a, dict(a, position=(40.0, 5.0, -60.0)), dict(a, position=(300.0, 10.0, 200.0), direction=(-0.4, -0.05, -0.9), far=3000.0),
            dict(a, position=(-200.0, 0.0, 100.0), direction=(0.3, 0.0, -0.95))]


def _frame_args(cam):
    return [cam] + scenes.shadow_cascade_args(cam, LIGHT, CASCADES)


def _frusta(args):
    return [lb.frustum_perspective(**a) if "fov" in a else lb.frustum_ortho(**a) for a in args]


def _transforms(rng, k):
    t = np.zeros(k, lb.TRANSFORM_DTYPE)
    t["pos"] = (rng.random((k, 3)) * 2.0 - 1.0) * EXTENT
    t["rot"] = scenes.random_unit_quats(rng, k)
    t["scale"] = rng.uniform(0.5, 2.0, (k, 3)).astype(np.float32)
    return t


class World:
    """A device-authoritative CullingSystem + SortKeys, the oracle's culling system, and the flat per-entity arrays the oracle's
    createSortKeys reads, for every id in [0, cap)."""

    def __init__(self, ctx, oracle, n=40_000, cap=None, seed=31, max_entities=None):
        self.ctx, self.oracle = ctx, oracle
        self.rng = np.random.default_rng(seed)
        cap = cap or n
        self.n, self.cap = n, cap
        scene = scenes.cull_scene(n, tuple(EXTENT), seed=seed, type_probs=(0.8, 0.08, 0.04, 0.08))
        sk = scenes.sortkey_setup(n, scene["types"], scene["pos"], seed=seed + 100, moved_fraction=0.0)
        self.sk = sk
        self.models = sk["models"]
        self.tr = np.zeros(cap, lb.TRANSFORM_DTYPE)
        self.tr[:n] = sk["transforms"]
        self.model_of = np.zeros(cap, np.uint32)
        self.model_of[:n] = sk["model_of"]
        self.lod = np.zeros(cap, np.float32)
        self.lod[:n] = sk["lod"]
        self.flags = np.zeros(cap, np.uint8)
        self.flags[:n] = sk["flags"]
        self.pf = np.full(cap, 0xffffffff, np.uint32)
        self.dsk = np.zeros(cap, np.uint32)
        self.dsk[:n] = sk["decal_sort_key"]
        self.dl = np.zeros(cap, np.uint8)
        self.dl[:n] = sk["decal_layer"]
        self.prev = np.zeros(cap, lb.TRANSFORM_DTYPE)
        self.listed, self.listed_set = [], set()  # m_moved_instances, at most once per entity (endFrame does the same for a second entry)
        self.alive = np.zeros(cap, bool)
        self.alive[:n] = True
        self.type = np.zeros(cap, np.uint8)
        self.type[:n] = scene["types"]
        self.br = (0.5 + 2.5 * self.rng.random(cap)).astype(np.float32)  # Model::getOriginBoundingRadius of each entity's model
        self.cs = lb.CullingSystem(ctx)
        self.cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
        self.cs.set_replicas(1)
        self.oc = oracle.OracleCulling()
        self.oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
        self.S = self.host_sortkeys(max_entities or n)

    def host_sortkeys(self, max_entities):
        """A SortKeys set up through whole-array uploads of the flat arrays' first max_entities entries."""
        m = max_entities
        S = lb.SortKeys(self.ctx, m, self.sk["max_sort_key"] + 1, max_keys=4 * self.cap, max_instances=4 * self.cap)
        S.setModels(self.sk["models"], self.sk["meshes"])
        S.setInstances(self.model_of[:m], self.lod[:m], self.flags[:m], self.pf[:m], self.dsk[:m], self.dl[:m])
        S.setTransforms(self.tr[:m])
        return S

    def _dev(self, *arrays):
        return [self.ctx.to_device(np.ascontiguousarray(a)) for a in arrays]

    def _free(self, ptrs):
        for p in ptrs:
            self.ctx.free_device(p)

    # ---- the culling side
    def cull_add(self, ids, types, pos):
        ids = np.asarray(ids, np.int32)
        types = np.asarray(types, np.uint8)
        rad = (0.5 + 4.5 * self.rng.random(len(ids))).astype(np.float32)
        d = self._dev(ids, types, pos, rad)
        self.cs.add_many_device(d[2], d[3], d[1], len(ids), dev_entities=d[0], max_entity=int(ids.max()))
        self._free(d)
        self.oc.add(ids, types, pos, rad)
        self.alive[ids], self.type[ids] = True, types

    def despawn(self, ids):
        ids = np.asarray(ids, np.int32)
        d = self._dev(ids)
        self.cs.remove_many_device(d[0], len(ids))
        self._free(d)
        self.oc.remove(ids)
        self.alive[ids] = False

    # ---- the sort-key side
    def spawn_sk(self, ids, models, t, dirty=None, max_entity=None):
        ids = np.asarray(ids, np.int32)
        models = np.asarray(models, np.uint32)
        d = self._dev(ids, models, t) + (self._dev(np.asarray(dirty, np.uint8)) if dirty is not None else [])
        try:
            self.S.spawnInstancesDevice(d[0], d[1], d[2], len(ids), int(ids.max()) if max_entity is None else max_entity, dev_dirty=d[3] if dirty is not None else None)
        finally:
            self._free(d)
        self.tr[ids] = t
        self.model_of[ids] = models
        self.lod[ids] = [spawn_lod(self.models, m) for m in models]
        fl = self.flags[ids] & ~np.uint8(MOVED | DIRTY)
        if dirty is not None:
            fl |= np.where(np.asarray(dirty) != 0, np.uint8(DIRTY), np.uint8(0))
        self.flags[ids] = fl
        self.pf[ids] = 0xffffffff
        self.prev[ids] = t

    def spawn(self, ids, models=None, t=None, dirty=None, max_entity=None):
        """A model-instance spawn as a frame issues it: add_many_device, then the sort keys' spawn."""
        k = len(ids)
        models = self.rng.integers(0, len(self.models), k).astype(np.uint32) if models is None else models
        t = _transforms(self.rng, k) if t is None else t
        self.cull_add(ids, np.zeros(k, np.uint8), t["pos"])
        self.spawn_sk(ids, models, t, dirty, max_entity)
        return models, t

    def spawn_decals(self, ids, max_entity=None):
        ids = np.asarray(ids, np.int32)
        k = len(ids)
        types = self.rng.choice(np.array([1, 3], np.uint8), k)
        self.cull_add(ids, types, (self.rng.random((k, 3)) * 2.0 - 1.0) * EXTENT)
        self.spawn_decals_sk(ids, self.rng.integers(0, 2000, k).astype(np.uint32), self.rng.choice(np.array([0, 1, 2, 3], np.uint8), k), max_entity)

    def spawn_decals_sk(self, ids, key, layer, max_entity=None):
        ids = np.asarray(ids, np.int32)
        k = len(ids)
        d = self._dev(ids, key, layer)
        try:
            self.S.spawnDecalsDevice(d[0], d[1], d[2], k, int(ids.max()) if max_entity is None else max_entity)
        finally:
            self._free(d)
        self.dsk[ids], self.dl[ids] = key, layer

    def move(self, ids, t=None):
        """onModelInstanceMoved on the device (moveDevice) + CullingSystem::set (set_many_device) for distinct live ids."""
        ids = np.asarray(ids, np.int32)
        k = len(ids)
        t = _transforms(self.rng, k) if t is None else t
        br = self.br[ids]
        d = self._dev(ids, t, br) + [self.ctx.to_device(np.zeros(3 * k)), self.ctx.to_device(np.zeros(k, np.float32))]
        self.S.moveDevice(d[0], d[1], k, d[2], d[3], d[4])
        self.cs.set_many_device(d[3], d[4], k, dev_entities=d[0], max_entity=int(ids.max()))
        self._free(d)
        rad = self.oracle.sphere_radius(np.ascontiguousarray(t).view(np.uint8).reshape(k, 56), br)
        self.oc.set(ids, np.ascontiguousarray(t["pos"]), rad)
        self.tr[ids] = t
        self.flags[ids] |= np.uint8(MOVED)
        for e in ids.tolist():
            if e not in self.listed_set:
                self.listed_set.add(e)
                self.listed.append(e)
        return t

    def live(self, type_=0):
        return np.nonzero(self.alive & (self.type == type_))[0].astype(np.int32)

    def dead(self):
        return np.nonzero(~self.alive)[0].astype(np.int32)

    # ---- a frame
    def views(self, args, frame):
        sk = self.sk
        ref = args[0]["position"]
        return [sortkeys.make_view(a["position"], ref, TIME_DELTA, 1.25, frame, k > 0, sk["max_sort_key"],
                                   *((sk["layer_to_bucket"], sk["depth_sorted_buckets"]) if k == 0 else (SHADOW_BUCKETS, ())))
                for k, a in enumerate(args)]

    def draw(self, cam, frame, what, S=None):
        """cull_views (main view + cascades) -> createSortKeysViews, every view against the oracle, then the lod / Pose::frame state.
        -> (results, outputs per view, visible MESH ids per view)"""
        S = S or self.S
        args = _frame_args(cam)
        frusta, views = _frusta(args), self.views(args, frame)
        self.cs.cull_views(frusta, want_counts=False)
        res = S.createSortKeysViews(self.cs, views)
        got = [S.readView(k, r) for k, r in enumerate(res)]
        vis = []
        for v, (f, view) in enumerate(zip(frusta, views)):
            oids, otys, _ = self.oc.cull(lb.culling.frustum_bytes(f))
            exp = self.oracle.create_sort_keys(oids, otys, self.tr, self.model_of, self.lod, self.flags, self.pf, self.dsk, self.dl,
                                               self.models, self.sk["meshes"], view)
            assert res[v].n_keys == len(exp["keys"]) and res[v].n_pose == len(exp["pose_list"]), f"{what} view {v}"
            _compare_view(got[v], exp, f"{what} view {v}")
            vis.append(oids[otys == 0])
        m = min(self.cap, S.max_entities)
        assert np.array_equal(got[0]["lod"][:m].view(np.uint32), self.lod[:m].view(np.uint32)), f"{what}: lod state"
        assert np.array_equal(got[0]["pose_frame"][:m], self.pf[:m]), f"{what}: Pose::frame"
        return res, got, vis

    def check_moved(self, what):
        got = self.S.movedList()
        assert len(got) == len(set(got.tolist())), f"{what}: an entity listed twice"
        assert sorted(got.tolist()) == sorted(self.listed), f"{what}: moved list"

    def end_frame(self, what):
        self.check_moved(what)
        self.S.endFrame()
        ids = np.asarray(self.listed, np.int64)
        if len(ids):
            self.flags[ids] &= np.uint8(~MOVED & 0xff)
            self.prev[ids] = self.tr[ids]
        self.listed, self.listed_set = [], set()
        m = min(self.cap, self.S.max_entities)
        _bits_equal(self.S.prevTransforms()[:m], self.prev[:m], f"{what}: prev_frame_transform")
        assert len(self.S.movedList()) == 0

    def close(self):
        self.S.close()
        self.cs.close()


# ------------------------------------------------------------------------------------------------------------------------ 1 + 6
def test_spawn_frames_match_oracle(ctx, oracle):
    """Four frames, moving camera: spawn instances (ids past the scene and ids despawned earlier) and decals, despawn, move (spawned ids
    too), cull_views -> createSortKeysViews -> endFrame.  Every view, the lod / Pose::frame state, the moved list and prev_frame_transform
    against the oracle; a spawned skinned instance joins the pose list of the first view that draws it."""
    k = 3000
    n = 40_000
    w = World(ctx, oracle, n=n, cap=n + 5 * k)
    skinned_models = np.nonzero(np.array([w.sk["meshes"]["skinned"][w.models["mesh_base"][m]] for m in range(len(w.models))]))[0]
    next_id = n
    spawned_drawn = 0
    for fno, cam in enumerate(_cams()):
        fresh = np.arange(next_id, next_id + k // 2, dtype=np.int32)
        next_id += k // 2
        dead = w.dead()
        dead = dead[dead < next_id - k // 2]
        reuse = w.rng.choice(dead, min(len(dead), k // 2), replace=False).astype(np.int32) if len(dead) else np.zeros(0, np.int32)
        ids = w.rng.permutation(np.concatenate([fresh, reuse])).astype(np.int32)
        models = w.rng.integers(0, len(w.models), len(ids)).astype(np.uint32)
        models[: len(ids) // 5] = w.rng.choice(skinned_models, len(ids) // 5)
        dirty = (w.rng.random(len(ids)) < 0.02).astype(np.uint8)
        # spawned in front of the camera, so that they are drawn
        t = _transforms(w.rng, len(ids))
        fwd = np.asarray(cam["direction"]) / np.linalg.norm(cam["direction"])
        t["pos"] = np.asarray(cam["position"]) + fwd * w.rng.uniform(20.0, 1500.0, (len(ids), 1)) + w.rng.normal(size=(len(ids), 3)) * 150.0
        w.spawn(ids, models, t, dirty if fno % 2 == 0 else None)
        decals = np.arange(next_id, next_id + k // 6, dtype=np.int32)
        next_id += k // 6
        w.spawn_decals(decals)
        gone = w.rng.choice(np.nonzero(w.alive)[0], k // 2, replace=False).astype(np.int32)
        w.despawn(gone)
        live = w.live()
        movers = np.union1d(w.rng.choice(live, k // 2, replace=False), w.rng.choice(np.intersect1d(ids, live), 200, replace=False)).astype(np.int32)
        w.move(movers)
        res, got, vis = w.draw(cam, 60 + fno, f"frame {fno}")
        # a spawned skinned instance: in the pose list of the first view that draws it
        sk_spawned = set(ids[np.isin(models, skinned_models)].tolist()) & set(np.nonzero(w.alive)[0].tolist())
        drawn = [_drawn(g) for g in got]
        for e in sk_spawned:
            first = next((v for v in range(len(got)) if e in drawn[v]), None)
            if first is not None:
                assert e in set(got[first]["pose_list"].tolist()), f"frame {fno}: spawned skinned {e} not in the pose list of view {first}"
                spawned_drawn += 1
        w.end_frame(f"frame {fno}")
    assert spawned_drawn > 100, spawned_drawn
    w.close()


def test_claimed_pose_is_claimed_again_after_a_respawn_in_the_same_frame(ctx, oracle):
    """Drawn (pose claimed), despawned, spawned again and drawn in the same frame number: the respawned skinned instance joins the pose
    list again, in the first view that draws it."""
    w = World(ctx, oracle, n=30_000, seed=41)
    cam = _cams()[0]
    _, got, vis = w.draw(cam, 80, "first draw")
    claimed = np.unique(np.concatenate([g["pose_list"] for g in got])).astype(np.int32)
    assert len(claimed) > 50
    again = w.rng.choice(claimed, 50, replace=False).astype(np.int32)
    t = w.tr[again].copy()
    models = w.model_of[again].copy()
    w.despawn(again)
    w.spawn(again, models, t)
    _, got, vis = w.draw(cam, 80, "second draw, same frame")
    drawn = [_drawn(g) for g in got]
    found = 0
    for e in again.tolist():
        first = next((v for v in range(len(got)) if e in drawn[v]), None)
        if first is not None:
            assert e in set(got[first]["pose_list"].tolist()), e
            found += 1
    assert found > 40, found
    w.end_frame("end")
    w.close()


# ------------------------------------------------------------------------------------------------------------------------ 2
def test_spawned_records_equal_whole_array_uploads(ctx, oracle):
    """The state a spawn frame reaches through the spawn calls and the same state uploaded whole (set_instances + set_transforms) give the
    same outputs view by view and the same lod / Pose::frame."""
    n = 30_000
    w = World(ctx, oracle, n=n, cap=n + 4000, seed=43, max_entities=n + 4000)
    cam = _cams()[1]
    w.draw(cam, 10, "before")
    w.spawn(np.arange(n, n + 3000, dtype=np.int32), dirty=(w.rng.random(3000) < 0.05).astype(np.uint8))
    reuse = w.rng.choice(w.live(), 800, replace=False).astype(np.int32)
    w.despawn(reuse)
    w.spawn(reuse)
    w.spawn_decals(np.arange(n + 3000, n + 3500, dtype=np.int32))
    H = w.host_sortkeys(w.cap)  # the flat arrays as the spawns left them, uploaded whole
    res, got, _ = w.draw(cam, 11, "spawned")
    views = w.views(_frame_args(cam), 11)
    rh = H.createSortKeysViews(w.cs, views)  # the same cull_views
    for v, r in enumerate(rh):
        h = H.readView(v, r)
        assert (r.n_keys, r.n_instances, r.n_pose, r.n_dirty) == (res[v].n_keys, res[v].n_instances, res[v].n_pose, res[v].n_dirty), v
        _compare_view(got[v], h, f"view {v} against the uploaded state")
    for f in ("lod", "pose_frame"):
        assert np.array_equal(got[0][f].view(np.uint32), h[f].view(np.uint32)), f
    H.close()
    w.close()


def test_lod_rule(ctx):
    """modelLoaded's LOD: every LOD's `to` -1 -> 4; LOD 0's only -> 3; gaps -> the highest LOD 3 .. 0 with one; none -> 3; LOD 0 only ->
    0; LOD 4 only -> 4 (LOD 4 is not looked at); an empty range whose `to` is not -1 counts, as in the reference."""
    cases = [  # (lod_from, lod_to, expected)
        ([0, 0, 0, 0, 0], [-1, -1, -1, -1, -1], 4.0),
        ([0, 1, 2, 3, 0], [-1, 1, 2, 3, -1], 3.0),
        ([0, 0, 1, 0, 0], [0, -1, 2, -1, -1], 2.0),
        ([0, 1, 2, 3, 4], [0, 1, 2, 3, 4], 3.0),
        ([0, 0, 0, 0, 0], [0, -1, -1, -1, -1], 0.0),
        ([0, 0, 0, 0, 5], [-1, -1, -1, -1, 5], 4.0),
        ([0, 3, 0, 0, 0], [0, 2, -1, -1, -1], 1.0),
    ]
    models = np.zeros(len(cases), sortkeys.SK_MODEL_DTYPE)
    for m, (f, t, _) in enumerate(cases):
        models[m]["lod_distances"] = [100.0, 400.0, 900.0, 1600.0]
        models[m]["lod_from"], models[m]["lod_to"] = f, t
        models[m]["mesh_base"], models[m]["mesh_count"] = 0, 6
    meshes = np.zeros(6, sortkeys.SK_MESH_DTYPE)
    meshes["sort_key"] = np.arange(6)
    S = lb.SortKeys(ctx, 64, 16)
    S.setModels(models, meshes)
    ids = np.arange(10, 10 + 3 * len(cases), 3, dtype=np.int32)
    mod = np.arange(len(cases), dtype=np.uint32)
    tr = np.zeros(len(ids), lb.TRANSFORM_DTYPE)
    d = [ctx.to_device(a) for a in (ids, mod, tr)]
    S.setInstances(lod=np.full(64, 0.5, np.float32))
    S.spawnInstancesDevice(d[0], d[1], d[2], len(ids), 63)
    for p in d:
        ctx.free_device(p)
    lod = S.read(sortkeys.SkResult())["lod"]
    assert lod[ids].tolist() == [c[2] for c in cases]
    assert np.all(np.delete(lod, ids) == np.float32(0.5)), "other records untouched"
    S.close()


# ------------------------------------------------------------------------------------------------------------------------ 4
def test_growth(ctx, oracle):
    """max_entities = the scene's 5000.  An id one past it, then one far past it, then several growths in a row, each in the middle of a
    frame with a non-empty moved list: the earlier records, lod, Pose::frame, the moved list and prev_frame_transform carry on; the latest
    view outputs still read; createSortKeysViews runs and matches the oracle where it refused before the growth."""
    n = 5000
    w = World(ctx, oracle, n=n, cap=200_000, seed=47)
    cam = _cams()[0]
    w.move(w.rng.choice(w.live(), 300, replace=False))
    res0, got0, _ = w.draw(cam, 20, "before growth")
    w.end_frame("frame 20")
    w.move(w.rng.choice(w.live(), 300, replace=False))  # the moved list of frame 21, non-empty across the growths below
    res0, got0, _ = w.draw(cam, 21, "frame 21, before growth")
    # the culling system gets id n first: createSortKeys refuses until the sort keys hold it
    t = _transforms(w.rng, 1)
    t["pos"] = np.asarray(cam["position"]) + np.array([0.0, 0.0, -30.0])
    w.cull_add([n], [0], t["pos"])
    with pytest.raises(LumixB200Error) as err:
        w.S.createSortKeysViews(w.cs, w.views(_frame_args(cam), 21))
    assert err.value.code == _lib.ERR_INVALID
    w.spawn_sk([n], [0], t)
    assert w.S.max_entities == 2 * n
    for k, r in enumerate(res0):  # the latest view outputs, copied over
        now = w.S.readView(k, r)
        for f in ("keys", "values", "group_count", "group_offset", "group_renderables", "instance_data", "pose_list", "dirty_list"):
            assert np.array_equal(now[f], got0[k][f]), f"view {k} {f} after the growth"
    w.check_moved("after one growth")
    w.spawn(np.array([20 * n + 3], np.int32))  # far past: 10000 -> 160000
    assert w.S.max_entities == 32 * n
    w.move(w.rng.choice(w.live(), 200, replace=False))
    w.draw(cam, 21, "frame 21 after two growths")
    w.end_frame("frame 21")
    # several growths inside one frame, moves in between, createSortKeys at the end
    w2 = World(ctx, oracle, n=n, cap=200_000, seed=53)
    w2.draw(cam, 30, "w2 first")
    for step, top in enumerate((n + 1, 3 * n, 7 * n + 5, 12 * n)):
        w2.move(w2.rng.choice(w2.live(), 100, replace=False))
        ids = np.unique(np.concatenate([[top], w2.rng.integers(n, top, 200)])).astype(np.int32)
        ids = ids[~w2.alive[ids]]
        w2.spawn(ids, max_entity=top + step)
        assert w2.S.max_entities >= top + step + 1
    w2.draw(cam, 31, "w2 after four growths")
    w2.end_frame("w2")
    w2.close()
    w.close()


# ------------------------------------------------------------------------------------------------------------------------ 5
def test_refusals_change_nothing(ctx, oracle):
    """Id -1, an id above max_entity, a duplicate, a model index equal to the table's count, NULL for each required pointer: each
    LB200_ERR_INVALID with valid entries in the same batch left unspawned; before set_models LB200_ERR_STATE.  The next frame, state and
    moved list equal the oracle's, which saw none of the refused calls."""
    n = 20_000
    w = World(ctx, oracle, n=n, cap=n + 100, seed=59, max_entities=n + 100)
    cam = _cams()[0]
    w.move(w.rng.choice(w.live(), 200, replace=False))
    _, got, _ = w.draw(cam, 5, "before")
    drawn = np.unique(np.concatenate([g["pose_list"] for g in got]))[:20].astype(np.int32)  # Pose::frame 5: a spawn would reset it
    assert len(drawn) == 20
    L = w.S.L
    n_models = len(w.models)

    def call(ids, models, max_entity, null=None, S=None):
        ids = np.asarray(ids, np.int32)
        models = np.asarray(models, np.uint32)
        d = w._dev(ids, models, _transforms(w.rng, len(ids)))
        args = [d[0], d[1], d[2]]
        if null is not None:
            args[null] = None
        rc = L.lb200_sortkeys_spawn_instances_device((S or w.S).h, *[_lib.vp(a) if a else None for a in args], None, C.c_uint32(len(ids)), C.c_uint32(max_entity))
        w._free(d)
        return rc

    m0 = np.zeros(len(drawn), np.uint32) + 1
    assert call(np.append(drawn, -1), np.append(m0, 0), n + 50) == _lib.ERR_INVALID
    assert call(np.append(drawn, n + 51), np.append(m0, 0), n + 50) == _lib.ERR_INVALID
    assert call(np.append(drawn, drawn[3]), np.append(m0, 0), n + 50) == _lib.ERR_INVALID
    assert call(drawn, np.append(m0[:-1], n_models), n + 50) == _lib.ERR_INVALID
    for null in range(3):
        assert call(drawn, m0, n + 50, null=null) == _lib.ERR_INVALID
    # the same refusals asking for a growth: refused before anything grows
    assert call(np.append(drawn, -1), np.append(m0, 0), 50 * n) == _lib.ERR_INVALID
    assert call(np.append(drawn, drawn[3]), np.append(m0, 0), 50 * n) == _lib.ERR_INVALID
    assert call(np.append(drawn, 3 * n), np.append(m0, n_models), 50 * n) == _lib.ERR_INVALID

    def decals(ids, max_entity, null=None):
        ids = np.asarray(ids, np.int32)
        d = w._dev(ids, np.zeros(len(ids), np.uint32), np.zeros(len(ids), np.uint8))
        args = [d[0], d[1], d[2]]
        if null is not None:
            args[null] = None
        rc = L.lb200_sortkeys_spawn_decals_device(w.S.h, *[_lib.vp(a) if a else None for a in args], C.c_uint32(len(ids)), C.c_uint32(max_entity))
        w._free(d)
        return rc

    for ids, top in ((np.append(drawn, -1), n + 50), (np.append(drawn, n + 51), n + 50), (np.append(drawn, drawn[0]), n + 50),
                     (np.append(drawn, -1), 50 * n), (np.append(drawn, drawn[0]), 50 * n)):
        assert decals(ids, top) == _lib.ERR_INVALID
    for null in range(3):
        assert decals(drawn, n + 50, null=null) == _lib.ERR_INVALID
    assert w.S.max_entities == n + 100, "a refused call grows nothing"
    # n = 0: LB200_OK before any other check, nothing launched
    bare = lb.SortKeys(ctx, 100, w.sk["max_sort_key"] + 1)
    launches = ctx.launches
    assert L.lb200_sortkeys_spawn_instances_device(bare.h, None, None, None, None, C.c_uint32(0), C.c_uint32(1 << 20)) == _lib.OK
    assert L.lb200_sortkeys_spawn_decals_device(bare.h, None, None, None, C.c_uint32(0), C.c_uint32(1 << 20)) == _lib.OK
    assert L.lb200_sortkeys_clear_dirty_device(bare.h, None, C.c_uint32(0)) == _lib.OK
    assert ctx.launches == launches and L.lb200_sortkeys_max_entities(bare.h) == 100
    assert call([1, 2], [0, 0], 99, S=bare) == _lib.ERR_STATE
    bare.close()
    w.check_moved("after the refusals")
    w.draw(cam, 5, "after the refusals, same frame")
    w.end_frame("end")
    w.close()


def test_records_from_spawns_alone(ctx, oracle):
    """A SortKeys that only ever saw set_models and spawn calls (no set_instances / set_transforms), created for 10 entities and grown by
    the spawns, runs createSortKeys and matches the oracle."""
    n = 20_000
    w = World(ctx, oracle, n=n, seed=71)
    w.S.close()
    w.S = lb.SortKeys(ctx, 10, w.sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
    w.S.setModels(w.sk["models"], w.sk["meshes"])
    inst = np.nonzero(w.type[:n] == 0)[0].astype(np.int32)
    other = np.nonzero(w.type[:n] != 0)[0]
    w.lod[other], w.pf[other] = 0.0, 0xffffffff  # records no spawn wrote: as create leaves them
    w.spawn_sk(inst, w.model_of[inst], w.tr[inst].copy(), dirty=((w.flags[inst] & DIRTY) != 0).astype(np.uint8), max_entity=n - 1)
    dec = np.nonzero((w.type[:n] == 1) | (w.type[:n] == 3))[0].astype(np.int32)
    w.spawn_decals_sk(dec, w.dsk[dec], w.dl[dec], max_entity=n - 1)
    assert w.S.max_entities >= n
    w.draw(_cams()[0], 9, "spawned records only")
    w.close()


# ------------------------------------------------------------------------------------------------------------------------ 7
def test_move_spawn_move_lists_once(ctx, oracle):
    """Move -> spawn -> move in one frame lists the entity once and end_frame takes the last transform; many such cycles in one frame keep
    the list within its capacity and match the oracle; a spawn clears MOVED (the spawned instance is drawn auto-instanced again)."""
    n = 8000
    w = World(ctx, oracle, n=n, seed=61)
    cam = _cams()[0]
    ids = w.rng.choice(w.live(), 500, replace=False).astype(np.int32)
    w.move(ids)
    w.spawn_sk(ids, w.model_of[ids], w.tr[ids].copy())
    w.check_moved("move -> spawn")
    w.draw(cam, 1, "move -> spawn: MOVED off")
    w.move(ids)
    w.check_moved("move -> spawn -> move")
    w.draw(cam, 1, "move -> spawn -> move")
    w.end_frame("one cycle")
    # every live mesh through 3 cycles in one frame: 3 x 6 k pushes would pass the 8 k capacity if a spawn let an entity be listed again
    live = w.live()
    for c in range(3):
        w.move(live)
        w.spawn_sk(live, w.model_of[live], w.tr[live].copy())
    w.move(live[::2])
    w.check_moved("three cycles")
    w.draw(cam, 2, "three cycles")
    w.end_frame("three cycles")
    w.close()


# ------------------------------------------------------------------------------------------------------------------------ 8
def test_clear_dirty(ctx, oracle):
    """Dirty instances are in the dirty list and not drawn; clearDirtyDevice (with out-of-range ids mixed in) takes them off it in the
    next frame and they are drawn, MOVED of the moved ones untouched."""
    n = 30_000
    w = World(ctx, oracle, n=n, seed=67)
    cam = _cams()[0]
    fresh = np.arange(n - 2000, n, dtype=np.int32)
    w.despawn(fresh)
    w.spawn(fresh, dirty=np.ones(len(fresh), np.uint8))
    _, got, _ = w.draw(cam, 3, "dirty")
    dirty = np.unique(np.concatenate([g["dirty_list"] for g in got])).astype(np.int32)
    assert len(dirty) > 100
    w.end_frame("f3")
    w.move(dirty[::3])
    d = w._dev(np.concatenate([dirty, [-1, 1 << 30]]).astype(np.int32))
    w.S.clearDirtyDevice(d[0], len(dirty) + 2)
    w._free(d)
    w.flags[dirty] &= np.uint8(~DIRTY & 0xff)
    _, got, _ = w.draw(cam, 4, "cleared")
    assert not (set(np.concatenate([g["dirty_list"] for g in got]).tolist()) & set(dirty.tolist()))
    drawn = set().union(*[_drawn(g) for g in got])
    assert len(drawn & set(dirty.tolist())) > 50
    w.check_moved("cleared")
    w.end_frame("f4")
    w.close()
