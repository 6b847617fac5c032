"""createSortKeys for all of a frame's views in one launch (SortKeys.createSortKeysViews, lb200_sortkeys_create_keys_views), held to the
oracle view by view.

The expected outputs come from oracle.create_sort_keys run view after view on the oracle's cull of each frustum, with one lod / pose_frame
pair updated in place: the order the call promises.  Per view the (key, value) pairs are compared as multisets (and sorted when asked),
group counts and offsets exactly, instance data matched through the renderable, pose and dirty lists as sets; after the call the shared lod
state bit for bit and Pose::frame exactly.
"""
import ctypes as C

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib, scenes, sortkeys

pytestmark = pytest.mark.gpu

LIGHT = (0.3, -0.8, 0.2)
CASCADES = (40.0, 200.0, 900.0, 2500.0)
SHADOW_BUCKETS = [0, 0xff, 0xff, 1]  # layer -> bucket of the shadow views: the main view's depth-sorted layer 1 is not drawn, layer 3 has its own bucket
TIME_DELTA = 0.15  # reaches both LOD branches: the 2.9 / 3.5 states of sortkey_setup snap, the others step


def _canon(keys, values):
    o = np.lexsort((values, keys))
    return keys[o], values[o]


def _compare_view(got, exp, what, sorted_keys=True):
    if sorted_keys:
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
    assert np.array_equal(np.sort(got["pose_list"]), np.sort(exp["pose_list"])), what
    assert np.array_equal(np.sort(got["dirty_list"]), np.sort(exp["dirty_list"])), what


class Frame:
    """A scene on the device (culling system + SortKeys) and in the oracle, with the oracle's lod / Pose::frame state beside the device's."""

    def __init__(self, ctx, oracle, n=60_000, seed=11, key_stride=1, scene=None, max_keys=None, max_instances=None):
        self.ctx, self.oracle = ctx, oracle
        self.scene = scene if scene is not None else scenes.cull_scene(n, (2500.0, 300.0, 2500.0), seed=seed, type_probs=(0.8, 0.08, 0.04, 0.08), big_fraction=0.002)
        n = len(self.scene["entities"])
        self.n = n
        sk = scenes.sortkey_setup(n, self.scene["types"], self.scene["pos"], seed=seed + 100)
        if key_stride > 1:  # sparse sort keys: more groups than a block keeps in shared memory (8192) -> group cursors in HBM
            sk["meshes"]["sort_key"] = sk["meshes"]["sort_key"] * key_stride + 7
            sk["max_sort_key"] = int(sk["meshes"]["sort_key"].max()) + 3
            assert sk["max_sort_key"] + 1 > 8192
        self.sk = sk
        self.cs = lb.CullingSystem(ctx)
        self.cs.add(self.scene["entities"], self.scene["types"], self.scene["pos"], self.scene["radius"])
        self.oc = oracle.OracleCulling()
        self.oc.add(self.scene["entities"], self.scene["types"], self.scene["pos"], self.scene["radius"])
        self.S = self.make_sortkeys(max_keys, max_instances)
        self.lod, self.pf = sk["lod"].copy(), sk["pose_frame"].copy()

    def make_sortkeys(self, max_keys=None, max_instances=None):
        sk, n = self.sk, self.n
        S = lb.SortKeys(self.ctx, n, sk["max_sort_key"] + 1, max_keys=max_keys or 4 * n, max_instances=max_instances or 4 * n)
        S.setModels(sk["models"], sk["meshes"])
        S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
        S.setTransforms(sk["transforms"])
        return S

    def reset_state(self, S=None):
        """lod / Pose::frame back to the scene's initial state, on the device and in the oracle."""
        (S or self.S).setInstances(lod=self.sk["lod"], pose_frame=self.sk["pose_frame"])
        self.lod, self.pf = self.sk["lod"].copy(), self.sk["pose_frame"].copy()

    def views(self, frusta_args, frame):
        """lb200_sk_view per frustum: the first is the main camera, the rest shadow views with buckets of their own (no depth-sorted bucket,
        layer 3 in bucket 1 alone); every view takes its LOD from the main camera."""
        ref = frusta_args[0]["position"]
        sk = self.sk
        return [sortkeys.make_view(a["position"], ref, TIME_DELTA, 1.25, frame, k > 0, sk["max_sort_key"], *((sk["layer_to_bucket"], sk["depth_sorted_buckets"]) if k == 0 else (SHADOW_BUCKETS, ())))
                for k, a in enumerate(frusta_args)]

    def expect(self, frusta, views, sort=True):
        """The oracle, view after view on one lod / pose_frame pair.  -> (expected outputs per view, visible MESH ids per view, lod changes per view)"""
        sk, out, vis, changed = self.sk, [], [], []
        for f, view in zip(frusta, views):
            oids, otys, _ = self.oc.cull(lb.culling.frustum_bytes(f))
            before = self.lod.copy()
            out.append(self.oracle.create_sort_keys(oids, otys, sk["transforms"], sk["model_of"], self.lod, sk["flags"], self.pf, sk["decal_sort_key"],
                                                    sk["decal_layer"], sk["models"], sk["meshes"], view, sort=sort))
            vis.append(set(oids[otys == 0].tolist()))
            changed.append(np.nonzero(before.view(np.uint32) != self.lod.view(np.uint32))[0])
        return out, vis, changed

    def run(self, frusta, views, sort=True, S=None):
        S = S or self.S
        self.cs.cull_views(frusta, want_counts=False)
        res = S.createSortKeysViews(self.cs, views, sort=sort)
        return res, [S.readView(k, r) for k, r in enumerate(res)]

    def check(self, frusta, views, what, sort=True):
        res, got = self.run(frusta, views, sort)
        exp, vis, changed = self.expect(frusta, views, sort)
        for v, (r, g, e) in enumerate(zip(res, got, exp)):
            assert r.n_keys == len(e["keys"]) and r.n_instances == len(e["group_renderables"]) and r.n_pose == len(e["pose_list"]), f"{what} view {v}"
            _compare_view(g, e, f"{what} view {v}", sort)
        lod = got[0]["lod"][:self.n]
        assert np.array_equal(lod.view(np.uint32), self.lod.view(np.uint32)), f"{what}: lod state"
        assert np.array_equal(got[0]["pose_frame"][:self.n], self.pf), f"{what}: Pose::frame"
        return res, got, exp, vis, changed

    def close(self):
        self.S.close()
        self.cs.close()


def _frame_args(cam, cascades=CASCADES):
    return [cam] + scenes.shadow_cascade_args(cam, LIGHT, cascades)


def _frusta(args):
    return [lb.frustum_perspective(**a) if "fov" in a else lb.frustum_ortho(**a) for a in args]


def _cams():
    a = dict(scenes.c1_frustum_args(), far=2500.0)
    return [a, dict(a, position=(40.0, 5.0, -60.0)), dict(a, position=(300.0, 10.0, 200.0), direction=(-0.4, -0.05, -0.9), far=3000.0)]


@pytest.fixture(scope="module")
def frame(ctx, oracle):
    F = Frame(ctx, oracle)
    yield F
    F.close()


def _over_frames(F, what):
    snap_shadow = step = shared_skinned = 0
    for fno, cam in enumerate(_cams()):  # moving camera, a new frame number each frame: lod and Pose::frame carry over
        args = _frame_args(cam)
        frusta, views = _frusta(args), F.views(args, 40 + fno)
        res, got, exp, vis, changed = F.check(frusta, views, f"{what} frame {fno}")
        assert res[0].n_keys > 100 and res[0].n_instances > 1000
        for v in range(1, len(views)):
            snap_shadow += len(changed[v])  # a shadow view changes lod in the snap branch only
        lod = F.lod[changed[0]]
        step += int(np.sum(lod != np.round(lod)))  # the main view's steps leave fractional states
        claimed = set()
        for v, g in enumerate(got):
            mine = set(g["pose_list"].tolist())
            assert not (mine & claimed), f"{what} frame {fno} view {v}: joins a pose list an earlier view already claimed"
            shared_skinned += len(claimed & vis[v])
            claimed |= mine
    assert snap_shadow > 0 and step > 0, (snap_shadow, step)
    assert shared_skinned > 0, "no skinned instance seen by two views"


def test_views_match_oracle_over_frames(frame):
    """Main view + four cascades over three frames of a 60 k-entity mixed-type scene."""
    frame.reset_state()
    _over_frames(frame, "smem groups")


def test_views_match_oracle_groups_in_hbm(ctx, oracle):
    """The same with more groups than a block keeps in shared memory: the group cursors live in HBM."""
    F = Frame(ctx, oracle, n=40_000, seed=13, key_stride=131)
    _over_frames(F, "hbm groups")
    F.close()


def _eight(cam):
    args = _frame_args(cam)
    extra = [dict(cam, direction=d, far=1800.0) for d in ((1.0, 0.0, -0.2), (-1.0, 0.0, 0.3), (0.2, -0.1, 1.0))]
    return args + extra


def test_view_counts(frame):
    """1 to 8 views against the oracle; one view equals select_view(0) + createSortKeys on an identical second object, state included."""
    args = _eight(_cams()[0])
    for n in range(1, 9):
        frame.reset_state()
        a = args[:n]
        frame.check(_frusta(a), frame.views(a, 70 + n), f"{n} views")
    a = args[:1]
    frusta, views = _frusta(a), frame.views(a, 90)
    frame.reset_state()
    S2 = frame.make_sortkeys()
    res, got = frame.run(frusta, views)
    frame.cs.select_view(0)
    r2 = S2.createSortKeys(frame.cs, views[0])
    plain = S2.read(r2)
    assert (res[0].n_keys, res[0].n_instances, res[0].n_pose, res[0].n_dirty, res[0].n_groups) == (r2.n_keys, r2.n_instances, r2.n_pose, r2.n_dirty, r2.n_groups)
    for k in ("group_count", "group_offset", "lod", "pose_frame"):
        assert np.array_equal(got[0][k], plain[k]), k
    _compare_view(got[0], plain, "one view against create_keys")
    S2.close()


def test_outputs_coexist(frame):
    """Views read in reverse order with a plain createSortKeys and another cull_views in between: every view's outputs stay; a views call
    leaves the plain outputs alone."""
    frame.reset_state()
    cam = _cams()[0]
    args = _frame_args(cam)
    frusta, views = _frusta(args), frame.views(args, 100)
    frame.cs.cull_device(frusta[0], want_counts=False)
    rp = frame.S.createSortKeys(frame.cs, views[0])
    plain = frame.S.read(rp)
    res, got = frame.run(frusta, views)
    again = frame.S.read(rp)
    for k in ("keys", "values", "group_count", "group_offset", "group_renderables", "instance_data", "pose_list", "dirty_list"):
        assert np.array_equal(plain[k], again[k]), f"plain {k} changed by a views call"
    frame.cs.cull_device(frusta[2], want_counts=False)
    frame.S.createSortKeys(frame.cs, views[2])
    other = _frame_args(_cams()[2])
    frame.cs.cull_views(_frusta(other), want_counts=False)
    for k in reversed(range(len(views))):
        now = frame.S.readView(k, res[k])
        for f in ("keys", "values", "group_count", "group_offset", "group_renderables", "instance_data", "pose_list", "dirty_list"):
            assert np.array_equal(now[f], got[k][f]), f"view {k} {f}"


def test_sort_off_then_on(frame):
    """sort=False then sort=True from the same state: per view the same pairs, sorted the second time."""
    args = _frame_args(_cams()[1])
    frusta, views = _frusta(args), frame.views(args, 110)
    frame.reset_state()
    r1, unsorted = frame.run(frusta, views, sort=False)
    frame.reset_state()
    r2, srt = frame.run(frusta, views, sort=True)
    for v in range(len(views)):
        assert r1[v].n_keys == r2[v].n_keys
        assert np.all(srt[v]["keys"][1:] >= srt[v]["keys"][:-1])
        a, b = _canon(unsorted[v]["keys"], unsorted[v]["values"]), _canon(srt[v]["keys"], srt[v]["values"])
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), v
    assert any(not np.all(u["keys"][1:] >= u["keys"][:-1]) for u in unsorted), "the unsorted pass came out sorted"


def test_launch_shapes(frame):
    """One block, every co-resident block, the default: the same outputs; get_launch reports the views launch."""
    args = _frame_args(_cams()[0])
    frusta, views = _frusta(args), frame.views(args, 120)
    ref = None
    try:
        for blocks in (1, -1, 0):
            frame.S.setLaunch(-1)
            frame.cs.cull_device(frusta[0], want_counts=False)
            frame.S.createSortKeys(frame.cs, views[0])  # a plain launch of every co-resident block before the views call
            full = frame.S.lastLaunch()[0]
            frame.S.setLaunch(blocks)
            frame.reset_state()
            res, got = frame.run(frusta, views)
            grid, in_smem, _ = frame.S.lastLaunch()
            assert in_smem
            if blocks == 1:
                assert grid == 1
            elif blocks == -1:
                assert grid == full
            else:
                assert 1 <= grid <= full
            if ref is None:
                ref = got
            for v in range(len(views)):
                _compare_view(got[v], ref[v], f"blocks {blocks} view {v}")
                assert np.array_equal(got[v]["group_offset"], ref[v]["group_offset"])
    finally:
        frame.S.setLaunch(0)


def test_capacity(frame):
    """One view over max_keys (then over max_instances): LB200_ERR_CAPACITY, and every view's needed sizes in the results."""
    args = _frame_args(_cams()[0])
    frusta, views = _frusta(args), frame.views(args, 130)
    frame.reset_state()
    need, _ = frame.run(frusta, views)
    keys = sorted(r.n_keys for r in need)
    inst = sorted(r.n_instances for r in need)
    assert keys[-1] > keys[-2] and inst[-1] > inst[-2]
    L = frame.S.L
    for max_keys, max_inst in ((keys[-2] + 1, 0), (0, inst[-2] + 1)):
        small = frame.make_sortkeys(max_keys=max_keys or 4 * frame.n, max_instances=max_inst or 4 * frame.n)
        arr = np.concatenate(views)
        res = (sortkeys.SkResult * len(views))()
        rc = L.lb200_sortkeys_create_keys_views(small.h, frame.cs.h, _lib.ptr(arr), C.c_uint32(len(views)), C.c_int(1), C.c_int(1), res)
        assert rc == _lib.ERR_CAPACITY
        for r, e in zip(res, need):
            assert (r.n_keys, r.n_instances, r.n_pose, r.n_dirty) == (e.n_keys, e.n_instances, e.n_pose, e.n_dirty)
        small.close()


def test_refusals(ctx, frame):
    """Every refusal, each leaving the earlier views' outputs readable."""
    L = frame.S.L
    args = _frame_args(_cams()[0])
    frusta, views = _frusta(args), frame.views(args, 140)
    frame.reset_state()
    res, got = frame.run(frusta, views)
    arr = np.concatenate(views)
    out = (sortkeys.SkResult * 9)()

    def call(S, cs, a, n):
        return L.lb200_sortkeys_create_keys_views(S.h, cs.h, _lib.ptr(a), C.c_uint32(n), C.c_int(1), C.c_int(1), out)

    def still_readable():
        for k in (0, len(views) - 1):
            now = frame.S.readView(k, res[k])
            assert np.array_equal(now["keys"], got[k]["keys"]) and np.array_equal(now["instance_data"], got[k]["instance_data"]), k

    nine = np.concatenate([arr, arr[:4]])
    for n in (0, 9, 4, 1):  # out of range, then different from the cull's 5
        assert call(frame.S, frame.cs, nine, n) == _lib.ERR_INVALID, n
        still_readable()
    bad = arr.copy()
    bad["max_sort_key"][3] += 1  # views disagree on the renderer-wide max sort key
    assert call(frame.S, frame.cs, bad, 5) == _lib.ERR_INVALID
    bad = arr.copy()
    bad["max_sort_key"][:] = frame.sk["max_sort_key"] + 10 ** 6  # >= max_groups
    assert call(frame.S, frame.cs, bad, 5) == _lib.ERR_INVALID
    bad = arr.copy()
    bad["max_sort_key"][:] = frame.sk["max_sort_key"] - 1  # below a sort key of the mesh table
    assert call(frame.S, frame.cs, bad, 5) == _lib.ERR_INVALID
    still_readable()
    # a model whose meshes leave the mesh table
    sk = frame.sk
    models = sk["models"].copy()
    models["mesh_base"][-1] = len(sk["meshes"])  # its mesh_count >= 1 meshes start at the end of the table
    S3 = frame.make_sortkeys()
    S3.setModels(models, sk["meshes"])
    assert call(S3, frame.cs, arr, 5) == _lib.ERR_INVALID
    S3.close()
    # entity range: a culling system whose ids pass max_entities
    small = lb.SortKeys(ctx, 100, sk["max_sort_key"] + 1)
    small.setModels(sk["models"], sk["meshes"])
    small.setTransforms(sk["transforms"][:100])
    assert call(small, frame.cs, arr, 5) == _lib.ERR_INVALID
    # before set_models / set_transforms
    bare = lb.SortKeys(ctx, frame.n, sk["max_sort_key"] + 1)
    assert call(bare, frame.cs, arr, 5) == _lib.ERR_STATE
    bare.setModels(sk["models"], sk["meshes"])
    assert call(bare, frame.cs, arr, 5) == _lib.ERR_STATE
    o = sortkeys.SkOutputs()
    assert L.lb200_sortkeys_view_outputs(bare.h, 0, C.byref(o)) == _lib.ERR_STATE  # no views call yet
    bare.close()
    assert L.lb200_sortkeys_view_outputs(frame.S.h, 5, C.byref(o)) == _lib.ERR_INVALID
    # no cull_views on the culling system; an empty one
    fresh = lb.CullingSystem(ctx)
    assert call(frame.S, fresh, arr, 5) == _lib.ERR_STATE
    fresh.cull_views(frusta)
    assert call(frame.S, fresh, arr, 5) == _lib.ERR_STATE
    fresh.close()
    still_readable()
    # view buffers released by set_replicas
    cs2 = lb.CullingSystem(ctx)
    cs2.add(frame.scene["entities"], frame.scene["types"], frame.scene["pos"], frame.scene["radius"])
    cs2.cull_views(frusta, want_counts=False)
    cs2.set_replicas(2)
    assert call(frame.S, cs2, arr, 5) == _lib.ERR_STATE
    cs2.close()
    still_readable()


def test_c2_main_view_and_default_cascades(ctx, oracle):
    """The 10 M-entity C2 scene, main view + default cascades, against the oracle."""
    F = Frame(ctx, oracle, scene=scenes.c2_scene(), max_keys=1 << 22, max_instances=1 << 22)
    args = _frame_args(scenes.c2_frustum_args(), scenes.DEFAULT_CASCADES)
    res, _, exp, _, _ = F.check(_frusta(args), F.views(args, 7), "c2")
    assert res[0].n_keys > 100_000 and sum(r.n_keys for r in res[1:]) > 0
    F.close()
