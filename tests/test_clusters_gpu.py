"""lb200_clusters_fill (fillClusters on the device) bit for bit against the restatement (oracle/oracle_clusters.c, pinned to the reference's
own code by tests/test_clusters_cpu.py) and, where it is built, against that code itself (oracle/_ref/libclusters_shim_b200.so), for the
light order the device's cull produced (read back through light_entities): lights[], clusters[], map[], the AtlasSorter list and the
uncast-in-atlas list."""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import clusters as lc
from lumixengine_b200 import scenes
from lumixengine_b200._lib import LumixB200Error
from oracle import pyclusters as pc
from test_clusters_cpu import restatement, unit_quat

pytestmark = pytest.mark.gpu

W, H = 1920, 1080


def light_records(rng, n, r, cast_fraction=0.3):
    pl = np.zeros(n, lc.POINT_LIGHT_DTYPE)
    pl["color"] = rng.uniform(0, 1, (n, 3)).astype(np.float32)
    pl["intensity"] = rng.uniform(0, 10, n).astype(np.float32)
    pl["fov"] = rng.uniform(0.1, 3.0, n).astype(np.float32)
    pl["attenuation_param"] = rng.uniform(0, 100, n).astype(np.float32)
    pl["range"] = r
    pl["flags"] = (rng.random(n) < cast_fraction).astype(np.uint32) | (2 * (rng.random(n) < 0.5)).astype(np.uint32)
    return pl


def probes(rng, n_env, n_refl, cam, spread=150.0):
    env = np.zeros(n_env, lc.CLUSTER_ENV_PROBE_DTYPE)
    env["pos"] = rng.uniform(-spread, spread, (n_env, 3)).astype(np.float32)
    env["outer_range"] = rng.uniform(1, 40, (n_env, 3)).astype(np.float32)
    env["sh_coefs"] = rng.normal(size=(n_env, 9, 4)).astype(np.float32)
    refl = np.zeros(n_refl, lc.CLUSTER_REFL_PROBE_DTYPE)
    refl["pos"] = rng.uniform(-spread, spread, (n_refl, 3)).astype(np.float32)
    refl["half_extents"] = rng.uniform(1, 40, (n_refl, 3)).astype(np.float32)
    return env, refl


class Scene:
    """Entities around the camera, a share of them LOCAL_LIGHT (type 2) with cull radius = range; culling system, sort keys with the
    transforms, clusters with the point lights and atlas entries."""

    def __init__(self, ctx, n=4000, light_fraction=0.3, seed=1, cam=(10.0, 5.0, -20.0), spread=300.0, r_range=(0.5, 30.0), n_atlas=20, pos=None, radius=None):
        rng = np.random.default_rng(seed)
        self.rng, self.cam, self.n = rng, np.asarray(cam, np.float64), n
        self.types = np.where(rng.random(n) < light_fraction, 2, 0).astype(np.uint8)
        self.pos = self.cam + rng.uniform(-spread, spread, (n, 3)) if pos is None else np.asarray(pos, np.float64)
        self.tr = np.zeros(n, lb.TRANSFORM_DTYPE)
        self.tr["pos"] = self.pos
        self.tr["rot"] = np.array([unit_quat(rng) for _ in range(n)], np.float32).reshape(n, 4)
        self.tr["scale"] = 1.0
        r = rng.uniform(*r_range, n).astype(np.float32) if radius is None else np.asarray(radius, np.float32)
        self.pl = light_records(rng, n, r)
        self.atlas = np.full(n, -1, np.int32)
        lights = np.flatnonzero(self.types == 2)
        pick = rng.choice(lights, min(n_atlas, len(lights)), replace=False) if len(lights) else np.zeros(0, np.int64)
        self.atlas[pick] = rng.integers(0, 37, len(pick))
        self.cs = lb.CullingSystem(ctx)
        self.cs.add(np.arange(n, dtype=np.int32), self.types, self.pos, self.pl["range"])
        self.sk = lb.SortKeys(ctx, n, 1)
        self.sk.setTransforms(self.tr)
        self.cl = lb.Clusters(ctx, n)
        if len(lights):
            self.cl.setPointLights(lights.astype(np.int32), self.pl[lights])
        if len(pick):
            self.cl.setAtlas(pick.astype(np.int32), self.atlas[pick])
        self.ctx = ctx

    def frustum(self, w=W, h=H, ortho=False, rot=(0.0, 0.0, 0.0, 1.0), far=2000.0):
        return lb.frustum_from_viewport(tuple(self.cam), rot, 1.0472, w, h, 0.1, far, is_ortho=ortho, ortho_size=200.0)

    def close(self):
        self.cl.close()
        self.sk.close()
        self.cs.close()


def points_of(f):
    return np.array([[f.points[i][c] for c in range(3)] for i in range(8)], np.float32).reshape(24)


def check_fill(S, f, res, env=None, refl=None, w=W, h=H, visible=None):
    """The device's outputs of the last fill against the restatement and the reference's code for its light order."""
    restatement()
    got = S.cl.read(res)
    ents = got["light_entities"]
    if visible is not None:
        assert np.array_equal(np.sort(ents), np.sort(visible)), "light_entities is not the cull's LOCAL_LIGHT segment"
    assert len(np.unique(ents)) == len(ents)
    args = (points_of(f), w, h, S.cam, ents, S.tr["pos"][ents], S.tr["rot"][ents], S.pl[ents], S.atlas[ents], env, refl)
    shadow = lc.shadow_list(res)
    uncast = np.array(res.uncast[:res.n_uncast], np.int32)
    for which in ("restatement", "shim"):
        if pc.load(which) is None:
            continue
        exp = pc.fill(*args, which=which)
        assert (res.n_lights, res.n_map, res.n_clusters) == (len(ents), len(exp["map"]), len(exp["clusters"])), which
        assert tuple(res.size) == exp["size"]
        assert np.array_equal(got["lights"].view(np.uint8), exp["lights"].view(np.uint8)), f"{which}: lights"
        assert np.array_equal(got["clusters"].view(np.uint8), exp["clusters"].view(np.uint8)), f"{which}: clusters"
        assert np.array_equal(got["map"], exp["map"]), f"{which}: map"
        assert np.array_equal(shadow.view(np.uint8), exp["shadow"].view(np.uint8)), f"{which}: shadow candidates"
        assert np.array_equal(uncast, exp["uncast"]), f"{which}: uncast lights in the atlas"
    return got


def visible_lights(ctx, S, res_cull, dev_ids):
    n, off = res_cull.type_count[2], res_cull.type_offset[2]
    return ctx.copy_to_host(dev_ids, off + n, np.uint32)[off:off + n].astype(np.int32) if n else np.zeros(0, np.int32)


@pytest.mark.parametrize("ortho", [False, True])
def test_lone_cull(ctx, ortho):
    S = Scene(ctx, seed=2 if ortho else 1)
    try:
        env, refl = probes(S.rng, 6, 9, S.cam)
        f = S.frustum(ortho=ortho)
        dev, cres = S.cs.cull_device(f)
        res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H), env, refl)
        assert res.n_lights > 50 and res.n_map > res.n_lights
        got = check_fill(S, f, res, env, refl, visible=visible_lights(ctx, S, cres, dev))
        # a second fill of the same cull gives the same bytes
        res2 = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H), env, refl)
        again = S.cl.read(res2)
        for k in ("lights", "clusters", "map", "light_entities"):
            assert np.array_equal(np.asarray(got[k]).view(np.uint8), np.asarray(again[k]).view(np.uint8)), k
        assert bytes(res) == bytes(res2)
    finally:
        S.close()


def test_cull_views_view_k_and_other_outputs_untouched(ctx):
    S = Scene(ctx, seed=3)
    try:
        rots = [(0.0, 0.0, 0.0, 1.0), tuple(unit_quat(S.rng)), tuple(unit_quat(S.rng))]
        frusta = [S.frustum(rot=r) for r in rots]
        views = S.cs.cull_views(frusta)
        # sort keys with models, as a frame has them, from the same transforms
        from lumixengine_b200 import sortkeys
        skin = scenes.sortkey_setup(S.n, S.types, S.pos, seed=5)
        S.tr = skin["transforms"]
        S.sk.close()
        S.sk = lb.SortKeys(ctx, S.n, skin["max_sort_key"] + 1, max_keys=4 * S.n, max_instances=4 * S.n)
        S.sk.setModels(skin["models"], skin["meshes"])
        S.sk.setInstances(skin["model_of"], skin["lod"], skin["flags"], skin["pose_frame"], skin["decal_sort_key"], skin["decal_layer"])
        S.sk.setTransforms(S.tr)
        v = sortkeys.make_view(tuple(S.cam), tuple(S.cam), 1.0 / 60.0, 1.0, 1, False, skin["max_sort_key"], skin["layer_to_bucket"], skin["depth_sorted_buckets"])
        skres = S.sk.createSortKeysViews(S.cs, [v] * 3)
        before = [S.sk.readView(k, skres[k]) for k in range(3)]
        ids_before = [ctx.copy_to_host(views[k][0], views[k][1].total, np.uint32) for k in range(3)]
        for k in (1, 2, 0):
            env, refl = probes(S.rng, 3, 4, S.cam)
            res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, frusta[k], W, H, view=k), env, refl)
            check_fill(S, frusta[k], res, env, refl, visible=visible_lights(ctx, S, views[k][1], views[k][0]))
        after = [S.sk.readView(k, skres[k]) for k in range(3)]
        for k in range(3):
            for name in before[k]:
                assert np.array_equal(np.asarray(before[k][name]).view(np.uint8), np.asarray(after[k][name]).view(np.uint8)), (k, name)
            assert np.array_equal(ids_before[k], ctx.copy_to_host(views[k][0], views[k][1].total, np.uint32))
        # view k past the call's count
        with pytest.raises(LumixB200Error):
            S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, frusta[0], W, H, view=3))
    finally:
        S.close()


def test_lights_moved_on_the_device(ctx):
    S = Scene(ctx, seed=4)
    try:
        lights = np.flatnonzero(S.types == 2).astype(np.int32)
        f = S.frustum()
        for frame in range(3):
            moved = S.rng.choice(lights, len(lights) // 3, replace=False).astype(np.int32)
            tr = S.tr[moved].copy()
            tr["pos"] += S.rng.uniform(-20, 20, (len(moved), 3))
            tr["rot"] = np.array([unit_quat(S.rng) for _ in moved], np.float32).reshape(-1, 4)
            de, dt = ctx.to_device(moved), ctx.to_device(tr)
            try:
                S.sk.moveDevice(de, dt, len(moved))
            finally:
                ctx.synchronize()
                ctx.free_device(de)
                ctx.free_device(dt)
            S.tr[moved] = tr
            S.cs.set(moved, tr["pos"], S.pl["range"][moved])
            dev, cres = S.cs.cull_device(f)
            res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))
            check_fill(S, f, res, visible=visible_lights(ctx, S, cres, dev))
            S.sk.endFrame()
    finally:
        S.close()


def test_patch_atlas_and_set_atlas(ctx):
    S = Scene(ctx, seed=5, n_atlas=30)
    try:
        f = S.frustum()
        S.cs.cull_device(f)
        res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))
        check_fill(S, f, res)
        shadow = lc.shadow_list(res)
        assert len(shadow) > 0 and res.n_uncast > 0
        idx = shadow["light_idx"][:10]
        new = np.arange(len(idx), dtype=np.int32) + 5
        S.cl.patchAtlas(idx, new)
        got = S.cl.read(res)
        assert np.array_equal(got["lights"]["atlas_idx"][idx], new.astype(np.uint32))
        others = np.setdiff1d(np.arange(res.n_lights), idx)
        refill = S.cl.read(S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H)))
        assert np.array_equal(refill["lights"]["atlas_idx"][others], got["lights"]["atlas_idx"][others])
        # the host's atlas step as the reference runs it: uncast entries removed, new entries for the candidates
        ents = np.array(res.uncast[:res.n_uncast], np.int32)
        S.cl.setAtlas(ents, np.full(len(ents), -1, np.int32))
        S.atlas[ents] = -1
        cand = shadow["entity"][:5]
        S.cl.setAtlas(cand, np.arange(5, dtype=np.int32))
        S.atlas[cand] = np.arange(5)
        res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))
        check_fill(S, f, res)
        assert res.n_uncast == 0
        # refusals change nothing
        for e, a in (([S.n], [1]), ([-1], [1]), ([0], [64]), ([0], [-2])):
            with pytest.raises(LumixB200Error):
                S.cl.setAtlas(np.array(e, np.int32), np.array(a, np.int32))
        with pytest.raises(LumixB200Error):
            S.cl.setAtlas(np.arange(65, dtype=np.int32) + 100, np.zeros(65, np.int32))
        with pytest.raises(LumixB200Error):
            S.cl.patchAtlas([res.n_lights], [0])
        res2 = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))
        assert bytes(res2) == bytes(res)
    finally:
        S.close()


def test_zero_lights_and_zero_probes(ctx):
    S = Scene(ctx, seed=6, light_fraction=0.0)
    try:
        f = S.frustum()
        S.cs.cull_device(f)
        res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))
        assert res.n_lights == 0 and res.n_map == 0 and res.n_shadow == 0 and res.n_uncast == 0
        got = check_fill(S, f, res)
        assert not got["clusters"].view(np.uint32).any()
        env, refl = probes(S.rng, 4, 0, S.cam)
        res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H), env, refl)
        check_fill(S, f, res, env, refl)
    finally:
        S.close()


def test_one_light_over_every_cluster_and_map_growth(ctx):
    cam = (0.0, 0.0, 0.0)
    pos = np.array([cam, (1.0, 2.0, -3.0), (-5.0, 1.0, 2.0), (2.0, -1.0, 1.0)], np.float64)
    S = Scene(ctx, n=4, light_fraction=1.0, seed=7, cam=cam, pos=pos, radius=np.full(4, 1e6, np.float32), n_atlas=0)
    try:
        f = S.frustum(w=64, h=64)
        S.cs.cull_device(f, type=2)
        one = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, 64, 64))
        got = check_fill(S, f, one, w=64, h=64)
        assert (got["clusters"]["lights_count"] == 4).all() and one.n_clusters == 16
        # 4096 x 4096: 65 536 clusters, every light in each: 262 144 entries, past the map's first capacity (65 536)
        f = S.frustum(w=4096, h=4096)
        S.cs.cull_device(f, type=2)
        n0 = ctx.launches
        res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, 4096, 4096))
        grown = ctx.launches - n0
        assert res.n_map == 4 * 65536
        check_fill(S, f, res, w=4096, h=4096)
        n0 = ctx.launches
        res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, 4096, 4096))
        assert ctx.launches - n0 == 4 and grown == 8
        check_fill(S, f, res, w=4096, h=4096)
    finally:
        S.close()


def test_launch_count_does_not_depend_on_lights(ctx):
    counts = []
    for n in (50, 20000):
        S = Scene(ctx, n=n, seed=8, r_range=(0.1, 0.5))
        try:
            f = S.frustum()
            S.cs.cull_device(f)
            S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))  # capacities settle
            n0 = ctx.launches
            res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))
            counts.append(ctx.launches - n0)
            check_fill(S, f, res)
        finally:
            S.close()
    assert counts == [4, 4]


def test_refusals(ctx):
    S = Scene(ctx, seed=9)
    try:
        f = S.frustum()
        S.cs.cull_device(f)
        res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))
        before = S.cl.read(res)
        for w, h in ((0, H), (W, 0), (4097, H), (W, 4097)):
            with pytest.raises(LumixB200Error) as e:
                S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, w, h))
            assert e.value.code == lb._lib.ERR_INVALID
        small = lb.SortKeys(ctx, S.n - 1, 1)
        small.setTransforms(S.tr[:S.n - 1])
        bare = lb.SortKeys(ctx, S.n, 1)
        small_cl = lb.Clusters(ctx, S.n - 1)
        try:
            for sk, cl in ((small, S.cl), (bare, S.cl), (S.sk, small_cl)):
                with pytest.raises(LumixB200Error) as e:
                    cl.fillClusters(sk, S.cs, lc.make_view(S.cam, f, W, H))
                assert e.value.code == lb._lib.ERR_INVALID
        finally:
            small.close()
            bare.close()
            small_cl.close()
        with pytest.raises(LumixB200Error) as e:  # no cull_views on this culling system
            S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H, view=0))
        assert e.value.code == lb._lib.ERR_STATE
        with pytest.raises(LumixB200Error):
            S.cl.setPointLights([0, 0], S.pl[:2])
        with pytest.raises(LumixB200Error):
            S.cl.setPointLights([S.n], S.pl[:1])
        # a culling system of another context, and one without a context: their ids are not on this stream
        other = lb.Context(0)
        try:
            for owner in (other, None):
                cs2 = lb.CullingSystem(owner)
                try:
                    cs2.add(np.arange(S.n, dtype=np.int32), S.types, S.pos, S.pl["range"])
                    if owner is not None:
                        cs2.cull_device(f)
                    with pytest.raises(LumixB200Error) as e:
                        S.cl.fillClusters(S.sk, cs2, lc.make_view(S.cam, f, W, H))
                    assert e.value.code == lb._lib.ERR_INVALID
                finally:
                    cs2.close()
        finally:
            other.close()
        # atlas indices outside -1 .. 63 are not patched
        for a in (64, -2):
            with pytest.raises(LumixB200Error) as e:
                S.cl.patchAtlas([0], [a])
            assert e.value.code == lb._lib.ERR_INVALID
        after = S.cl.read(res)
        for k in before:
            assert np.array_equal(np.asarray(before[k]).view(np.uint8), np.asarray(after[k]).view(np.uint8)), k
        fresh = lb.Clusters(ctx, 8)
        try:
            with pytest.raises(LumixB200Error) as e:
                fresh.patchAtlas([0], [0])
            assert e.value.code == lb._lib.ERR_STATE
        finally:
            fresh.close()
    finally:
        S.close()


def test_c2_main_view(ctx):
    """The C2 scene (10 M entities, 5 % LOCAL_LIGHT) with cull radius = range, its main view at 1920 x 1080."""
    sc = scenes.c2_scene()
    n = len(sc["entities"])
    rng = np.random.default_rng(11)
    cs = lb.CullingSystem(ctx)
    cs.add(sc["entities"], sc["types"], sc["pos"], sc["radius"])
    tr = np.zeros(n, lb.TRANSFORM_DTYPE)
    tr["pos"] = sc["pos"]
    tr["rot"] = (0.0, 0.0, 0.0, 1.0)
    tr["scale"] = 1.0
    sk = lb.SortKeys(ctx, n, 1, max_keys=1024, max_instances=1024)
    sk.setTransforms(tr)
    cl = lb.Clusters(ctx, n)
    try:
        lights = np.flatnonzero(sc["types"] == 2).astype(np.int32)
        pl = light_records(rng, len(lights), sc["radius"][lights], cast_fraction=0.2)
        cl.setPointLights(lights, pl)
        atlas = rng.choice(lights, 37, replace=False).astype(np.int32)
        cl.setAtlas(atlas, np.arange(37, dtype=np.int32))
        a = scenes.c2_frustum_args()
        f = lb.frustum_perspective(a["position"], a["direction"], a["up"], a["fov"], W / H, a["near"], a["far"])
        dev, cres = cs.cull_device(f)
        env, refl = probes(rng, 16, 16, np.zeros(3), spread=2000.0)
        res = cl.fillClusters(sk, cs, lc.make_view(a["position"], f, W, H), env, refl)
        assert res.n_lights > 50000 and res.n_shadow == 64

        class T:
            pass
        S = T()
        S.cl, S.cam, S.tr = cl, np.asarray(a["position"], np.float64), tr
        S.pl = np.zeros(n, lc.POINT_LIGHT_DTYPE)
        S.pl[lights] = pl
        S.atlas = np.full(n, -1, np.int32)
        S.atlas[atlas] = np.arange(37)
        check_fill(S, f, res, env, refl, visible=visible_lights(ctx, S, cres, dev))
    finally:
        cl.close()
        sk.close()
        cs.close()


def test_shadow_candidates_ties_nan_and_rising_priorities(ctx):
    """The AtlasSorter list on its two device paths: the selection of the 64 best casters (ties at one priority, -0 and +0, priorities
    rising along the light order) and the replay of the pushes once a caster's priority is NaN (fov 0 at the camera: 0 / 0)."""
    rng = np.random.default_rng(12)
    cam = np.array([10.0, 5.0, -20.0])
    n = 2000
    pos = cam + rng.uniform(-300, 300, (n, 3))
    pos[:300] = cam + (1.0, 2.0, -50.0)   # one position: equal priorities for equal fov and range
    pos[300:320] = cam                    # at the camera: distance 0
    radius = rng.uniform(0.5, 30.0, n).astype(np.float32)
    radius[:300] = 5.0
    S = Scene(ctx, n=n, light_fraction=1.0, seed=12, cam=tuple(cam), pos=pos, radius=radius, n_atlas=30)
    try:
        f = S.frustum()
        dev, cres = S.cs.cull_device(f)
        lights = np.arange(n, dtype=np.int32)

        def fill_with(fov, cast):
            S.pl["fov"] = fov
            S.pl["flags"] = np.where(cast, S.pl["flags"] | lc.CAST_SHADOWS, S.pl["flags"] & ~np.uint32(lc.CAST_SHADOWS))
            S.cl.setPointLights(lights, S.pl)
            res = S.cl.fillClusters(S.sk, S.cs, lc.make_view(S.cam, f, W, H))
            check_fill(S, f, res, visible=visible_lights(ctx, S, cres, dev))
            return res

        fov = rng.uniform(1e-6, 2e-6, n).astype(np.float32)   # below the 300 lights' priority whatever their distance and range
        fov[:300] = 1.0
        not_at_cam = np.ones(n, bool)
        not_at_cam[300:320] = False
        res = fill_with(fov, not_at_cam)                       # > 64 equal priorities at the top
        sh = lc.shadow_list(res)
        assert len(sh) == 64 and (sh["priority"] == sh["priority"][0]).all()
        zero = fov.copy()
        zero[:300] = 0.0                                       # +0 priorities, and -0 ones from a negative zero fov
        zero[:300:2] = -0.0
        fill_with(zero, not_at_cam)
        fov_nan = fov.copy()
        fov_nan[300:320] = 0.0                                 # 0 * r^3 / 0: NaN
        res = fill_with(fov_nan, np.ones(n, bool))             # NaN casters among 2,000: pushed out of the list again
        few = np.zeros(n, bool)
        few[:30] = few[300:320] = True
        res = fill_with(fov_nan, few)                          # 50 casters: the NaN ones stay in the list, where the pushes left them
        assert np.isnan(lc.shadow_list(res)["priority"]).sum() == 20
        # priorities rising along the light order of this cull: every caster beats the list so far
        ents = S.cl.read(res)["light_entities"]
        d = np.sqrt(((S.tr["pos"][ents] - cam) ** 2).sum(1))
        rising = S.pl["fov"].copy()
        rising[ents] = (np.arange(1, len(ents) + 1) * d / S.pl["range"][ents].astype(np.float64) ** 3).astype(np.float32)
        fill_with(rising, not_at_cam)
        fill_with(rising, np.ones(n, bool))                    # the same with the lights at the camera: 0 / 0 again, replayed
    finally:
        S.close()
