"""Skinning palettes of the instances createSortKeys claims (SortKeys.buildPalettes, lb200_sortkeys_build_palettes): PoseProcessor::push +
computeSkeletonDualQuats on the device for the pose lists create_keys / create_keys_views leave in HBM.

Every slice is compared bit for bit with the dual quaternions a DUAL_QUAT | POSE update of the same systems wrote for the instance that
lists the entity (and, for a sample, with the oracle's palettes of its pose); listed entities without an instance must get 0xffffffff,
slices must be disjoint, inside [0, n_bones), and add up to n_bones.
"""
import ctypes as C

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import _lib, scenes, sortkeys
from lumixengine_b200._lib import LumixB200Error
from bitexact import assert_bits_equal

pytestmark = pytest.mark.gpu

DQ, POSE = lb.PALETTE_DUAL_QUAT, lb.PALETTE_POSE
NONE = 0xffffffff
LIGHT = (0.3, -0.8, 0.2)


def _skeleton(bones, seed):
    return scenes.skeleton(seed=seed, parents=[-1]) if bones == 1 else scenes.skeleton(bones, seed=seed)


def _clips(sk, seed):
    return [scenes.clip(sk, frames=13, fps=30.0, seed=seed, const_fraction=0.3), scenes.clip(sk, frames=21, fps=24.0, seed=seed + 1, const_fraction=0.3)]


def _system(ctx, bones, entities, seed, max_instances=None):
    sk = _skeleton(bones, seed)
    clips = _clips(sk, seed + 50)
    a = lb.AnimationSystem(ctx, sk, clips, max_instances=max(1, max_instances or len(entities)))
    a.setInstances(*scenes.instance_times(len(entities), clips, seed=seed + 7))
    a.setEntities(entities)
    return a


class Scene:
    """A culled scene (meshes of skinned and static models, decals, MOVED and dirty instances) with the skinned mesh entities spread over
    animation systems; `animated` of them have an instance, the rest have no animation component."""

    def __init__(self, ctx, n=40_000, seed=3, bones=(1, 64, 196), animated=0.85, n_systems=None):
        self.ctx = ctx
        self.scene = scenes.cull_scene(n, (2500.0, 300.0, 2500.0), seed=seed, type_probs=(0.8, 0.08, 0.04, 0.08), big_fraction=0.002)
        self.n = n
        sk = scenes.sortkey_setup(n, self.scene["types"], self.scene["pos"], seed=seed + 100, skinned_fraction=0.3)
        self.sk = sk
        skinned_model = np.zeros(len(sk["models"]), bool)
        for m, md in enumerate(sk["models"]):
            skinned_model[m] = sk["meshes"]["skinned"][md["mesh_base"]:md["mesh_base"] + md["mesh_count"]].any()
        rng = np.random.default_rng(seed)
        skinned = np.nonzero((self.scene["types"] == 0) & skinned_model[sk["model_of"]])[0]
        ents = skinned[rng.random(len(skinned)) < animated].astype(np.int32)
        rng.shuffle(ents)
        k = n_systems or len(bones)
        self.systems = [_system(ctx, bones[s % len(bones)], ents[s::k], seed + 10 * s) for s in range(k)]
        self.entities = [ents[s::k] for s in range(k)]
        self.cs = lb.CullingSystem(ctx)
        self.cs.add(self.scene["entities"], self.scene["types"], self.scene["pos"], self.scene["radius"])
        self.S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
        self.S.setModels(sk["models"], sk["meshes"])
        self.S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
        self.S.setTransforms(sk["transforms"])

    def view(self, args, frame, shadow=False):
        sk = self.sk
        return sortkeys.make_view(args["position"], args["position"], 0.1, 1.0, frame, shadow, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])

    def pose(self, dt=0.05):
        lb.AnimationSystem.updateMany(self.systems, dt, DQ | POSE)

    def one_view(self, args, frame):
        self.cs.cull_device(lb.frustum_perspective(**args), want_counts=False)
        res = self.S.createSortKeys(self.cs, self.view(args, frame))
        return self.S.read(res)["pose_list"]

    def expected(self):
        """entity -> (system, instance) and the dual quaternions each system's update wrote."""
        owner = {}
        for s, ents in enumerate(self.entities):
            for i, e in enumerate(ents):
                owner[int(e)] = (s, i)
        return owner, [a.getDualQuats() for a in self.systems]

    def close(self):
        self.S.close()
        self.cs.close()
        for a in self.systems:
            a.close()


def _frusta(args):
    return [lb.frustum_perspective(**a) if "fov" in a else lb.frustum_ortho(**a) for a in args]


def _camera(x=0.0, z=0.0, dx=0.0):
    a = scenes.c1_frustum_args()
    a["position"] = (x, 0.0, z)
    a["direction"] = tuple(np.array([dx, 0.0, -1.0]) / np.linalg.norm([dx, 0.0, -1.0]))
    return a


def check(pal, listed, owner, dq, what):
    """Every listed entity's slice against the expectation; disjoint slices that add up to n_bones.  -> entities with a slice"""
    off, nb, got = pal["offset"], pal["n_bones"], pal["dual_quats"]
    listed = np.unique(np.asarray(listed, np.int64))
    has = np.array([int(e) in owner for e in listed], bool)
    assert np.all(off[listed[~has]] == NONE), f"{what}: a listed entity without an instance has an offset"
    used = np.zeros(nb, np.int32)
    for e in listed[has]:
        s, i = owner[int(e)]
        exp = dq[s][i]
        o = int(off[e])
        assert o != NONE and o + len(exp) <= nb, f"{what}: entity {e}: offset {o} with {len(exp)} bones outside [0, {nb})"
        used[o:o + len(exp)] += 1
        assert_bits_equal(got[o:o + len(exp)], exp, f"{what}: entity {e}")
    assert np.all(used == 1), f"{what}: slices overlap or leave gaps ({int((used != 1).sum())} bones)"
    return listed[has]


def test_one_view(ctx, oracle):
    sc = Scene(ctx)
    sc.pose()
    listed = sc.one_view(scenes.c2_frustum_args(), 1)
    owner, dq = sc.expected()
    sc.S.buildPalettes(sc.systems)
    pal = sc.S.readPalettes()
    built = check(pal, listed, owner, dq, "one view")
    assert len(built) > 100 and len(built) < len(np.unique(listed)), "the scene lists entities with and without instances"
    assert {sc.systems[owner[int(e)][0]].skeleton.bone_count for e in built} == {1, 64, 196}
    # a sample against the oracle's computeSkeletonDualQuats of the instance's absolute pose
    for e in built[::max(1, len(built) // 12)]:
        s, i = owner[int(e)]
        a = sc.systems[s]
        pos, rot = a.getPose(i, 1)
        exp, _ = oracle.palettes(a.skeleton, pos[0], rot[0])
        o = int(pal["offset"][e])
        assert_bits_equal(pal["dual_quats"][o:o + a.skeleton.bone_count], exp, f"oracle: entity {e}")
    sc.close()


@pytest.mark.parametrize("n_views", [1, 5, 8])
def test_views(ctx, n_views):
    sc = Scene(ctx, seed=5)
    sc.pose()
    cam = scenes.c2_frustum_args()
    args = ([cam] + scenes.shadow_cascade_args(cam, LIGHT, (40.0, 200.0, 900.0, 2500.0)) + [_camera(300.0 * k, 0.0, 0.4 * k) for k in (1, 2, 3)])[:n_views]
    sc.cs.cull_views(_frusta(args), want_counts=False)
    views = [sc.view(a, 3, shadow=k > 0) for k, a in enumerate(args)]
    res = sc.S.createSortKeysViews(sc.cs, views)
    lists = [sc.S.readView(k, r)["pose_list"] for k, r in enumerate(res)]
    all_listed = np.concatenate(lists)
    assert len(np.unique(all_listed)) == len(all_listed), "an entity joins one view's pose list"
    owner, dq = sc.expected()
    sc.S.buildPalettes(sc.systems, views=True)
    built = check(sc.S.readPalettes(), all_listed, owner, dq, f"{n_views} views")
    if n_views > 1:
        assert sum(len(x) for x in lists[1:]) > 0 and len(built) > 0
    sc.close()


def test_frames(ctx):
    sc = Scene(ctx, seed=7)
    prev = None
    for f in range(1, 6):
        sc.pose(dt=0.07)
        listed = sc.one_view(_camera(150.0 * f, -40.0 * f, 0.1 * f), f)
        owner, dq = sc.expected()
        sc.S.buildPalettes(sc.systems)
        pal = sc.S.readPalettes()
        built = check(pal, listed, owner, dq, f"frame {f}")
        if prev is not None:
            again = np.intersect1d(built, prev[0])
            assert len(again), "entities claimed in consecutive frames"
            moved = 0
            for e in again:
                s, i = owner[int(e)]
                B = len(dq[s][i])
                moved += not np.array_equal(pal["dual_quats"][pal["offset"][e]:pal["offset"][e] + B], prev[1][prev[2][e]:prev[2][e] + B])
            assert moved > 0, "the next frame's palettes follow the next frame's poses"
        prev = (built, pal["dual_quats"].copy(), pal["offset"].copy())
    sc.close()


def _ik_chain(sk):
    depth = np.zeros(sk.bone_count, np.int64)
    for b in range(sk.bone_count):
        depth[b] = 0 if sk.parents[b] < 0 else depth[sk.parents[b]] + 1
    return int(np.argmax(depth))


def test_modes_and_launches(ctx):
    """Clip-mode, sample-list, IK and root-motion systems in one update_many and one build, 70 systems: two launches of each kernel."""
    sc = Scene(ctx, seed=9, bones=(8, 17, 30), n_systems=70)
    rng = np.random.default_rng(1)
    for s, a in enumerate(sc.systems):
        n, clips, mode = len(sc.entities[s]), a.clips, s % 4
        if mode in (1, 2):
            counts = rng.integers(1, 3, n)
            off = np.concatenate([[0], np.cumsum(counts)]).astype(np.uint32)
            m = int(off[-1])
            ci = rng.integers(0, len(clips), m)
            t = rng.integers(0, 20000, m)
            w = rng.choice(np.array([1.0, 0.6], np.float32), m)
            if mode == 1:
                a.setSamples(off, ci, t, w, np.ones(m))
            else:
                ik_off = np.arange(n + 1, dtype=np.uint32)
                a.setStacks(off, ci, t, w, np.ones(m), ik_off, counts, np.full(n, _ik_chain(a.skeleton)), np.full(n, 2), np.full(n, 1.0, np.float32),
                            (rng.normal(size=(n, 3)) * 0.5).astype(np.float32))
        elif mode == 3:
            tr = [c.rootMotionTracks(0) for c in clips]
            a.setRootMotion(np.full(len(clips), 7), [x[0] for x in tr], [x[1] for x in tr])
    sc.pose()
    listed = sc.one_view(scenes.c2_frustum_args(), 1)
    owner, dq = sc.expected()
    before = ctx.launches
    sc.S.buildPalettes(sc.systems)
    assert ctx.launches - before == 4, "one map and one build launch per 64 systems"
    built = check(sc.S.readPalettes(), listed, owner, dq, "70 systems")
    assert len({owner[int(e)][0] % 4 for e in built}) == 4, "every mode builds"
    # fewer listed entities, same launches
    listed = sc.one_view(_camera(0.0, 0.0, 3.0), 2)
    before = ctx.launches
    sc.S.buildPalettes(sc.systems)
    assert ctx.launches - before == 4
    check(sc.S.readPalettes(), listed, owner, dq, "70 systems, another camera")
    sc.close()


def test_edges(ctx):
    sc = Scene(ctx, seed=11)
    sc.pose()
    args = scenes.c2_frustum_args()
    listed = sc.one_view(args, 1)
    owner, dq = sc.expected()
    sc.S.buildPalettes(sc.systems)
    built = check(sc.S.readPalettes(), listed, owner, dq, "first build")
    # two instances list one entity: a second system whose instance 0 lists an entity system 1 also lists
    e = int(next(x for x in built if owner[int(x)][0] == 1))
    s1, i1 = owner[e]
    twin = _system(ctx, sc.systems[1].skeleton.bone_count, np.array([e, -1], np.int32), seed=10 + 10 * s1)
    twin.update(0.05, DQ | POSE)
    sc.S.setInstances(pose_frame=np.full(sc.n, NONE, np.uint32))  # claim the same list again
    listed = sc.one_view(args, 1)
    sc.S.buildPalettes(sc.systems + [twin])
    pal = sc.S.readPalettes()
    o, B = int(pal["offset"][e]), sc.systems[1].skeleton.bone_count
    got = pal["dual_quats"][o:o + B]
    assert np.array_equal(got.view(np.uint32), dq[1][i1].view(np.uint32)) or np.array_equal(got.view(np.uint32), twin.getDualQuats()[0].view(np.uint32))
    twin.close()
    # set_entities between builds with a changed instance count: system 2 keeps its first half, system 0 lists its second half too
    keep = len(sc.entities[2]) // 2
    a2 = sc.systems[2]
    a2.setInstances(*scenes.instance_times(keep, a2.clips, seed=3))
    a2.setEntities(sc.entities[2][:keep])
    sc.entities[2] = sc.entities[2][:keep]
    sc.pose()
    owner, dq = sc.expected()
    sc.S.setInstances(pose_frame=np.full(sc.n, NONE, np.uint32))
    listed = sc.one_view(args, 2)
    before = sc.S.readPalettes()["offset"].copy()
    sc.S.buildPalettes(sc.systems)
    pal = sc.S.readPalettes()
    check(pal, listed, owner, dq, "after set_entities")
    # entities a build does not list keep their offsets
    listed2 = sc.one_view(_camera(0.0, 0.0, 4.0), 3)
    sc.S.buildPalettes(sc.systems)
    off2 = sc.S.readPalettes()["offset"]
    rest = np.setdiff1d(np.arange(sc.n), listed2)
    assert np.array_equal(off2[rest], pal["offset"][rest]), "offsets of unlisted entities are untouched"
    assert not np.array_equal(before, pal["offset"])
    sc.close()


def test_growth(ctx):
    """A spawn grows max_entities between create_keys_views and the build; then high ids join the lists and get their palettes."""
    sc = Scene(ctx, n=20_000, seed=13)
    sc.pose()
    cam = scenes.c2_frustum_args()
    sc.cs.cull_views(_frusta([cam]), want_counts=False)
    res = sc.S.createSortKeysViews(sc.cs, [sc.view(cam, 1)])
    listed = sc.S.readView(0, res[0])["pose_list"]
    sc.S.buildPalettes(sc.systems, views=True)
    # spawn skinned instances at ids past max_entities, in front of the camera
    n_new = 300
    ids = np.arange(3 * sc.n, 3 * sc.n + n_new, dtype=np.int32)
    skm = int(np.nonzero([sc.sk["meshes"]["skinned"][m["mesh_base"]] for m in sc.sk["models"]])[0][0])
    tr = np.zeros(n_new, lb.TRANSFORM_DTYPE)
    rng = np.random.default_rng(2)
    tr["pos"] = np.c_[rng.uniform(-50, 50, n_new), rng.uniform(-5, 5, n_new), rng.uniform(-60, -20, n_new)]
    tr["rot"] = (0, 0, 0, 1)
    tr["scale"] = 1
    d = [ctx.to_device(x) for x in (ids, np.full(n_new, skm, np.uint32), tr)]
    sc.S.spawnInstancesDevice(d[0], d[1], d[2], n_new, int(ids.max()))
    for p in d:
        ctx.free_device(p)
    assert sc.S.max_entities > ids.max()
    owner, dq = sc.expected()
    sc.S.buildPalettes(sc.systems, views=True)
    pal = sc.S.readPalettes()
    assert len(pal["offset"]) == sc.S.max_entities
    check(pal, listed, owner, dq, "after the growth")
    # the new ids culled, claimed and animated
    sc.cs.add(ids, 0, tr["pos"], 1.0)
    extra = _system(ctx, 64, ids[::2], seed=77)
    sc.systems.append(extra)
    sc.entities.append(ids[::2])
    sc.pose()
    sc.cs.cull_views(_frusta([cam]), want_counts=False)
    res = sc.S.createSortKeysViews(sc.cs, [sc.view(cam, 2)])
    listed = sc.S.readView(0, res[0])["pose_list"]
    assert np.isin(ids, listed).sum() > n_new // 2
    owner, dq = sc.expected()
    sc.S.buildPalettes(sc.systems, views=True)
    pal = sc.S.readPalettes()
    check(pal, listed, owner, dq, "high ids")
    high = ids[np.isin(ids, listed)]
    assert np.all(pal["offset"][high[high % 2 == ids[0] % 2]] != NONE) and np.all(pal["offset"][high[high % 2 != ids[0] % 2]] == NONE)
    sc.close()


def test_refusals(ctx):
    sc = Scene(ctx, n=10_000, seed=17)
    sc.pose()
    sc.one_view(scenes.c2_frustum_args(), 1)
    sc.S.buildPalettes(sc.systems)
    snap = sc.S.readPalettes()
    a, b = sc.systems[0], sc.systems[1]
    L = _lib.lib()
    out = _lib.SkPalettes()
    arr = (C.c_void_p * 2)(a.h, b.h)
    fresh = _system(ctx, 5, np.array([1, 2, 3], np.int32), seed=5)  # never updated: no absolute poses
    ctx2 = lb.Context(0)
    other = _system(ctx2, 5, np.array([4], np.int32), seed=6)
    other.update(0.1, POSE)
    cases = [
        ("NULL out", lambda: L.lb200_sortkeys_build_palettes(sc.S.h, arr, 2, 0, None), _lib.ERR_INVALID),
        ("NULL systems", lambda: L.lb200_sortkeys_build_palettes(sc.S.h, None, 2, 0, C.byref(out)), _lib.ERR_INVALID),
        ("NULL entry", lambda: sc.S.buildPalettes([a, None]), _lib.ERR_INVALID),
        ("listed twice", lambda: sc.S.buildPalettes([a, b, a]), _lib.ERR_INVALID),
        ("another context", lambda: sc.S.buildPalettes([a, other]), _lib.ERR_INVALID),
        ("no poses", lambda: sc.S.buildPalettes([a, fresh]), _lib.ERR_STATE),
        ("views before create_keys_views", lambda: sc.S.buildPalettes([a], views=True), _lib.ERR_STATE),
    ]
    for what, call, code in cases:
        try:
            rc = call()
        except LumixB200Error as err:
            rc = err.code
        assert rc == code, what
        now = sc.S.readPalettes()
        assert now["n_bones"] == snap["n_bones"] and np.array_equal(now["offset"], snap["offset"]), what
        assert_bits_equal(now["dual_quats"], snap["dual_quats"], what)
    S2 = lb.SortKeys(ctx, 100, 10)
    with pytest.raises(LumixB200Error) as e:
        S2.buildPalettes([a])
    assert e.value.code == _lib.ERR_STATE
    # set_entities refusals leave the table as it was
    with pytest.raises(LumixB200Error):
        a.setEntities(np.array([5, 6, 5], np.int32))
    with pytest.raises(LumixB200Error):
        a.setEntities(np.zeros(a.n + 10 ** 6, np.int32))
    a.setEntities(np.array([-1, -1, 7, 8], np.int32))  # negative ids may repeat
    S2.close()
    fresh.close()
    other.close()
    ctx2.close()
    sc.close()


def test_full_size(ctx):
    """100 k instances over three skeletons, one build against get_dual_quats."""
    n = 130_000
    sc = Scene(ctx, n=n, seed=19, bones=(64, 17, 1), animated=1.0)
    for s in range(3):  # top the systems up to 100 k instances with entities outside the scene
        need = {0: 60_000, 1: 30_000, 2: 10_000}[s] - len(sc.entities[s])
        if need > 0:
            extra = np.arange(n + 200_000 * (s + 1), n + 200_000 * (s + 1) + need, dtype=np.int32)
            ents = np.concatenate([sc.entities[s], extra]).astype(np.int32)
            a = sc.systems[s]
            sc.systems[s] = _system(ctx, a.skeleton.bone_count, ents, seed=19 + 10 * s)
            a.close()
            sc.entities[s] = ents
    assert sum(len(e) for e in sc.entities) >= 100_000
    sc.pose()
    listed = sc.one_view(scenes.c2_frustum_args(), 1)
    owner, dq = sc.expected()
    sc.S.buildPalettes(sc.systems)
    built = check(sc.S.readPalettes(), listed, owner, dq, "100 k instances")
    assert len(built) > 1000
    sc.close()
