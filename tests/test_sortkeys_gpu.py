"""GPU parity of the stage behind the cull — createSortKeys + radixSort on the device (csrc/sortkeys.cu, csrc/radix_sort.cu) — against the oracle:
sorted (key, value) pairs as a multiset, auto-instancing groups as sets with their 48-byte instance data matched by renderable, lod state,
pose and dirty lists, bit for bit."""
import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes, sortkeys

pytestmark = pytest.mark.gpu


def _canon_pairs(keys, values):
    o = np.lexsort((values, keys))
    return keys[o], values[o]


def _compare(got, exp, lod_exp, pf_exp, n_entities):
    assert np.all(got["keys"][1:] >= got["keys"][:-1]), "device keys are not sorted"
    gk, gv = _canon_pairs(got["keys"], got["values"])
    ek, ev = _canon_pairs(exp["keys"], exp["values"])
    assert np.array_equal(gk, ek) and np.array_equal(gv, ev)
    assert np.array_equal(got["group_count"], exp["group_count"]) and np.array_equal(got["group_offset"], exp["group_offset"])
    # same renderables per group (the group is a range), instance data matched through the renderable
    go, eo = np.argsort(got["group_renderables"], kind="stable"), np.argsort(exp["group_renderables"], kind="stable")
    assert np.array_equal(got["group_renderables"][go], exp["group_renderables"][eo])
    g_of = np.repeat(np.arange(len(exp["group_count"])), exp["group_count"])
    assert np.array_equal(g_of[go], g_of[eo])
    assert np.array_equal(got["instance_data"][go], exp["instance_data"][eo])
    assert np.array_equal(np.sort(got["pose_list"]), np.sort(exp["pose_list"]))
    assert np.array_equal(np.sort(got["dirty_list"]), np.sort(exp["dirty_list"]))
    assert np.array_equal(got["lod"][:n_entities].view(np.uint32), lod_exp.view(np.uint32))
    assert np.array_equal(got["pose_frame"][:n_entities], pf_exp)


@pytest.mark.parametrize("n,seed,is_shadow,key_stride", [(60_000, 11, False, 1), (25_000, 12, True, 1), (40_000, 13, False, 131)])
def test_sort_keys_match_oracle_over_frames(ctx, oracle, n, seed, is_shadow, key_stride):
    scene = scenes.cull_scene(n, (2500.0, 300.0, 2500.0), seed=seed, type_probs=(0.8, 0.08, 0.04, 0.08), big_fraction=0.002)
    sk = scenes.sortkey_setup(n, scene["types"], scene["pos"], seed=seed + 100)
    if key_stride > 1:  # sparse sort keys: more auto-instancer groups than a block keeps in shared memory (8192) -> the group cursors live in HBM
        sk["meshes"]["sort_key"] = sk["meshes"]["sort_key"] * key_stride + 7
        sk["max_sort_key"] = int(sk["meshes"]["sort_key"].max()) + 3
        assert sk["max_sort_key"] + 1 > 8192
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
    S.setModels(sk["models"][:1], sk["meshes"][:1])  # replaced by the larger tables below: the second call re-allocates both
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(sk["transforms"])
    lod, pf = sk["lod"].copy(), sk["pose_frame"].copy()
    a = scenes.c1_frustum_args()
    cams = [dict(a, far=2500.0), dict(a, far=2500.0), dict(a, position=(300.0, 10.0, 200.0), direction=(-0.4, -0.05, -0.9), far=3000.0)]
    for frame, cam in enumerate(cams):  # the lod smoothing state and Pose::frame carry over from frame to frame
        f = lb.frustum_perspective(**cam)
        view = sortkeys.make_view(cam["position"], cam["position"], 1.0 / 30.0, 1.25, 40 + frame, is_shadow, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
        cs.cull_device(f, want_counts=False)
        res = S.createSortKeys(cs, view)
        got = S.read(res)
        oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
        exp = oracle.create_sort_keys(oids, otys, sk["transforms"], sk["model_of"], lod, sk["flags"], pf, sk["decal_sort_key"], sk["decal_layer"], sk["models"], sk["meshes"], view)
        assert res.n_keys == len(exp["keys"]) > 100 and res.n_instances == len(exp["group_renderables"]) > 1000
        _compare(got, exp, lod, pf, n)
    S.close()
    cs.close()


def _sort_createsortkeys_output(ctx, n):
    """createSortKeys with its sort on a scene of n entities, all MOVED and all visible (few distinct keys in long runs, bucket << 56 | mesh
    sort key): the keys come out sorted and the (key, value) pairs are a permutation of the unsorted output of the same pass.  The order among
    equal keys is not checked here (the unsorted order is not reproducible); tests/test_radix_sort_gpu.py checks stability.  -> n_keys"""
    scene = scenes.cull_scene(n, (400.0, 100.0, 400.0), seed=2, type_probs=(1.0,))
    # every entity MOVED -> one key per visible mesh, keys = mesh sort key | bucket << 56: few distinct keys, long runs
    sk = scenes.sortkey_setup(n, scene["types"], scene["pos"], n_models=6, seed=9, skinned_fraction=0.0, moved_fraction=1.1, dirty_fraction=0.0)
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=8 * n, max_instances=n)
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(sk["transforms"])
    f = lb.frustum_ortho((0.0, 0.0, 2000.0), (0.0, 0.0, 1.0), (0.0, 1.0, 0.0), 2000.0, 2000.0, 0.0, 4000.0)  # everything visible
    view = sortkeys.make_view((0.0, 0.0, 0.0), (0.0, 0.0, 0.0), 1.0 / 60.0, 1.0, 3, False, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
    cs.cull_device(f, want_counts=False)
    lod0 = sk["lod"].copy()
    unsorted = S.read(S.createSortKeys(cs, view, sort=False))
    S.setInstances(lod=lod0, pose_frame=sk["pose_frame"])  # same state again
    cs.cull_device(f, want_counts=False)
    res = S.createSortKeys(cs, view, sort=True)
    got = S.read(res)
    assert res.n_keys > n and res.n_keys == len(unsorted["keys"])
    assert np.all(got["keys"][1:] >= got["keys"][:-1])
    a, b = _canon_pairs(got["keys"], got["values"]), _canon_pairs(unsorted["keys"], unsorted["values"])
    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
    assert len(np.unique(got["keys"])) < 100
    S.close()
    cs.close()
    return res.n_keys


def test_device_radix_sort_alone(ctx):
    """The sort behind createSortKeys on the keys of a 50 k-entity scene (register path): sorted and a permutation of the unsorted pass."""
    _sort_createsortkeys_output(ctx, 50_000)


def test_device_radix_sort_tiled_through_create_sort_keys(ctx):
    """The same on a 1.5 M-entity scene whose keys are more than the register path holds, so that createSortKeys' sort takes the tiled path."""
    n_keys = _sort_createsortkeys_output(ctx, 1_500_000)
    # createSortKeys launches as many sort blocks as are co-resident, like an unconstrained lb200_radix_sort_device: above grid * 8192 keys
    # the tiled path sorts
    cap = 1 << 20
    _, _, grid = lb.radix_sort(ctx, np.zeros(cap, np.uint64), np.zeros(cap, np.uint64), count=0)
    assert n_keys > grid * 512 * 16, f"{n_keys} keys stay on the register path of a {grid}-block sort"


def test_pose_to_attachment_to_cull_chain_on_device(ctx, oracle):
    """SURVEY 8f N4 closed on the device: this frame's poses -> updateBoneAttachment for a batch (render_module.cpp:377-405) -> the attached
    entities' new transforms stay in HBM -> onModelInstanceMoved's bookkeeping (MOVED flag, moved list, sphere for CullingSystem::set,
    :1544-1554) -> device re-binning -> cull -> createSortKeys (MOVED instances become DRAW_MESH keys) -> endFrame (:526-534: MOVED off,
    prev_frame_transform).  Every stage against the oracle fed with the same edits one by one."""
    n = 30_000
    scene = scenes.cull_scene(n, (1800.0, 200.0, 1800.0), seed=31, type_probs=(0.9, 0.04, 0.02, 0.04), big_fraction=0.002)
    sk = scenes.sortkey_setup(n, scene["types"], scene["pos"], seed=77, moved_fraction=0.0)
    cs = lb.CullingSystem(ctx)
    cs.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    S = lb.SortKeys(ctx, n, sk["max_sort_key"] + 1, max_keys=4 * n, max_instances=4 * n)
    S.setModels(sk["models"], sk["meshes"])
    S.setInstances(sk["model_of"], sk["lod"], sk["flags"], sk["pose_frame"], sk["decal_sort_key"], sk["decal_layer"])
    S.setTransforms(sk["transforms"])
    # posed instances
    skel = scenes.skeleton(40)
    clips = [scenes.clip(skel, frames=30, seed=s) for s in (3, 4)]
    n_inst = 120
    anim = lb.AnimationSystem(ctx, skel, clips, None, max_instances=n_inst)
    ci, tt = scenes.instance_times(n_inst, clips, seed=2)
    anim.setInstances(ci, tt)
    anim.update(1.0 / 60.0, lb.PALETTE_POSE)
    pos, rot = anim.getPose()
    # attachments: m distinct MESH entities follow bones of posed instances whose entity is some other entity of the scene
    rng = np.random.default_rng(9)
    mesh_ids = np.nonzero(scene["types"] == 0)[0]
    m = 2500
    att = rng.choice(mesh_ids, m, replace=False).astype(np.int32)
    parent_entity = rng.integers(0, n, m)
    inst = rng.integers(0, n_inst, m).astype(np.uint32)
    bone = rng.integers(0, 40, m).astype(np.uint32)
    rel = np.concatenate([(rng.normal(size=(m, 3)) * 0.5).astype(np.float32), scenes.random_unit_quats(rng, m)], axis=1).astype(np.float32)
    par = np.ascontiguousarray(sk["transforms"][parent_entity])
    scale = np.ascontiguousarray(sk["transforms"]["scale"][att])
    br = (0.5 + 2.0 * rng.random(m)).astype(np.float32)  # Model::getOriginBoundingRadius of the attached entities' models
    dev = {k: ctx.to_device(v) for k, v in dict(ent=att, inst=inst, bone=bone, rel=rel, par=par, scale=scale, br=br).items()}
    dev["out_tr"] = ctx.to_device(np.zeros(m, lb.TRANSFORM_DTYPE))
    dev["pos3"] = ctx.to_device(np.zeros((m, 3), np.float64))
    dev["rad"] = ctx.to_device(np.zeros(m, np.float32))
    anim.boneAttachmentsDevice(m, dev["inst"], dev["bone"], dev["rel"], dev["par"], dev["scale"], dev["out_tr"])
    S.moveDevice(dev["ent"], dev["out_tr"], m, dev["br"], dev["pos3"], dev["rad"])
    cs.set_replicas(1)
    cs.set_many_device(dev["pos3"], dev["rad"], m, dev_entities=dev["ent"], max_entity=n - 1)
    # the oracle's side of the same frame
    bone7 = np.concatenate([pos[inst, bone], rot[inst, bone]], axis=1).astype(np.float32)
    exp_tr = oracle.bone_attachments(np.ascontiguousarray(par).view(np.uint8).reshape(m, 56), bone7, rel, scale).view(lb.TRANSFORM_DTYPE).reshape(-1)
    got_tr = ctx.copy_to_host(dev["out_tr"], m, lb.TRANSFORM_DTYPE)
    for field in ("pos", "rot", "scale"):
        assert got_tr[field].tobytes() == exp_tr[field].tobytes()
    exp_rad = (br * np.max(exp_tr["scale"], axis=1)).astype(np.float32)
    assert np.array_equal(ctx.copy_to_host(dev["rad"], m, np.float32), exp_rad)
    oc.set(att, np.ascontiguousarray(exp_tr["pos"]), exp_rad)
    transforms2 = sk["transforms"].copy()
    transforms2[att] = exp_tr
    flags2 = sk["flags"].copy()
    flags2[att] |= sortkeys.MOVED
    lod, pf = sk["lod"].copy(), sk["pose_frame"].copy()
    a = scenes.c1_frustum_args()
    cam = dict(a, far=2500.0)
    f = lb.frustum_perspective(**cam)
    for frame, flags in ((0, flags2), (1, sk["flags"])):  # frame 1 comes after endFrame: MOVED is off again, the transforms stay
        view = sortkeys.make_view(cam["position"], cam["position"], 1.0 / 30.0, 1.0, 60 + frame, False, sk["max_sort_key"], sk["layer_to_bucket"], sk["depth_sorted_buckets"])
        cs.cull_device(f, want_counts=False)
        res = S.createSortKeys(cs, view)
        got = S.read(res)
        oids, otys, _ = oc.cull(lb.culling.frustum_bytes(f))
        exp = oracle.create_sort_keys(oids, otys, transforms2, sk["model_of"], lod, flags, pf, sk["decal_sort_key"], sk["decal_layer"], sk["models"], sk["meshes"], view)
        assert res.n_keys == len(exp["keys"]) > 100
        _compare(got, exp, lod, pf, n)
        if frame == 0:
            moved_visible = np.isin(att, oids).sum()
            assert moved_visible > 50, "the scene should have attached entities in view"
            S.endFrame()
            prev = S.prevTransforms()
            for field in ("pos", "rot", "scale"):
                assert prev[field][att].tobytes() == exp_tr[field].tobytes()
            rest = np.ones(n, bool)
            rest[att] = False
            assert not prev["pos"][rest].any()
    for p in dev.values():
        ctx.free_device(p)
    anim.close()
    S.close()
    cs.close()
