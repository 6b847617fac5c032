"""The drop-in boundary, executed: lumixengine_b200/host/culling_system_b200.cpp linked with the reference's own job system, allocators and
PageAllocator (oracle/_ref/libengine_shim_b200.so, built by oracle/build_ref.py from /root/reference + this repository's shim).  The GPU is
driven through the engine's abstract CullingSystem (culling_system.h:58-77): CullingSystem::create(allocator, page_allocator), add / set /
remove, cull() from job-system fibers for several views at once (pipeline.cpp:1036-1041), the CullResult page chain (one renderable
type per 4 KB page, <= 1020 ids, pages from the engine's PageAllocator) walked and freed by the caller (pipeline.cpp:1045)."""
import ctypes as C
import os

import numpy as np
import pytest

import lumixengine_b200 as lb
from lumixengine_b200 import scenes

pytestmark = pytest.mark.gpu
SO = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "oracle", "_ref", "libengine_shim_b200.so")


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


@pytest.fixture(scope="module")
def shim():
    if not os.path.exists(SO):
        pytest.skip("oracle/_ref/libengine_shim_b200.so not built (needs /root/reference at build time)")
    L = C.CDLL(SO)
    os.environ["LB200_ENGINE_SHIM_LOADED"] = "1"  # the engine's job system cannot be shut down on Linux: tests/conftest.py leaves with os._exit
    L.shim_create.restype = C.c_void_p
    L.shim_get_radius.restype = C.c_float
    assert L.shim_jobs_init(C.c_int(4)) == 4
    return L


def _cull_views(L, h, frusta, type, cap):
    fb = np.ascontiguousarray(np.stack([lb.culling.frustum_bytes(f) for f in frusta]))
    ids = np.zeros((len(frusta), cap), np.uint32)
    tys = np.zeros((len(frusta), cap), np.uint8)
    info = np.zeros((len(frusta), 4), np.uint32)
    L.shim_cull_views(C.c_void_p(h), _p(fb), C.c_uint32(len(frusta)), C.c_int(type), _p(ids), _p(tys), C.c_uint32(cap), _p(info))
    return [(ids[v, :info[v, 0]].copy(), tys[v, :info[v, 0]].copy(), info[v]) for v in range(len(frusta))]


def test_cull_through_the_engine_vtable_from_job_fibers(shim, oracle):
    L = shim
    n = 120_000
    scene = scenes.cull_scene(n, (3000.0, 300.0, 3000.0), seed=77, big_fraction=0.004, type_probs=(0.7, 0.15, 0.1, 0.05))
    h = L.shim_create()
    e, t, p, r = (np.ascontiguousarray(scene[k], d) for k, d in (("entities", np.int32), ("types", np.uint8), ("pos", np.float64), ("radius", np.float32)))
    L.shim_add(C.c_void_p(h), _p(e), _p(t), _p(p), _p(r), C.c_uint32(n))
    oc = oracle.OracleCulling()
    oc.add(scene["entities"], scene["types"], scene["pos"], scene["radius"])
    assert L.shim_is_added(C.c_void_p(h), C.c_int32(5)) == 1 and L.shim_get_radius(C.c_void_p(h), C.c_int32(5)) == np.float32(scene["radius"][5])
    a = scenes.c1_frustum_args()
    frusta = [lb.frustum_perspective(**dict(a, far=3500.0)),
              lb.frustum_perspective(**dict(a, position=(500.0, 30.0, 400.0), direction=(-0.6, -0.1, -0.8), far=2500.0)),
              lb.frustum_ortho((0.0, 1000.0, 0.0), (0.0, -1.0, 0.0), (0.0, 0.0, -1.0), 900.0, 900.0, 0.0, 2000.0),
              lb.frustum_perspective(**dict(a, position=(1e6, 0.0, 1e6), far=50.0))]  # sees nothing
    base_pages = L.shim_allocated_pages(C.c_void_p(h))

    def check(type_filter):
        views = _cull_views(L, h, frusta, type_filter, n)  # four views, four jobs at once
        for f, (ids, tys, info) in zip(frusta, views):
            oi, ot, _ = oc.cull(lb.culling.frustum_bytes(f), type_filter)
            assert info[2] == 0, "a result page broke the CullResult contract (count > 1020 or not 4 KB aligned)"
            assert len(ids) == len(oi)
            assert np.array_equal(np.sort(ids.astype(np.int64) * 256 + tys), np.sort(oi.astype(np.int64) * 256 + ot))
            if len(oi):
                assert info[1] >= -(-len(oi) // 1020) and info[3] == 0
        assert sum(len(v[0]) for v in views) > 20_000 or type_filter > 0
        assert L.shim_allocated_pages(C.c_void_p(h)) == base_pages, "CullResult::free left pages allocated"
    check(-1)
    check(1)
    # edits through the same interface (setPosition / setRadius / remove paths of culling_system.cpp:160-258), then again
    rng = np.random.default_rng(4)
    mv = rng.choice(n, 6000, replace=False).astype(np.int32)
    newp = scene["pos"][mv] + rng.normal(size=(len(mv), 3)) * np.array([400.0, 30.0, 400.0])
    newr = (rng.random(len(mv)) * 500).astype(np.float32)
    L.shim_set(C.c_void_p(h), _p(mv), _p(np.ascontiguousarray(newp)), _p(newr), C.c_uint32(len(mv)))
    oc.set(mv, newp, newr)
    gone = rng.choice(np.setdiff1d(np.arange(n, dtype=np.int32), mv), 3000, replace=False).astype(np.int32)
    L.shim_remove(C.c_void_p(h), _p(gone), C.c_uint32(len(gone)))
    oc.remove(gone)
    base_pages = L.shim_allocated_pages(C.c_void_p(h))
    check(-1)
    os.write(2, b"[test] all views checked\n")
    L.shim_destroy(C.c_void_p(h))


def _wshim(L):
    L.wshim_run.restype = C.c_int
    return L.wshim_run


@pytest.mark.parametrize("n,depth,fanout,reparent", [(20_000, 6, 3, 0), (60_000, 8, 4, 1)])
def test_world_patch_runs_inside_the_reference_world(shim, oracle, n, depth, fanout, reparent):
    """host/world_b200.inl inside the reference's own World (world.cpp + the patch, compiled by oracle/build_ref.py): root moves through
    World::setTransformsDeferredB200 + World::propagateHierarchyB200 (GPU) against the same moves through World::setTransform — the
    reference recursion transformEntity (world.cpp:255-282) — in a second World of the same process.  Every Transform bit for bit, and the
    `transformed` delegates (world.h:139, what RenderModule::onModelInstanceMoved hangs on) fire for the same entities the same number of
    times."""
    from lumixengine_b200.hierarchy import TRANSFORM_DTYPE
    parents, locals_, roots = scenes.hierarchy_forest(n, depth, fanout, seed=21 + depth)
    rng = np.random.default_rng(5)
    listens = (rng.random(n) < 0.7).astype(np.uint8)
    root_ids = np.nonzero(parents < 0)[0].astype(np.uint32)
    moved = rng.choice(root_ids, max(1, len(root_ids) // 2), replace=False).astype(np.uint32)  # half of the roots move, the other trees must stay put
    rounds = 3
    vals = np.zeros((rounds, len(moved)), TRANSFORM_DTYPE)
    for r in range(rounds):
        vals[r]["pos"] = roots[moved]["pos"] + rng.normal(size=(len(moved), 3)) * 50.0
        vals[r]["rot"] = scenes.random_unit_quats(rng, len(moved))
        vals[r]["scale"] = (0.7 + 0.6 * rng.random((len(moved), 3))).astype(np.float32)
    out_ref = np.zeros(n, TRANSFORM_DTYPE)
    out_b = np.zeros(n, TRANSFORM_DTYPE)
    calls_ref = np.zeros(n, np.uint32)
    calls_b = np.zeros(n, np.uint32)
    seconds = np.zeros(2)
    world_locals = np.zeros(n, TRANSFORM_DTYPE)
    rc = _wshim(shim)(_p(parents), _p(np.ascontiguousarray(locals_)), _p(np.ascontiguousarray(roots)), C.c_uint32(n), _p(listens),
                      _p(moved), _p(np.ascontiguousarray(vals)), C.c_uint32(len(moved)), C.c_uint32(rounds), C.c_int(reparent),
                      _p(out_ref), _p(out_b), _p(calls_ref), _p(calls_b), _p(seconds), _p(world_locals))
    assert rc == 0
    for field in ("pos", "rot", "scale"):
        assert out_ref[field].tobytes() == out_b[field].tobytes(), "World::propagateHierarchyB200 left other transforms than World::transformEntity"
    assert np.array_equal(calls_ref, calls_b), "the `transformed` delegates fired for other entities than under the reference recursion"
    assert calls_ref.sum() > 0 and (calls_ref[listens == 0] == 0).all()
    if not reparent:  # the reference World against the C restatement as well: same forest, last round's roots, and the local transforms as the
        # World holds them (World::setLocalTransform recomputes the local from the composed global, world.cpp:704-712 + 267-270)
        g = roots.copy()
        g[moved] = vals[-1]
        as_bytes = lambda a: np.ascontiguousarray(a).view(np.uint8).reshape(len(a), 56)
        want = oracle.propagate(parents, as_bytes(world_locals), as_bytes(g)).view(TRANSFORM_DTYPE).reshape(-1)
        # only under the moved roots: an unmoved node still holds the global composed from the local the caller passed in, while the World
        # keeps the recomputed local
        under_moved = np.zeros(n, bool)
        under_moved[moved] = True
        for i in range(n):  # parents come before their children
            if parents[i] >= 0:
                under_moved[i] = under_moved[parents[i]]
        assert under_moved.sum() > len(moved)
        for field in ("pos", "rot", "scale"):  # not the 4 padding bytes of the 56-byte Transform
            assert want[field][under_moved].tobytes() == out_ref[field][under_moved].tobytes()
    os.write(2, f"[test] world patch n={n}: reference recursion {seconds[0] * 1e3:.2f} ms, B200 path {seconds[1] * 1e3:.2f} ms (host time, {rounds} rounds)\n".encode())


def test_animation_binding_runs_over_reference_objects(shim):
    """host/animation_b200.inl (AnimablesB200, the batched AnimationModuleImpl::updateAnimables) over real Lumix::Model / Animation / Pose
    objects: poses delivered through lockPose / unlockPose and Animable::time after three frames, against the reference's own
    updateAnimable body (Animation::getRelativePose + Pose::computeAbsolute from its animation.cpp / pose.cpp) per animable, bit for bit."""
    from lumixengine_b200 import _lib
    sk = scenes.skeleton(48)
    clips = [scenes.clip(sk, frames=40, seed=s) for s in (5, 6, 7)]
    n = 700
    ci, tt = scenes.instance_times(n, clips, seed=3)
    ci = np.ascontiguousarray(ci, np.uint32)
    tt = np.ascontiguousarray(tt, np.uint32)
    sks = sk.as_struct(_lib.Skeleton)
    arr = (_lib.Clip * len(clips))(*[c.as_struct(_lib.Clip) for c in clips])
    B = sk.bone_count
    out = {k: np.zeros((n, B, w), np.float32) for k, w in (("pos_ref", 3), ("rot_ref", 4), ("pos_b", 3), ("rot_b", 4))}
    time_ref, time_b, info = np.zeros(n, np.uint32), np.zeros(n, np.uint32), np.zeros(4, np.uint32)
    shim.ashim_run.restype = C.c_int
    for dt, rounds in ((1.0 / 30.0, 3), (-0.05, 2)):
        rc = shim.ashim_run(C.byref(sks), arr, C.c_uint32(len(clips)), _p(ci), _p(tt), C.c_uint32(n), C.c_float(dt), C.c_uint32(rounds),
                            _p(out["pos_ref"]), _p(out["rot_ref"]), _p(time_ref), _p(out["pos_b"]), _p(out["rot_b"]), _p(time_b), _p(info))
        assert rc == 0 and info[2] == 0
        assert info[0] == info[1] == n * rounds and info[3] == n  # every animable locked and unlocked once per frame, poses left absolute
        assert np.array_equal(time_ref, time_b)
        assert not np.array_equal(time_ref, tt)
        assert out["pos_ref"].tobytes() == out["pos_b"].tobytes(), "AnimablesB200 delivered other bone positions than updateAnimable"
        assert out["rot_ref"].tobytes() == out["rot_b"].tobytes(), "AnimablesB200 delivered other bone rotations than updateAnimable"
        assert np.abs(out["pos_ref"]).max() > 0.1
